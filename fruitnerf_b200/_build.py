"""In-tree build of libfruitnerf_b200.so (sm_90a, H100) with nvcc.  Used by __graft_entry__.build().

The tensor-core path (impl = tcgen05 / auto) is the wgmma instantiation of the kernels in fnr_simt.cu (fnr_wgmma.cuh,
dispatch in fnr_api.cu).  The fused Blackwell kernels are kept outside the library under design/blackwell/."""
from __future__ import annotations

import os
import shutil
import subprocess
from pathlib import Path

CSRC = Path(__file__).resolve().parent / "csrc"
LIB = CSRC / "libfruitnerf_b200.so"
STAMP = CSRC / "libfruitnerf_b200.recipe"  # flags and sources LIB was built from
SOURCES = ["fnr_api.cu", "fnr_simt.cu", "fnr_proposal.cu", "fnr_optim.cu", "fnr_glue.cu", "fnr_nvls.cu", "fnr_cluster.cu",
           "fnr_fruit_split.cu", "fnr_render.cu", "fnr_mesh.cu", "fnr_poisson.cu", "fnr_measure.cu", "fnr_metrics.cu", "fnr_texture.cu",
           "fnr_decimate.cu", "fnr_unwrap.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-O2",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found")


def _stale(target: Path, deps) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False, defines=(), out_dir=None) -> Path:
    """Build the library; ``defines`` (e.g. ``["FNR_BWD_PHASE_TIMERS"]``) are passed as -D flags, and a diagnostic build
    with them should name its own ``out_dir`` for the objects and the library so that it never replaces the normal one."""
    flags = [*NVCC_FLAGS, *(f"-D{d}" for d in defines)]
    dest = Path(out_dir) if out_dir is not None else CSRC
    dest.mkdir(parents=True, exist_ok=True)
    lib, stamp = dest / LIB.name, dest / STAMP.name
    # objects built with other flags or sources (an older architecture, say) are stale whatever their mtimes
    recipe = " ".join([*flags, *SOURCES])
    if not stamp.exists() or stamp.read_text() != recipe:
        force = True
    headers = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + [CSRC.parent.parent / "include" / "fruitnerf_b200.h"]
    objs = []
    procs = []
    for src in SOURCES:
        obj = dest / (src[:-3] + ".o")
        objs.append(obj)
        if force or _stale(obj, [CSRC / src, *headers]):
            cmd = [_nvcc(), *flags, "-c", str(CSRC / src), "-o", str(obj)]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        log, _ = p.communicate()
        if verbose and log:
            print(log)
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{log}")
    if force or procs or _stale(lib, objs):
        cmd = [_nvcc(), "-shared", "-o", str(lib), *map(str, objs), "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}{r.stderr}")
        stamp.write_text(recipe)
    return lib


if __name__ == "__main__":
    import sys

    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
