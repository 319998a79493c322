"""C-ABI library: loads, exports every symbol include/fruitnerf_b200.h declares, and rejects bad
arguments with error codes (no compute calls: these run without a GPU)."""
import ctypes as C
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _declared_symbols():
    hdr = (ROOT / "include" / "fruitnerf_b200.h").read_text()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(fnr_[a-z_0-9]+)\s*\(", hdr)))


def test_header_symbols_are_exported(native_lib):
    from fruitnerf_b200 import _lib

    declared = _declared_symbols()
    assert declared, "no declarations parsed"
    for name in declared:
        assert hasattr(native_lib, name), f"{name} declared in include/fruitnerf_b200.h but not exported"
    assert sorted(_lib.EXPORTED_SYMBOLS) == declared
    assert native_lib.fnr_version() == 2


def test_struct_sizes_match_header(native_lib):
    """ctypes mirrors vs the C compiler's layout (compiled on the fly with gcc)."""
    import subprocess
    import tempfile

    from fruitnerf_b200 import _lib as L

    src = '#include <stdio.h>\n#include "fruitnerf_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n",' \
          "sizeof(fnr_field_desc),sizeof(fnr_field_params),sizeof(fnr_ray_batch),sizeof(fnr_render_out),sizeof(fnr_render_grads)," \
          "sizeof(fnr_render_saved),sizeof(fnr_export_params),sizeof(fnr_export_out),sizeof(fnr_nvls_desc));return 0;}\n"
    with tempfile.TemporaryDirectory() as td:
        c = Path(td) / "s.c"
        c.write_text(src)
        subprocess.run(["gcc", "-I", str(ROOT / "include"), str(c), "-o", str(Path(td) / "s")], check=True)
        sizes = list(map(int, subprocess.run([str(Path(td) / "s")], capture_output=True, text=True, check=True).stdout.split()))
    mirrors = [L.FieldDesc, L.FieldParams, L.RayBatch, L.RenderOut, L.RenderGrads, L.RenderSaved, L.ExportParams, L.ExportOut, L.NvlsDesc]
    assert sizes == [C.sizeof(m) for m in mirrors]


def test_invalid_arguments_return_error_codes(native_lib):
    from fruitnerf_b200 import _lib as L

    assert native_lib.fnr_render_forward(None, None, None, None, None) == -1
    assert b"desc is NULL" in native_lib.fnr_last_error()
    d = L.FieldDesc()  # all zeros: invalid hash grid
    assert native_lib.fnr_render_forward(C.byref(d), None, None, None, None) == -1
    d.num_levels, d.features_per_level, d.log2_hashmap_size, d.num_images, d.appearance_dim = 16, 2, 19, 3, 32
    d.geo_feat_dim = 7  # unsupported family
    assert native_lib.fnr_render_forward(C.byref(d), None, None, None, None) == -2
    assert b"unsupported FruitField shape" in native_lib.fnr_last_error()
    n = C.c_size_t(0)
    assert native_lib.fnr_render_backward_scratch_bytes(C.byref(d), 8, 8, C.byref(n)) == -2


def test_invalid_impl_is_rejected_by_every_field_entry_point(native_lib):
    from fruitnerf_b200 import _lib as L

    d = L.FieldDesc()  # fruit_nerf (small family) shape
    d.num_levels, d.features_per_level, d.log2_hashmap_size, d.num_images, d.appearance_dim = 16, 2, 19, 3, 32
    d.geo_feat_dim = 15
    for m, dims in ((d.base, (32, 64, 16)), (d.semantic, (15, 64, 64)), (d.color, (63, 64, 64, 3))):
        m.n_layers = len(dims) - 1
        for i, v in enumerate(dims):
            m.dims[i] = v
    d.impl = 7
    calls = {
        "fnr_render_forward": lambda: native_lib.fnr_render_forward(C.byref(d), None, None, None, None),
        "fnr_render_backward": lambda: native_lib.fnr_render_backward(C.byref(d), None, None, None, None, None, None, 0, None),
        "fnr_export_forward": lambda: native_lib.fnr_export_forward(C.byref(d), None, None, None, None, 0.0, 1.0, 0, 1, 0, None,
                                                                    None, None),
    }
    for name, call in calls.items():
        assert call() == -1, name
        assert b"invalid impl" in native_lib.fnr_last_error(), name


def test_ops_refuse_cpu_tensors(native_lib):
    import torch

    from fruitnerf_b200 import _lib as L
    from fruitnerf_b200 import ops

    from .util import make_field, make_state

    sd, spec = make_state("small", log2T=10)
    field = make_field("small", sd, spec, "cpu")
    o = torch.zeros(2, 3)
    with pytest.raises(L.FruitNerfNativeError, match="no CPU fallback"):
        ops.render(field.kernel_shape(), field.kernel_params(), o, o, torch.zeros(2, 4), torch.ones(2, 4), None,
                   field.position_mode(), L.FNR_APP_ZEROS)
