"""fnr_render_backward's scratch: its size for the simt and the tensor-core implementations, and the refusal of scratch too
small for the tensor-core path.  These calls return before any device work, so they run without a GPU (the pointers below
are never dereferenced)."""
import ctypes as C

import pytest

from fruitnerf_b200 import _lib as L

FAMILIES = {
    "small": (15, ((32, 64, 16), (15, 64, 64), (63, 64, 64, 3))),
    "big": (30, ((32, 64, 31), (30, 128, 128, 64), (78, 64, 64, 3))),
}


def _desc(family, impl, log2T=19):
    geo, mlps = FAMILIES[family]
    d = L.FieldDesc()
    d.num_levels, d.features_per_level, d.log2_hashmap_size, d.num_images, d.appearance_dim = 16, 2, log2T, 7, 32
    d.geo_feat_dim = geo
    for m, dims in zip((d.base, d.semantic, d.color), mlps):
        m.n_layers = len(dims) - 1
        for i, v in enumerate(dims):
            m.dims[i] = v
    d.impl = impl
    return d


def _scratch_bytes(lib, desc, R, S):
    n = C.c_size_t(0)
    assert lib.fnr_render_backward_scratch_bytes(C.byref(desc), R, S, C.byref(n)) == 0
    return n.value


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("R,S", [(4096, 192), (1, 1), (37, 77), (0, 5)])
def test_scratch_bytes_simt_vs_tensor_core(native_lib, family, R, S):
    """simt: the per-point upstream gradients (5 floats) plus alignment.  The small family's tensor-core backward: also the
    [16][N] float2 encoding gradients of the level-major scatter, plus alignment; the big family's scatters inline."""
    n = R * S
    simt = _scratch_bytes(native_lib, _desc(family, L.FNR_IMPL_SIMT), R, S)
    assert simt == n * 5 * 4 + 256
    extra = 256 + n * 16 * 2 * 4 if family == "small" else 0
    for impl in (L.FNR_IMPL_AUTO, L.FNR_IMPL_TCGEN05):
        assert _scratch_bytes(native_lib, _desc(family, impl), R, S) == simt + extra


def test_tensor_core_backward_refuses_scratch_sized_for_simt(native_lib):
    """fruit_nerf's tensor-core backward needs the encoding-gradient buffer: simt-sized scratch is refused up front."""
    fake = 256  # 16-byte aligned, never dereferenced
    R, S = 64, 48
    params = L.FieldParams()
    params.hash_table = params.head_w = params.head_b = params.app_embedding = fake
    for arr in (params.base_w, params.base_b, params.sem_w, params.sem_b, params.col_w, params.col_b):
        for i in range(L.FNR_MAX_LAYERS):
            arr[i] = fake
    rays = L.RayBatch(R, S, fake, fake, fake, fake, fake)
    saved = L.RenderSaved(fake, fake, fake, fake, fake, fake)
    up = L.RenderGrads(fake, None, fake, None, None, None, None)
    simt_bytes = _scratch_bytes(native_lib, _desc("small", L.FNR_IMPL_SIMT), R, S)
    for impl in (L.FNR_IMPL_AUTO, L.FNR_IMPL_TCGEN05):
        desc = _desc("small", impl)
        need = _scratch_bytes(native_lib, desc, R, S)
        for have in (simt_bytes, need - 1):
            rc = native_lib.fnr_render_backward(C.byref(desc), C.byref(params), C.byref(rays), C.byref(saved), C.byref(up),
                                                C.byref(params), fake, have, None)
            assert rc == -1, (impl, have)
            assert b"scratch too small" in native_lib.fnr_last_error()
