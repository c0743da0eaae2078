"""CPU checks of the deterministic render and loss (no device needed): the new C-ABI entry points refuse null, misaligned
and undersized arguments before any launch, their workspace queries follow the documented layout, the operators'
deterministic=None follows torch.use_deterministic_algorithms, and the legacy tile scatter-add (float atomics where tile
positions repeat) goes through torch's nondeterminism alert."""
import ctypes as C
import warnings

import pytest
import torch

GS_EINVAL, GS_ENOMEM = -1, -3
W, H = 64, 48
T = (W // 16) * (H // 16)
FAKE = 0x10000          # 256-byte aligned, never dereferenced: every call below fails validation first


@pytest.fixture(scope="module")
def lib():
    from gs_b200 import build, _lib
    build.build()
    return _lib.load()


@pytest.fixture
def det_flag():
    """torch.use_deterministic_algorithms set by the test and restored afterwards."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


def _err(lib):
    return lib.gs_last_error().decode().lower()


def _fwd(lib, num_views=1, view_start=None, P=4, R=8, sorted_u=FAKE, ids_unsorted=FAKE, ids_sorted=FAKE):
    p = [FAKE] * 7
    return lib.gs_render_forward_det(num_views, view_start, P, R, H, W, *p[:7], FAKE, ids_unsorted, FAKE, ids_sorted,
                                     sorted_u, FAKE, 1 << 20, FAKE, FAKE, FAKE, FAKE, None, None, FAKE, 1 << 24, None)


def test_render_forward_det_rejects_bad_arguments(lib):
    assert _fwd(lib, num_views=2) == GS_EINVAL and "view_start" in _err(lib)      # NULL view_start is one view only
    assert _fwd(lib, P=-1) == GS_EINVAL
    assert _fwd(lib, sorted_u=None) == GS_EINVAL and "null" in _err(lib)
    assert _fwd(lib, ids_unsorted=None) == GS_EINVAL and "null" in _err(lib)
    assert _fwd(lib, sorted_u=FAKE + 2) == GS_EINVAL and "aligned" in _err(lib)
    assert _fwd(lib, ids_sorted=FAKE + 1) == GS_EINVAL and "aligned" in _err(lib)
    bad_views = (C.c_int32 * 3)(1, 2, 3)                                               # view_start[0] != 0
    assert _fwd(lib, num_views=2, view_start=bad_views) == GS_EINVAL


def _bwd(lib, P=4, R=8, seg=FAKE, seg_bytes=None, det_ws=FAKE, det_bytes=None, order=FAKE, grads=FAKE, sorted_u=FAKE,
         num_views=1):
    seg_bytes = lib.gs_render_seg_bytes(R, T * num_views) if seg_bytes is None else seg_bytes
    det_bytes = lib.gs_render_det_bytes(R, P) if det_bytes is None else det_bytes
    return lib.gs_render_backward_det(num_views, P, R, H, W, FAKE, FAKE, FAKE, FAKE, FAKE, sorted_u, order, FAKE, FAKE,
                                      FAKE, FAKE, seg, seg_bytes, det_ws, det_bytes, grads, FAKE, FAKE, None)


def test_render_backward_det_rejects_bad_arguments(lib):
    from gs_b200 import _lib
    assert _bwd(lib, num_views=0) == GS_EINVAL
    assert _bwd(lib, R=-1) == GS_EINVAL
    assert _bwd(lib, R=1 << 31) == GS_EINVAL
    assert _bwd(lib, order=None) == GS_EINVAL and "null" in _err(lib)
    assert _bwd(lib, grads=None) == GS_EINVAL and "null" in _err(lib)
    assert _bwd(lib, sorted_u=None) == GS_EINVAL and "null" in _err(lib)
    assert _bwd(lib, order=FAKE + 2) == GS_EINVAL and "aligned" in _err(lib)
    assert _bwd(lib, det_ws=FAKE + 16) == GS_EINVAL and "256-byte" in _err(lib)
    assert _bwd(lib, det_ws=None) == GS_EINVAL
    # no deterministic form without the segment workspace (the tile-parallel backward), nor with the debug tile kernel
    assert _bwd(lib, seg=None) == GS_EINVAL and "segment workspace" in _err(lib)
    prev = _lib.debug_set(_lib.DEBUG_BWD_TILE)
    try:
        assert _bwd(lib) == GS_EINVAL and "gs_debug_bwd_tile" in _err(lib)
    finally:
        _lib.debug_set(prev)
    assert _bwd(lib, seg_bytes=lib.gs_render_seg_bytes(8, T) - 1) == GS_ENOMEM
    assert _bwd(lib, det_bytes=lib.gs_render_det_bytes(8, 4) - 1) == GS_ENOMEM and "det_ws" in _err(lib)


def test_loss_forward_det_rejects_bad_arguments(lib):
    tb = lib.gs_loss_temp_bytes_det(H, W)
    assert lib.gs_loss_forward_det(H, W, 0, H, 0, H, FAKE, FAKE, FAKE, FAKE, tb - 257, None) == GS_ENOMEM   # the query adds 256 spare bytes
    assert lib.gs_loss_forward_det(H, W, 0, H, 0, H, FAKE, FAKE, FAKE, FAKE + 4, tb, None) == GS_EINVAL
    assert "8-byte" in _err(lib)
    assert lib.gs_loss_forward_det(H, W, 0, H, 0, H, FAKE, None, FAKE, FAKE, tb, None) == GS_EINVAL
    assert lib.gs_loss_forward_det(H, W, 0, H, 0, H, None, FAKE, FAKE, FAKE, tb, None) == GS_EINVAL
    assert lib.gs_loss_forward_det(H, W, 5, 5, 5, 5, FAKE, FAKE, FAKE, FAKE, tb, None) == GS_EINVAL
    rows4 = (C.c_int32 * 8)(0, H, 0, H, 0, 16, 0, 16)
    gts = (C.c_void_p * 2)(FAKE, FAKE)
    tbb = lib.gs_loss_temp_bytes_batched_det(2, rows4, W)
    assert lib.gs_loss_forward_batched_det(2, H, W, rows4, FAKE, gts, FAKE, FAKE, tbb - 257, None) == GS_ENOMEM
    assert lib.gs_loss_forward_batched_det(65, H, W, rows4, FAKE, gts, FAKE, FAKE, tbb, None) == GS_EINVAL
    assert lib.gs_loss_forward_batched_det(2, H, W, rows4, FAKE, (C.c_void_p * 2)(FAKE, None), FAKE, FAKE, tbb,
                                           None) == GS_EINVAL


def _up(v, a=256):
    return (v + a - 1) // a * a


@pytest.mark.parametrize("R,P", [(0, 0), (1, 1), (7, 3), (1000, 999), (5_700_000, 2_000_000), ((1 << 31) - 1, (1 << 31) - 1)])
def test_render_det_bytes(lib, R, P):
    """A 256-byte header (the long-range counter), 36 bytes (9 floats) per instance and twice 4 bytes (the depth rank and
    the long-range list) per splat, each in whole 256-byte blocks."""
    assert lib.gs_render_det_bytes(R, P) == 256 + _up(36 * R) + 2 * _up(4 * P)
    assert lib.gs_render_det_bytes(-5, -1) == 256


@pytest.mark.parametrize("rows,width", [(1, 1), (32, 32), (33, 33), (1080, 1920), (137, 1959)])
def test_loss_det_bytes(lib, rows, width):
    """The deterministic temp is the atomic form's header and maps, then 16 bytes (two fp64 partials) per 32x32 CTA."""
    ctas = -(-rows // 32) * -(-width // 32)
    assert lib.gs_loss_temp_bytes_det(rows, width) == 256 + _up(36 * rows * width) + 16 * ctas + 256
    assert lib.gs_loss_temp_bytes_det(rows, width) >= lib.gs_loss_temp_bytes(rows, width)
    # batched: one slot per CTA of the grid, which every view spans at the tallest strip's height
    r4 = [0, rows, 0, rows, 0, 0, 0, 0, 3, 3 + (rows + 1) // 2, 3, 3 + (rows + 1) // 2]
    rows4 = (C.c_int32 * 12)(*r4)
    sum_rows = rows + (rows + 1) // 2
    expect = 2 * 8 * 64 + _up(36 * sum_rows * width) + 16 * 3 * ctas + 256
    assert lib.gs_loss_temp_bytes_batched_det(3, rows4, width) == expect
    assert lib.gs_loss_temp_bytes_batched_det(3, rows4, width) >= lib.gs_loss_temp_bytes_batched(3, rows4, width)


def test_deterministic_none_follows_the_torch_flag(det_flag):
    from gs_b200 import ops
    torch.use_deterministic_algorithms(False)
    assert ops.deterministic_enabled() is False and ops.deterministic_enabled(None) is False
    assert ops.deterministic_enabled(True) is True
    torch.use_deterministic_algorithms(True)
    assert ops.deterministic_enabled() is True and ops.deterministic_enabled(False) is False
    torch.use_deterministic_algorithms(True, warn_only=True)
    assert ops.deterministic_enabled() is True


def test_trainer_refuses_determinism_with_a_moving_division():
    """Determinism holds for a fixed strip division; the load balancer moves strips by measured times."""
    from gs_b200 import pipeline
    with pytest.raises(ValueError, match="load_balance"):
        pipeline.Trainer({"means3D": torch.zeros((4, 3))}, [], None, "cpu", rank=0, world=2, deterministic=True)


def _merge_args():
    pos = torch.zeros((2, 2), dtype=torch.int64)                # both tiles at the same position: added atomically
    tiles = torch.zeros((2, 3, 16, 16))
    return pos, tiles, 32, 32, (0, 16, 0, 16), (0, 1, 0, 1)


def test_legacy_scatter_add_raises_under_the_flag(det_flag):
    from gs_b200 import ops
    torch.use_deterministic_algorithms(True)
    with pytest.raises(RuntimeError, match="merge_image_tiles_by_pos does not have a deterministic implementation"):
        ops.merge_image_tiles_by_pos(*_merge_args())


def test_legacy_scatter_add_warns_under_warn_only(det_flag):
    from gs_b200 import ops
    torch.use_deterministic_algorithms(True, warn_only=True)
    with warnings.catch_warnings(record=True) as got:
        warnings.simplefilter("always")
        with pytest.raises(ValueError, match="CUDA tensor"):   # warned, then refused for the CPU tensor as always
            ops.merge_image_tiles_by_pos(*_merge_args())
    assert any("merge_image_tiles_by_pos does not have a deterministic implementation" in str(w.message) for w in got)
    torch.use_deterministic_algorithms(False)
    with warnings.catch_warnings(record=True) as got:
        warnings.simplefilter("always")
        with pytest.raises(ValueError, match="CUDA tensor"):
            ops.merge_image_tiles_by_pos(*_merge_args())
    assert not any("deterministic" in str(w.message) for w in got)
