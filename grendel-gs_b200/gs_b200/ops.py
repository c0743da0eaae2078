"""Autograd operators over the C ABI: the host-side mirror of the reference's
`diff_gaussian_rasterization` wrappers (SURVEY.md section 8b).

  preprocess_gaussians  /root/reference/gaussian_renderer/__init__.py:949-958
  render_gaussians      /root/reference/gaussian_renderer/__init__.py:1271-1282
  get_local2j_ids_bool  /root/reference/gaussian_renderer/workload_division.py:721-744
"""
import contextlib
import ctypes as C
import os

import torch

from . import _lib, statlog

BLOCK_X, BLOCK_Y, ONE_DIM_BLOCK_SIZE = 16, 16, 256


# torch.cuda.current_stream() costs ~20 us of Python per call and every operator asks for it: a caller that runs a whole
# step on one stream (pipeline.Trainer.step) pins the handle here for the duration of the step (None = ask torch)
STEP_STREAM = None


def _stream():
    return STEP_STREAM if STEP_STREAM is not None else torch.cuda.current_stream().cuda_stream


def _f32c(t, name):
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (this operator has no CPU path)")
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    return t.contiguous()


class LazyMs:
    """Elapsed milliseconds between two CUDA events, resolved on first numeric use.

    cuda_args["stats_collector"]["forward_render_time"/"backward_render_time"] must be readable as
    numbers by finish_strategy_final (/root/reference/gaussian_renderer/workload_division.py:953-957).
    Resolving lazily removes two host syncs per camera from the step; set GS_B200_EAGER_TIMING=1 to
    store plain floats instead."""

    __slots__ = ("_s", "_e", "_v")

    def __init__(self, start, end):
        self._s, self._e, self._v = start, end, None

    def value(self):
        if self._v is None:
            self._e.synchronize()
            self._v = float(self._s.elapsed_time(self._e))
            self._s = self._e = None
        return self._v

    def __float__(self):
        return self.value()

    def __add__(self, o):
        return self.value() + float(o)

    __radd__ = __add__

    def __sub__(self, o):
        return self.value() - float(o)

    def __rsub__(self, o):
        return float(o) - self.value()

    def __mul__(self, o):
        return self.value() * float(o)

    __rmul__ = __mul__

    def __truediv__(self, o):
        return self.value() / float(o)

    def __rtruediv__(self, o):
        return float(o) / self.value()

    def __lt__(self, o):
        return self.value() < float(o)

    def __gt__(self, o):
        return self.value() > float(o)

    def __repr__(self):
        return repr(self.value())

    def __format__(self, spec):
        return format(self.value(), spec)


def _timed(collector, key, start, end):
    if collector is None:
        return
    v = LazyMs(start, end)
    collector[key] = v.value() if os.environ.get("GS_B200_EAGER_TIMING") == "1" else v


def _screen_outputs(lead, dev):
    """Empty (means2D, depths, radii, conic_opacity, rgb, clamped) of a preprocess forward; lead = (P,) or (B, P)."""
    f32 = torch.float32
    return (torch.empty((*lead, 2), dtype=f32, device=dev), torch.empty(lead, dtype=f32, device=dev),
            torch.empty(lead, dtype=torch.int32, device=dev), torch.empty((*lead, 4), dtype=f32, device=dev),
            torch.empty((*lead, 3), dtype=f32, device=dev), torch.empty(lead, dtype=torch.uint8, device=dev))


# stored SH coefficients K -> max_sh_degree: the reference's --sh_degree D keeps (D+1)^2 coefficients per Gaussian
# (scene/gaussian_model.py:51-53, 150-156)
_STORED_DEGREE = {1: 0, 4: 1, 9: 2, 16: 3}


def stored_sh_degree(K, what):
    """max_sh_degree of a model storing K SH coefficients per Gaussian; ValueError naming `what` for any other K."""
    if K not in _STORED_DEGREE:
        raise ValueError(f"{what}: a model stores (D+1)^2 SH coefficients, D = 0..3 (1, 4, 9 or 16), got {K}")
    return _STORED_DEGREE[K]


def _stored_degree(K, sh_degree, what):
    """stored_sh_degree, and a ValueError (before any launch) for an active sh_degree outside 0..max_sh_degree."""
    D = stored_sh_degree(K, what)
    if not 0 <= int(sh_degree) <= D:
        raise ValueError(f"active sh_degree {sh_degree} is outside 0..{D}, the degree the model stores ({K} coefficients)")
    return D


# The reference's --zhx_time keys (analyze_statistic.py:1972-1991) per operator call, and the gs_profile stage
# (gs_profile_stage_name) each one is read from.  None: the fork times the three statistics sums (81-83) as stages of their
# own; here they are fused into the blend forward (stage 70), so their keys read 0.  Stage 24 is written with the time of
# k_count_tiles, which covers the reference's 21-24; 24 is the column analyze_statistic.py sums.
REFERENCE_STAGE_KEYS = {
    "preprocess forward": (("10 preprocess time", "10 preprocess"),),
    "render forward": (("24 updateDistributedStatLocally.updateTileTouched time", "21-24 count local tiles"),
                       ("30 InclusiveSum time", "30 InclusiveSum"), ("40 duplicateWithKeys time", "40 duplicateWithKeys"),
                       ("50 SortPairs time", "50 SortPairs"), ("60 identifyTileRanges time", "60 identifyTileRanges"),
                       ("70 render time", "70 render"), ("81 sum_n_render time", None),
                       ("82 sum_n_consider time", None), ("83 sum_n_contrib time", None)),
    "render backward": (("b10 render time", "b10 render"),),
    "preprocess backward": (("b20 preprocess time", "b20 preprocess"),),
}


def reference_stage_times(call, stages):
    """[(reference key, ms)] of one operator call (a REFERENCE_STAGE_KEYS key) from _lib.profile_read() output; a stage
    without launches (no instances: nothing to sort) reads 0."""
    return [(key, 0.0 if st is None else float(stages.get(st, (0.0, 0))[0])) for key, st in REFERENCE_STAGE_KEYS[call]]


@contextlib.contextmanager
def _gpu_time(log, call):
    """--zhx_time around one operator call's launches: on a logging call (log.time) the profiler is switched on for the
    block, its stages are read back (a host sync, on logging iterations only), the profiler is put back as it was -- any
    times it held are handed back to its own reader -- and the call's block is appended to the gpu_time log.  Otherwise
    nothing at all happens."""
    if log is None or not log.time:
        yield
        return
    was_on = _lib.PROFILE_ON
    held = _lib.profile_read() if was_on else {}
    _lib.profile_enable(True)
    stages = {}
    try:
        yield
        stages = _lib.profile_read()
    finally:
        _lib.profile_enable(was_on)
        if was_on:
            _lib.profile_carry(held)
            _lib.profile_carry(stages)
    statlog.append(log.path("gpu_time"), statlog.gpu_time_text(
        log.iteration, f"rk={log.global_rank}, ws={log.world_size}, {call}", reference_stage_times(call, stages)))


def _grad_or_zeros(g, shape, dev):
    """An incoming gradient as contiguous fp32, or zeros where autograd passes None for an unused output."""
    return torch.zeros(shape, dtype=torch.float32, device=dev) if g is None else _f32c(g, "grad")


class _PreprocessGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, scales, rotations, shs, opacities, rs, log):
        ctx.set_materialize_grads(False)   # undefined output gradients arrive as None, not as zero-filled tensors
        means3D, scales, rotations = _f32c(means3D, "means3D"), _f32c(scales, "scales"), _f32c(rotations, "rotations")
        shs, opacities = _f32c(shs, "shs"), _f32c(opacities, "opacities")
        P = means3D.shape[0]
        if shs.dim() != 3 or shs.shape[2] != 3:
            raise ValueError(f"shs must be (P,K,3) (scene/gaussian_model.py:122-125), got {tuple(shs.shape)}")
        max_deg = _stored_degree(shs.shape[1], rs.sh_degree, "shs")
        if tuple(means3D.shape) != (P, 3) or tuple(scales.shape) != (P, 3) or tuple(rotations.shape) != (P, 4) \
                or opacities.numel() != P or shs.shape[0] != P:
            raise ValueError("inconsistent Gaussian parameter shapes")
        dev = means3D.device
        vm, pm, cp = _f32c(rs.viewmatrix, "viewmatrix"), _f32c(rs.projmatrix, "projmatrix"), _f32c(rs.campos, "campos")
        means2D, depths, radii, conic_opacity, rgb, clamped = _screen_outputs((P,), dev)
        with _gpu_time(log, "preprocess forward"):
            _lib.call("gs_preprocess_forward_sh", P, int(rs.sh_degree), max_deg, means3D.data_ptr(), scales.data_ptr(),
                      float(rs.scale_modifier), rotations.data_ptr(), opacities.data_ptr(), shs.data_ptr(), vm.data_ptr(),
                      pm.data_ptr(), cp.data_ptr(), int(rs.image_width), int(rs.image_height), float(rs.tanfovx),
                      float(rs.tanfovy), means2D.data_ptr(), depths.data_ptr(), radii.data_ptr(),
                      conic_opacity.data_ptr(), rgb.data_ptr(), clamped.data_ptr(), _stream())
        ctx.rs, ctx.max_deg, ctx.log = rs, max_deg, log
        ctx.cam = (vm, pm, cp)
        ctx.save_for_backward(means3D, scales, rotations, shs, radii, clamped)
        ctx.mark_non_differentiable(radii, depths)
        return means2D, rgb, conic_opacity, radii, depths

    @staticmethod
    def backward(ctx, g_means2D, g_rgb, g_conic_opacity, _g_radii, _g_depths):
        means3D, scales, rotations, shs, radii, clamped = ctx.saved_tensors
        rs = ctx.rs
        vm, pm, cp = ctx.cam
        P = means3D.shape[0]
        dev = means3D.device
        g_means2D, g_rgb = _grad_or_zeros(g_means2D, (P, 2), dev), _grad_or_zeros(g_rgb, (P, 3), dev)
        g_conic_opacity = _grad_or_zeros(g_conic_opacity, (P, 4), dev)
        d_means3D = torch.empty((P, 3), dtype=torch.float32, device=dev)
        d_scales = torch.empty((P, 3), dtype=torch.float32, device=dev)
        d_rot = torch.empty((P, 4), dtype=torch.float32, device=dev)
        d_opac = torch.empty((P, 1), dtype=torch.float32, device=dev)
        d_shs = torch.empty(tuple(shs.shape), dtype=torch.float32, device=dev)
        with _gpu_time(ctx.log, "preprocess backward"):
            _lib.call("gs_preprocess_backward_sh", P, int(rs.sh_degree), ctx.max_deg, means3D.data_ptr(),
                      scales.data_ptr(), float(rs.scale_modifier), rotations.data_ptr(), shs.data_ptr(), vm.data_ptr(),
                      pm.data_ptr(), cp.data_ptr(), int(rs.image_width), int(rs.image_height), float(rs.tanfovx),
                      float(rs.tanfovy), radii.data_ptr(), clamped.data_ptr(), g_means2D.data_ptr(),
                      g_conic_opacity.data_ptr(), g_rgb.data_ptr(), d_means3D.data_ptr(), d_scales.data_ptr(),
                      d_rot.data_ptr(), d_opac.data_ptr(), d_shs.data_ptr(), _stream())
        return d_means3D, d_scales, d_rot, d_shs, d_opac, None, None


def preprocess_gaussians(means3D, scales, rotations, shs, opacities, raster_settings, cuda_args=None):
    """-> (means2D (P,2) pixels, rgb (P,3), conic_opacity (P,4), radii (P) int32, depths (P)).
    shs (P,K,3): the K = (D+1)^2 coefficients of a model stored at degree D = 0..3; raster_settings.sh_degree <= D.
    cuda_args: the reference's dict; with zhx_time "True" on a logging iteration (statlog.request) this call and its
    backward append stages 10 and b20 to the gpu_time log."""
    return _PreprocessGaussians.apply(means3D, scales, rotations, shs, opacities, raster_settings,
                                      statlog.request(cuda_args))


# the raw preprocess operator's argument order, the C ABI's (GaussianParams attributes; GaussianParams.raw_parameters)
RAW_ORDER = ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")


def _raw_camera(B, rs, cams):
    """What the launch reads of the B views' cameras.  One view: (viewmatrix, projmatrix, campos, tanfovx, tanfovy), the
    device matrices and host tangents the single-camera kernels take, from its settings rs or, without them, from the row
    of the (1,40) table cams (the two tangents are read back to the host: a sync).  More views: the (B,40) device table
    cams, or cams() when it is a callable (the table is then built only here)."""
    if B == 1 and rs is not None:
        return (_f32c(rs.viewmatrix, "viewmatrix"), _f32c(rs.projmatrix, "projmatrix"), _f32c(rs.campos, "campos"),
                float(rs.tanfovx), float(rs.tanfovy))
    cams = _f32c(cams() if callable(cams) else cams, "cams")
    if tuple(cams.shape) != (B, 40):
        raise ValueError(f"cams must be ({B},40) (pack_cameras), got {tuple(cams.shape)}")
    if B > 1:
        return cams
    tanfovx, tanfovy = cams[0, 35:37].tolist()
    return cams[0, :16], cams[0, 16:32], cams[0, 32:35], tanfovx, tanfovy


def _launch_raw(direction, B, cam, P, meta, max_deg, params, *tail):
    """gs_preprocess_{direction}_raw_sh (B = 1) or gs_preprocess_{direction}_batched_sh (B > 1); params: the six raw
    parameters, tail: the direction's remaining tensors in the entry point's order."""
    W, H, D, mod = meta
    xyz, f_dc, f_rest, scaling, rotation, opacity = (t.data_ptr() for t in params)
    body = (P, D, max_deg, xyz, f_dc, f_rest, scaling, mod, rotation, opacity)
    tail = [t.data_ptr() for t in tail]
    if B == 1:
        vm, pm, cp, tanfovx, tanfovy = cam
        _lib.call(f"gs_preprocess_{direction}_raw_sh", *body, vm.data_ptr(), pm.data_ptr(), cp.data_ptr(), W, H, tanfovx,
                  tanfovy, *tail, _stream())
    else:
        _lib.call(f"gs_preprocess_{direction}_batched_sh", B, *body, cam.data_ptr(), W, H, *tail, _stream())


class _PreprocessRaw(torch.autograd.Function):
    """preprocess_gaussians' outputs for B views from the six RAW GaussianModel parameters
    (scene/gaussian_model.py:219-228), the activations of :109-129 inside the kernel -> (means2D (B,P,2), rgb (B,P,3),
    conic_opacity (B,P,4), radii (B,P) int32, depths (B,P)).  meta = (image_width, image_height, active sh_degree,
    scale_modifier), shared by the views; rs, cams: the views' cameras (_raw_camera).

    B > 1 is ONE batched launch over the (B,40) camera table, which reads every Gaussian once.  B = 1 launches the
    single-camera kernels instead: both give equal outputs there, and the single-camera backward is the faster one,
    0.357-0.361 ms for k_preprocess_bwd<true,16> against 0.410-0.413 ms for k_preprocess_bwd_batched<16> at c2
    (DESIGN.md section 5)."""

    @staticmethod
    def forward(ctx, xyz, f_dc, f_rest, scaling, rotation, opacity, B, rs, cams, meta):
        ctx.set_materialize_grads(False)   # undefined output gradients arrive as None, not as zero-filled tensors
        P = xyz.shape[0]
        if tuple(f_dc.shape) != (P, 1, 3) or f_rest.dim() != 3 or f_rest.shape[0] != P or f_rest.shape[2] != 3:
            raise ValueError("features must be (P,1,3) and (P,K-1,3) (scene/gaussian_model.py:219-228)")
        if tuple(xyz.shape) != (P, 3) or tuple(scaling.shape) != (P, 3) or tuple(rotation.shape) != (P, 4) \
                or opacity.numel() != P:
            raise ValueError("inconsistent Gaussian parameter shapes")
        max_deg = _stored_degree(f_rest.shape[1] + 1, meta[2], "_features_dc + _features_rest")
        params = [_f32c(t, name) for t, name in zip((xyz, f_dc, f_rest, scaling, rotation, opacity), RAW_ORDER)]
        cam = _raw_camera(B, rs, cams)
        means2D, depths, radii, conic_opacity, rgb, clamped = _screen_outputs((B, P), xyz.device)
        _launch_raw("forward", B, cam, P, meta, max_deg, params, means2D, depths, radii, conic_opacity, rgb, clamped)
        ctx.cam, ctx.meta, ctx.max_deg = cam, meta, max_deg
        ctx.save_for_backward(*params, radii, clamped)
        ctx.mark_non_differentiable(radii, depths)
        return means2D, rgb, conic_opacity, radii, depths

    @staticmethod
    def backward(ctx, g_means2D, g_rgb, g_conic_opacity, _g_radii, _g_depths):
        *params, radii, clamped = ctx.saved_tensors
        B, P = radii.shape
        grads = [_grad_or_zeros(g, (B, P, n), radii.device)
                 for g, n in ((g_means2D, 2), (g_conic_opacity, 4), (g_rgb, 3))]
        d = [torch.empty_like(t) for t in params]
        _launch_raw("backward", B, ctx.cam, P, ctx.meta, ctx.max_deg, params, radii, clamped, *grads, *d)
        return (*d, None, None, None, None)


def preprocess_gaussians_raw(xyz, features_dc, features_rest, scaling, rotation, opacity, raster_settings):
    """Same outputs as preprocess_gaussians, from the six RAW GaussianModel parameters
    (scene/gaussian_model.py:219-228); the activations of :109-129 run inside the kernel.  features_rest (P,K-1,3),
    (P,0,3) for a model stored at degree 0.  The one-view case of preprocess_gaussians_batched, with the camera read
    from raster_settings."""
    rs = raster_settings
    out = _PreprocessRaw.apply(xyz, features_dc, features_rest, scaling, rotation, opacity, 1, rs, None,
                               (int(rs.image_width), int(rs.image_height), int(rs.sh_degree), float(rs.scale_modifier)))
    return tuple(t.squeeze(0) for t in out)


def preprocess_gaussians_batched(xyz, features_dc, features_rest, scaling, rotation, opacity, cams, image_width,
                                 image_height, sh_degree, scale_modifier=1.0):
    """All B cameras at once from the RAW GaussianModel parameters (features_rest (P,K-1,3) as in
    preprocess_gaussians_raw).  cams: pack_cameras(...) (B,40); at B = 1 its two tangents are read back to the host for
    the single-camera kernels (a sync that preprocess_gaussians_raw, given the view's settings, does not need).
    -> (means2D (B,P,2), rgb (B,P,3), conic_opacity (B,P,4), radii (B,P) int32, depths (B,P)); slice k equals the
    single-camera operator's output for camera k."""
    return _PreprocessRaw.apply(xyz, features_dc, features_rest, scaling, rotation, opacity, cams.shape[0], None, cams,
                                (int(image_width), int(image_height), int(sh_degree), float(scale_modifier)))


def deterministic_enabled(deterministic=None):
    """The operators' `deterministic` argument: None follows torch.use_deterministic_algorithms (PyTorch's switch: an op
    runs a deterministic implementation or raises), True / False force the choice for one call."""
    return torch.are_deterministic_algorithms_enabled() if deterministic is None else bool(deterministic)


def _tiles(rs):
    return (int(rs.image_height) + BLOCK_Y - 1) // BLOCK_Y, (int(rs.image_width) + BLOCK_X - 1) // BLOCK_X


def _seg_workspace(R, num_tiles, dev, needed):
    """Segment workspace linking a render forward to its backward (gs_render_seg_bytes); None for forward-only calls."""
    if not needed or R == 0:
        return None, 0
    nb = _lib.query("gs_render_seg_bytes", R, num_tiles)
    return torch.empty((nb,), dtype=torch.uint8, device=dev), nb


# Instance-count hints: the render reads its instance count R back from the device (the operator's one host sync, as in
# the reference, which sizes its buffers from num_rendered).  Behind that sync the GPU is idle until the next launch, so
# everything the launch needs is allocated BEFORE the sync from the previous call's R of the same shape (+8 %); only when
# the hint is missing or too small are the buffers allocated after the read-back.
_R_HINT = {}


class _InstanceBuffers:
    """det: also sorted_u (cap), kept with the rest until the backward has run (the deterministic backward's workspace,
    _det_workspace, follows the same capacity)."""
    __slots__ = ("cap", "tiles", "ids", "sort_temp", "sb", "seg", "segb", "sorted_u")

    def __init__(self, cap, num_tiles, dev, needs_grad, det=False):
        self.cap = _q(cap)
        self.tiles = torch.empty((2, self.cap), dtype=torch.int32, device=dev)
        self.ids = torch.empty((2, self.cap), dtype=torch.int32, device=dev)
        self.sb = _lib.query("gs_render_sort_temp_bytes", self.cap)
        self.sort_temp = torch.empty((self.sb,), dtype=torch.uint8, device=dev)
        self.seg, self.segb = _seg_workspace(self.cap, num_tiles, dev, needs_grad)
        self.sorted_u = torch.empty((self.cap,), dtype=torch.int32, device=dev) if det else None

    def row(self, t, r):
        return t.data_ptr() + 4 * self.cap * r


def _det_workspace(ib, Pq, dev):
    """Instance-gradient rows (36 B per instance), the depth rank and the long-range list (8 B per splat) of
    gs_render_backward_det, sized
    from the instance buffers' quantised capacity and the quantised splat count."""
    return torch.empty((_lib.query("gs_render_det_bytes", ib.cap, Pq),), dtype=torch.uint8, device=dev)


def _instance_buffers_before_sync(key, num_tiles, dev, needs_grad, det=False):
    est = _R_HINT.get(key)
    return None if est is None else _InstanceBuffers(est + est // 12 + 4096, num_tiles, dev, needs_grad, det)


def _instance_buffers_after_sync(key, pre, R, num_tiles, dev, needs_grad, det=False):
    _R_HINT[key] = R
    if pre is not None and R <= pre.cap and (R > 0 or pre.seg is None):
        return pre
    return _InstanceBuffers(R, num_tiles, dev, needs_grad, det)


def _q(n):
    """Buffer sizes that follow a data-dependent count (received splats, instances) are rounded up to 1/16 steps of their
    leading power of two: when the strips of a view move, the counts change a little every step, and exact sizes would
    hand the caching allocator a new size -- eventually a cudaMalloc and a device synchronisation -- every few steps."""
    n = max(int(n), 1)
    q = 1 << max(10, n.bit_length() - 5)
    return (n + q - 1) // q * q


def _grad_block(P, dev):
    """dL/dmeans2D (P,2), dL/dconic_opacity (P,4), dL/drgb (P,3) as consecutive blocks of ONE allocation: the backward
    zeroes them with one memset instead of three (it accumulates into them with RED.ADD)."""
    buf = torch.empty((9 * _q(P),), dtype=torch.float32, device=dev)   # conic first: its rows are read as float4
    return buf[4 * P:6 * P].view(P, 2), buf[:4 * P].view(P, 4), buf[6 * P:9 * P].view(P, 3)


class _RenderGaussians(torch.autograd.Function):
    """The B cameras of a batch in ONE pass (gs_render_*_batched): the splats of all cameras concatenated (camera k = rows
    [view_start[k], view_start[k+1])), masks (B,T), images (B,3,H,W).  view_start None: render_gaussians' one camera,
    view_start = [0, P], whose outputs are allocated without the view axis."""

    @staticmethod
    def forward(ctx, means2D, conic_opacity, rgb, depths, radii, compute_locally, view_start, rs, collector, want_ts, log,
                det):
        ctx.set_materialize_grads(False)   # undefined output gradients arrive as None, not as zero-filled tensors
        means2D, conic_opacity, rgb = _f32c(means2D, "means2D"), _f32c(conic_opacity, "conic_opacity"), _f32c(rgb, "rgb")
        depths = _f32c(depths, "depths")
        if radii.dtype != torch.int32:
            radii = radii.to(torch.int32)
        radii = radii.contiguous()
        single = view_start is None
        if single:
            view_start = [0, means2D.shape[0]]
        B = len(view_start) - 1
        P = int(view_start[B])
        if not 1 <= B <= MAX_VIEWS:
            raise ValueError(f"1..{MAX_VIEWS} views per batched render, got {B}")
        if means2D.shape[0] != P:
            raise ValueError(f"view_start ends at {P} but {means2D.shape[0]} splats were passed")
        H, W = int(rs.image_height), int(rs.image_width)
        ty, tx = _tiles(rs)
        T = ty * tx
        dev = means2D.device
        if compute_locally is None:
            cl = torch.ones((B * T,), dtype=torch.uint8, device=dev)
        else:
            if compute_locally.numel() != B * T:
                raise ValueError(f"compute_locally must have {B}x{ty}x{tx} entries, got {tuple(compute_locally.shape)}")
            cl = compute_locally.contiguous()
            cl = cl.view(torch.uint8) if cl.dtype == torch.bool else cl.to(torch.uint8)
        bg = _f32c(rs.bg, "bg")
        s = _stream()
        vs = _i32_array(view_start)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        Pq = _q(P)
        offsets = torch.empty((Pq,), dtype=torch.int32, device=dev)
        order = torch.empty((Pq,), dtype=torch.int32, device=dev)
        rec = torch.empty((Pq, 12), dtype=torch.float32, device=dev)
        tb = _lib.query("gs_render_count_temp_bytes", Pq)
        temp = torch.empty((tb,), dtype=torch.uint8, device=dev)
        ranges = torch.empty((B * T, 2), dtype=torch.int32, device=dev)
        lead = () if single else (B,)
        image = torch.empty((*lead, 3, H, W), dtype=torch.float32, device=dev)
        final_T = torch.empty((B, H, W), dtype=torch.float32, device=dev)
        n_contrib = torch.empty((B, H, W), dtype=torch.int32, device=dev)
        stats = torch.empty((*lead, 3), dtype=torch.int64, device=dev)
        log_tiles = log is not None and log.debug
        ts = torch.empty((*lead, ty, tx, 3), dtype=torch.int64, device=dev) if want_ts or log_tiles else None
        needs_grad = means2D.requires_grad or conic_opacity.requires_grad or rgb.requires_grad
        det = det and needs_grad    # a forward-only render is the same bits either way
        with _gpu_time(log, "render forward"):   # the count, the sort and the blend of this call (stages 24-70)
            R = C.c_int64(0)
            ticket = C.c_void_p()
            _lib.call("gs_render_count_launch", B, vs, P, H, W, means2D.data_ptr(), conic_opacity.data_ptr(),
                      rgb.data_ptr(), depths.data_ptr(), radii.data_ptr(), cl.data_ptr(), order.data_ptr(),
                      offsets.data_ptr(), rec.data_ptr(), temp.data_ptr(), tb, C.byref(ticket), s)
            # not P: the splat count of a strip varies from step to step, R follows it smoothly
            key = (B, H, W, needs_grad) if not det else (B, H, W, needs_grad, "det")
            pre = _instance_buffers_before_sync(key, B * T, dev, needs_grad, det)   # host work while the count / sort / scan run
            _lib.call("gs_render_count_read", ticket, C.byref(R), s)   # the operator's one host sync
            R = int(R.value)
            if collector is not None:   # the call's instance count, under the reference's name for it
                collector["num_rendered"] = R
            ib = _instance_buffers_after_sync(key, pre, R, B * T, dev, needs_grad, det)
            seg = ib.seg if R > 0 else None
            if det:
                _lib.call("gs_render_forward_det", B, vs, P, R, H, W, means2D.data_ptr(), radii.data_ptr(), cl.data_ptr(),
                          order.data_ptr(), offsets.data_ptr(), rec.data_ptr(), bg.data_ptr(), ib.row(ib.tiles, 0),
                          ib.row(ib.ids, 0), ib.row(ib.tiles, 1), ib.row(ib.ids, 1), ib.sorted_u.data_ptr(),
                          ib.sort_temp.data_ptr(), ib.sb, ranges.data_ptr(), image.data_ptr(), final_T.data_ptr(),
                          n_contrib.data_ptr(), stats.data_ptr(), _lib.ptr(ts), _lib.ptr(seg),
                          ib.segb if seg is not None else 0, s)
            else:
                _lib.call("gs_render_forward_batched_ts", B, vs, R, H, W, means2D.data_ptr(), radii.data_ptr(),
                          cl.data_ptr(), order.data_ptr(), offsets.data_ptr(), rec.data_ptr(), bg.data_ptr(),
                          ib.row(ib.tiles, 0), ib.row(ib.ids, 0), ib.row(ib.tiles, 1), ib.row(ib.ids, 1),
                          ib.sort_temp.data_ptr(), ib.sb, ranges.data_ptr(), image.data_ptr(), final_T.data_ptr(),
                          n_contrib.data_ptr(), stats.data_ptr(), _lib.ptr(ts), _lib.ptr(seg),
                          ib.segb if seg is not None else 0, s)
            ev1.record()
        if log_tiles:
            statlog.append(log.path("n_contrib"), statlog.n_contrib_text(
                log.iteration, log.local_rank, log.world_size, H, W, cl.cpu(), ranges.cpu(), ts.cpu()))
        _timed(collector, "forward_render_time", ev0, ev1)
        ids_sorted = ib.ids[1]    # a view: the (tile, id) scratch stays alive until the backward has run (16 B / instance)
        ctx.rs, ctx.R, ctx.P, ctx.B, ctx.collector, ctx.seg, ctx.log = rs, R, P, B, collector, seg, log
        # deterministic backward: the depth order and offsets of the count, the slots of the sort and the row workspace
        ctx.det = (order, offsets, ib.sorted_u, _det_workspace(ib, Pq, dev)) if det else None
        ctx.save_for_backward(rec, bg, cl, ranges, ids_sorted, final_T, n_contrib)
        outs = (stats[0], stats[1], stats[2]) if single else (stats,)   # n_render, n_consider, n_contrib
        if want_ts:
            outs += (ts,)
        ctx.mark_non_differentiable(*outs)
        return (image, *outs)

    @staticmethod
    def backward(ctx, g_image, *_unused):
        rec, bg, cl, ranges, ids_sorted, final_T, n_contrib = ctx.saved_tensors
        rs, R, P, B = ctx.rs, ctx.R, ctx.P, ctx.B
        H, W = int(rs.image_height), int(rs.image_width)
        dev = rec.device
        g_image = torch.zeros((B, 3, H, W), dtype=torch.float32, device=dev) if g_image is None else _f32c(g_image, "grad")
        d_means2D, d_conic, d_rgb = _grad_block(P, dev)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        seg = ctx.seg
        with _gpu_time(ctx.log, "render backward"):
            if ctx.det is not None:
                _render_backward_det(ctx.det, B, P, R, H, W, rec, bg, cl, ranges, ids_sorted, final_T, n_contrib,
                                     g_image, seg, d_means2D, d_conic, d_rgb)
            else:
                _lib.call("gs_render_backward_batched", B, P, R, H, W, rec.data_ptr(), bg.data_ptr(), cl.data_ptr(),
                          ranges.data_ptr(), ids_sorted.data_ptr(), final_T.data_ptr(), n_contrib.data_ptr(),
                          g_image.data_ptr(), _lib.ptr(seg), 0 if seg is None else seg.numel(),
                          d_means2D.data_ptr(), d_conic.data_ptr(), d_rgb.data_ptr(), _stream())
        ctx.seg = ctx.det = None
        ev1.record()
        _timed(ctx.collector, "backward_render_time", ev0, ev1)
        return d_means2D, d_conic, d_rgb, None, None, None, None, None, None, None, None, None


def _render_backward_det(det, B, P, R, H, W, rec, bg, cl, ranges, ids_sorted, final_T, n_contrib, g_image, seg, d_means2D,
                         d_conic, d_rgb):
    """gs_render_backward_det: stores per instance, sums per splat in a fixed order, writes every gradient row."""
    order, offsets, sorted_u, det_ws = det
    _lib.call("gs_render_backward_det", B, P, R, H, W, rec.data_ptr(), bg.data_ptr(), cl.data_ptr(), ranges.data_ptr(),
              ids_sorted.data_ptr(), _lib.ptr(sorted_u), order.data_ptr(), offsets.data_ptr(), final_T.data_ptr(),
              n_contrib.data_ptr(), g_image.data_ptr(), _lib.ptr(seg), 0 if seg is None else seg.numel(),
              _lib.ptr(det_ws), 0 if det_ws is None else det_ws.numel(), d_means2D.data_ptr(), d_conic.data_ptr(),
              d_rgb.data_ptr(), _stream())


def render_gaussians(means2D, conic_opacity, rgb, depths, radii, compute_locally, raster_settings, cuda_args=None,
                     extended_compute_locally=None, *, tile_stats=False, deterministic=None):
    """-> (image (3,H,W) with non-local tiles exactly 0, n_render, n_consider, n_contrib), and with tile_stats=True also
    (TILE_Y, TILE_X, 3) int64: per tile the list length, the entries walked and the entries blended summed over the tile's
    in-image pixels (gs_render_forward_ts; non-local tiles read 0).

    deterministic: None follows torch.use_deterministic_algorithms.  When on and a gradient is needed, the backward
    stores every (splat, tile) instance's gradient and sums them per splat in a fixed order (gs_render_backward_det):
    two runs give the same bits.  The forward's outputs are bit-identical either way.

    cuda_args: the reference's dict.  Its stats_collector receives the call's forward / backward render times and its
    instance count R ("num_rendered").  On a logging iteration (statlog.request) zhx_time "True" appends stages 24-83 of
    this call and b10 of its backward to the gpu_time log, and zhx_debug "True" appends this call's per-tile lines and
    summary to the n_contrib log.

    extended_compute_locally: the live path passes None (workload_division.py:802-803); the legacy render()
    (gaussian_renderer/__init__.py:458-507) passes the local tile region dilated by one tile
    (workload_division.py:142-156, 435-448).  What the fork's CUDA code did with it is not observable (its source is an
    absent submodule) and every in-tree consumer of the result requires the image to be exactly zero outside
    compute_locally (loss_distribution.py:1875), so the mask is validated -- a (TILE_Y, TILE_X) boolean mask that covers
    compute_locally -- and the blend stays confined to compute_locally."""
    if extended_compute_locally is not None:
        ty, tx = _tiles(raster_settings)
        if extended_compute_locally.numel() != ty * tx:
            raise ValueError(f"extended_compute_locally must have {ty}x{tx} entries, got {tuple(extended_compute_locally.shape)}")
        if compute_locally is not None and bool((compute_locally.reshape(-1).bool() & ~extended_compute_locally.reshape(-1).bool()).any()):
            raise ValueError("extended_compute_locally must cover compute_locally")
    collector = None
    if isinstance(cuda_args, dict):
        collector = cuda_args.setdefault("stats_collector", {})
    return _RenderGaussians.apply(means2D, conic_opacity, rgb, depths, radii, compute_locally, None, raster_settings,
                                  collector, bool(tile_stats), statlog.request(cuda_args),
                                  deterministic_enabled(deterministic))


MAX_VIEWS = 64   # GS_MAX_VIEWS


def _i32_array(vals):
    return (C.c_int32 * len(vals))(*[int(v) for v in vals])


def render_gaussians_batched(means2D, conic_opacity, rgb, depths, radii, compute_locally, view_start, raster_settings,
                             cuda_args=None, *, tile_stats=False, deterministic=None):
    """All B cameras of a batch in one pass.  means2D (N,2), conic_opacity (N,4), rgb (N,3), depths (N), radii (N):
    the splats of the B cameras concatenated, camera k = rows [view_start[k], view_start[k+1]) (len(view_start) = B+1);
    compute_locally (B, TILE_Y*TILE_X) (None = everything local); the cameras share the image size and background of
    `raster_settings` (their view / projection matrices were consumed by the preprocess).
    -> (images (B,3,H,W) with non-local tiles exactly 0, stats (B,3) int64 = n_render / n_consider / n_contrib), and
    with tile_stats=True also (B, TILE_Y, TILE_X, 3) int64: slice k is render_gaussians(..., tile_stats=True)'s for
    camera k.  cuda_args["stats_collector"] and deterministic: as in render_gaussians."""
    collector = None
    if isinstance(cuda_args, dict):
        collector = cuda_args.setdefault("stats_collector", {})
    return _RenderGaussians.apply(means2D, conic_opacity, rgb, depths, radii, compute_locally,
                                  [int(v) for v in view_start], raster_settings, collector, bool(tile_stats), None,
                                  deterministic_enabled(deterministic))


_LOSS_W = {}


class _FusedL1SSIM(torch.autograd.Function):
    """Per-strip (Ll1, ssim) of loss_distribution.py:2536-2585 for the B views of `images` (B,3,H,W) in two kernels
    instead of ~20 (gs_loss_*_batched[_gt_full][_det]).

    single: the per-camera calls, `images` is the one view's (3,H,W) image; its ground truth is checked even without
    rows, and the strip form refuses an empty window (gs_loss_forward's contract).  Without lambda_dssim the (B,2) sums
    are returned, or for a single view the two 0-dim sums.  With it, one view's (1 - lambda) Ll1 + lambda (1 - ssim) is
    ONE autograd node (train_internal.py:166-189 forms it with five elementwise kernels and as many in the backward): one
    dot product with a cached weight vector, and the backward hands (g (1 - lambda), -g lambda) to the kernel."""

    @staticmethod
    def forward(ctx, images, gts, rows4, det, gt_full, single, lambda_dssim):
        ctx.set_materialize_grads(False)   # undefined output gradients arrive as None, not as zero-filled tensors
        images = _f32c(images, "images")
        B, _, H, W = (1, *images.shape) if single else images.shape
        if len(gts) != B or len(rows4) != B:
            raise ValueError("one ground-truth strip and one (row0,row1,count_row0,count_row1) per view")
        what = "images (3, H, W)" if gt_full else "strips (3, rows, W)"
        keep = []
        for k, (gt, r) in enumerate(zip(gts, rows4)):
            rows = int(r[1]) - int(r[0])
            if rows == 0 and not single:
                keep.append(None)
                continue
            if gt is None or gt.dtype != torch.uint8 or not gt.is_cuda:
                raise TypeError(f"gt {what} must be CUDA uint8 tensors")
            gt = gt.contiguous()
            want = (3, H, W) if gt_full else (3, rows, W)
            if tuple(gt.shape) != want:
                raise ValueError(f"gt {k} must be {want}, got {tuple(gt.shape)}")
            if rows == 0 and not gt_full:   # a single view's strip form: gs_loss_forward refuses an empty strip
                raise _lib.GsError(f"a strip needs rows: [{r[0]}, {r[1]}) is empty")
            keep.append(gt)
        ctx.w = None
        if lambda_dssim is not None:
            key = (images.device, lambda_dssim)
            if key not in _LOSS_W:
                _LOSS_W[key] = torch.tensor([1.0 - lambda_dssim, -lambda_dssim], dtype=torch.float32, device=images.device)
            ctx.w = _LOSS_W[key]
        flat = _i32_array([int(v) for r in rows4 for v in r])
        gptr = (C.c_void_p * B)(*[None if g is None else g.data_ptr() for g in keep])
        sfx = "_det" if det else ""
        tb = _lib.query("gs_loss_temp_bytes_batched" + sfx, B, flat, W)
        temp = torch.empty((tb,), dtype=torch.uint8, device=images.device)
        out = torch.empty((2,) if single else (B, 2), dtype=torch.float32, device=images.device)
        full = "_gt_full" if gt_full else ""
        _lib.call("gs_loss_forward_batched" + full + sfx, B, H, W, flat, images.data_ptr(), gptr, out.data_ptr(),
                  temp.data_ptr(), tb, _stream())
        ctx.rows4, ctx.gts, ctx.full, ctx.pair = flat, keep, full, single and lambda_dssim is None
        ctx.save_for_backward(images, temp)
        if ctx.w is not None:
            return torch.dot(out, ctx.w) + lambda_dssim
        return (out[0], out[1]) if ctx.pair else out

    @staticmethod
    def backward(ctx, *g):
        images, temp = ctx.saved_tensors
        B, (H, W) = len(ctx.gts), images.shape[-2:]
        if ctx.pair:
            g_l1, g_ssim = (torch.zeros((), device=images.device) if x is None else x.to(torch.float32) for x in g)
            p_l1, p_ssim = g_l1.data_ptr(), g_ssim.data_ptr()
        elif g[0] is None:
            return None, None, None, None, None, None, None
        else:
            gw = g[0].to(torch.float32)
            if ctx.w is not None:
                gw = gw * ctx.w      # (g (1 - lambda), -g lambda)
            # the kernel reads the B Ll1 gradients and the B ssim gradients as two contiguous vectors
            if B == 1:
                p_l1 = gw.data_ptr()
                p_ssim = p_l1 + 4 * gw.stride(-1)
            else:
                gw = gw.reshape(B, 2).t().contiguous()
                p_l1, p_ssim = gw.data_ptr(), gw.data_ptr() + 4 * B
        d_images = torch.empty_like(images)
        gptr = (C.c_void_p * B)(*[None if t is None else t.data_ptr() for t in ctx.gts])
        _lib.call("gs_loss_backward_batched" + ctx.full, B, H, W, ctx.rows4, images.data_ptr(), gptr, temp.data_ptr(),
                  p_l1, p_ssim, d_images.data_ptr(), _stream())
        return d_images, None, None, None, None, None, None


def fused_l1_ssim_batched(images, gts_u8, rows4, *, deterministic=None, gt_full=False):
    """The strip losses of the B cameras of a batch in one launch.  images (B,3,H,W); gts_u8: list of B CUDA uint8
    strips (3,rows,W) (None where rows == 0); rows4: B tuples (row0, row1, count_row0, count_row1).
    -> (B,2) = (Ll1, ssim_loss) per camera, both normalised by 3*H*W; zeros for cameras without rows.
    deterministic: None follows torch.use_deterministic_algorithms; when on, the per-CTA partial sums are added in a fixed
    order (gs_loss_forward_batched_det), the same bits on every run.
    gt_full: gts_u8 are the views' whole (3,H,W) images, read in place at rows [row0, row1) (gs_loss_*_batched_gt_full):
    the same bits as passing the strips gt[:, row0:row1, :], without copying them out."""
    return _FusedL1SSIM.apply(images, list(gts_u8), [tuple(int(v) for v in r) for r in rows4],
                              deterministic_enabled(deterministic), bool(gt_full), False, None)


def eval_sums_batched(images, gts, rows, gt_row0):
    """The per-tile-row metric sums of training_report (train_internal.py:461-478) for the B views of `images` (B,3,H,W)
    fp32 (gs_eval_sums_batched).  rows: B pairs (row0, row1) of local pixel rows (row0 a multiple of 16, row1 too or H;
    row0 == row1: none); gts: B CUDA uint8 (3, R, W) ground truths holding image rows [gt_row0[v], gt_row0[v] + R), read
    in place -- a whole resident image with gt_row0 0, or a strip with gt_row0 = row0 -- (None where a view has no rows).
    -> (B, TILE_Y, 3, 2) fp64 slots: per tile row and channel (sum |clamp(x,0,1) - g/255|, sum of its square) over that
    row's pixels, +0.0 outside the local rows.  A slot does not depend on the batch, the rank or the strip boundaries, so
    summing the slots of the ranks gives the same bits as one rank.  No autograd."""
    images = _f32c(images, "images")
    if images.dim() != 4 or images.shape[1] != 3:
        raise ValueError(f"images must be (B, 3, H, W), got {tuple(images.shape)}")
    B, _, H, W = images.shape
    if not (len(gts) == len(rows) == len(gt_row0) == B):
        raise ValueError("one ground truth, one (row0, row1) and one gt_row0 per view")
    keep, g_rows = [], []
    for k, (gt, r) in enumerate(zip(gts, rows)):
        if int(r[1]) == int(r[0]) and gt is None:
            keep.append(None)
            g_rows.append(0)
            continue
        if gt is None or gt.dtype != torch.uint8 or not gt.is_cuda or gt.device != images.device:
            raise TypeError(f"gt {k} must be a uint8 tensor on {images.device}")
        gt = gt.contiguous()
        if gt.dim() != 3 or gt.shape[0] != 3 or gt.shape[2] != W:
            raise ValueError(f"gt {k} must be (3, rows, {W}), got {tuple(gt.shape)}")
        keep.append(gt)
        g_rows.append(int(gt.shape[1]))
    slots = torch.empty((B, (H + BLOCK_Y - 1) // BLOCK_Y, 3, 2), dtype=torch.float64, device=images.device)
    _lib.call("gs_eval_sums_batched", B, H, W, images.data_ptr(),
              (C.c_void_p * B)(*[None if g is None else g.data_ptr() for g in keep]), _i32_array(gt_row0),
              _i32_array(g_rows), _i32_array([r[0] for r in rows]), _i32_array([r[1] for r in rows]), slots.data_ptr(),
              _stream())
    return slots


def eval_finalize(slots, H, W):
    """(B, TILE_Y, 3, 2) fp64 slots (eval_sums_batched, summed over the ranks) -> (B, 2) fp64 (L1, PSNR) per view:
    L1 = sum of |.| / (3 H W) and PSNR = the mean over the channels of 20 log10(1 / sqrt(MSE_c)) (gs_eval_finalize)."""
    if slots.dtype != torch.float64 or not slots.is_cuda:
        raise TypeError("slots must be a CUDA float64 tensor")
    B = slots.shape[0]
    if tuple(slots.shape) != (B, (int(H) + BLOCK_Y - 1) // BLOCK_Y, 3, 2):
        raise ValueError(f"slots must be (B, TILE_Y, 3, 2) for H = {H}, got {tuple(slots.shape)}")
    slots = slots.contiguous()
    out = torch.empty((B, 2), dtype=torch.float64, device=slots.device)
    _lib.call("gs_eval_finalize", B, int(H), int(W), slots.data_ptr(), out.data_ptr(), _stream())
    return out


SSIM_HALO = 5   # rows of the 11 x 11 SSIM window on each side of a pixel


def _u8_buffer(t, k, what, channels, W, device):
    if t is None or t.dtype != torch.uint8 or not t.is_cuda or t.device != device:
        raise TypeError(f"{what} {k} must be a uint8 tensor on {device}")
    if not t.is_contiguous() or t.dim() != 3 or t.shape[0] != channels or t.shape[2] != W:
        raise ValueError(f"{what} {k} must be a contiguous ({channels}, rows, {W}) tensor, got {tuple(t.shape)}")
    return int(t.shape[1])


def quantize_u8_batched(images, rows, outs, out_row0):
    """render.py's clamp + save_image's 8-bit quantization of rows [row0, row1) of each of the B views of `images`
    (B,3,H,W) fp32, written in place into outs[v] (gs_quantize_u8_batched): a contiguous CUDA uint8 (3, R, W) buffer that
    holds image rows [out_row0[v], out_row0[v] + R) -- a window's first three channels, say (None where a view has no
    rows).  q = uint8(clamp(fl(fl(clamp(x,0,1) * 255) + 0.5), 0, 255)), truncated, with the multiply and the add rounded
    separately as torch's mul(255).add_(0.5) rounds them; a NaN render gives 0.  No autograd.  -> outs."""
    images = _f32c(images, "images")
    if images.dim() != 4 or images.shape[1] != 3:
        raise ValueError(f"images must be (B, 3, H, W), got {tuple(images.shape)}")
    B, _, H, W = images.shape
    if not (len(outs) == len(rows) == len(out_row0) == B):
        raise ValueError("one output, one (row0, row1) and one out_row0 per view")
    o_rows = [0 if (o is None and int(r[1]) == int(r[0])) else _u8_buffer(o, k, "out", 3, W, images.device)
              for k, (o, r) in enumerate(zip(outs, rows))]
    _lib.call("gs_quantize_u8_batched", B, H, W, images.data_ptr(), _i32_array([r[0] for r in rows]),
              _i32_array([r[1] for r in rows]), (C.c_void_p * B)(*[None if o is None else o.data_ptr() for o in outs]),
              _i32_array(out_row0), _i32_array(o_rows), _stream())
    return outs


def image_metric_sums_batched(windows, win_row0, rows, H):
    """The per-tile-row sums of metrics.py's SSIM and PSNR (metrics.py:26-80) for B views of height H
    (gs_image_metric_sums_batched).  rows: B pairs (row0, row1) of local pixel rows (row0 a multiple of 16, row1 too or H;
    row0 == row1: none); windows: B contiguous CUDA uint8 (6, R, W) windows holding image rows
    [win_row0[v], win_row0[v] + R) of the 8-bit render (channels 0-2, quantize_u8_batched) and of the ground truth
    (channels 3-5), covering rows [max(0, row0 - 5), min(H, row1 + 5)) (None where a view has no rows).
    -> (B, TILE_Y, 2) fp64 slots: per tile row (sum of the fp64 SSIM map, sum of (q - g)^2) over that row's pixels, +0.0
    outside the local rows.  A slot does not depend on the batch, the rank or the strip boundaries, so summing the slots of
    the ranks gives the same bits as one rank.  No autograd."""
    B = len(windows)
    if not (len(win_row0) == len(rows) == B) or not 1 <= B <= MAX_VIEWS:
        raise ValueError(f"1..{MAX_VIEWS} views, with one window, one win_row0 and one (row0, row1) each")
    live = [w for w in windows if w is not None]
    if not live:
        raise ValueError("no view has a window")
    dev, W = live[0].device, int(live[0].shape[-1])
    w_rows = [0 if (w is None and int(r[1]) == int(r[0])) else _u8_buffer(w, k, "window", 6, W, dev)
              for k, (w, r) in enumerate(zip(windows, rows))]
    slots = torch.empty((B, (int(H) + BLOCK_Y - 1) // BLOCK_Y, 2), dtype=torch.float64, device=dev)
    _lib.call("gs_image_metric_sums_batched", B, int(H), W,
              (C.c_void_p * B)(*[None if w is None else w.data_ptr() for w in windows]), _i32_array(win_row0),
              _i32_array(w_rows), _i32_array([r[0] for r in rows]), _i32_array([r[1] for r in rows]), slots.data_ptr(),
              _stream())
    return slots


def image_metric_finalize(slots, H, W):
    """(B, TILE_Y, 2) fp64 slots (image_metric_sums_batched, summed over the ranks) -> (B, 2) fp64 (SSIM, PSNR) per view:
    SSIM = the map's sum / (3 H W) and PSNR = 20 log10(1 / sqrt(S / (255^2 3 H W))), +inf for S = 0
    (gs_image_metric_finalize)."""
    if slots.dtype != torch.float64 or not slots.is_cuda:
        raise TypeError("slots must be a CUDA float64 tensor")
    B = slots.shape[0]
    if tuple(slots.shape) != (B, (int(H) + BLOCK_Y - 1) // BLOCK_Y, 2):
        raise ValueError(f"slots must be (B, TILE_Y, 2) for H = {H}, got {tuple(slots.shape)}")
    slots = slots.contiguous()
    out = torch.empty((B, 2), dtype=torch.float64, device=slots.device)
    _lib.call("gs_image_metric_finalize", B, int(H), int(W), slots.data_ptr(), out.data_ptr(), _stream())
    return out


def get_local2j_ids_bool(image_height, image_width, rank, world_size, means2D, radii, dist_global_strategy,
                         cuda_args=None):
    """(P, world_size) bool: does splat i touch rank j's flattened tile range.  `rank` is unused (kept for
    signature parity with workload_division.py:727-738)."""
    means2D = _f32c(means2D.detach(), "means2D")
    radii = radii.to(torch.int32).contiguous()
    strat = dist_global_strategy.to(device=means2D.device, dtype=torch.int32).contiguous()
    if strat.numel() != world_size + 1:
        raise ValueError("dist_global_strategy must have world_size+1 entries")
    P = means2D.shape[0]
    out = torch.empty((P, world_size), dtype=torch.bool, device=means2D.device)
    _lib.call("gs_get_local2j_ids_bool", P, int(image_height), int(image_width), int(world_size), means2D.data_ptr(),
              radii.data_ptr(), strat.data_ptr(), out.data_ptr(), _stream())
    return out


def get_local2j_ids_bool_adjust_mode6(image_height, image_width, rank, world_size, means2D, radii, rectangles,
                                      cuda_args=None):
    """Legacy variant (workload_division.py:471-484): rank j owns tile rectangle (y_l, y_r, x_l, x_r)."""
    means2D = _f32c(means2D.detach(), "means2D")
    radii = radii.to(torch.int32).contiguous()
    rects = rectangles.to(device=means2D.device, dtype=torch.int32).contiguous()
    P = means2D.shape[0]
    out = torch.empty((P, world_size), dtype=torch.bool, device=means2D.device)
    _lib.call("gs_get_local2j_ids_bool_rects", P, int(image_height), int(image_width), int(world_size),
              means2D.data_ptr(), radii.data_ptr(), rects.data_ptr(), out.data_ptr(), _stream())
    return out


def get_block_XY():
    """(BLOCK_X, BLOCK_Y, ONE_DIM_BLOCK_SIZE) as compiled into the library (arguments/__init__.py:254-257)."""
    a, b, c = C.c_int(), C.c_int(), C.c_int()
    _lib.call("gs_get_block_xy", C.byref(a), C.byref(b), C.byref(c))
    return a.value, b.value, c.value


def fused_l1_ssim(image, gt_u8, row0, row1, count_row0=None, count_row1=None, *, deterministic=None):
    """-> (Ll1, ssim_loss) 0-dim tensors, both normalised by 3*H*W of the FULL image.
    Rows [row0,row1) of `image` (and the (3,row1-row0,W) uint8 `gt_u8`) form the window the 11x11 SSIM filter sees;
    only rows [count_row0,count_row1) (default: the whole window) are summed -- pass a window widened by exchanged halo
    rows to make strip losses add up to the full-image loss (border-pixel exchange, loss_distribution.py:601-972).
    deterministic: as in fused_l1_ssim_batched."""
    c0 = int(row0) if count_row0 is None else int(count_row0)
    c1 = int(row1) if count_row1 is None else int(count_row1)
    return _FusedL1SSIM.apply(image, [gt_u8], [(int(row0), int(row1), c0, c1)], deterministic_enabled(deterministic),
                              False, True, None)


def fused_loss(image, gt_u8, row0, row1, lambda_dssim, count_row0=None, count_row1=None, *, deterministic=None,
               gt_full=False):
    """-> 0-dim loss (1 - lambda) Ll1 + lambda (1 - ssim) of the strip rows [row0, row1) (same window / count-row
    semantics as fused_l1_ssim; deterministic as in fused_l1_ssim_batched).  gt_full: gt_u8 is the whole (3,H,W) image,
    read in place (as in fused_l1_ssim_batched)."""
    c0 = int(row0) if count_row0 is None else int(count_row0)
    c1 = int(row1) if count_row1 is None else int(count_row1)
    return _FusedL1SSIM.apply(image, [gt_u8], [(int(row0), int(row1), c0, c1)], deterministic_enabled(deterministic),
                              bool(gt_full), True, float(lambda_dssim))


# ---------------------------------------------------------------------------------------------------------
# legacy tile-mask / tile-exchange helpers (SURVEY.md 8a rows L3-L4; never called by the shipped trainer)
# ---------------------------------------------------------------------------------------------------------
def _mask_u8(m):
    if not m.is_cuda:
        raise ValueError("compute_locally must be a CUDA tensor")
    m = m.contiguous()
    return m.view(torch.uint8) if m.dtype == torch.bool else m.to(torch.uint8)


def get_touched_locally(compute_locally, image_height, image_width, extension_distance):
    """(TILE_Y, TILE_X) bool: tiles within `extension_distance` tiles of a locally computed tile
    (/root/reference/gaussian_renderer/loss_distribution.py:136-141)."""
    cl = _mask_u8(compute_locally)
    ty, tx = (int(image_height) + BLOCK_Y - 1) // BLOCK_Y, (int(image_width) + BLOCK_X - 1) // BLOCK_X
    if cl.numel() != ty * tx:
        raise ValueError("compute_locally does not match the image's tile grid")
    out = torch.empty((ty, tx), dtype=torch.bool, device=cl.device)
    _lib.call("gs_get_touched_locally", ty, tx, int(extension_distance), cl.data_ptr(), out.data_ptr(), _stream())
    return out


def get_pixels_compute_locally_and_in_rect(compute_locally, image_height, image_width, min_y, max_y, min_x, max_x):
    """(max_y-min_y, max_x-min_x) bool pixel mask: is the pixel's tile computed locally (loss_distribution.py:205-213)."""
    cl = _mask_u8(compute_locally)
    out = torch.empty((int(max_y) - int(min_y), int(max_x) - int(min_x)), dtype=torch.bool, device=cl.device)
    _lib.call("gs_get_pixels_compute_locally_and_in_rect", int(image_height), int(image_width), cl.data_ptr(), int(min_y),
              int(max_y), int(min_x), int(max_x), out.data_ptr(), _stream())
    return out


def _alert_scatter_add(caller):
    """gs_image_tiles_scatter_add adds with float atomics where tile positions repeat: under
    torch.use_deterministic_algorithms it raises (or warns, with warn_only=True) through torch's own alert, as index_add_
    on CUDA does."""
    from torch._prims_common import alert_not_deterministic
    alert_not_deterministic(caller)


class _LoadImageTilesByPos(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rect, pos, H, W, pixels_rect, tiles_rect):
        ctx.set_materialize_grads(False)   # undefined output gradients arrive as None, not as zero-filled tensors
        rect = _f32c(rect, "local_image_rect")
        pos = pos.to(device=rect.device, dtype=torch.int64).contiguous().reshape(-1, 2)
        n = pos.shape[0]
        _, rh, rw = rect.shape
        tiles = torch.empty((n, 3, BLOCK_Y, BLOCK_X), dtype=torch.float32, device=rect.device)
        _lib.call("gs_image_tiles_gather", n, pos.data_ptr(), rect.data_ptr(), rh, rw, int(pixels_rect[0]),
                  int(pixels_rect[2]), int(H), int(W), tiles.data_ptr(), _stream())
        ctx.save_for_backward(pos)
        ctx.meta = (rh, rw, int(pixels_rect[0]), int(pixels_rect[2]), int(H), int(W))
        return tiles

    @staticmethod
    def backward(ctx, g):
        (pos,) = ctx.saved_tensors
        rh, rw, y0, x0, H, W = ctx.meta
        if g is None:
            return None, None, None, None, None, None
        g = _f32c(g, "grad")
        _alert_scatter_add("load_image_tiles_by_pos backward")
        out = torch.zeros((3, rh, rw), dtype=torch.float32, device=g.device)
        _lib.call("gs_image_tiles_scatter_add", pos.shape[0], pos.data_ptr(), g.data_ptr(), rh, rw, y0, x0, H, W,
                  out.data_ptr(), _stream())
        return out, None, None, None, None, None


class _MergeImageTilesByPos(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, tiles, H, W, pixels_rect, tiles_rect):
        ctx.set_materialize_grads(False)   # undefined output gradients arrive as None, not as zero-filled tensors
        _alert_scatter_add("merge_image_tiles_by_pos")
        tiles = _f32c(tiles, "tiles")
        pos = pos.to(device=tiles.device, dtype=torch.int64).contiguous().reshape(-1, 2)
        rh, rw = int(pixels_rect[1]) - int(pixels_rect[0]), int(pixels_rect[3]) - int(pixels_rect[2])
        out = torch.zeros((3, rh, rw), dtype=torch.float32, device=tiles.device)
        _lib.call("gs_image_tiles_scatter_add", pos.shape[0], pos.data_ptr(), tiles.data_ptr(), rh, rw,
                  int(pixels_rect[0]), int(pixels_rect[2]), int(H), int(W), out.data_ptr(), _stream())
        ctx.save_for_backward(pos)
        ctx.meta = (rh, rw, int(pixels_rect[0]), int(pixels_rect[2]), int(H), int(W))
        return out

    @staticmethod
    def backward(ctx, g):
        (pos,) = ctx.saved_tensors
        rh, rw, y0, x0, H, W = ctx.meta
        if g is None:
            return None, None, None, None, None, None
        g = _f32c(g, "grad")
        n = pos.shape[0]
        tiles = torch.empty((n, 3, BLOCK_Y, BLOCK_X), dtype=torch.float32, device=g.device)
        _lib.call("gs_image_tiles_gather", n, pos.data_ptr(), g.data_ptr(), rh, rw, y0, x0, H, W, tiles.data_ptr(),
                  _stream())
        return None, tiles, None, None, None, None


def load_image_tiles_by_pos(local_image_rect, all_pos_send_to_j, image_height, image_width, touched_pixels_rect,
                            touched_tiles_rect):
    """(3,h,w) local rect -> (n,3,16,16) tiles at GLOBAL tile positions (n,2); differentiable
    (/root/reference/gaussian_renderer/loss_distribution.py:168-175)."""
    return _LoadImageTilesByPos.apply(local_image_rect, all_pos_send_to_j, image_height, image_width,
                                      touched_pixels_rect, touched_tiles_rect)


def merge_image_tiles_by_pos(all_pos_recv_from_i, all_tiles_recv_from_i, image_height, image_width, touched_pixels_rect,
                             touched_tiles_rect):
    """(n,3,16,16) tiles at GLOBAL tile positions -> (3,h,w) local rect, zero elsewhere; differentiable
    (loss_distribution.py:188-195)."""
    return _MergeImageTilesByPos.apply(all_pos_recv_from_i, all_tiles_recv_from_i, image_height, image_width,
                                       touched_pixels_rect, touched_tiles_rect)


# ---------------------------------------------------------------------------------------------------------
# the camera table of preprocess_gaussians_batched
# ---------------------------------------------------------------------------------------------------------
def pack_cameras(settings_list):
    """(B,40) float32 device tensor: viewmatrix[16], projmatrix[16], campos[3], tanfovx, tanfovy, 3 pad per camera."""
    rows = []
    for rs in settings_list:
        dev = rs.viewmatrix.device
        tail = torch.tensor([float(rs.tanfovx), float(rs.tanfovy), 0.0, 0.0, 0.0], dtype=torch.float32, device=dev)
        rows.append(torch.cat([rs.viewmatrix.reshape(-1).float(), rs.projmatrix.reshape(-1).float(),
                               rs.campos.reshape(-1).float(), tail]))
    return torch.stack(rows).contiguous()
