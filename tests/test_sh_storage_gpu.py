"""-m gpu: models that store fewer SH coefficients (--sh_degree D_max = 0, 1, 2 in the reference: K = (D_max+1)^2
coefficients per Gaussian, scene/gaussian_model.py:51-53, 150-156) against the degree-3 path on the same inputs with the
coefficients zero-padded to 16.

The K = 16 kernels multiply every coefficient beyond the active degree by a zero basis value, so the padding adds +0 to
every colour sum, and its gradients are exactly 0 (Adam then leaves the padded coefficients at 0).  A K-coefficient
kernel does the same fp32 operations minus those terms, so its outputs must equal the padded call's BIT FOR BIT: the
six _sh preprocess entry points (outputs NaN-filled, a NaN guard after every SH gradient), the operators, and the sparse
gradient rows of 11 + 3 K floats.  A short training run with densification matches the padded run up to the blend
backward's atomic-order noise (see test_training_run_equals_the_padded_run).  The degree-3 path itself is pinned to the
CPU oracle by test_projection_gpu.py and test_gpu_parity.py.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import gpu_util as gu
import proj_cases as pc
from gs_b200 import _lib, densify, ops, pipeline
from gs_b200.optim import FusedAdam

pytestmark = pytest.mark.gpu

W, H = 197, 131
SIZES = (1, 129, 20011)         # ragged tails of 1, 1 and 43 splats: not a multiple of 4 (no TMA at K = 1 and 9)
GUARD = 256


def _K(D):
    return (D + 1) ** 2


def bits_equal(a, b):
    """Bit-identical tensors (fp32 compared as int32, so -0 != +0 and NaN patterns count)."""
    if a.shape != b.shape:
        return False
    if a.dtype == torch.float32:
        a, b = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    return torch.equal(a, b)


class Guarded:
    """NaN-filled fp32 output of `shape` followed by GUARD NaNs that the kernel must not touch."""

    def __init__(self, *shape):
        n = int(np.prod(shape))
        self.buf = torch.full((n + GUARD,), float("nan"), device=gu.DEV)
        self.t = self.buf[:n].view(shape)

    def intact(self):
        return bool(torch.isnan(self.buf[-GUARD:]).all())


def _screen(lead):
    return dict(means2D=gu.nan(*lead, 2), depths=gu.nan(*lead),
                radii=torch.full(lead, -7, dtype=torch.int32, device=gu.DEV), conic_opacity=gu.nan(*lead, 4),
                rgb=gu.nan(*lead, 3), clamped=torch.full(lead, 0xAB, dtype=torch.uint8, device=gu.DEV))


def _scr_ptrs(o):
    return [o[k].data_ptr() for k in ("means2D", "depths", "radii", "conic_opacity", "rgb", "clamped")]


def _assert_screen_equal(got, ref, what):
    for k in ref:
        assert bits_equal(got[k], ref[k]), (what, k)


def _scene(D_max, D, P, seed):
    cam = pc.golden_camera(seed % pc.N_GOLDEN, W, H, sh_degree=D)
    sc, _ = pc.region_scene(cam, P, seed=seed)
    K = _K(D_max)
    padded = dict(sc, shs=sc["shs"].copy())
    padded["shs"][:, K:] = 0.0
    stored = dict(sc, shs=np.ascontiguousarray(padded["shs"][:, :K]))
    return cam, stored, padded


def _raw_stored(raw16, K):
    """The raw parameters of a K-coefficient model: _features_rest (P,K-1,3) (an empty (P,0,3) tensor at K = 1)."""
    rest = raw16[2][:, :K - 1].contiguous() if K > 1 else torch.empty((raw16[0].shape[0], 0, 3), device=gu.DEV)
    return [raw16[0], raw16[1], rest, raw16[3], raw16[4], raw16[5]]


def _grads(P, lead, seed):
    rng = np.random.default_rng(seed)
    return [gu.to_dev(rng.normal(size=(*lead, s)).astype(np.float32)) for s in (2, 4, 3)]


@pytest.mark.parametrize("P", SIZES)
@pytest.mark.parametrize("D_max", range(4))
def test_plain_and_raw_entry_points_equal_the_padded_call(D_max, P):
    """gs_preprocess_{forward,backward}_sh and _raw_sh with K stored coefficients, every active degree <= D_max, the posed
    cameras and region scenes of proj_cases: every output == the degree-3 entry point on the zero-padded coefficients, bit
    for bit; dL/dSH == its first K coefficients, nothing written past them.  At D_max = 3 this compares the new entry
    points with the old ones on the same data."""
    K = _K(D_max)
    for D in range(D_max + 1):
        seed = 97 * D_max + 13 * D + P
        cam, stored, padded = _scene(D_max, D, P, seed)
        c = gu.cam_dev(cam)
        sm = 0.6 + 0.1 * D
        # ---- plain forward / backward ----
        ref, d16, _ = gu.preprocess_forward(padded, cam, sm)
        dK = {k: gu.to_dev(v, torch.float32) for k, v in stored.items()}
        got = _screen((P,))
        _lib.call("gs_preprocess_forward_sh", P, D, D_max, dK["means3D"].data_ptr(), dK["scales"].data_ptr(), sm,
                  dK["rotations"].data_ptr(), dK["opacities"].data_ptr(), dK["shs"].data_ptr(), c["V"].data_ptr(),
                  c["PM"].data_ptr(), c["cp"].data_ptr(), W, H, float(cam["tanfovx"]), float(cam["tanfovy"]),
                  *_scr_ptrs(got), gu.stream())
        torch.cuda.synchronize()
        _assert_screen_equal(got, ref, ("plain forward", D_max, D))
        assert int((ref["radii"] > 0).sum()) > 0 or P == 1
        gm, gc, gr = _grads(P, (P,), seed + 1)
        rb = gu.preprocess_backward(d16, c, cam, ref, gm, gc, gr, sm)
        out = dict(means3D=gu.nan(P, 3), scales=gu.nan(P, 3), rotations=gu.nan(P, 4), opacities=gu.nan(P, 1))
        dsh = Guarded(P, K, 3)
        _lib.call("gs_preprocess_backward_sh", P, D, D_max, dK["means3D"].data_ptr(), dK["scales"].data_ptr(), sm,
                  dK["rotations"].data_ptr(), dK["shs"].data_ptr(), c["V"].data_ptr(), c["PM"].data_ptr(),
                  c["cp"].data_ptr(), W, H, float(cam["tanfovx"]), float(cam["tanfovy"]), got["radii"].data_ptr(),
                  got["clamped"].data_ptr(), gm.data_ptr(), gc.data_ptr(), gr.data_ptr(), out["means3D"].data_ptr(),
                  out["scales"].data_ptr(), out["rotations"].data_ptr(), out["opacities"].data_ptr(), dsh.t.data_ptr(),
                  gu.stream())
        torch.cuda.synchronize()
        for k in out:
            assert bits_equal(out[k], rb[k]), ("plain backward", D_max, D, k)
        assert bits_equal(dsh.t, rb["shs"][:, :K]) and dsh.intact(), ("plain dL/dSH", D_max, D)
        assert bool((rb["shs"][:, K:] == 0).all())
        # ---- _raw forward / backward ----
        raw16 = gu.raw_parameters(padded)
        rawK = _raw_stored(raw16, K)
        refr = gu.preprocess_forward_raw(raw16, cam, sm)
        gotr = _screen((P,))
        _lib.call("gs_preprocess_forward_raw_sh", P, D, D_max, *(t.data_ptr() for t in rawK[:4]), sm,
                  rawK[4].data_ptr(), rawK[5].data_ptr(), c["V"].data_ptr(), c["PM"].data_ptr(), c["cp"].data_ptr(),
                  W, H, float(cam["tanfovx"]), float(cam["tanfovy"]), *_scr_ptrs(gotr), gu.stream())
        torch.cuda.synchronize()
        _assert_screen_equal(gotr, refr, ("raw forward", D_max, D))
        rbr = gu.preprocess_backward_raw(raw16, cam, refr, gm, gc, gr, sm)
        outr = [Guarded(*t.shape) for t in rawK]
        _lib.call("gs_preprocess_backward_raw_sh", P, D, D_max, *(t.data_ptr() for t in rawK[:4]), sm,
                  rawK[4].data_ptr(), rawK[5].data_ptr(), c["V"].data_ptr(), c["PM"].data_ptr(), c["cp"].data_ptr(),
                  W, H, float(cam["tanfovx"]), float(cam["tanfovy"]), gotr["radii"].data_ptr(),
                  gotr["clamped"].data_ptr(), gm.data_ptr(), gc.data_ptr(), gr.data_ptr(),
                  *(o.t.data_ptr() for o in outr), gu.stream())
        torch.cuda.synchronize()
        for q in (0, 1, 3, 4, 5):
            assert bits_equal(outr[q].t, rbr[q]) and outr[q].intact(), ("raw backward", D_max, D, q)
        assert bits_equal(outr[2].t, rbr[2][:, :K - 1]) and outr[2].intact(), ("raw dL/drest", D_max, D)
        assert bool((rbr[2][:, K - 1:] == 0).all())


@pytest.mark.parametrize("B", [1, 6, 64])
@pytest.mark.parametrize("D_max", range(4))
def test_batched_entry_points_equal_the_padded_call(D_max, B):
    """gs_preprocess_{forward,backward}_batched_sh over B posed cameras (the six of cameras.npz, repeated): == the
    degree-3 batched call on the padded coefficients, bit for bit, for every active degree and P in SIZES."""
    K = _K(D_max)
    for P in SIZES:
        for D in range(D_max + 1):
            seed = 31 * D_max + 7 * D + P + B
            cam, stored, padded = _scene(D_max, D, P, seed)
            cams = [pc.golden_camera(k % pc.N_GOLDEN, W, H, sh_degree=D) for k in range(B)]
            packed = ops.pack_cameras([pipeline.DeviceCamera(cc, gu.DEV).settings(D) for cc in cams])
            raw16 = gu.raw_parameters(padded)
            rawK = _raw_stored(raw16, K)
            ref, got = _screen((B, P)), _screen((B, P))
            for name, raw, o, extra in (("gs_preprocess_forward_batched", raw16, ref, ()),
                                        ("gs_preprocess_forward_batched_sh", rawK, got, (D_max,))):
                _lib.call(name, B, P, D, *extra, *(t.data_ptr() for t in raw[:4]), 1.0, raw[4].data_ptr(),
                          raw[5].data_ptr(), packed.data_ptr(), W, H, *_scr_ptrs(o), gu.stream())
            torch.cuda.synchronize()
            _assert_screen_equal(got, ref, ("batched forward", D_max, D, P))
            gm, gc, gr = _grads(P, (B, P), seed + 1)
            rb = [gu.nan(*t.shape) for t in raw16]
            gb = [Guarded(*t.shape) for t in rawK]
            for name, raw, o, extra, fwd in (("gs_preprocess_backward_batched", raw16, rb, (), ref),
                                             ("gs_preprocess_backward_batched_sh", rawK, [g.t for g in gb], (D_max,), got)):
                _lib.call(name, B, P, D, *extra, *(t.data_ptr() for t in raw[:4]), 1.0, raw[4].data_ptr(),
                          raw[5].data_ptr(), packed.data_ptr(), W, H, fwd["radii"].data_ptr(), fwd["clamped"].data_ptr(),
                          gm.data_ptr(), gc.data_ptr(), gr.data_ptr(), *(t.data_ptr() for t in o), gu.stream())
            torch.cuda.synchronize()
            for q in (0, 1, 3, 4, 5):
                assert bits_equal(gb[q].t, rb[q]) and gb[q].intact(), ("batched backward", D_max, D, P, q)
            assert bits_equal(gb[2].t, rb[2][:, :K - 1]) and gb[2].intact(), ("batched dL/drest", D_max, D, P)
            assert bool((rb[2][:, K - 1:] == 0).all())


def test_operators_take_the_stored_coefficients():
    """preprocess_gaussians (and the drop-in GaussianRasterizer), _raw and _batched accept K in {1, 4, 9, 16} stored
    coefficients, return gradients in the input's shape equal to the padded call's, and raise ValueError before any launch
    for any other K and for an active degree above the stored one."""
    import diff_gaussian_rasterization as dgr
    P = 3001
    for D_max in range(4):
        K = _K(D_max)
        D = D_max
        cam, stored, padded = _scene(D_max, D, P, 11 + D_max)
        dcam = pipeline.DeviceCamera(cam, gu.DEV)
        rs = dcam.settings(D)
        res = {}
        for tag, sc in (("K", stored), ("16", padded)):
            t = {k: gu.to_dev(v, torch.float32).requires_grad_(True) for k, v in sc.items()}
            r = dgr.GaussianRasterizer(raster_settings=rs)
            m2, rgb, co, radii, depths = r.preprocess_gaussians(t["means3D"], t["scales"], t["rotations"], t["shs"],
                                                                t["opacities"], {})
            (m2.sum() + (rgb * rgb).sum() + co.sum()).backward()
            res[tag] = (m2, rgb, co, radii, depths, t)
        for a, b in zip(res["K"][:5], res["16"][:5]):
            assert bits_equal(a.detach(), b.detach())
        tK, t16 = res["K"][5], res["16"][5]
        assert tuple(tK["shs"].grad.shape) == (P, K, 3)
        assert bits_equal(tK["shs"].grad, t16["shs"].grad[:, :K])
        for k in ("means3D", "scales", "rotations", "opacities"):
            assert bits_equal(tK[k].grad, t16[k].grad), k
        # raw and batched operators: gradients of _features_rest in its own shape
        raw16 = [t.clone().requires_grad_(True) for t in gu.raw_parameters(padded)]
        rawK = [t.clone().requires_grad_(True) for t in _raw_stored([t.detach() for t in raw16], K)]
        packed = ops.pack_cameras([rs, pipeline.DeviceCamera(pc.golden_camera(2, W, H), gu.DEV).settings(D)])
        for raw in (raw16, rawK):
            o1 = ops.preprocess_gaussians_raw(*raw, rs)
            o2 = ops.preprocess_gaussians_batched(*raw, packed, W, H, D)
            (o1[0].sum() + o1[1].sum() + o2[0].sum() + (o2[1] * o2[1]).sum() + o2[2].sum()).backward()
        assert tuple(rawK[2].grad.shape) == (P, K - 1, 3)
        assert bits_equal(rawK[2].grad, raw16[2].grad[:, :K - 1])
        for q in (0, 1, 3, 4, 5):
            assert bits_equal(rawK[q].grad, raw16[q].grad), q
        # refused before a launch: an active degree above the stored one, and any other coefficient count
        if D_max < 3:
            hi = dcam.settings(D_max + 1)
            x = {k: gu.to_dev(v, torch.float32) for k, v in stored.items()}
            with pytest.raises(ValueError):
                ops.preprocess_gaussians(x["means3D"], x["scales"], x["rotations"], x["shs"], x["opacities"], hi)
            with pytest.raises(ValueError):
                ops.preprocess_gaussians_raw(*[t.detach() for t in rawK], hi)
            with pytest.raises(ValueError):
                ops.preprocess_gaussians_batched(*[t.detach() for t in rawK], packed, W, H, D_max + 1)
    x = {k: gu.to_dev(v, torch.float32) for k, v in padded.items()}
    raw = gu.raw_parameters(padded)
    for bad in (0, 2, 5, 15, 17):            # K = bad coefficients in the plain form, bad + 1 in the split forms
        with pytest.raises(ValueError):
            ops.preprocess_gaussians(x["means3D"], x["scales"], x["rotations"], torch.zeros((P, bad, 3), device=gu.DEV),
                                     x["opacities"], pipeline.DeviceCamera(cam, gu.DEV).settings(0))
        rest = torch.zeros((P, bad - 1 if bad else 1, 3), device=gu.DEV)
        with pytest.raises(ValueError):
            ops.preprocess_gaussians_raw(raw[0], raw[1], rest, raw[3], raw[4], raw[5],
                                         pipeline.DeviceCamera(cam, gu.DEV).settings(0))
    with pytest.raises(ValueError):
        ops.preprocess_gaussians_raw(*raw, pipeline.DeviceCamera(cam, gu.DEV).settings(4))


@pytest.mark.parametrize("D_max", range(4))
def test_batched_one_view_equals_the_single_camera_operator(D_max):
    """preprocess_gaussians_batched over a one-view table == preprocess_gaussians_raw with that camera's settings, bit for
    bit (-0 and +0 told apart): the five outputs and the six parameter gradients, for a model storing K = 1, 4, 9 or 16
    coefficients.  Both run the single-camera kernels at B = 1."""
    K, P, mod = _K(D_max), SIZES[-1], 0.8
    cam, _, padded = _scene(D_max, D_max, P, 5 + D_max)
    rs = pipeline.DeviceCamera(cam, gu.DEV).settings(D_max)
    rs.scale_modifier = mod
    gm, gc, gr = _grads(P, (P,), 6 + D_max)
    res = []
    for batched in (True, False):
        raw = [t.clone().requires_grad_(True) for t in _raw_stored(gu.raw_parameters(padded), K)]
        if batched:
            out = [t[0] for t in ops.preprocess_gaussians_batched(*raw, ops.pack_cameras([rs]), W, H, D_max, mod)]
        else:
            out = ops.preprocess_gaussians_raw(*raw, rs)
        ((out[0] * gm).sum() + (out[2] * gc).sum() + (out[1] * gr).sum()).backward()
        res.append(([t.detach() for t in out], [t.grad for t in raw]))
    assert int((res[1][0][3] > 0).sum()) > 1000
    for q, (a, b) in enumerate(zip(res[0][0] + res[0][1], res[1][0] + res[1][1])):
        assert bits_equal(a, b), (D_max, q)


# ---------------------------------------------------------------------------------------------------------------------
# a short training run: Trainer.step + FusedAdam, the active degree raised along the way, one densify_and_prune
# ---------------------------------------------------------------------------------------------------------------------
TW, TH = 256, 192
SCHEDULE = (0, 0, 1, 2, 3, 3)          # active degree per step (capped at the stored degree)
DENSIFY_AFTER = 3


def _training_run(sc, D_max, one_view, noise, top, shared=None):
    cams = [pc.golden_camera(5, TW, TH, uid=0), pc.golden_camera(4, TW, TH, uid=1)]
    gts = [torch.from_numpy(pc.syn.make_gt_image(TW, TH, seed=5 + k)).pin_memory() for k in range(2)]
    tr = pipeline.Trainer(sc, cams, gts, torch.device("cuda", 0), max_sh_degree=D_max)
    opt = FusedAdam(tr.optimizer_groups(), lr=0.0, eps=1e-15)
    losses, counts = [], None
    for it, deg in enumerate(SCHEDULE):
        tr.params.active_sh_degree = min(deg, top)
        losses.append(tr.step(views=[it % 2] if one_view else None, resident=False))
        opt.step(grad_scale=1.0 if one_view else 0.5)
        if it == DENSIFY_AFTER:
            p = tr.params
            if shared is None:     # the statistics and thresholds of the first run, handed to the second
                accum = p._xyz.grad.norm(dim=1, keepdim=True)
                extent = float(torch.exp(p._scaling).max(dim=1).values.median()) / 0.01
                shared = (accum, float(torch.quantile(accum, 0.8)), extent)
            accum, max_grad, extent = shared
            res = densify.densify_and_prune(opt, accum, torch.ones_like(accum), max_grad, 0.005, extent, 0.01, 0,
                                            noise=noise)
            tr.adopt_parameters(res)
            counts = res["counts"]
    state = {}
    for g in opt.param_groups:
        prm = g["params"][0]
        st = opt.state[prm]
        state[g["name"]] = (prm.detach(), st["exp_avg"], st["exp_avg_sq"])
    return losses, counts, state, shared


@pytest.mark.parametrize("one_view", [False, True], ids=["fused_batched", "one_view"])
@pytest.mark.parametrize("D_max", [0, 1, 2])
def test_training_run_equals_the_padded_run(D_max, one_view):
    """Six Trainer.steps over two posed cameras with FusedAdam, the active degree raised 0 -> D_max, one
    densify_and_prune (clones and splits, the same noise and statistics) after the fourth, the K-coefficient model against
    the padded degree-3 model.  The first step's loss is bit-identical (preprocess, binning, blend and loss forward are
    deterministic); from the first backward on, the blend backward's atomic adds reach the same sums in a varying order
    (test_gpu_parity.test_block_cull_is_invisible), so two runs of even the same model differ in the last bits: the
    later losses agree to 1e-5 relative, parameters and moments under test_gpu_parity's bar (1e-4 relative + 1e-4 x
    RMS, all but 1e-3 of the entries), densify counts exactly.  The padded coefficients and their moments stay exactly 0.
    one_view: each step trains one of the two views (the per-camera preprocess) instead of both in one batch."""
    K = _K(D_max)
    cam = pc.golden_camera(5, TW, TH)
    sc, _ = pc.region_scene(cam, 30000, seed=77 + D_max, mix=pc.MILD)
    padded = dict(sc, shs=sc["shs"].copy())
    padded["shs"][:, K:] = 0.0
    stored = dict(padded, shs=np.ascontiguousarray(padded["shs"][:, :K]))
    noise = torch.randn((2 * 30000, 3), generator=torch.Generator().manual_seed(D_max)).to(gu.DEV)
    lK, cK, sK, shared = _training_run(stored, D_max, one_view, noise, D_max)
    l16, c16, s16, _ = _training_run(padded, 3, one_view, noise, D_max, shared)
    same = all(bits_equal(sK[n][q], s16[n][q][:, :K - 1] if n == "f_rest" else s16[n][q]) for n in sK for q in range(3))
    print(f"[sh-storage] D_max {D_max} one_view={one_view}: losses {lK} vs padded {l16}; densify counts {cK}; parameters and "
          f"moments bit-identical: {same}")
    assert lK[0] == l16[0]
    np.testing.assert_allclose(lK, l16, rtol=1e-5, atol=0)
    assert cK == c16 and cK[1] > 0 and cK[3] > 0            # clones and splits both happened
    for name in sK:
        for q in range(3):
            a, b = sK[name][q], s16[name][q]
            if name == "f_rest":
                assert tuple(a.shape[1:]) == (K - 1, 3)
                assert bool((b[:, K - 1:] == 0).all()), (name, q)
                b = b[:, :K - 1]
            assert a.shape == b.shape, (name, q)
            frac, _ = gu.rel_report(f"sh-storage.D{D_max}.{name}.{q}", gu.npy(a), gu.npy(b))
            assert frac <= 1e-3, (name, q)


# ---------------------------------------------------------------------------------------------------------------------
# sparse gradient rows of 11 + 3 K floats
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rest", [0, 9, 24, 45])
@pytest.mark.parametrize("R", [2, 3])
def test_sparse_grad_rows_simulated(R, rest):
    """R replicas in one process: mask -> OR -> scan -> gs_sparse_grad_pack_rows -> rows summed in rank order ->
    gs_sparse_grad_unpack_rows.  Rows of 14 + rest = 11 + 3 K floats hold the touched gradients; touched rows end up with the sum
    (what dense synchronisation gives them), untouched rows keep their own gradient.  At rest = 0 the rest gradient is an
    empty tensor (possibly a NULL pointer); at rest = 45 the _rows entry points equal gs_sparse_grad_pack / _unpack."""
    P = 4099
    widths = (3, 3, rest, 3, 4, 1)
    rng = np.random.default_rng(R * 1000 + rest)
    s = gu.stream()
    grads, mask = [], np.zeros(P, np.uint8)
    for r in range(R):
        touched = rng.random(P) < 0.1
        g = [rng.integers(-64, 64, size=(P, w)).astype(np.float32) / 8 for w in widths]   # exact sums in any order
        g[0][~touched] = 0.0
        grads.append([gu.to_dev(a) for a in g])
        m = torch.empty((P,), dtype=torch.uint8, device=gu.DEV)
        _lib.call("gs_sparse_grad_mask", P, grads[r][0].data_ptr(), m.data_ptr(), s)
        mask |= gu.npy(m)
    orig = [[t.clone() for t in g] for g in grads]
    mask_d = gu.to_dev(mask)
    pos = torch.empty((P,), dtype=torch.int32, device=gu.DEV)
    colstart = torch.empty((2,), dtype=torch.int32, device=gu.DEV)
    tb = _lib.query("gs_route_scan_temp_bytes", P, 1)
    temp = torch.empty((tb,), dtype=torch.uint8, device=gu.DEV)
    _lib.call("gs_route_scan", P, 1, mask_d.data_ptr(), pos.data_ptr(), colstart.data_ptr(), temp.data_ptr(), tb, s)
    n = int(gu.npy(colstart)[1])
    idx = torch.from_numpy(np.nonzero(mask)[0]).to(gu.DEV)
    ROW = 14 + rest
    total = torch.zeros((n, ROW), device=gu.DEV)
    for r in range(R):
        rows = Guarded(n, ROW)
        ptrs = (C.c_void_p * 6)(*[t.data_ptr() for t in grads[r]])
        _lib.call("gs_sparse_grad_pack_rows", P, rest, mask_d.data_ptr(), pos.data_ptr(), ptrs, rows.t.data_ptr(), s)
        torch.cuda.synchronize()
        exp = torch.cat([t[idx].reshape(n, w) for t, w in zip(grads[r], widths)], 1)
        bad = rows.t != exp
        assert bits_equal(rows.t, exp), (r, n, int(bad.sum()), torch.nonzero(bad)[:4].tolist(),
                                         rows.t[bad][:4].tolist(), exp[bad][:4].tolist())
        assert rows.intact(), r
        if rest == 45:
            old = torch.empty((n, 59), device=gu.DEV)
            _lib.call("gs_sparse_grad_pack", P, mask_d.data_ptr(), pos.data_ptr(), ptrs, old.data_ptr(), s)
            assert bits_equal(old, rows.t)
        total += rows.t
    for r in range(R):
        ptrs = (C.c_void_p * 6)(*[t.data_ptr() for t in grads[r]])
        _lib.call("gs_sparse_grad_unpack_rows", P, rest, mask_d.data_ptr(), pos.data_ptr(), total.data_ptr(), ptrs, s)
        torch.cuda.synchronize()
        for q in range(6):
            dense = sum(orig[rr][q] for rr in range(R))
            exp = orig[r][q].clone()
            exp[idx] = dense[idx]
            assert bits_equal(grads[r][q], exp), (r, q)


def _grad_sync_worker(rank, world, port, D, q):
    try:
        _grad_sync_check(rank, world, port, D, q)
    except Exception as e:      # reported, so that the parent does not wait for a result that never comes
        q.put((rank, False, repr(e)))
        raise


def _grad_sync_check(rank, world, port, D, q):
    import torch.distributed as dist
    from gs_b200 import grad_sync
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    P = 2003
    g = torch.Generator().manual_seed(40 + rank)
    shapes = [(3,), (1, 3), (_K(D) - 1, 3), (3,), (4,), (1,)]
    ok = True
    grads = [torch.randint(-64, 64, (P,) + s, generator=g).float() / 8 for s in shapes]   # exact sums in any order
    grads[0][torch.rand((P,), generator=g) < 0.7] = 0.0
    a = [torch.zeros((P,) + s, device="cuda:0", requires_grad=True) for s in shapes]
    b = [torch.zeros((P,) + s, device="cuda:0", requires_grad=True) for s in shapes]
    for x, y, t in zip(a, b, grads):
        x.grad, y.grad = t.to("cuda:0"), t.to("cuda:0")
    n = grad_sync.sync_gradients_fused_sparse(a)
    grad_sync.sync_gradients_densely(b)
    touched = b[0].grad.ne(0).any(dim=1)
    ok = ok and n == int(touched.sum())
    for x, y, t in zip(a, b, grads):
        exp = t.to("cuda:0").clone()
        exp[touched] = y.grad[touched]
        ok = ok and bits_equal(x.grad, exp)
    q.put((rank, bool(ok), n))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("D", [0, 1])
@pytest.mark.parametrize("world", [2, 3])
def test_fused_sparse_sync_over_gloo(world, D):
    """grad_sync.sync_gradients_fused_sparse over a real gloo group of 2 / 3 processes for a model stored at degree 0 or 1
    (rows of 14 and 23 floats): touched Gaussians get the sum dense synchronisation gives them, the others keep their own
    gradient (gaussian_model.py:1350-1391)."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29850 + 10 * D + world
    procs = [ctx.Process(target=_grad_sync_worker, args=(r, world, port, D, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok, _ in res), res
    assert len({n for *_, n in res}) == 1 and res[0][2] > 0
