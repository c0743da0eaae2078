"""Populations built to order for the densification tests: Gaussians placed exactly at, and one representable step
either side of, every threshold the step decides on.

Every decision of densify_and_prune compares an fp32 value with an fp32 threshold:
  * grad = accum / denom against fl32(max_grad) (clone: |grad|, split: grad; NaN -> 0, x / 0 -> +-inf);
  * the largest scale exp(log-scale) against dense_thr = fl32(percent_dense * extent) (clone <=, split >);
  * the largest scale against big_thr = fl32(0.1 * extent) (world-size prune, only with a screen-size limit), for an
    original and for a split child, whose scale is exp(log(exp(log-scale) / 1.6));
  * sigmoid(logit) against fl32(min_opacity).
A raw parameter reaches only the values exp / sigmoid produce from fp32 inputs -- near 0.05 consecutive log-scales are
about three fp32 steps apart after exp -- so the values are found by searching raw log-scales and logits on the
device, with torch.exp / torch.sigmoid, the libdevice functions the kernel calls, for the target bits.  The thresholds
themselves are then moved onto those values (and one ulp either side) through extent and min_opacity.

A case is a dict: the raw state (numpy; six parameters, their Adam moments for the groups that have optimizer state,
send_to_gpui_cnt, xyz_gradient_accum, denom), noise (2 P, 3), the scalars, `label` (per Gaussian; "" for background
rows) and the family.  `near` counts the near-threshold Gaussians; the builder refuses a case whose family it could not
populate.
"""
import numpy as np
import torch

F = np.float32
NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
SHAPES = {"xyz": (3,), "f_dc": (1, 3), "f_rest": (15, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}
MAX_GRAD, MIN_OPACITY, PD = 2e-4, 0.005, 0.01


def ulp_step(v, direction):
    return np.nextafter(F(v), F(np.inf) if direction > 0 else F(-np.inf))


def preimages(fn, targets, r0, slope, dev, k=96):
    """Raw fp32 inputs r near r0 (float64 estimates, one per target) with fn(r) == target, just below and just above.
    fn: torch elementwise function evaluated on `dev`; slope: |d fn / dr| at r0.  The grid steps r by about half an
    output ulp, so every fp32 input in the window is visited.  -> (at, below, above) fp32 arrays of raw inputs; `at` is
    NaN where no input maps exactly onto the target; fn(below) is the largest output < target, fn(above) the smallest >."""
    T = np.asarray(targets, F)
    step = 0.5 * np.spacing(np.abs(T)).astype(np.float64) / np.abs(np.asarray(slope, np.float64))
    r = (np.asarray(r0, np.float64)[:, None] + np.arange(-k, k + 1)[None, :] * step[:, None]).astype(F)
    out = fn(torch.from_numpy(r).to(dev)).cpu().numpy()
    at = np.full(T.shape, np.nan, F)
    below, above = np.zeros(T.shape, F), np.zeros(T.shape, F)
    for i in range(T.size):
        eq = np.nonzero(out[i] == T[i])[0]
        if eq.size:
            at[i] = r[i, eq[eq.size // 2]]
        lo, hi = np.nonzero(out[i] < T[i])[0], np.nonzero(out[i] > T[i])[0]
        assert lo.size and hi.size, "search window does not bracket the target"
        below[i] = r[i, lo[np.argmax(out[i, lo])]]
        above[i] = r[i, hi[np.argmin(out[i, hi])]]
    return at, below, above


def exp_pre(targets, dev):
    T = np.asarray(targets, np.float64)
    return preimages(torch.exp, targets, np.log(T), T, dev)


def child_scale(r):
    """The split child's scale as the reference forms it: get_scaling / (0.8 N), stored through log, read through exp."""
    return torch.exp(torch.log(torch.exp(r) / (0.8 * 2)))


def child_pre(targets, dev):
    T = np.asarray(targets, np.float64)
    return preimages(child_scale, targets, np.log(1.6 * T), T, dev)


def sigmoid_pre(targets, dev):
    T = np.asarray(targets, np.float64)
    return preimages(torch.sigmoid, targets, np.log(T / (1 - T)), T * (1 - T), dev)


def extent_for(T, factor):
    """A double extent with fl32(factor * extent) == T (the reference's threshold lands exactly on T)."""
    e = float(T) / factor
    for _ in range(64):
        v = F(factor * e)
        if v == F(T):
            return e
        e = np.nextafter(e, np.inf if v < F(T) else -np.inf)
    raise AssertionError("no extent reaches the threshold")


def old_thresholds(extent, pd):
    """The thresholds formed from fp32-rounded extent / percent_dense (what a float-typed interface computes)."""
    return F(float(F(pd)) * float(F(extent))), F(0.1 * float(F(extent)))


class Pop:
    """A population under construction: random background rows plus rows placed at chosen decision values."""

    def __init__(self, seed, n_bg, extent, world=2, pd=PD, max_grad=MAX_GRAD, min_opacity=MIN_OPACITY, screen=True):
        self.rng = np.random.default_rng(seed)
        self.extent, self.pd, self.max_grad, self.min_opacity, self.screen = extent, pd, max_grad, min_opacity, screen
        self.world = world
        self.rows, self.labels = [], []
        self.dense = F(pd * extent)
        for _ in range(n_bg):
            hot = self.rng.random() < 0.4
            m = np.log(float(self.dense)) + self.rng.normal() * 1.2
            self.add("", m, grad=(F(self.rng.uniform(2.5, 8) * max_grad), F(1)) if hot else None,
                     logit=F(self.rng.normal() * 3.0))

    def add(self, label, log_scale_max, grad=None, logit=None, rot=None, xyz=None, spread=(0.3, 2.0)):
        """One Gaussian whose largest log-scale is `log_scale_max` (the other two axes lie `spread` below it, in a random
        axis order).  grad: (accum, denom) or None (cold: 0 / 1).  logit default: opaque."""
        rng = self.rng
        s = np.array([log_scale_max, log_scale_max - rng.uniform(*spread), log_scale_max - rng.uniform(*spread)], F)
        s[0] = F(log_scale_max)
        s = s[rng.permutation(3)]
        accum, denom = grad if grad is not None else (F(0), F(1))
        row = {"xyz": rng.normal(size=3) * 2.0 if xyz is None else xyz, "f_dc": rng.normal(size=(1, 3)),
               "f_rest": rng.normal(size=(15, 3)) * 0.1, "opacity": [F(3.0) if logit is None else logit],
               "scaling": s, "rotation": rng.normal(size=4) if rot is None else rot,
               "xyz_gradient_accum": [accum], "denom": [denom]}
        self.rows.append({k: np.asarray(v, F) for k, v in row.items()})
        self.labels.append(label)

    def hot(self, factor=4.0):
        return (F(factor * self.max_grad), F(1))

    def finish(self, name, family, stateless=(), shuffle=True, noise=None):
        P = len(self.rows)
        order = self.rng.permutation(P) if shuffle else np.arange(P)
        st = {k: np.stack([self.rows[i][k] for i in order]).astype(F) for k in self.rows[0]}
        for k in NAMES:
            if k in stateless:
                continue
            st[k + ".exp_avg"] = (self.rng.normal(size=st[k].shape) * 1e-3).astype(F)
            st[k + ".exp_avg_sq"] = (self.rng.random(size=st[k].shape) * 1e-6).astype(F)
        st["send_to_gpui_cnt"] = self.rng.integers(0, 1 << 40, size=(P, self.world), dtype=np.int64)
        labels = np.array(self.labels, dtype=object)[order]
        return dict(name=name, family=family, state=st, label=labels,
                    noise=self.rng.normal(size=(2 * P, 3)).astype(F) if noise is None else noise,
                    max_grad=self.max_grad, min_opacity=self.min_opacity, extent=self.extent, pd=self.pd,
                    screen=self.screen, near=int(sum(1 for s in labels if s)))


def _place(pop, tag, raws, grad):
    """Rows at each of (at, below, above) raw log-scales that exist, three of each."""
    for where, r in zip(("at", "below", "above"), raws):
        if np.isfinite(r):
            for _ in range(3):
                pop.add(f"{tag}_{where}", float(r), grad=grad)


def grad_cases(dev):
    """grad at fl32(max_grad) and one ulp either side (denom 1 and 3), of both signs, with small (clone) and large
    (split) scales; 0/0, +x/0 and -x/0."""
    out = []
    for screen in (True, False):
        pop = Pop(10 + screen, 120, 5.0, screen=screen)
        g = F(pop.max_grad)
        small, large = np.log(float(pop.dense)) - 1.0, np.log(float(pop.dense)) + 1.0
        for gv, where in ((ulp_step(g, -1), "below"), (g, "at"), (ulp_step(g, 1), "above")):
            for sign in (1, -1):
                for grad in ((F(sign * gv), F(1)), _accum_for(F(sign * gv))):
                    for m, size in ((small, "small"), (large, "large")):
                        pop.add(f"grad_{where}_{'pos' if sign > 0 else 'neg'}_{size}", m, grad=grad)
        for accum, tag in ((F(0), "nan"), (F(1e-3), "posinf"), (F(-1e-3), "neginf")):
            for m in (small, large):
                pop.add(f"grad_{tag}", m, grad=(accum, F(0)))
        out.append(pop.finish(f"grad_screen{int(screen)}", "grad"))
    # max_grad = 0: a zero gradient is selected, a NaN one (0 / 0, set to 0 by the reference) too
    pop = Pop(12, 40, 5.0, max_grad=0.0)
    for m in (np.log(float(pop.dense)) - 1.0, np.log(float(pop.dense)) + 1.0):
        for grad, tag in (((F(0), F(0)), "nan"), ((F(0), F(2)), "zero"), ((F(-1e-30), F(1)), "neg")):
            for _ in range(3):
                pop.add(f"grad_thr0_{tag}", m, grad=grad)
    out.append(pop.finish("grad_max_grad_0", "grad"))
    return out


def _accum_for(target, denoms=(3, 5, 6, 7, 9)):
    """(accum, denom) with fl32(accum / denom) == target, denom > 1 (IEEE division: the same on every device)."""
    for denom in denoms:
        a0 = F(float(target) * denom)
        cand = [a0]
        for d in (1, -1):
            a = a0
            for _ in range(4):
                a = ulp_step(a, d)
                cand.append(a)
        for a in cand:
            if F(a / F(denom)) == target:
                return a, F(denom)
    raise AssertionError("no accum reaches the target gradient")


def dense_cases(dev, n_random_extents=6):
    """Largest scale at dense_thr and one step either side: at extent 5.0 (dense_thr = 0.05f), with the threshold moved
    onto a reachable scale and one ulp either side of it, and at random extents in [0.5, 50] whose fl32(pd * extent)
    differs from the product of the fp32-rounded inputs."""
    out = []
    # extent 5.0: the scales exp reaches nearest to 0.05f (0.05f itself only if exp reaches it)
    pop = Pop(20, 100, 5.0)
    raws = exp_pre([pop.dense], dev)
    _place(pop, "dense", [raws[0][0], raws[1][0], raws[2][0]], pop.hot())
    out.append(pop.finish("dense_extent5", "dense"))
    # a reachable scale v; thresholds v, v + 1 ulp, v - 1 ulp
    v = F(torch.exp(torch.tensor([np.log(0.031)], dtype=torch.float32, device=dev)).item())
    r_v = exp_pre([v], dev)[0][0]
    assert np.isfinite(r_v)
    for shift in (0, 1, -1):
        T = v if shift == 0 else ulp_step(v, shift)
        pop = Pop(21 + shift, 100, extent_for(T, PD))
        assert pop.dense == T
        at, below, above = exp_pre([v], dev)
        _place(pop, f"dense_shift{shift}", [at[0], below[0], above[0]], pop.hot())
        out.append(pop.finish(f"dense_thr_v{shift:+d}ulp", "dense"))
    # random extents whose threshold rounds differently from fl32(fl32(pd) * fl32(extent))
    rng = np.random.default_rng(23)
    ext = rng.uniform(0.5, 50.0, size=4000)
    diff = np.array([F(PD * e) != old_thresholds(e, PD)[0] for e in ext])
    ext = ext[diff]
    T_new = np.array([F(PD * e) for e in ext], F)
    T_old = np.array([old_thresholds(e, PD)[0] for e in ext], F)
    at_new = exp_pre(T_new, dev)
    at_old = exp_pre(T_old, dev)
    found = 0
    for i in range(ext.size):
        if found == n_random_extents:
            break
        if not (np.isfinite(at_new[0][i]) or np.isfinite(at_old[0][i])):
            continue
        pop = Pop(100 + i, 80, float(ext[i]))
        _place(pop, "dense_new", [at_new[0][i], at_new[1][i], at_new[2][i]], pop.hot())
        _place(pop, "dense_old", [at_old[0][i], at_old[1][i], at_old[2][i]], pop.hot())
        out.append(pop.finish(f"dense_extent{ext[i]:.6f}", "dense_rounding"))
        found += 1
    assert found == n_random_extents, "too few extents with a reachable threshold"
    return out


def big_cases(dev):
    """Originals (cold, and hot-and-split) with their largest scale at big_thr and one ulp either side, screen-size
    limit on and off; split children whose scale exp(log(s / 1.6)) sits at big_thr and one step either side, placed
    between children that survive (the noise rank must advance past the pruned ones); big_thr of extents that round
    differently."""
    out = []
    v = F(torch.exp(torch.tensor([np.log(0.43)], dtype=torch.float32, device=dev)).item())
    for screen in (True, False):
        for shift in (0, 1, -1):
            T = v if shift == 0 else ulp_step(v, shift)
            pop = Pop(30 + 3 * screen + shift, 100, extent_for(T, 0.1), screen=screen)
            at, below, above = exp_pre([v], dev)
            _place(pop, f"big_orig_cold{shift}", [at[0], below[0], above[0]], None)
            _place(pop, f"big_orig_hot{shift}", [at[0], below[0], above[0]], pop.hot())
            out.append(pop.finish(f"big_orig_screen{int(screen)}_{shift:+d}ulp", "big_orig"))
    # children: a value a child reaches, thresholds on it and one ulp either side
    c = F(child_scale(torch.tensor([np.log(0.6)], dtype=torch.float32, device=dev)).item())
    for shift in (0, 1, -1):
        T = c if shift == 0 else ulp_step(c, shift)
        pop = Pop(40 + shift, 60, extent_for(T, 0.1), screen=True)
        at, below, above = child_pre([c], dev)
        for where, r in zip(("at", "below", "above"), (at[0], below[0], above[0])):
            if not np.isfinite(r):
                continue
            for _ in range(3):
                pop.add(f"big_child{shift}_{where}", float(r), grad=pop.hot(), spread=(0.05, 0.5))
                pop.add("", float(r) - 0.6, grad=pop.hot())      # a split neighbour whose children survive
        out.append(pop.finish(f"big_child_{shift:+d}ulp", "big_child"))
    # extents whose big_thr rounds differently from fl32(0.1 * fl32(extent))
    rng = np.random.default_rng(43)
    ext = rng.uniform(0.5, 50.0, size=4000)
    ext = ext[np.array([F(0.1 * e) != old_thresholds(e, PD)[1] for e in ext])]
    T_new = np.array([F(0.1 * e) for e in ext], F)
    T_old = np.array([old_thresholds(e, PD)[1] for e in ext], F)
    pre_new, pre_old = exp_pre(T_new, dev), exp_pre(T_old, dev)
    found = 0
    for i in range(ext.size):
        if found == 3:
            break
        if not (np.isfinite(pre_new[0][i]) or np.isfinite(pre_old[0][i])):
            continue
        pop = Pop(200 + i, 60, float(ext[i]), screen=True)
        _place(pop, "big_new", [pre_new[0][i], pre_new[1][i], pre_new[2][i]], None)
        _place(pop, "big_old", [pre_old[0][i], pre_old[1][i], pre_old[2][i]], None)
        out.append(pop.finish(f"big_extent{ext[i]:.6f}", "big_rounding"))
        found += 1
    assert found == 3, "too few extents with a reachable world-size threshold"
    return out


def opacity_cases(dev):
    """sigmoid(logit) at min_opacity and one ulp either side (min_opacity moved onto a value sigmoid reaches), for
    survivors, clones and split originals / children."""
    out = []
    v = F(torch.sigmoid(torch.tensor([np.log(0.0052 / (1 - 0.0052))], dtype=torch.float32, device=dev)).item())
    for shift in (0, 1, -1):
        T = v if shift == 0 else ulp_step(v, shift)
        pop = Pop(50 + shift, 100, 5.0, min_opacity=float(T))
        at, below, above = sigmoid_pre([v], dev)
        for where, r in zip(("at", "below", "above"), (at[0], below[0], above[0])):
            if not np.isfinite(r):
                continue
            for grad, m in ((None, -3.0), (pop.hot(), -4.0), (pop.hot(), -2.0)):
                pop.add(f"opacity{shift}_{where}", m, grad=grad, logit=r)
        out.append(pop.finish(f"opacity_{shift:+d}ulp", "opacity"))
    return out


def whole_cases(dev):
    """Whole-population outcomes: everything pruned, nothing selected, everything split, and clone / split / prune
    interleaved row by row in index order."""
    out = []
    pop = Pop(60, 0, 5.0)
    for i in range(300):
        pop.add("all_pruned", -3.0 + 0.01 * i, grad=pop.hot() if i % 2 else None, logit=F(-12.0))
    out.append(pop.finish("all_pruned", "whole"))
    pop = Pop(61, 0, 5.0)
    for i in range(300):
        pop.add("none_selected", -3.0 + 0.01 * (i % 50), grad=(F(1e-5), F(2)) if i % 3 else None)
    out.append(pop.finish("none_selected", "whole"))
    pop = Pop(62, 0, 5.0, screen=False)
    for i in range(300):
        pop.add("all_split", -1.5 + 0.002 * i, grad=pop.hot(1.0 + i))
    out.append(pop.finish("all_split", "whole"))
    pop = Pop(63, 0, 5.0)
    small, large = np.log(0.05) - 0.7, np.log(0.05) + 0.7
    kinds = [("clone", small, pop.hot(), None), ("split", large, pop.hot(), None), ("keep", large, None, None),
             ("pruned", small, None, F(-12.0)), ("pruned_split", large, pop.hot(), F(-12.0)),
             ("big", np.log(0.9), None, None), ("pruned_clone", small, pop.hot(), F(-12.0))]
    for i in range(700):
        name, m, g, lg = kinds[(i * 5 + i // 7) % len(kinds)]
        pop.add("interleave_" + name, m, grad=g, logit=lg)
    out.append(pop.finish("interleaved", "whole", shuffle=False))
    return out


def position_cases(dev):
    """Children's positions: unnormalised quaternions with norms 1e-3 .. 1e3, scales 1e-4 .. 1e2, draws up to |z| = 6."""
    pop = Pop(70, 0, 0.001, screen=False)      # dense_thr = 1e-5: every hot Gaussian splits
    rng = pop.rng
    n = 600
    for i in range(n):
        q = rng.normal(size=4)
        q *= 10.0 ** rng.uniform(-3, 3) / np.linalg.norm(q)
        pop.add("positions", np.log(10.0 ** rng.uniform(-4, 2)), grad=pop.hot(), rot=q,
                xyz=rng.normal(size=3) * 10.0 ** rng.uniform(-2, 3), spread=(0.0, 6.0))
    noise = rng.normal(size=(2 * n, 3)).astype(F)
    noise[::7] = rng.choice([-6.0, 6.0], size=noise[::7].shape) * rng.uniform(0.9, 1.0, size=noise[::7].shape)
    return [pop.finish("positions", "positions", noise=noise)]


def shape_case(P, seed, world, stateless=(), name=None):
    """A random population of P Gaussians (about a fifth cloned, a fifth split, some pruned) built vectorised."""
    rng = np.random.default_rng(seed)
    st = {"xyz": rng.normal(size=(P, 3)) * 2.0, "f_dc": rng.normal(size=(P, 1, 3)),
          "f_rest": rng.standard_normal(size=(P, 15, 3), dtype=F) * 0.1, "opacity": rng.normal(size=(P, 1)) * 2.5,
          "scaling": rng.normal(size=(P, 3)) + np.log(0.05), "rotation": rng.normal(size=(P, 4))}
    denom = rng.integers(0, 7, size=(P, 1)).astype(F)
    st["xyz_gradient_accum"] = rng.random(size=(P, 1)) * 6e-4 * denom
    st["denom"] = denom
    st = {k: np.asarray(v, F) for k, v in st.items()}
    for k in NAMES:
        if k in stateless:
            continue
        st[k + ".exp_avg"] = rng.standard_normal(size=st[k].shape, dtype=F) * F(1e-3)
        st[k + ".exp_avg_sq"] = rng.random(size=st[k].shape, dtype=F) * F(1e-6)
    st["send_to_gpui_cnt"] = rng.integers(-(1 << 40), 1 << 40, size=(P, world), dtype=np.int64)
    return dict(name=name or f"P{P}_w{world}", family="shapes", state=st, label=np.full(P, "", dtype=object),
                noise=rng.standard_normal(size=(2 * P, 3), dtype=F), max_grad=MAX_GRAD, min_opacity=MIN_OPACITY,
                extent=5.0, pd=PD, screen=bool(seed % 2), near=0)


SHAPES_P = ((1, 1, 1), (255, 2, 3), (256, 3, 16), (257, 4, 1), (4099, 5, 3))
BIG_P = 1 << 20 | 3


def shape_cases():
    out = [shape_case(P, seed, world) for P, seed, world in SHAPES_P]
    out.append(shape_case(4099, 6, 2, stateless=("f_dc", "rotation"), name="P4099_partial_state"))
    return out


def all_cases(dev):
    return (grad_cases(dev) + dense_cases(dev) + big_cases(dev) + opacity_cases(dev) + whole_cases(dev)
            + position_cases(dev) + shape_cases())
