"""-m gpu: gs_adam_step (through gs_b200.optim.FusedAdam) against torch.optim.Adam on the same device -- the
multi-tensor (foreach) path torch takes by default for CUDA parameters -- bit for bit in p, exp_avg and exp_avg_sq.

The reference divides every gradient by bsz (`param.grad /= bsz`, a multiply by the fp32 reciprocal on CUDA) and then
steps torch.optim.Adam; FusedAdam takes grad_scale = 1 / bsz instead.  The cases put every per-tensor input in a
different place: each tensor has its own group with its own lr, betas and eps (the sqrt lr-scale mode's betas^bsz and
eps / sqrt(bsz) among them, and beta1 <= 0.5, where torch's lerp takes its other form), step counters loaded at
0, 1, 9, 999 and 29999 into both optimizers, 9 to 17 tensors (FusedAdam launches 8 at a time), numel 0, 1, 3, 4, 5 and
ragged tails, one tensor 4 bytes off a 16-byte boundary next to float4-aligned ones, tensors without a gradient, and
gradients that are exactly zero (v = 0, the denominator is eps), 1e-20 (g^2 is denormal), around 1e18, or of mixed sign.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"

NUMELS = (0, 1, 3, 4, 5, 7, 1023, 4097, 20011, 9, 6, 2, 65539, 13, 1, 4, 8)
GRAD_KINDS = ("normal", "zero", "tiny", "huge", "mixed")


def hyper(k, bsz):
    """Distinct lr / betas / eps for tensor k: the defaults, the sqrt lr-scale mode's and arbitrary values."""
    table = [(1e-3, (0.9, 0.999), 1e-15),
             (0.05, (0.9 ** bsz, 0.999 ** bsz), 1e-15 / math.sqrt(bsz)),
             (0.0025, (0.8, 0.99), 1e-8),
             (0.0025 / 20, (0.95, 0.9999), 1e-12),
             (0.005, (0.3, 0.97), 1e-6),                  # 1 - beta1 >= 0.5: torch's lerp takes end - (end - x)(1 - w)
             (0.001, (0.9 ** 16, 0.999 ** 16), 1e-15 / 4.0),
             (0.00016 * 4.2, (0.5, 0.5), 1e-15),
             (0.1, (0.0, 0.0), 1e-10),
             (1.0, (0.99, 0.999999), 1e-3)]
    lr, betas, eps = table[k % len(table)]
    return lr * (1.0 + 0.01 * k), betas, eps


def grad_of(kind, shape, gen):
    if kind == "zero":
        return torch.zeros(shape)
    if kind == "tiny":
        return torch.full(shape, 1e-20) * torch.sign(torch.randn(shape, generator=gen))
    if kind == "huge":
        return torch.randn(shape, generator=gen) * 1e18
    if kind == "mixed":
        g = torch.randn(shape, generator=gen)
        return g * torch.pow(10.0, torch.randint(-12, 6, shape, generator=gen).float())
    return torch.randn(shape, generator=gen) * 0.01


def build(n_tensors, bsz, step0, seed):
    """Two identical parameter sets (FusedAdam's, torch's) with loaded state: step0 == 0 leaves the state empty."""
    gen = torch.Generator().manual_seed(seed)
    base = torch.randn((NUMELS[3] + 1,), generator=gen)
    sets = []
    for _ in range(2):
        params = []
        for k in range(n_tensors):
            if k == 3:     # 4 bytes past a 16-byte boundary: the kernel's scalar path for this tensor only
                buf = torch.empty((NUMELS[k] + 1,), device=DEV)
                buf.copy_(base.to(DEV))
                p = buf[1:]
            else:
                p = torch.empty((NUMELS[k],), device=DEV)
            params.append(p)
        sets.append(params)
    gen = torch.Generator().manual_seed(seed + 1)
    for k in range(n_tensors):
        if k == 3:
            continue
        init = torch.randn((NUMELS[k],), generator=gen).to(DEV)
        for params in sets:
            params[k].copy_(init)
    out = []
    for params in sets:
        ps = [p.requires_grad_(True) for p in params]
        groups = [{"params": [p], "lr": hyper(k, bsz)[0], "betas": hyper(k, bsz)[1], "eps": hyper(k, bsz)[2],
                   "name": f"t{k}"} for k, p in enumerate(ps)]
        out.append((ps, groups))
    assert out[0][0][3].data_ptr() % 16 == 4
    state = []
    if step0 > 0:
        gen = torch.Generator().manual_seed(seed + 2)
        for k in range(n_tensors):
            m = torch.randn((NUMELS[k],), generator=gen) * 1e-3
            v = torch.rand((NUMELS[k],), generator=gen) * 1e-6
            state.append((m, v))
    return out, state


def load_state(opt, params, state, step0):
    for p, (m, v) in zip(params, state):
        opt.state[p] = {"step": torch.tensor(float(step0)), "exp_avg": m.to(DEV).clone(), "exp_avg_sq": v.to(DEV).clone()}


def bits(t):
    return t.detach().cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("step0", [0, 1, 9, 999, 29999])
@pytest.mark.parametrize("bsz", [1, 3, 4, 6])
def test_fused_adam_equals_torch_adam_bit_for_bit(bsz, step0):
    from gs_b200.optim import FusedAdam
    n_tensors = 9 + (bsz * 7 + step0) % 9          # 9 .. 17 tensors: two or three launches
    sets, state = build(n_tensors, bsz, step0, seed=bsz * 100 + step0 % 97)
    (pf, gf), (pt, gt) = sets
    fused = FusedAdam(gf, lr=0.0, eps=1e-15)
    ref = torch.optim.Adam(gt, lr=0.0, eps=1e-15)
    if step0:
        load_state(fused, pf, state, step0)
        load_state(ref, pt, state, step0)
    gen = torch.Generator().manual_seed(7 + bsz)
    for s in range(3):
        for k in range(n_tensors):
            if (k + s) % 5 == 4:                     # no gradient this step: the tensor and its step counter stay put
                pf[k].grad = pt[k].grad = None
                continue
            g = grad_of(GRAD_KINDS[(k + s) % len(GRAD_KINDS)], (NUMELS[k],), gen).to(DEV)
            pf[k].grad = g.clone()
            pt[k].grad = g.clone()
            pt[k].grad /= bsz                        # the reference's division, on the device
        fused.step(grad_scale=1.0 / bsz)
        ref.step()
        for k in range(n_tensors):
            a, b = fused.state.get(pf[k]), ref.state.get(pt[k])
            assert (a is None) == (b is None), k
            if a is None:
                continue
            assert float(a["step"]) == float(b["step"]), k
            for what, x, y in (("p", pf[k], pt[k]), ("exp_avg", a["exp_avg"], b["exp_avg"]),
                               ("exp_avg_sq", a["exp_avg_sq"], b["exp_avg_sq"])):
                bx, by = bits(x), bits(y)
                assert np.array_equal(bx, by), (f"step {s} tensor {k} ({NUMELS[k]} elements, {hyper(k, bsz)}) {what}: "
                                                f"{int((bx != by).sum())} differ")
