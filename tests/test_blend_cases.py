"""CPU checks of tests/blend_cases.py: every regime is populated where the case says, the fp64 decision walk agrees with
both oracles on every pixel it calls decision-safe and leaves few out, and the fp64 oracle's blend backward equals
torch autograd of tests/torch_ref.render on the constructed cases (clamp straight-through, saturation, the floor)."""
import numpy as np
import pytest
import torch

import blend_cases as bc
import torch_ref
from oracle.oracle import Oracle

CASES = {c["name"]: c for c in bc.all_cases()}


@pytest.fixture(scope="module")
def o32():
    return Oracle(np.float32, threads=4)


@pytest.fixture(scope="module")
def o64():
    return Oracle(np.float64, threads=4)


def fwd(o, c, dtype):
    a = [np.asarray(c[k], dtype) for k in ("means2D", "conic_opacity", "rgb")]
    return o.render_forward(c["H"], c["W"], *a, c["depths"], c["radii"], c["cl"], c["bg"])


@pytest.mark.parametrize("name", list(CASES))
def test_decision_walk_agrees_with_both_oracles(o32, o64, name):
    c = CASES[name]
    f32, f64 = fwd(o32, c, np.float32), fwd(o64, c, np.float64)
    assert np.array_equal(f32["ids"], f64["ids"]) and np.array_equal(f32["ranges"], f64["ranges"])
    w = bc.decision_walk(c, f32)
    safe = ~w["ambiguous"]
    assert w["ambiguous"].mean() <= 1e-2, w["ambiguous"].sum()
    assert np.array_equal(w["n_contrib"][safe], f64["n_contrib"][safe].astype(np.int64))
    assert np.array_equal(w["n_contrib"][safe], f32["n_contrib"][safe].astype(np.int64))


def test_regions_are_populated(o32):
    gx, _ = bc.tiles_of(64, 48)
    for name in ("saturation_bg0", "saturation_bg1"):
        c = CASES[name]
        f = fwd(o32, c, np.float32)
        w = bc.decision_walk(c, f)
        term, nc, safe = w["term"], w["n_contrib"], ~w["ambiguous"]
        for t, target in enumerate(bc.SAT_TARGETS):
            ty, tx = divmod(t, gx)
            sl = (slice(ty * 16, ty * 16 + 16), slice(tx * 16, tx * 16 + 16))
            tt, nn, ss = term[sl], nc[sl], safe[sl]
            assert ((tt == target) & ss).any(), (name, target)           # saturates exactly at the chosen entry
            assert ((tt < 0) & (nn > target) & ss).any(), (name, target)  # never saturates, blends past it
        assert c["bg"] == (0.0, 0.0, 0.0) or min(c["bg"]) > 0
    c = CASES["lengths_mask_all"]
    f = fwd(o32, c, np.float32)
    assert tuple(int(v) for v in f["ranges"][:, 1] - f["ranges"][:, 0]) == bc.LENGTHS
    m = dict(all=12, checkerboard=6, single=1, none=0)
    for k, n in m.items():
        assert int(CASES[f"lengths_mask_{k}"]["cl"].sum()) == n
    c = CASES["clamp"]
    co, m2 = c["conic_opacity"], c["means2D"]
    hi = co[:, 3] > 0.99
    assert (co[:, 3] == 1.0).any() and hi.sum() > 100
    assert (hi & (m2 == np.round(m2)).all(1)).sum() > 50                  # centred exactly on a pixel: o G = o
    c = CASES["floor"]
    o, m2 = c["conic_opacity"][:, 3], c["means2D"]
    on_px = (m2 == np.round(m2)).all(1)
    for v in bc.FLOOR_OPACITIES:
        assert ((o == v) & on_px).any() and ((o == v) & ~on_px).any(), v
    assert (o == bc.INV255).any() and (o == np.nextafter(bc.INV255, np.float32(0))).any()
    for name in ("ragged_1x1", "ragged_15x17", "ragged_17x33", "ragged_33x15", "ragged_33x1"):
        c = CASES[name]
        for lab in ("whole_image", "off_screen_reach", "off_screen_empty", "culled"):
            assert (c["label"] == lab).any(), (name, lab)
        f = fwd(o32, c, np.float32)
        gx_, gy_ = bc.tiles_of(c["W"], c["H"])
        whole = int(np.nonzero(c["label"] == "whole_image")[0][0])
        assert (f["ids"] == whole).sum() == gx_ * gy_                     # its rect covers every tile
        reach = np.nonzero(c["label"] == "off_screen_reach")[0]
        assert np.isin(reach, f["ids"]).all()
        m2 = c["means2D"][reach]
        assert ((m2[:, 0] < 0) | (m2[:, 0] >= c["W"]) | (m2[:, 1] < 0) | (m2[:, 1] >= c["H"])).all()
        assert not np.isin(np.nonzero((c["label"] == "off_screen_empty") | (c["label"] == "culled"))[0], f["ids"]).any()
    c = CASES["ties"]
    d = c["depths"]
    assert len(np.unique(d)) == 5 and (d == np.float32(1.5)).sum() > 20
    f = fwd(o32, c, np.float32)
    for t in range(4):   # within a tile, equal depth bits keep index order
        ids = f["ids"][f["ranges"][t, 0]:f["ranges"][t, 1]]
        key = d[ids].view(np.uint32).astype(np.int64) * (1 << 20) + ids
        assert (np.diff(key) > 0).all()
    c = CASES["band_edge"]
    co = c["conic_opacity"][c["label"] == "band_edge"].astype(np.float64)
    reach2 = 2.0 * np.log(255.0 * co[:, 3]) / co[:, 0]           # squared radius of the alpha = 1/255 circle
    assert len(co) == 600 and (np.abs(reach2 / 9.0 - 1.0) <= 3e-6).all()
    c = CASES["degenerate"]
    co = c["conic_opacity"][c["label"] == "degenerate"]
    det = co[:, 0] * co[:, 2] - co[:, 1] * co[:, 1]
    assert (det == 0).any() and (det < 0).any() and len(det) > 30


@pytest.mark.parametrize("name", ["clamp", "floor", "saturation_bg1", "ragged_15x17", "degenerate", "ties"])
def test_fp64_oracle_matches_torch_autograd(o64, name):
    """The fp64 oracle's hand-written blend backward == autograd of torch_ref.render (the clamp straight-through) on
    the oracle's own decisions."""
    c = CASES[name]
    f = fwd(o64, c, np.float64)
    g = c["dL"].astype(np.float64)
    rb = o64.render_backward(c["H"], c["W"], *[np.asarray(c[k], np.float64) for k in ("means2D", "conic_opacity", "rgb")],
                             c["bg"], f, g)
    t = [torch.tensor(np.asarray(c[k], np.float64), requires_grad=True) for k in ("means2D", "conic_opacity", "rgb")]
    img = torch_ref.render(*t, c["bg"], c["H"], c["W"], f)
    np.testing.assert_allclose(img.detach().numpy(), f["image"], rtol=1e-9, atol=1e-12)
    (img * torch.tensor(g)).sum().backward()
    W, H = c["W"], c["H"]
    for k, a, b in (("means2D", rb["means2D"], t[0].grad.numpy() * np.array([W / 2, H / 2])),
                    ("conic_opacity", rb["conic_opacity"], t[1].grad.numpy()), ("rgb", rb["rgb"], t[2].grad.numpy())):
        scale = np.abs(b).max() + 1e-300
        np.testing.assert_allclose(a, b, rtol=1e-7, atol=1e-9 * scale, err_msg=k)
    if name == "clamp":
        assert (f["image"] != 0).any() and (np.abs(rb["conic_opacity"][c["conic_opacity"][:, 3] > 0.99, 3]) > 0).any()
