"""CPU checks of the per-view training loss report: the rank-order sum and the (1 - lambda) Ll1 + lambda (1 - ssim)
formation of Trainer.train_losses (pipeline.sum_over_ranks / loss_table / loss_entries) on hand-made gathered records,
and the training log's loss lines (statlog.train_loss_text, statlog.EpochLoss) against restated copies of the reference's
parsers (analyze_statistic.py:2746-2790), checked verbatim against its source when the reference checkout is present."""
import os
import re

import numpy as np
import pytest
import torch

from gs_b200 import pipeline, statlog

ANALYZE = "/root/reference/analyze_statistic.py"
# draw_iteration_loss (analyze_statistic.py:2782-2784) and draw_epoch_loss (:2753-2754), restated
REG_EXP1 = r"iteration (\d+) image: \w+ loss: (\d+\.\d+)"
REG_EXP2 = r"iteration\[(\d+),\d+\) loss: \[(.*)\] image: \[('\w+')(, '\w+')*\]"
EPOCH_TEST = 'if line.startswith("epoch "):'
EPOCH_VALUE = 'epoch_loss.append(float(line.split(" ")[-1]))'


def parse_iteration_lines(text):
    """draw_iteration_loss's loop body: -> [(iteration, [losses])]."""
    reg_exp1, reg_exp2 = re.compile(REG_EXP1), re.compile(REG_EXP2)
    out = []
    for line in text.splitlines(keepends=True):
        m = reg_exp1.match(line) or reg_exp2.match(line)
        if m:
            out.append((int(m.group(1)), [float(x) for x in m.group(2).split(", ")]))
    return out


def parse_epoch_lines(text):
    return [float(line.split(" ")[-1]) for line in text.splitlines(keepends=True) if line.startswith("epoch ")]


def bits32(a):
    return np.asarray(a, dtype=np.float32).view(np.int32)


def test_the_restated_parsers_are_the_reference_source():
    if not os.path.exists(ANALYZE):
        pytest.skip("the reference checkout is not present")
    src = open(ANALYZE).read()
    for s in (f'reg_exp1 = re.compile(r"{REG_EXP1}")', f'reg_exp2 = re.compile(r"{REG_EXP2}")', EPOCH_TEST, EPOCH_VALUE):
        assert s in src, s


# 1. the rank-order sum
def test_sum_over_ranks_is_a_left_fold_in_rank_order():
    # a float32 sum that depends on the order: (1e8 - 1e8) + 1 = 1, but 1e8 + (-1e8 + 1) = 0
    g = torch.tensor([[[1e8, 0.5]], [[-1e8, 0.25]], [[1.0, 0.125]]], dtype=torch.float32)
    got = pipeline.sum_over_ranks(g)
    want = (g[0] + g[1]) + g[2]
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    other = g[0] + (g[1] + g[2])
    assert not torch.equal(got, other)            # the order is visible, and it is rank order
    assert got[0, 0].item() == 1.0 and got[0, 1].item() == 0.875
    assert torch.equal(pipeline.sum_over_ranks(g[:1]), g[0])   # one rank: its record as it is


def test_views_whole_on_one_rank_keep_their_bits():
    """Local sampling: a view is rendered whole by one rank, the others hold +0.0, so the sum is that rank's value."""
    rng = np.random.default_rng(0)
    W, k = 4, 3
    vals = rng.random((W * k, 2), dtype=np.float32) * np.float32([0.3, 1.0])
    g = np.zeros((W, W * k, 2), dtype=np.float32)
    for p in range(W * k):
        g[p // k, p] = vals[p]
    got = pipeline.sum_over_ranks(torch.from_numpy(g)).numpy()
    assert np.array_equal(bits32(got), bits32(vals))


# 2. the per-view loss and the entries
LAM = 0.2


def reference_loss(l1, ssim, lam):
    """train_internal.py:220-222 in float32: (1 - lambda) * Ll1 + lambda * (1 - ssim)."""
    l1, ssim = np.float32(l1), np.float32(ssim)
    return np.float32(np.float32(1.0 - lam) * l1) + np.float32(np.float32(lam) * np.float32(np.float32(1.0) - ssim))


def test_loss_table_forms_the_reference_loss():
    rng = np.random.default_rng(1)
    n = 97
    g = torch.from_numpy(rng.random((2, n, 2), dtype=np.float32) * np.float32([0.2, 0.5]))
    index = torch.from_numpy(rng.integers(0, 1000, n))
    rows = pipeline.loss_table(g, index, LAM)
    assert rows.dtype == torch.float64 and tuple(rows.shape) == (n, 4)
    pairs = (g[0] + g[1]).numpy()
    assert rows[:, 0].tolist() == index.tolist()
    assert np.array_equal(rows[:, 1:3].numpy(), pairs.astype(np.float64))   # float32 values, widened exactly
    want = np.array([reference_loss(a, b, LAM) for a, b in pairs], dtype=np.float32)
    assert np.array_equal(bits32(rows[:, 3].numpy().astype(np.float32)), bits32(want))
    assert np.array_equal(rows[:, 3].numpy(), want.astype(np.float64))
    # +0.0 records (a view no rank has a strip of) give Ll1 = ssim = 0 and loss = lambda
    z = pipeline.loss_table(torch.zeros((3, 1, 2)), torch.zeros((1,), dtype=torch.int64), LAM)
    assert z[0, 1:].tolist() == [0.0, 0.0, float(np.float32(LAM) * np.float32(1.0))]


def test_ragged_steps_split_into_entries():
    """Steps of 1, 3, 64 and 2 views over three ranks: a strip-divided view has partials on several ranks, a whole view
    on one; the entries list the steps oldest first with their views in batch order."""
    rng = np.random.default_rng(2)
    steps = [(1, 1), (2, 3), (3, 64), (4, 2)]
    n = sum(b for _, b in steps)
    W = 3
    g = np.zeros((W, n, 2), dtype=np.float32)
    owners = []
    for p in range(n):
        ranks = [p % W] if p % 2 else sorted(rng.choice(W, size=int(rng.integers(2, W + 1)), replace=False))
        owners.append(ranks)
        for r in ranks:
            g[r, p] = rng.random(2, dtype=np.float32) * np.float32([0.1, 0.3])
    index = rng.integers(0, 50, n)
    rows = pipeline.loss_table(torch.from_numpy(g), torch.from_numpy(index), LAM).tolist()
    entries = pipeline.loss_entries(rows, steps)
    assert [(e["iteration"], len(e["views"])) for e in entries] == steps
    p = 0
    for e in entries:
        for q in range(len(e["views"])):
            s = np.float32(0.0) + g[0, p]
            for r in range(1, W):
                s = s + g[r, p]
            assert e["views"][q] == int(index[p])
            assert (e["l1"][q], e["ssim"][q]) == (float(s[0]), float(s[1]))
            assert e["loss"][q] == float(reference_loss(s[0], s[1], LAM))
            if len(owners[p]) == 1:   # whole on one rank: its own value
                assert (e["l1"][q], e["ssim"][q]) == tuple(float(v) for v in g[owners[p][0], p])
            p += 1
    assert all(isinstance(v, float) for e in entries for k in ("l1", "ssim", "loss") for v in e[k])
    assert pipeline.loss_entries([], []) == []


# 3. the log lines
def test_train_loss_line_parses_back():
    losses = [np.float32(0.33102712), 0.2134300001, np.float64(0.243), 1e-7, 0.5]
    names = ["00297", "DSC08048", "a_b", "x", "00001"]
    text = statlog.train_loss_text(3006, 5, losses, names)
    assert text.startswith("iteration[3006,3011) loss: [0.331027, 0.21343, 0.243, 0.0, 0.5] image: "
                           "['00297', 'DSC08048', 'a_b', 'x', '00001']") and text.endswith("\n")
    assert re.compile(REG_EXP2).match(text)
    assert parse_iteration_lines(text) == [(3006, [0.331027, 0.21343, 0.243, 0.0, 0.5])]
    one = statlog.train_loss_text(1, 1, [torch.tensor(0.1234565)], ["img"])
    assert one == f"iteration[1,2) loss: [{round(float(torch.tensor(0.1234565)), 6)}] image: ['img']\n"
    assert parse_iteration_lines(one) == [(1, [round(float(torch.tensor(0.1234565)), 6)])]


def test_iteration_lines_of_a_run_parse_in_order():
    rng = np.random.default_rng(3)
    text, want, it = "", [], 1
    for bsz in (1, 4, 16, 3):
        losses = rng.random(bsz).astype(np.float32)
        text += statlog.train_loss_text(it, bsz, losses, [f"{it + q:05d}" for q in range(bsz)])
        want.append((it, [round(float(v), 6) for v in losses]))
        it += bsz
    assert parse_iteration_lines(text) == want


def test_epoch_lines():
    acc = statlog.EpochLoss(3)
    assert acc.update([0.5, 0.25]) == ""
    t = acc.update([0.75, 0.125, 0.25, 0.125, 1.0])   # completes epochs 1 and 2, keeps one loss pending
    assert t == f"epoch 1 loss: {(0.5 + 0.25 + 0.75) / 3}\nepoch 2 loss: {(0.125 + 0.25 + 0.125) / 3}\n"
    assert parse_epoch_lines(t) == [(0.5 + 0.25 + 0.75) / 3, (0.125 + 0.25 + 0.125) / 3]
    assert acc.iteration_loss == [1.0] and len(acc.epoch_loss) == 2
    assert acc.update(np.array([0.0, 0.5], dtype=np.float32)) == "epoch 3 loss: 0.5\n"
    one = statlog.EpochLoss(1)
    assert parse_epoch_lines(one.update([0.1, 0.2])) == [0.1, 0.2]
    with pytest.raises(ValueError):
        statlog.EpochLoss(0)


def test_lines_write_through_append(tmp_path):
    path = str(tmp_path / "logs" / "python_ws=1_rk=0.log")
    acc = statlog.EpochLoss(2)
    for it, losses in ((1, [0.25, 0.5]), (3, [0.125, 0.375])):
        statlog.append(path, statlog.train_loss_text(it, 2, losses, ["a", "b"]))
        statlog.append(path, acc.update(losses))
    text = open(path).read()
    assert parse_iteration_lines(text) == [(1, [0.25, 0.5]), (3, [0.125, 0.375])]
    assert parse_epoch_lines(text) == [0.375, 0.25]
