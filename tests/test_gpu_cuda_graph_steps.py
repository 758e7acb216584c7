"""CUDA-graph steps with the learning rate in device memory (GraphedTrainStep(device_lr=True), --cuda-graph-steps):
the _lr_dev kernel entry points against the by-value ones, graph replays over a changing schedule against eager
train_step calls (all-device tables, host tables, host tables with a row cache), and the command line's graphed
runs against the reference's recorded runs."""
import os
import re

import numpy as np
import pytest
import torch

from test_gpu_host_tables import DEV, LN, _batches, _state, _st, L

import test_gpu_bin_records as bin_cli
import test_gpu_criteo_dataset as kaggle_cli
import test_gpu_criteo_days as days_cli
from test_criteo_days_host import write_days

pytestmark = pytest.mark.gpu
_LOSS = re.compile(r"Finished training it .* loss ([0-9.]+)")
_REPORT = re.compile(r"CUDA-graph steps: (\d+) train steps replayed, (\d+) eager .*; (\d+) test batches replayed, "
                     r"(\d+) eager")


def _engine(host=(), gemm="tc", cache=0):
    from dlrm_b200.engine import Engine

    D = 32
    F = len(LN) + 1
    top = [D + F * (F - 1) // 2, 64, 1]
    e = Engine(D, LN, [13, 64, D], top, sigmoid_top=len(top) - 2, device=DEV, max_batch=256, gemm=gemm,
               host_tables=list(host), host_cache_rows=cache)
    e.init_params(seed=3)
    return e


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad", "adagrad"])
@pytest.mark.parametrize("gemm", ["simt", "tc"])
def test_device_lr_updates_are_bit_identical_to_by_value(opt, gemm):
    """Tables 1 and 3 (200 and 40 rows) take the tiny-table kernels, the others the list path; simt steps the dense
    parameters with dense_update, tc with dense_update_pack.  The by-value lr handed to the _lr_dev calls is wrong on
    purpose: only the device float may reach the kernels."""
    bs = _batches(3, seed=7)
    res = []
    for mode in ("value", "device"):
        e = _engine(gemm=gemm)
        e.ensure_optimizer_state(opt)
        assert any(e.is_small(k) for k in range(len(LN))) and not all(e.is_small(k) for k in range(len(LN)))
        losses = []
        for i, b in enumerate(bs):
            lr = 0.05 / (i + 1)
            if mode == "device":
                e.lr_dev = torch.full((1,), lr, dtype=torch.float32, device=DEV)
                losses.append(e.train_step(b.X, b.sparse, b.target, 1e3, opt).clone())
                e.lr_dev = None
            else:
                losses.append(e.train_step(b.X, b.sparse, b.target, lr, opt).clone())
        torch.cuda.synchronize()
        res.append((torch.stack(losses), _state(e, opt)))
    assert torch.equal(res[0][0], res[1][0])
    for a, b in zip(res[0][1], res[1][1]):
        assert torch.equal(a, b)


def _schedule(n):
    """Warm-up over 3 steps, one flat step, then quadratic decay: every replay sees another rate."""
    out = []
    for c in range(1, n + 1):
        out.append(0.08 * c / 3 if c <= 3 else 0.08 if c == 4 else 0.08 * ((n + 1 - c) / (n - 3)) ** 2 + 1e-4)
    return out


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad", "adagrad"])
@pytest.mark.parametrize("host,cache", [((), 0), ((0, 2, 4), 0), ((0, 2, 4), 64)])
def test_device_lr_replays_equal_eager_steps(opt, host, cache):
    """N replays over a changing schedule (lr_decay > 0 for the Adagrad variants) == N eager train_step calls with the
    same rates: losses, tables, accumulators, dense parameters and the host row cache's counters.  An eager step at
    another batch size runs between replays, on the same engine."""
    from dlrm_b200.engine import GraphedTrainStep

    bs = _batches(9, seed=11)
    odd = _batches(1, B=100, seed=12)[0]
    lrs = _schedule(8)
    decay = 0.1 if opt != "sgd" else 0.0
    res = []
    for mode in ("eager", "graph"):
        e = _engine(host, "tc", cache)
        for b in bs:
            e.prepare(b.sparse, True)
        if mode == "graph":
            st = bs[8]
            g = GraphedTrainStep(e, st, 0.5, opt, warmup=0, device_lr=True)
            assert e.opt_step == 0
        losses = []
        for i in range(8):
            if i == 4:        # the short batch: eager in both runs
                losses.append(e.train_step(odd.X, odd.sparse, odd.target, lrs[i], opt, lr_decay=decay).clone())
            b = bs[i]
            if mode == "eager":
                losses.append(e.train_step(b.X, b.sparse, b.target, lrs[i], opt, lr_decay=decay).clone())
            else:
                st.buf.copy_(b.buf)
                losses.append(g.replay(lrs[i], decay).clone())
        assert e.opt_step == 9
        stats = e.host_cache_stats() if host else None
        torch.cuda.synchronize()
        res.append((torch.stack(losses), _state(e, opt), stats))
        assert L().dlrm_b200_check_device_errors(_st()) == 0
    assert torch.equal(res[0][0], res[1][0])
    for a, b in zip(res[0][1], res[1][1]):
        assert torch.equal(a, b)
    assert res[0][2] == res[1][2]
    if cache:
        assert res[1][2]["hits"] > 0


def test_baked_graph_refuses_a_learning_rate():
    from dlrm_b200.engine import GraphedTrainStep

    e = _engine(gemm="simt")
    st = _batches(1)[0]
    g = GraphedTrainStep(e, st, 0.01, "sgd", warmup=0)
    with pytest.raises(ValueError, match="baked in"):
        g.replay(0.02)


# ---------------------------------------------------------------------------------------------- command line
def _report(text):
    m = _REPORT.search(text)
    assert m, text[-2000:]
    return [int(v) for v in m.groups()]


def _compare(got_txt, want_txt, other, atol):
    want, got = want_txt.splitlines(), got_txt.splitlines()
    want_loss = [float(_LOSS.match(ln).group(1)) for ln in want if _LOSS.match(ln)]
    got_loss = [float(_LOSS.match(ln).group(1)) for ln in got if _LOSS.match(ln)]
    assert len(got_loss) == len(want_loss) > 0
    np.testing.assert_allclose(got_loss, want_loss, rtol=0, atol=atol)
    assert [ln for ln in got if other.search(ln)] == [ln for ln in want if other.search(ln)]


@pytest.mark.parametrize("tag", ["A", "B", "C"])
def test_cli_kaggle_graphed_matches_the_reference_run(tag):
    got = kaggle_cli._cli(tag, ["--gemm=simt", "--cuda-graph-steps"])
    want = open(os.path.join(kaggle_cli.GOLD, "cli_kaggle_%s.txt" % tag)).read()
    _compare(got, want, re.compile(r"Sparse fea|Randomized|Defined|Split data|Testing at|accuracy|^recall "), 1e-5)
    assert _report(got)[0] > 0 and _report(got)[2] > 0


@pytest.mark.parametrize("tag", ["K", "T1", "T2", "T3"])
def test_cli_days_graphed_matches_the_reference_run(tmp_path, tag):
    raw = write_days(tmp_path, "kaggle" if tag == "K" else "terabyte")
    extra = ["--gemm=simt", "--cuda-graph-steps"] + (
        ["--load-model=" + os.path.join(days_cli.GOLD, "cli_days_T1_ref.pt")] if tag == "T3" else [])
    got = days_cli._cli(tag, raw, extra)
    want = open(os.path.join(days_cli.GOLD, "cli_days_%s.txt" % tag)).read()
    other = re.compile(r"Sparse features|Testing at|accuracy|^recall |Saved at|Training state|Testing state|"
                       r"Testing for inference")
    if tag == "T3":         # inference only: no loss lines
        assert [ln for ln in got.splitlines() if other.search(ln)] == \
            [ln for ln in want.splitlines() if other.search(ln)]
    else:
        _compare(got, want, other, 1e-5)
    assert _report(got)[2] > 0


def test_cli_bin_graphed_matches_the_reference_run():
    got = bin_cli._cli(["--gemm=simt", "--cuda-graph-steps"])
    want = open(os.path.join(bin_cli.GOLD, "cli_bin_A.txt")).read()
    want_loss = [float(v) for v in re.findall(r"loss ([0-9.]+)", want)]
    got_loss = [float(v) for v in re.findall(r"Finished training it .* loss ([0-9.]+)", got)]
    np.testing.assert_allclose(got_loss, want_loss, rtol=0, atol=2e-5)
    assert re.findall(r"Testing at - .*", got) == re.findall(r"Testing at - .*", want)
    w, g = bin_cli._metrics(want), bin_cli._metrics(got)
    assert len(g) == len(w) == 8
    unit = np.array([1e-4] * 6 + [1e-3] * 2)
    for a, b in zip(g, w):
        assert (np.abs(np.array(a) - np.array(b)) <= unit * 1.0001).all(), (a, b)
    assert _report(got)[0] > 0


def test_cli_short_last_batches_run_eager_and_are_counted():
    """30 train batches of 37 samples and test batches of 45 leave a short last batch in both splits."""
    got = kaggle_cli._cli("A", ["--gemm=simt", "--cuda-graph-steps", "--mini-batch-size=37",
                                "--test-mini-batch-size=45", "--nepochs=1"])
    from dlrm_b200 import criteo

    np.random.seed(727)
    train = criteo.CriteoDataset("kaggle", -1, 0.0, "total", "train", kaggle_cli.RAW, kaggle_cli.PRO)
    test = criteo.CriteoDataset("kaggle", -1, 0.0, "total", "test", kaggle_cli.RAW, kaggle_cli.PRO, data=train)
    assert len(train) % 37 and len(test) % 45
    n_train, n_test = -(-len(train) // 37), -(-len(test) // 45)
    passes = len(re.findall(r"Testing at", got))
    assert passes > 0
    assert _report(got) == [n_train - 1, 1, passes * (n_test - 1), passes]
    assert all(np.isfinite(float(v)) for v in _LOSS.findall(got))


@pytest.mark.parametrize("first", ["graph", "eager"])
def test_cli_checkpoints_resume_across_modes(tmp_path, first):
    """Epoch 0 in one mode, saved; epoch 1 resumed from the checkpoint in the other: the losses of epoch 1 are the
    recorded 2-epoch run's."""
    ck = str(tmp_path / "ck.pt")
    flag = {"graph": ["--cuda-graph-steps"], "eager": []}
    second = "eager" if first == "graph" else "graph"
    kaggle_cli._cli("A", ["--gemm=simt", "--nepochs=1", "--test-freq=-1", "--save-model=" + ck] + flag[first])
    got = kaggle_cli._cli("A", ["--gemm=simt", "--test-freq=-1", "--load-model=" + ck] + flag[second])
    want = open(os.path.join(kaggle_cli.GOLD, "cli_kaggle_A.txt")).read().splitlines()
    want_loss = [float(_LOSS.match(ln).group(1)) for ln in want if _LOSS.match(ln) and "of epoch 1," in ln]
    got_loss = [float(_LOSS.match(ln).group(1)) for ln in got.splitlines() if _LOSS.match(ln)]
    assert len(got_loss) == len(want_loss) > 0
    np.testing.assert_allclose(got_loss, want_loss, rtol=0, atol=1e-5)
    if second == "graph":
        assert _report(got)[0] > 0
