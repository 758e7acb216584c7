"""Learned weighted pooling on the GPU: the fused update's v_W_l step (row_weights / row_weight_sum of
dlrm_emb_bwd_table_t) against the float64 restatement (oracle/learned_f64.py) on every update path, DLRM_Net training
against the live reference's recorded runs (tests/golden/cfg0_learned.npz), graph replays against eager steps, and the
command line against the reference command line (tests/golden/cli_cfg0_W*)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from golden_util import Golden
from oracle.learned_f64 import OPT_ADAGRAD, learned_step_f64
from oracle.sparse_f64 import OPT_RWSADAGRAD, OPT_SGD

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
_OPT = {"sgd": OPT_SGD, "rwsadagrad": OPT_RWSADAGRAD, "adagrad": OPT_ADAGRAD}
LN = [5000, 3000, 200]          # two list-path tables, one tiny table (<= 256 rows: the two-pass update)


def _sparse(rng, B):
    """Bags of 0..10 uniform rows, then: row 7 of table 0 in 40 bags (a list longer than 32, the fixed-point sum),
    rows 1..5 of tables 0 and 1 in 2..20 bags each; every row of the tiny table occurs many times."""
    from dlrm_b200.engine import sparse_from_reference

    offs, idxs = [], []
    for k, n in enumerate(LN):
        lens = rng.integers(0, 11, size=B)
        bags = [list(rng.integers(0, n, size=int(m))) for m in lens]
        if k < 2:
            for r, c in ((7, 40 if k == 0 else 0), (1, 2), (2, 5), (3, 12), (4, 20), (5, 32)):
                for b in rng.choice(B, size=c, replace=False):
                    bags[b].append(r)
        idx = np.array([r for bag in bags for r in bag], dtype=np.int64)
        off = np.concatenate([[0], np.cumsum([len(b) for b in bags])[:-1]]).astype(np.int64)
        offs.append(off)
        idxs.append(idx)
    sp = sparse_from_reference([torch.from_numpy(o) for o in offs], [torch.from_numpy(i) for i in idxs], DEV)
    return sp, offs, idxs


def _learned_engine(D, dtype, opt, learned=True):
    from dlrm_b200.engine import Engine

    F = len(LN) + 1
    e = Engine(D, LN, [13, D], [D + F * (F - 1) // 2, 16, 1], sigmoid_top=1, device=DEV, max_batch=512, gemm="simt",
               emb_dtype=dtype, learned_row_weights=learned)
    e.init_params(seed=5)
    e.ensure_optimizer_state(opt)
    return e


def _acc_of(e, opt, k):
    return {"sgd": None, "rwsadagrad": lambda: e.momentum_of(k), "adagrad": lambda: e.accumulator_ew(k)}[opt]


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad", "adagrad"])
@pytest.mark.parametrize("dtype,D", [("fp32", 128), ("fp32", 16), ("fp32", 256), ("fp16", 128)])
@pytest.mark.parametrize("lr_dev", [False, True])
def test_update_matches_float64(opt, dtype, D, lr_dev):
    """D = 16 / 128: the lean kernel, D = 256: the general kernel, the 200-row table: the two-pass kernels; fp16 rows
    are widened for the dot product and stored with stochastic rounding.  Rows, row accumulators, v and its sum within
    fp32 (fp16: one fp16 ulp) of the float64 step; untouched rows and entries bit-identical to the inputs."""
    rng = np.random.default_rng(D + len(opt))
    B = 512
    e = _learned_engine(D, dtype, opt)
    sp, offs, idxs = _sparse(rng, B)
    with torch.no_grad():
        e.row_weights.copy_(torch.from_numpy(rng.uniform(0.5, 1.5, e.total_rows).astype(np.float32)))
        if e.row_weight_sum is not None:
            e.row_weight_sum.copy_(torch.from_numpy(rng.uniform(0.0, 1e-3, e.total_rows).astype(np.float32)))
        for k in range(len(LN)):
            a = _acc_of(e, opt, k)
            if a is not None:
                a().copy_(torch.from_numpy(rng.uniform(0.0, 1e-3, tuple(a().shape)).astype(np.float32)))
    dY = torch.from_numpy(rng.standard_normal((B, len(LN), D)).astype(np.float32) * 0.1).to(DEV)
    before = ([e.table(k).float().cpu().numpy() for k in range(len(LN))],
              [None if _acc_of(e, opt, k) is None else _acc_of(e, opt, k)().cpu().numpy() for k in range(len(LN))],
              e.row_weights.cpu().numpy(),
              None if e.row_weight_sum is None else e.row_weight_sum.cpu().numpy())
    lr = 0.05
    e.emb_link(sp)
    if lr_dev:          # the by-value rate is wrong on purpose: only the device float may reach the kernels
        e.lr_dev = torch.full((1,), lr, dtype=torch.float32, device=DEV)
    e.emb_update(sp, dY, len(LN) * D, D, optimizer=opt, lr=1e3 if lr_dev else lr)
    e.lr_dev = None
    torch.cuda.synchronize()
    assert int(e.head.abs().sum().item()) == 0
    W0, A0, V0, S0 = before
    rtol, atol = (2e-3, 1e-4) if dtype == "fp16" else (1e-4, 1e-6)
    for k in range(len(LN)):
        lo, hi = int(e.row_base[k]), int(e.row_base[k + 1])
        W2, A2, V2, S2, rows = learned_step_f64(W0[k], A0[k], V0[lo:hi], None if S0 is None else S0[lo:hi],
                                                idxs[k], offs[k], idxs[k].size, dY[:, k, :].cpu().numpy(),
                                                _OPT[opt], lr, 1e-10)
        got_w = e.table(k).float().cpu().numpy()
        got_v = e.row_weights[lo:hi].cpu().numpy()
        np.testing.assert_allclose(got_w[rows], W2[rows], rtol=rtol, atol=atol)
        np.testing.assert_allclose(got_v[rows], V2[rows], rtol=1e-4, atol=1e-6)
        if A0[k] is not None:
            np.testing.assert_allclose(_acc_of(e, opt, k)().cpu().numpy()[rows], A2[rows], rtol=1e-4, atol=1e-12)
        if S0 is not None:
            np.testing.assert_allclose(e.row_weight_sum[lo:hi].cpu().numpy()[rows], S2[rows], rtol=1e-4, atol=1e-12)
        un = np.setdiff1d(np.arange(LN[k]), rows)
        assert un.size > 0 or k == 2
        assert np.array_equal(got_w[un], W0[k][un]) and np.array_equal(got_v[un], V0[lo:hi][un])
        if A0[k] is not None:
            assert np.array_equal(_acc_of(e, opt, k)().cpu().numpy()[un], A0[k][un])
        if S0 is not None:
            assert np.array_equal(e.row_weight_sum[lo:hi].cpu().numpy()[un], S0[lo:hi][un])


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad", "adagrad"])
@pytest.mark.parametrize("D", [16, 128, 256])
def test_weights_of_one_leave_the_rows_of_the_unweighted_update(opt, D):
    """v = 1 scales S exactly: the rows and accumulators equal those of the row_weights == NULL kernels bit for bit."""
    rng = np.random.default_rng(3)
    B = 512
    sp, _, _ = _sparse(rng, B)
    dY = torch.from_numpy(rng.standard_normal((B, len(LN), D)).astype(np.float32) * 0.1).to(DEV)
    res = []
    for learned in (False, True):
        e = _learned_engine(D, "fp32", opt, learned)
        e.emb_link(sp)
        e.emb_update(sp, dY, len(LN) * D, D, optimizer=opt, lr=0.05)
        torch.cuda.synchronize()
        res.append([e.table(k).clone() for k in range(len(LN))] +
                   [_acc_of(e, opt, k)().clone() for k in range(len(LN)) if _acc_of(e, opt, k) is not None])
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_duplicate_filter_and_peer_update_refuse_row_weights():
    from dlrm_b200 import _lib

    d = (_lib.EmbBwdTable * 1)()
    v = torch.ones(8, device=DEV)
    w = torch.zeros(8, 16, device=DEV)
    idx = torch.zeros(1, dtype=torch.int64, device=DEV)
    d[0].weight, d[0].indices, d[0].offsets, d[0].nnz, d[0].rows = w.data_ptr(), idx.data_ptr(), idx.data_ptr(), 1, 8
    d[0].row_weights = v.data_ptr()
    lib = _lib.lib()
    flags = torch.zeros(4, dtype=torch.uint8, device=DEV)
    dd = _lib.EmbDedup(flags.data_ptr(), 0, flags.data_ptr(), flags.data_ptr())
    link = torch.zeros(4, dtype=torch.int32, device=DEV)
    dy = torch.zeros(16, device=DEV)
    import ctypes as C

    rc = lib.dlrm_b200_emb_bwd_update(d, 1, 16, 1, 8, 0, link.data_ptr(), dy.data_ptr(), 16, 0, 0, 0.1, 1e-10,
                                      C.byref(dd), torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and b"duplicate filter" in lib.dlrm_b200_last_error()
    peers = (C.c_void_p * 1)(dy.data_ptr())
    rc = lib.dlrm_b200_emb_bwd_update_p2p(d, 1, 16, 1, 8, 0, link.data_ptr(), peers, 1, 1, 16, 0, 0, 0.1, 1e-10,
                                          None, torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and b"row_weights" in lib.dlrm_b200_last_error()


# ---------------------------------------------------------------------------------------------- DLRM_Net
def _net(g):
    from dlrm_b200.dlrm_net import DLRM_Net

    np.random.seed(1)
    net = DLRM_Net(g.m_spa, np.array(g.ln_emb), np.array(g.ln_bot), np.array(g.ln_top), arch_interaction_op="dot",
                   sigmoid_bot=-1, sigmoid_top=len(g.ln_top) - 2, loss_function="bce", device=DEV, gemm="tc",
                   max_batch=g.B, weighted_pooling="learned")
    p = g.params()
    sd = {}
    for k, W in enumerate(p["emb"]):
        sd[f"emb_l.{k}.weight"] = torch.from_numpy(W)
    for k, v in enumerate(p["v_W_l"]):
        sd[f"v_W_l.{k}"] = torch.from_numpy(v)
    for nm in ("bot", "top"):
        for i, (W, b) in enumerate(p[nm]):
            sd[f"{nm}_l.{2 * i}.weight"] = torch.from_numpy(W)
            sd[f"{nm}_l.{2 * i}.bias"] = torch.from_numpy(b)
    assert list(net.state_dict().keys()) == list(sd.keys())     # the reference's keys, in its order
    net.load_state_dict(sd)
    return net


def _batch(g, s):
    X, off, idx, T = g.batch(s)
    return (torch.from_numpy(X), torch.from_numpy(np.stack(off)), [torch.from_numpy(i) for i in idx],
            torch.from_numpy(T))


@pytest.mark.parametrize("optname", ["sgd", "rwsadagrad", "adagrad"])
def test_module_training_follows_the_reference(optname):
    from dlrm_b200 import optim as fused

    g = Golden("cfg0_learned")
    net = _net(g)
    assert isinstance(net.v_W_l, torch.nn.ParameterList)
    names = [n for n, _ in net.named_parameters()]
    assert names[g.T:2 * g.T] == [f"v_W_l.{k}" for k in range(g.T)]
    cls = {"sgd": fused.SGD, "rwsadagrad": fused.RWSAdagrad, "adagrad": fused.Adagrad}[optname]
    opt = cls(net.parameters(), lr=float(g[f"{optname}_lr"]))
    losses = []
    for s in range(g.nsteps):
        X, lS_o, lS_i, T = _batch(g, s)
        E = net.loss_fn(net(X, lS_o, lS_i), T.to(DEV))
        losses.append(float(E.item()))
        opt.zero_grad()
        E.backward()
        opt.step()
        if not g.has(f"{optname}{s}_emb0"):
            continue
        tol = dict(rtol=1e-3, atol=2e-5 if s == 0 else 2e-4)
        st = opt.state_dict()["state"] if optname != "sgd" else {}
        for k in range(g.T):
            np.testing.assert_allclose(net.emb_l[k].weight.detach().cpu().numpy(), g[f"{optname}{s}_emb{k}"], **tol)
            np.testing.assert_allclose(net.v_W_l[k].detach().cpu().numpy(), g[f"{optname}{s}_v{k}"], **tol)
            if optname == "rwsadagrad":
                assert set(st[k]) == {"step", "momentum"} and set(st[g.T + k]) == {"step", "sum"}
                np.testing.assert_allclose(st[k]["momentum"].cpu().numpy(), g[f"{optname}{s}_mom{k}"], rtol=2e-3,
                                           atol=1e-7)
            if optname == "adagrad":
                np.testing.assert_allclose(st[k]["sum"].cpu().numpy(), g[f"{optname}{s}_acc{k}"], rtol=2e-3, atol=1e-7)
            if optname != "sgd":
                assert tuple(st[g.T + k]["sum"].shape) == (g.ln_emb[k],)
                np.testing.assert_allclose(st[g.T + k]["sum"].cpu().numpy(), g[f"{optname}{s}_vsum{k}"], rtol=2e-3,
                                           atol=1e-7)
    np.testing.assert_allclose(losses, g[f"{optname}_losses"], rtol=0, atol=2e-5 if optname == "sgd" else 3e-4)


def test_backward_without_a_fused_optimizer_names_them():
    g = Golden("cfg0_learned")
    net = _net(g)
    X, lS_o, lS_i, T = _batch(g, 0)
    with pytest.raises(RuntimeError, match="fused optimizers"):
        net.loss_fn(net(X, lS_o, lS_i), T.to(DEV)).backward()


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad", "adagrad"])
def test_graphed_steps_with_device_lr_equal_eager_steps(opt):
    """GraphedTrainStep(device_lr=True) replays over a changing schedule == eager train_step calls: losses, tables,
    accumulators, v and its sum, bit for bit."""
    from dlrm_b200.data import make_batch, to_device_packed
    from dlrm_b200.engine import Engine, GraphedTrainStep

    rng = np.random.default_rng(9)
    bs = [to_device_packed(make_batch(rng, LN, 256, lmax=6), DEV) for _ in range(7)]
    lrs = [0.02, 0.04, 0.06, 0.05, 0.03, 0.01]
    decay = 0.1 if opt != "sgd" else 0.0
    v0 = torch.from_numpy(rng.uniform(0.5, 1.5, sum(LN)).astype(np.float32))
    res = []
    for mode in ("eager", "graph"):
        D, F = 32, len(LN) + 1
        e = Engine(D, LN, [13, 64, D], [D + F * (F - 1) // 2, 64, 1], sigmoid_top=1, device=DEV, max_batch=256,
                   gemm="tc", learned_row_weights=True)
        e.init_params(seed=3)
        with torch.no_grad():
            e.row_weights.copy_(v0)
        e.ensure_optimizer_state(opt)
        for b in bs:
            e.prepare(b.sparse, True)
        if mode == "graph":
            st = bs[6]
            gs = GraphedTrainStep(e, st, 0.5, opt, warmup=0, device_lr=True)
        losses = []
        for i, lr in enumerate(lrs):
            if mode == "eager":
                losses.append(e.train_step(bs[i].X, bs[i].sparse, bs[i].target, lr, opt, lr_decay=decay).clone())
            else:
                st.buf.copy_(bs[i].buf)
                losses.append(gs.replay(lr, decay).clone())
        torch.cuda.synchronize()
        state = [e.tables.clone(), e.row_weights.clone(), e.dense.clone()]
        if e.row_weight_sum is not None:
            state.append(e.row_weight_sum.clone())
        if opt == "adagrad":
            state.append(e.acc_ew.clone())
        res.append((torch.stack(losses), state))
    assert torch.equal(res[0][0], res[1][0])
    for a, b in zip(res[0][1], res[1][1]):
        assert torch.equal(a, b)
    assert not torch.equal(res[0][1][1], torch.ones_like(res[0][1][1]))


# ---------------------------------------------------------------------------------------------- command line
_CLI_BASE = ["--arch-sparse-feature-size=16", "--arch-embedding-size=1000-1000-1000", "--arch-mlp-bot=13-512-256-64-16",
             "--arch-mlp-top=512-256-1", "--mini-batch-size=128", "--data-generation=random", "--num-batches=6",
             "--print-freq=1", "--learning-rate=0.1", "--numpy-rand-seed=727", "--use-gpu"]


def _flags(tag):
    return open(os.path.join(ROOT, "tests", "golden", f"cli_cfg0_{tag}.flags")).read().split()


def _cli(args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py")] + args, capture_output=True,
                       text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def _compare_lines(got_txt, tag, atol):
    want = [ln for ln in open(os.path.join(ROOT, "tests", "golden", f"cli_cfg0_{tag}.txt")).read().splitlines()]
    got = [ln for ln in got_txt.splitlines() if re.match(r"Finished| accuracy|Testing at|Saving model", ln)]
    assert len(got) == len(want), got_txt
    for a, b in zip(got, want):
        if a.startswith("Finished"):
            la, lb = float(a.rsplit(" ", 1)[1]), float(b.rsplit(" ", 1)[1])
            assert a.rsplit(" ", 1)[0] == b.rsplit(" ", 1)[0] and abs(la - lb) < atol, (a, b)
        elif a.startswith("Saving model"):
            assert b.startswith("Saving model")
        else:
            assert a == b


@pytest.mark.parametrize("tag,atol", [("W2", 3e-4), ("W3", 3e-4)])
def test_cli_adagrad_variants_follow_the_reference(tag, atol):
    _compare_lines(_cli(_CLI_BASE + _flags(tag)), tag, atol)


def test_cli_test_pass_and_checkpoint_follow_the_reference(tmp_path):
    """W1 (sgd, --test-freq=3): the printed lines equal the reference's, and the checkpoint written here has the
    reference checkpoint's keys, shapes and order, with v_W_l.{k} of shape [n_k] after the tables."""
    ck = str(tmp_path / "ours.pt")
    _compare_lines(_cli(_CLI_BASE + _flags("W1") + ["--save-model=" + ck]), "W1", 2e-5)
    ref = torch.load(os.path.join(ROOT, "tests", "golden", "cli_cfg0_W1_ref.pt"), map_location="cpu",
                     weights_only=False)
    ours = torch.load(ck, map_location="cpu", weights_only=False)
    assert set(ours) == set(ref)
    assert list(ours["state_dict"]) == list(ref["state_dict"])
    assert [k for k in ref["state_dict"] if k.startswith("v_W_l")] == ["v_W_l.0", "v_W_l.1", "v_W_l.2"]
    for k, v in ref["state_dict"].items():
        assert tuple(ours["state_dict"][k].shape) == tuple(v.shape)
        np.testing.assert_allclose(ours["state_dict"][k].numpy(), v.numpy(), rtol=0, atol=1e-4)
    assert ours["opt_state_dict"]["param_groups"][0]["params"] == ref["opt_state_dict"]["param_groups"][0]["params"]


def test_cli_loads_a_reference_checkpoint_and_trains_on(tmp_path):
    """The reference's W1 checkpoint (v_W_l trained by the reference) loads for inference -- the accuracy it recorded
    -- and resumes training: batches 1-6 are skipped, 7-9 train."""
    ck = os.path.join(ROOT, "tests", "golden", "cli_cfg0_W1_ref.pt")
    flags = [f for f in _flags("W1") if not f.startswith("--test-freq")]
    out = _cli(_CLI_BASE + flags + ["--load-model=" + ck, "--inference-only"])
    ref = torch.load(ck, map_location="cpu", weights_only=False)
    assert " accuracy %.3f %%" % (100 * float(ref["test_acc"])) in out
    base = [a for a in _CLI_BASE if not a.startswith("--num-batches")]
    out = _cli(base + flags + ["--num-batches=9", "--load-model=" + ck])
    losses = re.findall(r"Finished training it (\d+)/9 of epoch 0, .* loss ([0-9.]+)", out)
    assert [int(i) for i, _ in losses] == [7, 8, 9] and all(np.isfinite(float(v)) for _, v in losses)


def test_cli_dataset_path_graphed_equals_eager():
    """--weighted-pooling=learned on the preprocessed Kaggle path (recorded run A's flags), --optimizer=rwsadagrad:
    CUDA-graph steps print the eager run's test lines and its losses within rounding (the graphed loss comes from the
    fused head), and replay every full-size batch."""
    import test_gpu_criteo_dataset as kaggle_cli

    extra = ["--gemm=simt", "--weighted-pooling=learned", "--optimizer=rwsadagrad"]
    eager = kaggle_cli._cli("A", extra)
    graph = kaggle_cli._cli("A", extra + ["--cuda-graph-steps"])
    loss = re.compile(r"Finished training it .* loss ([0-9.]+)")
    le, lg = [float(v) for v in loss.findall(eager)], [float(v) for v in loss.findall(graph)]
    assert len(le) == len(lg) > 0
    np.testing.assert_allclose(lg, le, rtol=0, atol=1e-5)
    other = re.compile(r"Testing at|accuracy")
    assert [ln for ln in graph.splitlines() if other.search(ln)] == [ln for ln in eager.splitlines() if other.search(ln)]
    assert int(re.search(r"CUDA-graph steps: (\d+) train steps replayed", graph).group(1)) > 0
