"""Training steps at CHANGING batch sizes on one engine, every step against the float64 step of oracle/dlrm_numpy.py
taken from the same parameters.

The weight-gradient GEMMs of the tensor-core back end reduce over the batch in split-K slabs.  A plan never launches
an empty split, so for 9 <= ceil(B / 64) <= 14 it writes fewer slabs than the 8 the engine asks for; whatever folds
the slabs must fold the ones the plan wrote.  An engine that has only ever seen one batch size cannot tell: the slabs
it never wrote still hold the zeros they were allocated with.

The reference takes its ReLU masks from the engine's own forward activations (relu_masks of dlrm_backward), so a
pre-activation within rounding of zero is not a disagreement and the bounds below are the GEMM error model's:
a gradient element is off by at most EPS[gemm] of its tensor's largest element, and that error goes through the
optimizer's derivative.  Worst err / bound ratios are printed."""
import copy
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import dlrm_numpy as O

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
# exact in fp32.  Adagrad's first step moves every dense parameter by lr, whatever its gradient: small enough to keep
# the model out of saturation over a sequence; SGD's is large enough to lift lr * (gradient error) above an ulp
LRS = {"sgd": 2.0 ** -3, "rwsadagrad": 2.0 ** -10}
# gradient error relative to the largest element of its tensor: bf16x3 drops lo*lo (2^-16 per product) and carries
# activations / gradients as (hi, lo) pairs (2^-17); plain bf16 operands round at 2^-9 through up to 7 GEMMs; fp32
EPS = {"tc": 2e-4, "tc_bf16": 5e-2, "simt": 2e-5}
LOSS_TOL = {"tc": 1e-5, "tc_bf16": 2e-2, "simt": 1e-5}       # of max(1, loss)


def _shape(D, ln_emb, ln_bot, tail):
    F = len(ln_emb) + 1
    return D, ln_emb, ln_bot, [D + F * (F - 1) // 2] + tail


SHAPES = {
    "cfg0": _shape(16, [1000, 1000, 1000], [13, 512, 256, 64, 16], [512, 256, 1]),
    # MLPerf MLP widths over 26 small tables (some take the dense small-table update, some the row lists):
    # 32 and 36 tiles in the first two top layers -> 4 slabs asked, 3 written at 9 k blocks
    "cfg2": _shape(128, [60 + 37 * k for k in range(26)], [13, 512, 256, 128], [1024, 512, 256, 1]),
    # a 1280 x 1537 weight gradient: 130 tiles, one slab, beside layers that ask for 8
    "wide": _shape(32, [500, 300, 70], [13, 96, 32], [1536, 1280, 1]),
}
SEQUENCES = [
    ("tc", "cfg0", [1024, 700]), ("tc", "cfg0", [1024, 700, 1024]), ("tc", "cfg0", [2048, 576, 640, 896, 513]),
    ("tc", "cfg0", [700]), ("tc", "cfg0", [128, 1, 128]), ("tc", "cfg0", [300, 8, 63, 64, 65]),
    ("tc", "cfg2", [1024, 700]), ("tc", "cfg2", [2048, 576, 640, 896, 513]),
    ("tc", "wide", [1024, 700, 1024]), ("tc", "wide", [300, 8, 63, 64, 65]),
    ("tc_bf16", "cfg0", [1024, 700]), ("tc_bf16", "cfg2", [2048, 576, 640, 896, 513]),
    ("simt", "cfg0", [1024, 700]), ("simt", "cfg0", [128, 1, 128]),
]


def _batch(rng, ln_emb, ln_bot, B):
    X, off, idx = O.random_batch(rng, ln_emb, B, ln_bot[0], 6)
    return X, off, idx, np.round(rng.random((B, 1))).astype(np.float32)


# ------------------------------------------------------------------------------------------ the float64 step
def _ref_step(params, state, batch, opt, relu_masks=None):
    """One float64 step in place on (params, state); returns the backward's results."""
    X, off, idx, tgt = batch
    return O.train_step(params, state, X.astype(np.float64), off, idx, tgt.astype(np.float64), lr=LRS[opt], optimizer=opt,
                        loss="bce", dtype=np.float64, relu_masks=relu_masks)


def _ulp(x):
    return 2.0 ** -22 * np.abs(x)


def _ratio(got, want, bound, what):
    from oracle.dense_f64 import check_within

    return check_within(got, want, bound, what)


def compare_step(got, before, after, r, batch, opt, eps, D):
    """got / before / after: dict(params, state) of the implementation after the step and of the float64 model before
    and after it; r: the reference backward.  Returns the worst err / bound ratio of every family."""
    worst, LR = {}, LRS[opt]

    def note(fam, v):
        worst[fam] = max(worst.get(fam, 0.0), v)

    for nm in ("bot", "top"):
        for i, grads in enumerate(r[nm + "_grads"]):
            for j, kind in enumerate("Wb"):
                g = grads[j]
                dg = eps * np.abs(g).max()
                p2, what = after["params"][nm][i][j], "%s %s%d" % (nm, kind, i)
                if opt == "sgd":
                    bound = LR * dg + _ulp(p2)
                else:   # p -= lr g / (sqrt(s + g^2) + eps): |d/dg| <= 1 / sqrt(s2); two steps are at most 2 lr apart
                    s2 = after["state"][nm][i][j]
                    bound = LR * np.minimum(2.5, 2.0 * dg / np.sqrt(np.maximum(s2, 1e-300))) + _ulp(p2)
                    note("dense state", _ratio(got["state"][nm][i][j], s2, 2 * np.abs(g) * dg + dg * dg + _ulp(s2),
                                               what + " state"))
                note("dense", _ratio(got["params"][nm][i][j], p2, bound, what))
    _, off, idx, _ = batch
    for k in range(len(idx)):
        rows, g = O.coalesce(*O.sparse_grad(idx[k], off[k], r["d_ly"][k]))
        dg = eps * np.abs(g).max()
        w2 = after["params"]["emb"][k][rows]
        if opt == "sgd":
            bound = LR * dg + 4 * _ulp(w2)      # a row met n times may be rounded n times
        else:   # w -= lr g / (sqrt(m) + eps), m += mean_d g^2: |g_j| <= sqrt(D m), so both factors move by dg / sqrt(m)
            m2, m0 = after["state"]["mom"][k][rows], before["state"]["mom"][k][rows]
            rel = dg / np.sqrt(np.maximum(m2, 1e-300))
            bound = LR * np.minimum(2.0 * np.sqrt(D), (1.0 + np.sqrt(D)) * rel)[:, None] + 4 * _ulp(w2)
            note("accumulator", _ratio(got["state"]["mom"][k][rows], m2,
                                       2 * np.sqrt(m2 - m0) * dg + dg * dg + _ulp(m2), "accumulator %d" % k))
        note("emb rows", _ratio(got["params"]["emb"][k][rows], w2, bound, "table %d" % k))
        untouched = np.ones(after["params"]["emb"][k].shape[0], bool)
        untouched[rows] = False
        assert np.array_equal(got["params"]["emb"][k][untouched], before["params"]["emb"][k][untouched]), k
    return worst


# ------------------------------------------------------------------------------------------ the engine's side
def _engine(shape, gemm, max_batch, params):
    from dlrm_b200.engine import Engine

    D, ln_emb, ln_bot, ln_top = shape
    e = Engine(D, ln_emb, ln_bot, ln_top, loss="bce", sigmoid_top=len(ln_top) - 2, device=DEV, max_batch=max_batch,
               gemm=gemm)
    e.load_params(params)
    return e


def _dev(batch):
    from dlrm_b200.engine import sparse_from_reference

    X, off, idx, tgt = batch
    sp = sparse_from_reference([torch.from_numpy(o) for o in off], [torch.from_numpy(i) for i in idx], DEV)
    return torch.from_numpy(X).to(DEV), sp, torch.from_numpy(tgt).to(DEV)


def _snapshot(e):
    """Parameters and optimizer state of the engine as float64 numpy, in the oracle's layout."""
    f = lambda t: t.detach().double().cpu().numpy()
    zeros = torch.zeros_like(e.dense)
    st = e.dense_state if e.dense_state is not None else zeros
    params = dict(emb=[f(e.table(k)) for k in range(e.T)], bot=[], top=[], v_W_l=None)
    state = dict(step=e.opt_step, mom=[], bot=[], top=[])
    mom = e.momentum
    for k in range(e.T):
        lo, hi = int(e.row_base[k]), int(e.row_base[k + 1])
        state["mom"].append(f(mom[lo:hi]) if mom is not None else np.zeros(hi - lo))
    sl = {(name, i, kind): (o, shape) for name, i, kind, o, shape in e.dense_slices}
    for nm in ("bot", "top"):
        for i in range(len(e.W[nm])):
            view = lambda t, kind: f(t[sl[(nm, i, kind)][0]:][:int(np.prod(sl[(nm, i, kind)][1]))]).reshape(sl[(nm, i, kind)][1])
            params[nm].append((view(e.dense, "W"), view(e.dense, "b")))
            state[nm].append((view(st, "W"), view(st, "b")))
    return dict(params=params, state=state)


def _relu_outputs(e, B):
    """Post-activation outputs of every ReLU layer as the engine's last forward left them, with the sign its backward
    tested: the hi half of the next tensor-core layer's operand pair (the dgrad epilogue masks on mask_hi > 0; -0.0,
    subnormal hi and the other edges are tests/test_gpu_gemm_tc_edges.py's), or the fp32 activation buffers."""
    out = {}
    for nm, ln, acts in (("bot", e.ln_bot, e.bot_act), ("top", e.ln_top, e.top_act)):
        nl, ys = len(ln) - 1, []
        for i in range(nl):
            if nm == "top" and i == nl - 1:
                ys.append(None)                                    # the sigmoid output
            elif nm == "bot" and i == nl - 1:
                ys.append(e.Tbuf[:B, 0, :].double().cpu().numpy())
            elif e.tc and i + 1 < e.ntc[nm]:
                ys.append(e.tc_in[nm][i + 1][0][:B, :ln[i + 1]].double().cpu().numpy())
            else:
                ys.append(acts[i][:B, :ln[i + 1]].double().cpu().numpy())
        out[nm] = ys
    return out


def _run_sequence(gemm, shape, seq, opt, seed=0):
    D, ln_emb, ln_bot, ln_top = shape
    rng = np.random.default_rng(seed)
    e = _engine(shape, gemm, max(seq), O.random_params(rng, D, ln_emb, ln_bot, ln_top))
    worst = {}
    for step, B in enumerate(seq):
        batch = _batch(rng, ln_emb, ln_bot, B)
        before = _snapshot(e)
        X, sp, T = _dev(batch)
        loss = float(e.train_step(X, sp, T, LRS[opt], opt).item())
        torch.cuda.synchronize()
        got = _snapshot(e)
        after = copy.deepcopy(before)
        r = _ref_step(after["params"], after["state"], batch, opt, _relu_outputs(e, B))
        assert abs(loss - float(r["loss"])) <= LOSS_TOL[gemm] * max(1.0, float(r["loss"])), (step, B, loss, float(r["loss"]))
        try:
            w = compare_step(got, before, after, r, batch, opt, EPS[gemm], D)
        except AssertionError as err:
            raise AssertionError("step %d (B=%d) of %s: %s" % (step, B, seq, err)) from None
        for k, v in w.items():
            worst[k] = max(worst.get(k, 0.0), v)
        assert int(e.head.abs().sum().item()) == 0, "row-list heads not reset"
    print("%s %s: worst err/bound %s" % (gemm, seq, {k: "%.3g" % v for k, v in sorted(worst.items())}))
    return e


@gpu
@pytest.mark.parametrize("gemm,shape,seq", SEQUENCES, ids=["%s-%s-%s" % (g, s, "_".join(map(str, q))) for g, s, q in SEQUENCES])
def test_batch_sequence_vs_float64_step(gemm, shape, seq):
    _run_sequence(gemm, SHAPES[shape], seq, "rwsadagrad")


@gpu
@pytest.mark.parametrize("gemm", ["tc", "simt"])
def test_batch_sequence_sgd(gemm):
    """SGD: the parameter error is lr times the gradient error, nothing to condition."""
    _run_sequence(gemm, SHAPES["cfg0"], [1024, 700, 576], "sgd")


# ------------------------------------------------------------------------------------------ the invariant itself
@gpu
@pytest.mark.parametrize("shape", ["cfg2", "wide"])
def test_engine_folds_the_slabs_its_plans_write(shape):
    """For every k-block count 1..32 of the weight-gradient GEMMs and the batch sizes either side of each boundary."""
    sh = SHAPES[shape]
    rng = np.random.default_rng(1)
    e = _engine(sh, "tc", 2049, O.random_params(rng, *sh))
    seen = set()
    for B in sorted({b for kb in range(1, 33) for b in (64 * kb - 1, 64 * kb, 64 * kb + 1)}):
        e._tc_setup(B)
        for key, plan in e.tc_plans["wgrad"].items():
            info = plan.info()
            num_kb = (B + 63) // 64
            ask = int(plan.desc.split_k)
            per = -(-num_kb // min(ask, num_kb))
            assert info["splits"] == -(-num_kb // per), (B, key, info)
            assert e.tc_splits[key] == info["splits"], (B, key, e.tc_splits[key], info)
            seen.add((ask, info["splits"]))
        assert e.dense_grad.numel() >= max(e.tc_splits.values()) * e.dense_numel
    assert any(a != s for a, s in seen), "no batch size of the sweep made a plan write fewer slabs than asked"


@gpu
@pytest.mark.parametrize("gemm", ["tc", "tc_bf16"])
@pytest.mark.parametrize("B", [700, 576, 2048, 65])
def test_step_does_not_depend_on_what_the_gradient_slabs_held(gemm, B):
    """NaN in every gradient slab before the step == zeros before the step, bit for bit."""
    sh = SHAPES["cfg2"]
    D, ln_emb, ln_bot, ln_top = sh
    res = []
    for fill in (0.0, float("nan")):
        rng = np.random.default_rng(2)
        e = _engine(sh, gemm, B, O.random_params(rng, D, ln_emb, ln_bot, ln_top))
        X, sp, T = _dev(_batch(rng, ln_emb, ln_bot, B))
        e.prepare(sp, True, batch=B)
        e.dense_grad.fill_(fill)
        loss = e.train_step(X, sp, T, LRS["rwsadagrad"], "rwsadagrad").clone()
        torch.cuda.synchronize()
        res.append((loss, e.dense.clone(), e.dense_state.clone(), e.tables.clone()))
    for a, b in zip(*res):
        assert bool(torch.isfinite(b.float()).all()), "a never-written gradient slab reached the parameters"
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------ forward / eval between
@gpu
def test_forward_at_one_batch_train_at_another():
    sh = SHAPES["cfg0"]
    D, ln_emb, ln_bot, ln_top = sh
    rng = np.random.default_rng(3)
    params = O.random_params(rng, D, ln_emb, ln_bot, ln_top)
    big, small, warm = (_batch(rng, ln_emb, ln_bot, b) for b in (2048, 700, 2048))
    e = _engine(sh, "tc", 2048, params)
    Xw, spw, Tw = _dev(warm)
    e.train_step(Xw, spw, Tw, LRS["sgd"], "sgd")            # every slab written once
    Xb, spb, _ = _dev(big)
    for _ in range(2):
        p = e.forward(Xb, spb).double().cpu().numpy()
        snap = _snapshot(e)
        want = O.dlrm_forward(snap["params"], big[0].astype(np.float64), big[1], big[2], dtype=np.float64)
        np.testing.assert_allclose(p, want, rtol=0, atol=1e-5)
        X, sp, T = _dev(small)
        e.train_step(X, sp, T, LRS["sgd"], "sgd")
        torch.cuda.synchronize()
        got, after = _snapshot(e), copy.deepcopy(snap)
        r = _ref_step(after["params"], after["state"], small, "sgd", _relu_outputs(e, 700))
        compare_step(got, snap, after, r, small, "sgd", EPS["tc"], D)


@gpu
def test_module_evaluated_at_one_batch_trained_at_another():
    """DLRM_Net: training steps at 1024 and 700, and between them the module in eval() at a test batch of 2048, once
    under no_grad and once with grad enabled (the reference's inference loop runs without no_grad; the module then
    also threads the row lists of a training forward, the harder case).  The tensor-core module follows the fp32
    CUDA-core one (no slabs) within the bf16x3 drift."""
    from dlrm_b200 import optim as fused
    from dlrm_b200.dlrm_net import DLRM_Net

    D, ln_emb, ln_bot, ln_top = SHAPES["cfg0"]
    rng = np.random.default_rng(4)
    params = O.random_params(rng, D, ln_emb, ln_bot, ln_top)
    sd = {"emb_l.%d.weight" % k: torch.from_numpy(W) for k, W in enumerate(params["emb"])}
    for nm in ("bot", "top"):
        for i, (W, b) in enumerate(params[nm]):
            sd["%s_l.%d.weight" % (nm, 2 * i)], sd["%s_l.%d.bias" % (nm, 2 * i)] = torch.from_numpy(W), torch.from_numpy(b)
    batches = [_batch(rng, ln_emb, ln_bot, b) for b in (1024, 700, 700, 700)]
    ev = _batch(rng, ln_emb, ln_bot, 2048)
    t = lambda b: (torch.from_numpy(b[0]), torch.from_numpy(np.stack(b[1])), [torch.from_numpy(i) for i in b[2]])
    out = {}
    for gemm in ("tc", "simt"):
        net = DLRM_Net(D, np.array(ln_emb), np.array(ln_bot), np.array(ln_top), arch_interaction_op="dot",
                       arch_interaction_itself=False, sigmoid_bot=-1, sigmoid_top=len(ln_top) - 2, loss_threshold=0.0,
                       loss_function="bce", device=DEV, gemm=gemm, max_batch=2048)
        net.load_state_dict(sd)
        opt = fused.SGD(net.parameters(), lr=0.1)
        losses, evals = [], []
        for b in batches:
            net.train()
            E = net.loss_fn(net(*t(b)), torch.from_numpy(b[3]).to(DEV))
            losses.append(float(E.item()))
            opt.zero_grad()
            E.backward()
            opt.step()
            net.eval()
            with torch.no_grad():
                evals.append(net(*t(ev)).cpu().numpy())
            again = net(*t(ev)).detach().cpu().numpy()
            assert np.array_equal(again, evals[-1])
        out[gemm] = (losses, evals)
    np.testing.assert_allclose(out["tc"][0], out["simt"][0], rtol=0, atol=2e-5)
    for a, b in zip(out["tc"][1], out["simt"][1]):
        np.testing.assert_allclose(a, b, rtol=0, atol=5e-5)


@gpu
def test_graph_captured_after_a_batch_size_change_equals_eager():
    from dlrm_b200.data import DeviceBatch, make_batch
    from dlrm_b200.engine import GraphedTrainStep

    sh = SHAPES["cfg0"]
    D, ln_emb, ln_bot, ln_top = sh
    params = O.random_params(np.random.default_rng(5), D, ln_emb, ln_bot, ln_top)
    first = make_batch(np.random.default_rng(50), ln_emb, 1024, 13, 6)
    hbs = [make_batch(np.random.default_rng(51 + i), ln_emb, 700, 13, 6) for i in range(3)]
    res = []
    for mode in ("eager", "graph"):
        e = _engine(sh, "tc", 1024, params)
        s0 = DeviceBatch(first.layout, DEV)
        s0.load(first, non_blocking=False)
        losses = [float(e.train_step(s0.X, s0.sparse, s0.target, LRS["sgd"], "sgd").item())]
        st = DeviceBatch(hbs[0].layout, DEV)
        st.load(hbs[0], non_blocking=False)
        gs = GraphedTrainStep(e, st, LRS["sgd"], "sgd", warmup=0) if mode == "graph" else None
        for hb in hbs:
            st.load(hb, non_blocking=False)
            out = gs.replay() if gs else e.train_step(st.X, st.sparse, st.target, LRS["sgd"], "sgd")
            losses.append(float(out.item()))
        torch.cuda.synchronize()
        res.append((losses, e.dense.clone(), e.tables.clone()))
    assert res[0][0] == res[1][0]
    assert torch.equal(res[0][1], res[1][1]) and torch.equal(res[0][2], res[1][2])


@gpu
def test_cli_tail_batch_and_second_epoch_follow_the_fp32_run():
    """1724 samples in batches of 1024: a 700-sample tail, then a second epoch.  The tensor-core run's printed losses
    stay within the bf16x3 drift of the fp32 CUDA-core run, which has no slabs to fold."""
    got = {}
    for gemm in ("tc", "simt"):
        cmd = [sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py"), "--arch-sparse-feature-size=16",
               "--arch-embedding-size=1000-1000-1000", "--arch-mlp-bot=13-512-256-64-16", "--arch-mlp-top=512-256-1",
               "--mini-batch-size=1024", "--data-size=1724", "--nepochs=2", "--data-generation=random",
               "--print-freq=1", "--learning-rate=0.1", "--numpy-rand-seed=727", "--use-gpu", "--gemm", gemm]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        got[gemm] = [float(m.group(1)) for m in re.finditer(r"Finished training it \d+/2 of epoch \d, .* loss ([0-9.]+)",
                                                            r.stdout)]
        assert len(got[gemm]) == 4, r.stdout
    print("cli losses", got)
    np.testing.assert_allclose(got["tc"], got["simt"], rtol=0, atol=1e-4)


# ------------------------------------------------------------------------------------------ the comparison bites
def _sub_batch(batch, lo):
    X, off, idx, tgt = batch
    return X[lo:], [o[lo:] - o[lo] for o in off], [i[o[lo]:] for i, o in zip(idx, off)], tgt[lo:]


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad"])
def test_comparison_rejects_a_step_that_folds_two_stale_slabs(opt):
    """Host only.  A step at B = 700 whose dense gradients also contain slabs 6 and 7 of the previous step at
    B = 1024 (samples 768..1023, each slab 128 samples) is rejected by compare_step at the tensor-core tolerance; the
    same step computed in fp32 is accepted."""
    D, ln_emb, ln_bot, ln_top = _shape(16, [200, 100], [13, 64, 16], [64, 32, 1])
    rng = np.random.default_rng(6)
    p32 = O.random_params(rng, D, ln_emb, ln_bot, ln_top)
    prev, cur = _batch(rng, ln_emb, ln_bot, 1024), _batch(rng, ln_emb, ln_bot, 700)
    to64 = lambda p: dict(emb=[W.astype(np.float64) for W in p["emb"]], v_W_l=None,
                          **{nm: [(W.astype(np.float64), b.astype(np.float64)) for W, b in p[nm]] for nm in ("bot", "top")})
    st32 = O.new_state(p32)
    O.train_step(p32, st32, *prev, lr=np.float32(LRS[opt]), optimizer=opt, loss="bce")
    before = dict(params=to64(p32), state=dict(step=1, mom=[m.astype(np.float64) for m in st32["mom"]],
                                               **{nm: [(a.astype(np.float64), b.astype(np.float64)) for a, b in st32[nm]]
                                                  for nm in ("bot", "top")}))
    after = copy.deepcopy(before)
    r = _ref_step(after["params"], after["state"], cur, opt)
    # the honest fp32 step
    g32 = copy.deepcopy(st32)
    q32 = copy.deepcopy(p32)
    O.train_step(q32, g32, *cur, lr=np.float32(LRS[opt]), optimizer=opt, loss="bce", relu_masks=dict(
        bot=r["fwd"]["bot_acts"], top=r["fwd"]["top_acts"]))
    good = dict(params=to64(q32), state=dict(mom=g32["mom"], bot=g32["bot"], top=g32["top"]))
    compare_step(good, before, after, r, cur, opt, EPS["tc"], D)
    # the same with the stale slabs: a gradient over the previous batch's last 256 samples, a quarter of its mean
    X, off, idx, tgt = _sub_batch(prev, 768)
    stale = O.dlrm_backward(before["params"], X.astype(np.float64), off, idx, tgt.astype(np.float64), dtype=np.float64)
    bad = copy.deepcopy(before)
    for nm in ("bot", "top"):
        for i, (W, b) in enumerate(bad["params"][nm]):
            for p, s, g, gs in zip((W, b), bad["state"][nm][i], r[nm + "_grads"][i], stale[nm + "_grads"][i]):
                gg = g + 0.25 * gs
                if opt == "sgd":
                    O.sgd_dense(p, gg, LRS[opt])
                else:
                    O.adagrad_dense(p, s, gg, LRS[opt], step=2)
    bad["params"]["emb"], bad["state"]["mom"] = after["params"]["emb"], after["state"]["mom"]
    with pytest.raises(AssertionError, match="err/bound"):
        compare_step(bad, before, after, r, cur, opt, EPS["tc"], D)
