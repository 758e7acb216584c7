"""Engine parity with the wgmma (bf16x3 split) GEMM back end against the live-reference goldens:
the north_star gate "forward logits within 1e-5 of the reference CPU forward" on tensor cores."""
import numpy as np
import pytest
import torch

from golden_util import Golden, O
from test_gpu_parity import DEV, _dev_batch, _robust_close

pytestmark = pytest.mark.gpu
TC_CASES = ["cfg0", "cfg0_itself_thr", "mini_cfg1"]


def _grad_close(got, want, what):
    """Gradients flow through ReLU masks: a pre-activation within rounding of 0 flips a whole term
    on/off relative to the reference, so a handful of entries differ by one term while the bulk
    agrees to bf16x3 accuracy.  Compare with robust statistics relative to the tensor's scale."""
    err = np.abs(np.asarray(got, np.float64) - np.asarray(want, np.float64)).ravel()
    sc = float(np.abs(want).max()) + 1e-12
    assert np.median(err) <= 2e-5 * sc + 1e-7, (what, "median", np.median(err) / sc)
    assert np.quantile(err, 0.99) <= 5e-3 * sc, (what, "p99", np.quantile(err, 0.99) / sc)
    assert err.max() <= 0.25 * sc, (what, "max", err.max() / sc)


def _engine(g, gemm):
    from dlrm_b200.engine import Engine

    e = Engine(g.m_spa, g.ln_emb, g.ln_bot, g.ln_top, op=g.op, itself=g.itself, sigmoid_bot=-1,
               sigmoid_top=len(g.ln_top) - 2, loss=g.loss, loss_threshold=g.thr, device=DEV, max_batch=g.B,
               gemm=gemm)
    e.load_params(g.params())
    return e


@pytest.mark.parametrize("name", TC_CASES + ["cfg0_weighted"])
def test_tc_forward_within_1e5_of_reference(name):
    g = Golden(name)
    e = _engine(g, "tc")
    X, sp, T = _dev_batch(g, 0)
    out = e.forward(X, sp).cpu().numpy()
    err = np.abs(out - g["f_out"]).max()
    print(name, "tc bf16x3 forward max|err| vs reference =", err)
    np.testing.assert_allclose(out, g["f_out"], rtol=0, atol=1e-5)
    Tb = e.Tbuf[:g.B].cpu().numpy()
    np.testing.assert_allclose(Tb[:, 0, :], g["f_x"], rtol=5e-5, atol=5e-6)
    for k in range(g.T):
        if g.has(f"f_ly{k}") and not g.weighted:
            assert np.array_equal(Tb[:, 1 + k, :], g[f"f_ly{k}"])


@pytest.mark.parametrize("name", TC_CASES)
def test_tc_bf16_forward_error_reported(name):
    """Plain bf16 operands (perf mode): NOT claimed to meet 1e-5; bound it loosely and print it."""
    g = Golden(name)
    e = _engine(g, "tc_bf16")
    X, sp, T = _dev_batch(g, 0)
    out = e.forward(X, sp).cpu().numpy()
    err = np.abs(out - g["f_out"]).max()
    print(name, "tc bf16 forward max|err| vs reference =", err)
    assert err < 2e-2


@pytest.mark.parametrize("name", TC_CASES)
def test_tc_backward_vs_reference(name):
    g = Golden(name)
    e = _engine(g, "tc")
    X, sp, T = _dev_batch(g, 0)
    e.forward(X, sp)
    e.backward(X, sp, T)
    assert abs(float(e.loss_buf.item()) - float(g["f_loss"])) < 5e-6
    P = e.dense_numel
    for nm in ("bot", "top"):
        ln = e.ln_bot if nm == "bot" else e.ln_top
        for i in range(len(ln) - 1):
            ns = e.tc_splits.get((nm, i), 1) if i < e.ntc[nm] else 1
            oW, ob = e._dense_off[(nm, i, "W")], e._dense_off[(nm, i, "b")]
            nW, nb = ln[i + 1] * ln[i], ln[i + 1]
            dW = sum(e.dense_grad[s * P + oW:s * P + oW + nW] for s in range(ns)).view(ln[i + 1], ln[i])
            db = sum(e.dense_grad[s * P + ob:s * P + ob + nb] for s in range(ns))
            for got, want in (g.dense_grad(f"g_{nm}W{i}", dW.cpu().numpy()), (db.cpu().numpy(), g[f"g_{nm}b{i}"])):
                _grad_close(got, want, (nm, i))
    dT = e.dT[:g.B].cpu().numpy()
    _, off, idx, _ = g.batch(0)
    for k in range(g.T):
        if g.has(f"g_emb{k}_rows"):
            rows, vals = O.coalesce(*O.sparse_grad(idx[k], off[k], dT[:, 1 + k, :]))
            _grad_close(vals, g[f"g_emb{k}_vals"], ("emb", k))


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad"])
@pytest.mark.parametrize("name", TC_CASES)
def test_tc_train_steps_vs_reference(name, opt):
    g = Golden(name)
    e = _engine(g, "tc")
    lr = float(g[f"{opt}_lr"])
    losses = []
    for s in range(g.nsteps):
        X, sp, T = _dev_batch(g, s)
        losses.append(float(e.train_step(X, sp, T, lr, optimizer=opt).item()))
        if s == 0:  # after ONE step the rows / accumulators are a well-conditioned function of the batch-0 gradients
            for k in range(g.T):
                if g.has(f"{opt}1_emb{k}_rows"):
                    rows = g[f"{opt}1_emb{k}_rows"]
                    np.testing.assert_allclose(e.table(k)[torch.from_numpy(rows).to(DEV)].cpu().numpy(),
                                               g[f"{opt}1_emb{k}_vals"], rtol=1e-3, atol=5e-6)
                assert abs(float(e.table(k).double().sum().item()) - float(g[f"{opt}1_emb{k}_sum"])) < 2e-3
                if opt == "rwsadagrad":
                    m = e.momentum[int(e.row_base[k]):int(e.row_base[k + 1])].cpu().numpy()
                    np.testing.assert_allclose(m, g[f"{opt}1_mom{k}"], rtol=2e-3, atol=1e-10)
    assert int(e.head.abs().sum().item()) == 0, "row-list heads not reset"
    tight = opt == "sgd"
    np.testing.assert_allclose(losses, g[f"{opt}_losses"], rtol=0, atol=2e-5 if tight else 3e-4)
    X, sp, T = _dev_batch(g, g.nsteps)
    pa = e.forward(X, sp).cpu().numpy()
    _robust_close(pa, g[f"{opt}_p_after"], 3e-5 if tight else 5e-4, 2e-4 if tight else 5e-3, "p_after")
    for k in range(g.T):        # rows after all steps (Adagrad: robust, the normalised update amplifies rounding)
        if g.has(f"{opt}_emb{k}_rows"):
            rows = torch.from_numpy(g[f"{opt}_emb{k}_rows"]).to(DEV)
            _robust_close(e.table(k)[rows].cpu().numpy(), g[f"{opt}_emb{k}_vals"], 2e-6 if tight else 2e-5,
                          2e-5 if tight else 2.5 * lr, f"emb{k}")
    for nm in ("bot", "top"):
        for i in range(len(e.W[nm])):
            _robust_close(e.b[nm][i].cpu().numpy(), g[f"{opt}_{nm}b{i}"], 2e-6 if tight else 2e-5,
                          2e-5 if tight else 2.5 * lr, f"{nm}b{i}")


@pytest.mark.parametrize("gemm", ["simt", "tc"])
def test_cuda_graph_step_equals_eager(gemm):
    """GraphedTrainStep (packed static batch, whole step in one CUDA graph) == eager train_step."""
    from dlrm_b200.data import DeviceBatch, make_batch
    from dlrm_b200.engine import Engine, GraphedTrainStep

    rng = np.random.default_rng(3)
    D, ln_emb, ln_bot = 128, [3000, 500, 40], [13, 64, 128]
    ln_top = [D + 4 * 3 // 2, 64, 32, 1]
    B = 192
    params = O.random_params(rng, D, ln_emb, ln_bot, ln_top)
    hbs = [make_batch(np.random.default_rng(10 + i), ln_emb, B, 13, 10) for i in range(4)]
    res = []
    for mode in ("eager", "graph"):
        e = Engine(D, ln_emb, ln_bot, ln_top, loss="bce", sigmoid_top=len(ln_top) - 2, device=DEV, max_batch=B,
                   gemm=gemm)
        e.load_params(params)
        st = DeviceBatch(hbs[0].layout, DEV)
        st.load(hbs[0], non_blocking=False)
        losses = []
        if mode == "graph":
            gs = GraphedTrainStep(e, st, 0.01, "sgd", warmup=0)   # warmup=0: identical update count
            # capture itself does not execute; replay for every batch
            for hb in hbs:
                st.load(hb, non_blocking=False)
                losses.append(float(gs.replay().item()))
        else:
            for hb in hbs:
                st.load(hb, non_blocking=False)
                losses.append(float(e.train_step(st.X, st.sparse, st.target, 0.01, "sgd").item()))
        res.append((losses, e.dense.clone(), e.tables.clone()))
    np.testing.assert_allclose(res[0][0], res[1][0], rtol=0, atol=1e-6)
    assert torch.allclose(res[0][1], res[1][1], rtol=0, atol=1e-6)
    assert torch.allclose(res[0][2], res[1][2], rtol=0, atol=1e-6)


def test_pipelined_multi_step_graph_equals_sequential():
    """GraphedTrainSteps: K steps per graph, the embedding update of step j overlapping step j+1's bottom
    MLP on the side stream -> same losses and parameters as K sequential train_step() calls."""
    from dlrm_b200.data import DeviceBatch, make_batch
    from dlrm_b200.engine import Engine, GraphedTrainSteps

    rng = np.random.default_rng(4)
    # rows are shared between consecutive steps; per-row lists stay <= 32 members (deterministic order)
    D, ln_emb, ln_bot = 128, [2000, 600, 300], [13, 64, 128]
    ln_top = [D + 4 * 3 // 2, 64, 32, 1]
    B, K = 160, 3
    params = O.random_params(rng, D, ln_emb, ln_bot, ln_top)
    hbs = [make_batch(np.random.default_rng(20 + i), ln_emb, B, 13, 10) for i in range(2 * K)]
    res = []
    for mode in ("eager", "graph"):
        e = Engine(D, ln_emb, ln_bot, ln_top, loss="bce", sigmoid_top=len(ln_top) - 2, device=DEV, max_batch=B,
                   gemm="tc")
        e.load_params(params)
        stages = [DeviceBatch(hbs[0].layout, DEV) for _ in range(K)]
        losses = []
        if mode == "graph":
            for j, st in enumerate(stages):
                st.load(hbs[j], non_blocking=False)
            e.prepare(stages[0].sparse, True)
            gs = GraphedTrainSteps.__new__(GraphedTrainSteps)   # capture without warm-up steps
            gs.eng, gs.stages, gs.lr, gs.optimizer, gs.K = e, stages, 0.02, "rwsadagrad", K
            e.ensure_optimizer_state("rwsadagrad")
            gs.losses = torch.zeros(K, device=DEV)
            torch.cuda.synchronize()
            gs.graph = torch.cuda.CUDAGraph()
            n0 = e.n_launch
            with torch.cuda.graph(gs.graph):
                gs._eager()
            gs.kernels_per_replay = e.n_launch - n0
            for r in range(2):
                for j, st in enumerate(stages):
                    st.load(hbs[r * K + j], non_blocking=False)
                losses += gs.replay().cpu().tolist()
        else:
            st = stages[0]
            for hb in hbs:
                st.load(hb, non_blocking=False)
                losses.append(float(e.train_step(st.X, st.sparse, st.target, 0.02, "rwsadagrad").item()))
        torch.cuda.synchronize()
        res.append((losses, e.dense.clone(), e.tables.clone(), e.momentum.clone()))
    np.testing.assert_allclose(res[0][0], res[1][0], rtol=0, atol=1e-6)
    assert torch.allclose(res[0][1], res[1][1], rtol=0, atol=1e-6)
    assert torch.allclose(res[0][2], res[1][2], rtol=0, atol=1e-6)
    assert torch.allclose(res[0][3], res[1][3], rtol=0, atol=1e-7)
