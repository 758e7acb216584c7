"""Pin the numpy oracle (oracle/dlrm_numpy.py) against fixtures generated from the
LIVE reference (oracle/make_goldens.py).  CPU only."""
import numpy as np
import pytest

from golden_util import ALL_CASES, Golden, O

TOL = dict(rtol=2e-5, atol=2e-6)


@pytest.mark.parametrize("name", ALL_CASES)
def test_forward_stages(name):
    g = Golden(name)
    p = g.params()
    X, off, idx, T = g.batch(0)
    f = O.dlrm_forward(p, X, off, idx, keep=True, **g.kw())
    # embedding bags: bit-exact (sequential fp32 order == reference CPU kernel)
    for k in range(g.T):
        if g.has(f"f_ly{k}"):
            if g.weighted:
                np.testing.assert_allclose(f["ly"][k], g[f"f_ly{k}"], rtol=1e-6, atol=1e-7)
            else:
                assert np.array_equal(f["ly"][k], g[f"f_ly{k}"]), f"table {k} not bit-exact"
    np.testing.assert_allclose(f["x"], g["f_x"], **TOL)
    np.testing.assert_allclose(f["R"], g["f_R"], **TOL)
    np.testing.assert_allclose(f["p"], g["f_p"], rtol=0, atol=1e-6)
    np.testing.assert_allclose(f["z"], g["f_out"], rtol=0, atol=1e-6)
    L = O.loss_forward(f["z"], T, g.loss)
    assert abs(float(L) - float(g["f_loss"])) < 2e-6


@pytest.mark.parametrize("name", ALL_CASES)
def test_backward_grads(name):
    g = Golden(name)
    p = g.params()
    X, off, idx, T = g.batch(0)
    r = O.dlrm_backward(p, X, off, idx, T, loss=g.loss, **g.kw())
    for nm in ("bot", "top"):
        for i, (dW, db) in enumerate(r[nm + "_grads"]):
            np.testing.assert_allclose(*g.dense_grad(f"g_{nm}W{i}", dW), rtol=2e-4, atol=2e-7)
            np.testing.assert_allclose(db, g[f"g_{nm}b{i}"], rtol=2e-4, atol=2e-7)
    for k in range(g.T):
        if not g.has(f"g_emb{k}_rows"):
            continue
        ind, val = O.sparse_grad(idx[k], off[k], r["d_ly"][k])
        if g.weighted:  # d out / d W[row] = psw * d_ly
            val = val * p["v_W_l"][k][ind][:, None]
        rows, vals = O.coalesce(ind, val)
        assert np.array_equal(rows, g[f"g_emb{k}_rows"])
        np.testing.assert_allclose(vals, g[f"g_emb{k}_vals"], rtol=2e-4, atol=2e-7)


def _robust_close(a, b, atol_med, atol_max, what):
    """Adagrad's first steps divide by |g|: entries whose gradient is ~0 are
    ill-conditioned (sign flips move them by 2*lr).  Compare with robust statistics."""
    err = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).ravel()
    assert np.median(err) <= atol_med, f"{what}: median err {np.median(err)}"
    assert np.quantile(err, 0.999) <= atol_max, f"{what}: p99.9 err {np.quantile(err, 0.999)}"


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad"])
@pytest.mark.parametrize("name", ALL_CASES)
def test_optimizer_step1_from_golden_grads(name, opt):
    """Optimizer restatement alone: feed the reference's own batch-0 grads."""
    g = Golden(name)
    p = g.params()
    st = O.new_state(p)
    lr = float(g[f"{opt}_lr"])
    for k in range(g.T):
        if not g.has(f"g_emb{k}_rows"):
            continue
        rows, vals = g[f"g_emb{k}_rows"], g[f"g_emb{k}_vals"]
        if opt == "sgd":
            O.sgd_sparse(p["emb"][k], rows, vals, lr)
        else:
            O.rwsadagrad_sparse(p["emb"][k], st["mom"][k], rows, vals, lr)
            np.testing.assert_allclose(st["mom"][k], g[f"{opt}1_mom{k}"], rtol=2e-6, atol=1e-12)
        tr = g[f"{opt}1_emb{k}_rows"]
        np.testing.assert_allclose(p["emb"][k][tr], g[f"{opt}1_emb{k}_vals"], rtol=2e-6, atol=1e-7)
        assert abs(p["emb"][k].astype(np.float64).sum() - float(g[f"{opt}1_emb{k}_sum"])) < 1e-3
    for nm in ("bot", "top"):
        for i, (W, b) in enumerate(p[nm]):
            for arr, key, s in ((W, "W", st[nm][i][0]), (b, "b", st[nm][i][1])):
                if not g.has(f"{opt}1_{nm}{key}{i}"):
                    continue
                grad = g[f"g_{nm}{key}{i}"]
                if opt == "sgd":
                    O.sgd_dense(arr, grad, lr)
                else:
                    O.adagrad_dense(arr, s, grad, lr)
                np.testing.assert_allclose(arr, g[f"{opt}1_{nm}{key}{i}"], rtol=2e-6, atol=1e-7)


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad"])
@pytest.mark.parametrize("name", [c for c in ALL_CASES if c != "cfg0_weighted"])
def test_train_steps(name, opt):
    g = Golden(name)
    p = g.params()
    st = O.new_state(p)
    lr = float(g[f"{opt}_lr"])
    losses = []
    for s in range(g.nsteps):
        X, off, idx, T = g.batch(s)
        r = O.train_step(p, st, X, off, idx, T, lr=lr, optimizer=opt, loss=g.loss, **g.kw())
        losses.append(float(r["loss"]))
    tight = opt == "sgd"
    np.testing.assert_allclose(losses, g[f"{opt}_losses"], rtol=0, atol=5e-6 if tight else 2e-4)
    X, off, idx, T = g.batch(g.nsteps)
    pa = O.dlrm_forward(p, X, off, idx, **g.kw())
    _robust_close(pa, g[f"{opt}_p_after"], 2e-5 if tight else 5e-4, 1e-4 if tight else 5e-3, "p_after")
    for k in range(g.T):
        if g.has(f"{opt}_emb{k}_rows"):
            rows = g[f"{opt}_emb{k}_rows"]
            _robust_close(p["emb"][k][rows], g[f"{opt}_emb{k}_vals"], 1e-6 if tight else 2e-5,
                          1e-5 if tight else 2.5 * lr, f"emb{k}")
        if opt == "rwsadagrad":
            _robust_close(st["mom"][k], g[f"{opt}_mom{k}"], 1e-9, 1e-6, f"mom{k}")
    for nm in ("bot", "top"):
        for i in range(len(p[nm])):
            _robust_close(p[nm][i][1], g[f"{opt}_{nm}b{i}"], 1e-6 if tight else 2e-5,
                          1e-5 if tight else 2.5 * lr, f"{nm}b{i}")
            if g.has(f"{opt}_{nm}W{i}"):
                _robust_close(p[nm][i][0], g[f"{opt}_{nm}W{i}"], 1e-6 if tight else 2e-5,
                              1e-5 if tight else 2.5 * lr, f"{nm}W{i}")


def test_empty_and_ragged_bags():
    rng = np.random.default_rng(0)
    W = rng.standard_normal((50, 8)).astype(np.float32)
    idx = np.array([3, 4, 4, 49, 0], dtype=np.int64)
    off = np.array([0, 0, 2, 2, 5], dtype=np.int64)  # bags: [], [3,4], [], [4,49,0], []
    out = O.emb_bag_sum(W, idx, off)
    assert np.array_equal(out[0], np.zeros(8, np.float32))
    assert np.array_equal(out[1], W[3] + W[4])
    assert np.array_equal(out[2], np.zeros(8, np.float32))
    assert np.array_equal(out[3], (W[4] + W[49]) + W[0])
    assert np.array_equal(out[4], np.zeros(8, np.float32))
    # no bags at all
    assert O.emb_bag_sum(W, np.zeros(0, np.int64), np.zeros(0, np.int64)).shape == (0, 8)


# ---- the torch-CPU port used as the timed CPU baseline on the GPU box
@pytest.mark.parametrize("name", [c for c in ALL_CASES if c != "cfg0_weighted"])
def test_torch_port_matches_reference(name):
    import torch

    from oracle.torch_cpu_port import CpuDLRM, RowWiseAdagradCPU

    g = Golden(name)
    m = CpuDLRM(g.m_spa, g.ln_emb, g.ln_bot, g.ln_top, op=g.op, itself=g.itself, loss=g.loss,
                loss_threshold=g.thr)
    m.load(g.params())

    def tb(s):
        X, off, idx, T = g.batch(s)
        return (torch.from_numpy(X), [torch.from_numpy(o) for o in off], [torch.from_numpy(i) for i in idx],
                torch.from_numpy(T))

    X, o, i, T = tb(0)
    with torch.no_grad():
        p = m(X, o, i).numpy()
    assert np.array_equal(p, g["f_out"]), "same ATen ops -> identical forward"
    opt = RowWiseAdagradCPU(m.parameters(), lr=float(g["rwsadagrad_lr"]))
    losses = []
    for s in range(g.nsteps):
        X, o, i, T = tb(s)
        E = m.loss_fn(m(X, o, i), T)
        losses.append(E.item())
        opt.zero_grad()
        E.backward()
        opt.step()
    np.testing.assert_allclose(losses, g["rwsadagrad_losses"], rtol=0, atol=1e-6)
    X, o, i, T = tb(g.nsteps)
    with torch.no_grad():
        pa = m(X, o, i).numpy()
    np.testing.assert_allclose(pa, g["rwsadagrad_p_after"], rtol=0, atol=1e-6)
