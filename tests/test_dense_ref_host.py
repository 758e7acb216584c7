"""The float64 restatements of the dense-path kernels (oracle/dense_f64.py), checked on the CPU: against torch float64
autograd at small shapes (an independent derivation), against fp32 evaluations in the kernels' operation order (the
bounds must hold for an honest fp32 kernel), and with negative controls: at the bounds the GPU tests use, the
comparator must reject plausible wrong kernels.  No GPU needed."""
import numpy as np
import pytest
import torch

from oracle import dense_f64 as O

RTOL = 1e-9     # float64 restatement vs float64 autograd: only the association of the sums differs


def _close(a, b, rtol=RTOL):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(1.0, float(np.abs(b).max())) if b.size else 1.0
    assert np.allclose(a, b, rtol=rtol, atol=rtol * scale), float(np.abs(a - b).max())


def _act_t(x, kind):
    return torch.relu(x) if kind == O.ACT_RELU else torch.sigmoid(x) if kind == O.ACT_SIGMOID else x


def _f32(rng, *shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float32)


# ------------------------------------------------------------------------------------------------ float64 autograd
@pytest.mark.parametrize("F,D,itself,mask0", [(1, 3, 0, 0), (1, 2, 1, 1), (2, 1, 0, 2), (4, 3, 1, 1), (5, 8, 0, 2),
                                              (6, 4, 1, 0), (9, 2, 0, 1)])
def test_interaction_matches_autograd(F, D, itself, mask0):
    rng = np.random.default_rng(F * 10 + D)
    B = 3
    xpre = rng.standard_normal((B, D))
    xpre[:, 0] = 0.0                                   # exact zeros of a relu output
    ly = rng.standard_normal((B, F - 1, D))
    xp_t = torch.tensor(xpre, requires_grad=True)
    ly_t = torch.tensor(ly, requires_grad=True)
    x_t = _act_t(xp_t, mask0)
    T_t = torch.cat([x_t[:, None, :], ly_t], dim=1)
    Z = torch.bmm(T_t, T_t.transpose(1, 2))
    li, lj = torch.tril_indices(F, F, offset=0 if itself else -1)
    R_t = torch.cat([x_t, Z[:, li, lj]], dim=1)
    dR = rng.standard_normal(R_t.shape)
    R_t.backward(torch.tensor(dR))
    T = T_t.detach().numpy()
    R, _ = O.interact_fwd(T, itself)
    _close(R, R_t.detach().numpy())
    dT, _ = O.interact_bwd(T, dR, itself, mask0)
    _close(dT[:, 0, :], xp_t.grad.numpy())
    _close(dT[:, 1:, :], ly_t.grad.numpy())


def _torch_head(hpre, act_prev, w, b, t, ws, act_last, kind, thr):
    clampd, lo, hi = O.clamp_limits(thr)
    hp = torch.tensor(hpre, requires_grad=True)
    W = torch.tensor(w, requires_grad=True)
    bb = torch.tensor(b, requires_grad=True)
    zpre = _act_t(hp, act_prev) @ W + bb
    zpre.retain_grad()
    p = _act_t(zpre, act_last)
    z = torch.clamp(p, lo, hi) if clampd else p
    tt = torch.tensor(t)
    if kind == O.LOSS_MSE:
        loss = torch.nn.functional.mse_loss(z, tt)
    elif kind == O.LOSS_BCE:
        loss = torch.nn.functional.binary_cross_entropy(z, tt)
    else:   # dlrm_s_pytorch.py loss_fn_wrap, "wbce"
        loss = (torch.tensor(ws)[tt.long()] * torch.nn.functional.binary_cross_entropy(z, tt, reduction="none")).mean()
    loss.backward()
    return [v.detach().numpy() for v in (p, loss, zpre.grad, W.grad, bb.grad, hp.grad)]


@pytest.mark.parametrize("act_last", [0, 1, 2])
@pytest.mark.parametrize("act_prev", [0, 1, 2])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_head_and_loss_match_autograd(act_last, act_prev, kind):
    rng = np.random.default_rng(act_last * 9 + act_prev * 3 + kind)
    B, K = 19, 7
    hpre = rng.standard_normal((B, K))
    w = rng.uniform(0.05, 0.3, K)
    b = np.array([0.2])
    if act_prev == O.ACT_NONE:
        hpre = np.abs(hpre)          # keeps the identity last layer's p inside (0, 1) for BCE
    t = rng.integers(0, 2, B).astype(np.float64)
    if kind == O.LOSS_MSE:
        t = rng.uniform(0, 1, B)
    ws = np.array([0.3, 2.5])
    thr = 0.0 if act_last == O.ACT_SIGMOID else 0.05     # BCE needs z in [0, 1]
    p_t, loss_t, gz_t, dW_t, db_t, gprev_t = _torch_head(hpre, act_prev, w, b, t, ws, act_last, kind, thr)
    h = O.act(hpre, act_prev)
    p, _ = O.head_p(h, w, b, act_last)
    _close(p, p_t)
    per, g, _, _ = O.loss_terms(p, t, ws, kind, thr, act_last)
    _close(per.mean(), loss_t)
    _close(g, gz_t)
    bw = O.head_backward(h, w, g, act_prev, 1)
    _close(bw["dW"][0], dW_t)
    _close(bw["db"][0], db_t)
    _close(bw["gprev"][0], gprev_t)


def test_bce_saturation_and_clamp_boundary_match_autograd():
    """p exactly 0 and 1 (log clamped at -100, the 1e-12 floor) and p exactly at thr / 1 - thr (inclusive mask)."""
    thr = 0.45
    _, lo, hi = O.clamp_limits(thr)
    for th, pv in ((0.0, [0.0, 1.0, 0.0, 1.0, 0.5]), (thr, [lo, hi, 0.2, 0.9, 0.5])):
        p = np.array(pv)
        t = np.array([1.0, 0.0, 0.0, 1.0, 1.0])
        for kind in (O.LOSS_BCE, O.LOSS_WBCE):
            _, loss_t, gz_t, _, _, _ = _torch_head(p[:, None], 0, np.ones(1), np.zeros(1), t, np.array([0.3, 2.5]),
                                                   O.ACT_NONE, kind, th)
            per, g, _, _ = O.loss_terms(p, t, [0.3, 2.5], kind, th, O.ACT_NONE)
            _close(per.mean(), loss_t, 1e-7)
            _close(g, gz_t, 1e-7)      # the kernels' floor is fp32(1e-12), ATen's the double 1e-12
            if th:
                assert g[0] != 0 and g[1] != 0 and g[2] == 0 and g[3] == 0


def test_act_bwd_matches_autograd():
    rng = np.random.default_rng(3)
    thr = 0.45
    _, lo, hi = O.clamp_limits(thr)
    for kind in (0, 1, 2):
        zpre = rng.standard_normal(40)
        y = O.act(zpre, kind)
        y[:3] = [lo, hi, 0.0] if kind != O.ACT_SIGMOID else y[:3]
        zt = torch.tensor(zpre, requires_grad=True)
        yt = _act_t(zt, kind)
        gy = rng.standard_normal(40)
        for th in (thr, 0.0, 1.5):
            clampd, a, b = O.clamp_limits(th)
            if zt.grad is not None:
                zt.grad = None
            out = torch.clamp(yt, a, b) if clampd else yt
            out.backward(torch.tensor(gy), retain_graph=True)
            if kind == O.ACT_SIGMOID or not clampd:
                g, _ = O.act_bwd(gy, yt.detach().numpy(), kind, th)
                _close(g, zt.grad.numpy())
        g, _ = O.act_bwd(gy, y, kind, thr)
        if kind == O.ACT_NONE:
            assert g[0] == gy[0] and g[1] == gy[1] and g[2] == 0.0     # inclusive clamp mask


def test_dense_step_matches_torch_optimizers():
    rng = np.random.default_rng(4)
    p0, g, s0 = rng.standard_normal(50), rng.standard_normal(50), rng.uniform(0, 2, 50)
    lr, eps = 0.125, 1e-8
    for opt in (O.OPT_SGD, O.OPT_RWSADAGRAD):
        pt = torch.nn.Parameter(torch.tensor(p0))
        if opt == O.OPT_SGD:
            o = torch.optim.SGD([pt], lr=lr)
        else:
            o = torch.optim.Adagrad([pt], lr=lr, eps=float(np.float32(eps)))
            o.state[pt]["sum"].copy_(torch.tensor(s0))
        pt.grad = torch.tensor(g)
        o.step()
        p1, s1 = O.dense_step(p0, g, s0, opt, lr, eps)
        _close(p1, pt.detach().numpy(), 1e-12)
        if opt == O.OPT_RWSADAGRAD:
            _close(s1, o.state[pt]["sum"].numpy(), 1e-12)


def test_fold_pack_and_split_reference():
    rng = np.random.default_rng(5)
    slabs = [_f32(rng, 6, 9) for _ in range(3)]
    f = O.fold_slabs_f32(slabs)
    want = (torch.from_numpy(slabs[0]) + torch.from_numpy(slabs[1])) + torch.from_numpy(slabs[2])
    assert np.array_equal(f.view(np.uint32), want.numpy().view(np.uint32))
    W, b = _f32(rng, 4, 5), _f32(rng, 4)
    P = O.pack_layer(W, b)
    assert np.array_equal(P[:, :5], W) and np.array_equal(P[:, 5], b)
    # round to nearest even on ties, subnormals kept, lo the exact remainder
    x = np.array([0x3F808000, 0x3F818000, 0x3F80C000, 0x00008000, 0x00018000, 0x80000000, 0x7F7F8000,
                  0x7F7F7FFF], np.uint32).view(np.float32)
    hi, lo = O.split_bf16(x)
    assert hi.tolist() == [0x3F80, 0x3F82, 0x3F81, 0x0000, 0x0002, 0x8000, 0x7F80, 0x7F7F]
    y = np.concatenate([_f32(rng, 200), (rng.uniform(-1, 1, 50) * 2.0 ** -130).astype(np.float32)])
    hi, lo = O.split_bf16(y)
    bf = lambda u: (u.astype(np.uint32) << 16).view(np.float32).astype(np.float64)  # noqa: E731
    assert np.all(np.abs(bf(hi) + bf(lo) - y) <= 2.0 ** -16 * np.abs(y) + 2.0 ** -134)   # bf16 subnormal step 2^-133


@pytest.mark.parametrize("act_kind", [0, 1, 2])
def test_linear_matches_autograd(act_kind):
    rng = np.random.default_rng(6 + act_kind)
    M, N, K = 7, 5, 6
    Xpre, W, b = rng.standard_normal((M, K)), rng.standard_normal((N, K)), rng.standard_normal(N)
    xt = torch.tensor(Xpre, requires_grad=True)
    Wt, bt = torch.tensor(W, requires_grad=True), torch.tensor(b, requires_grad=True)
    X = _act_t(xt, act_kind)
    Y = _act_t(torch.nn.functional.linear(X, Wt, bt), act_kind)
    dY = rng.standard_normal((M, N))
    Y.backward(torch.tensor(dY))
    Xv = X.detach().numpy()
    Yr, _ = O.linear_fwd(Xv, W, b, act_kind)
    _close(Yr, Y.detach().numpy())
    dpre = dY * O.act_grad(Yr, act_kind)      # the gradient entering the layer's GEMMs
    dX, _ = O.linear_dgrad(dpre, W, Xv, act_kind)
    _close(dX, xt.grad.numpy())
    (dW, _), (db, _) = O.linear_wgrad(dpre, Xv)
    _close(dW, Wt.grad.numpy())
    _close(db, bt.grad.numpy())


# ------------------------------------------------------------------------------------------------ positive controls
def _fma(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def _interact_fwd_f32(T, itself):
    B, F, D = T.shape
    li, lj = O.tril_pairs(F, itself)
    z = np.zeros((B, li.size), np.float32)
    for d in range(D):
        z = _fma(T[:, li, d], T[:, lj, d], z)
    return np.concatenate([T[:, 0, :], z], axis=1)


def _interact_bwd_f32(T, dR, itself, mask0):
    B, F, D = T.shape
    S = O.interact_S(dR, F, D, itself).astype(np.float32)       # exact: copies and doublings of fp32 values
    dT = np.zeros_like(T)
    for i in range(F):
        acc = dR[:, :D].copy() if i == 0 else np.zeros((B, D), np.float32)
        for j in range(F):
            acc = _fma(S[:, i, j][:, None], T[:, j, :], acc)
        dT[:, i, :] = acc
    x = T[:, 0, :]
    if mask0 == O.ACT_RELU:
        dT[:, 0, :] = np.where(x > 0, dT[:, 0, :], np.float32(0))
    elif mask0 == O.ACT_SIGMOID:
        dT[:, 0, :] = dT[:, 0, :] * ((np.float32(1) - x) * x)
    return dT


@pytest.mark.parametrize("F,D", [(4, 16), (9, 17), (27, 64)])
def test_fp32_evaluation_in_kernel_order_is_within_bounds(F, D):
    rng = np.random.default_rng(F + D)
    B = 6
    T = _f32(rng, B, F, D)
    T[:, 0, :] = np.abs(T[:, 0, :]) / 4
    R, Rb = O.interact_fwd(T, 1)
    assert O.check_within(_interact_fwd_f32(T, 1), R, Rb, "fwd") <= 1
    dR = _f32(rng, B, R.shape[1])
    for mask0 in (0, 1, 2):
        dT, dTb = O.interact_bwd(T, dR, 1, mask0)
        assert O.check_within(_interact_bwd_f32(T, dR, 1, mask0), dT, dTb, "bwd") <= 1
    X, W = _f32(rng, 5, 300), _f32(rng, 3, 300)
    Y, Yb = O.linear_fwd(X, W, None, O.ACT_NONE)
    acc = np.zeros((5, 3), np.float32)
    for k in range(300):
        acc = _fma(X[:, None, k], W[None, :, k], acc)
    assert O.check_within(acc, Y, Yb, "gemm") <= 1
    p, g = rng.uniform(0, 1, 64).astype(np.float32), _f32(rng, 64)
    s = rng.uniform(0, 1, 64).astype(np.float32)
    for opt in (O.OPT_SGD, O.OPT_RWSADAGRAD):
        p1, _ = O.dense_step_f32(p, g, s, opt, 0.01, 1e-8)
        p64, _ = O.dense_step(p, g, s, opt, 0.01, 1e-8)
        assert O.check_within(p1, p64, O.gamma(5) * np.abs(p64) + O.gamma(5) * 0.01 * np.abs(g) * 10, "step") <= 1


def test_gamma_and_comparator():
    assert O.gamma(1) == pytest.approx(2.0 ** -24, rel=1e-6)
    assert O.gamma(1000) > 1000 * 2.0 ** -24
    r, at = O.worst_ratio(np.array([1.0, 2.0, 3.5]), np.array([1.0, 2.0, 3.0]), np.array([1.0, 1.0, 0.25]))
    assert r == 2.0 and at == (2,)
    assert O.worst_ratio([np.nan], [1.0], [1e9])[0] == np.inf
    assert O.worst_ratio([1.0], [1.0], [0.0])[0] == 0.0
    assert O.worst_ratio([1.0 + 1e-16], [1.0], [0.0])[0] == 0.0   # equal after the float64 cast
    assert O.worst_ratio([1.5], [1.0], [0.0])[0] == np.inf
    assert O.ulp_diff(np.float32(1.0), np.nextafter(np.float32(1.0), np.float32(2))) == 1
    assert O.ulp_diff(np.float32(0.0), np.float32(-0.0)) == 0
    with pytest.raises(AssertionError, match="err/bound"):
        O.check_within([2.0], [1.0], [0.5], "x")


# ------------------------------------------------------------------------------------------------ negative controls
def _rejects(got, want, bound):
    r, _ = O.worst_ratio(got, want, bound)
    assert r > 1.0, r
    return r


def test_negative_controls_interaction():
    rng = np.random.default_rng(7)
    B, F, D = 4, 5, 16
    T = _f32(rng, B, F, D)
    for itself in (0, 1):
        R, Rb = O.interact_fwd(T, itself)
        li, lj = O.tril_pairs(F, itself)
        # lower triangle in column-major order (pair (i, j) stored in the slot of another pair)
        order = np.lexsort((li, lj))
        Zw = R[:, D:][:, order]
        _rejects(np.concatenate([R[:, :D], Zw], 1), R, Rb)
        # off-by-one pair index
        _rejects(np.concatenate([R[:, :D], np.roll(R[:, D:], 1, axis=1)], 1), R, Rb)
    # the itself diagonal left out of the forward
    R1, R1b = O.interact_fwd(T, 1)
    li, lj = O.tril_pairs(F, 1)
    wrong = R1.copy()
    wrong[:, D:][:, li == lj] = 0.0
    _rejects(wrong, R1, R1b)
    # backward: diagonal missing / not doubled; mask on the wrong feature
    dR = _f32(rng, B, R1.shape[1])
    dT, dTb = O.interact_bwd(T, dR, 1, O.ACT_NONE)
    S = O.interact_S(dR, F, D, 1)
    for diag_scale in (0.0, 0.5):
        Sw = S.copy()
        idx = np.arange(F)
        Sw[:, idx, idx] *= diag_scale
        w = np.matmul(Sw, T.astype(np.float64))
        w[:, 0, :] += dR[:, :D]
        _rejects(w, dT, dTb)
    Tm = T.copy()
    Tm[:, 0, :] = rng.uniform(0, 1, (B, D)).astype(np.float32)
    Tm[:, 1, :] = rng.uniform(0, 1, (B, D)).astype(np.float32)
    for mask0 in (O.ACT_RELU, O.ACT_SIGMOID):
        Tm[:, 0, ::3] = 0.0
        good, gb = O.interact_bwd(Tm, dR, 1, mask0)
        raw, _ = O.interact_bwd(Tm, dR, 1, O.ACT_NONE)
        wrong = raw.copy()
        wrong[:, 1, :] *= O.act_grad(Tm[:, 1, :], mask0)
        _rejects(wrong, good, gb)


def test_negative_controls_loss_and_head():
    thr = 0.45
    _, lo, hi = O.clamp_limits(thr)
    p = np.array([lo, hi, 0.5, 0.47], np.float32)
    t = np.array([1.0, 0.0, 1.0, 0.0])
    per, g, per_b, g_b = O.loss_terms(p, t, None, O.LOSS_BCE, thr, O.ACT_NONE)
    # clamp mask made exclusive: p exactly at thr / 1 - thr would lose its gradient
    pf = p.astype(np.float64)
    excl = np.where((pf > lo) & (pf < hi), g, 0.0)
    _rejects(excl, g, g_b)
    # WBCE weights swapped
    rng = np.random.default_rng(8)
    p2 = rng.uniform(0.05, 0.95, 64).astype(np.float32)
    t2 = rng.integers(0, 2, 64).astype(np.float64)
    per, g, per_b, g_b = O.loss_terms(p2, t2, [0.3, 2.5], O.LOSS_WBCE, 0.0, O.ACT_SIGMOID)
    per_w, g_w, _, _ = O.loss_terms(p2, t2, [2.5, 0.3], O.LOSS_WBCE, 0.0, O.ACT_SIGMOID)
    _rejects(g_w, g, g_b)
    loss, lb = O.loss_reduce_bound(per, per_b, O.head_depth(64, 16), 64)
    _rejects(per_w.mean(), loss, lb)
    # one sample's term dropped from the loss sum, and a head that forgets one column of the dot product
    _rejects(per[1:].sum() / 64, loss, lb)
    h, w = _f32(rng, 8, 40), _f32(rng, 40, scale=0.2)
    pr, pb = O.head_p(h, w, np.zeros(1), O.ACT_SIGMOID)
    pw, _ = O.head_p(h[:, 1:], w[1:], np.zeros(1), O.ACT_SIGMOID)
    _rejects(pw, pr, pb)
    # BCE without the -100 clamp (p exactly 0) is infinite
    _, gz0, _, _ = O.loss_terms(np.array([0.0], np.float32), np.array([1.0]), None, O.LOSS_BCE, 0.0, O.ACT_NONE)
    per0, _, per0_b, _ = O.loss_terms(np.array([0.0], np.float32), np.array([1.0]), None, O.LOSS_BCE, 0.0, O.ACT_NONE)
    assert per0[0] == 100.0 and np.isfinite(gz0[0])
    _rejects(np.array([np.inf]), per0, per0_b)


def test_negative_controls_dense_update_and_pack():
    rng = np.random.default_rng(9)
    N, K, S = 6, 11, 3
    slabs = [_f32(rng, N * K + N) for _ in range(S)]
    g = O.fold_slabs_f32(slabs)
    dropped = O.fold_slabs_f32(slabs[:-1])
    # the fold is compared bit for bit; the step within one ulp
    assert O.worst_ratio(dropped, g, 0.0)[0] > 1
    p, s = _f32(rng, N * K + N), rng.uniform(0, 1, N * K + N).astype(np.float32)
    want, _ = O.dense_step_f32(p, g, s, O.OPT_SGD, 0.5, 1e-8)
    got, _ = O.dense_step_f32(p, dropped, s, O.OPT_SGD, 0.5, 1e-8)
    assert O.ulp_diff(got, want).max() > 1
    # the bias column not packed
    W, b = _f32(rng, N, K), _f32(rng, N)
    hi, lo = O.split_bf16(O.pack_layer(W, b))
    hi_w, lo_w = O.split_bf16(O.pack_layer(W, np.zeros(N, np.float32)))
    assert not np.array_equal(hi_w, hi) and np.array_equal(hi_w[:, :K], hi[:, :K])


def test_negative_controls_gemm():
    rng = np.random.default_rng(10)
    M, N, K = 9, 7, 64
    X, W = _f32(rng, M, K), _f32(rng, N, K)
    Y, Yb = O.linear_fwd(X, W, None, O.ACT_NONE)
    Yw, _ = O.linear_fwd(X[:, :-1], W[:, :-1], None, O.ACT_NONE)          # last k dropped
    _rejects(Yw, Y, Yb)
    dY = _f32(rng, M, N)
    Xa = rng.uniform(0, 1, (M, K)).astype(np.float32)
    dX, dXb = O.linear_dgrad(dY, W, Xa, O.ACT_SIGMOID)
    raw, _ = O.linear_dgrad(dY, W, Xa, O.ACT_NONE)
    _rejects(raw, dX, dXb)                                                 # mask not applied
    (dW, dWb), (db, dbb) = O.linear_wgrad(dY, X)
    (dWw, _), (dbw, _) = O.linear_wgrad(dY[1:], X[1:])                     # first row of the batch dropped
    _rejects(dWw, dW, dWb)
    _rejects(dbw, db, dbb)
