"""Float64 restatements of the dense-path kernels, written from the ABI comments of include/dlrm_b200.h, and the
rounding-error bounds their tests compare against.  Independent of the product: nothing here imports dlrm_b200.

Operations (inputs are fp32 values, every result is float64):
  interaction  R[b] = [x; <T_i, T_j> for j < i (+ j == i when itself)], strict lower triangle in row-major order;
               dT[b] = (dZ + dZ^T) T[b] + dR[b, :D] on feature 0, feature 0 times act'(x)
  head / loss  ATen semantics: z = clamp(p, thr, 1 - thr) iff 0 < thr < 1 (inclusive gradient mask), BCE log terms
               clamped at -100, backward (z - t) / max((1 - z) z, 1e-12), WBCE weight ws[int(t)], mean over n
  act_bwd      gz = gy * [thr <= y <= 1 - thr] * act'(y)
  dense step   SGD p -= lr g;  RWSAdagrad s += g g, p -= lr g / (sqrt(s) + eps);  split-K slabs folded in slab order
  pack         [W | b] as (hi, lo) bf16: hi = bf16(x), lo = bf16(x - hi), both round-to-nearest-even
  linear       Y = act(X W^T + b);  dX = (dY W) * act'(Xact);  dW = dY^T X, db = sum_m dY

Bounds use the standard model fl(a op b) = (a op b)(1 + d), |d| <= u = 2^-24, and gamma_n = n u / (1 - n u): a
sum of m terms evaluated through a chain (or tree) of depth n has |error| <= gamma_n * sum |terms|.
"""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24                 # unit roundoff of fp32
TINY = 2.0 ** -126             # smallest normal fp32: 1 / (1 + expf(-z)) is 0 once expf overflows (z < -88.7)
ACT_NONE, ACT_RELU, ACT_SIGMOID = 0, 1, 2
LOSS_MSE, LOSS_BCE, LOSS_WBCE = 0, 1, 2
OPT_SGD, OPT_RWSADAGRAD = 0, 1


def gamma(n: int) -> float:
    nu = n * U
    assert nu < 1.0
    return nu / (1.0 - nu)


def f64(x):
    return np.asarray(x, dtype=np.float64)


# ---------------------------------------------------------------------------------------------- comparator
def worst_ratio(got, want, bound):
    """(largest |got - want| / bound, its index).  Where bound == 0 the values must be equal; a NaN or an infinity
    that `want` does not have counts as an infinite ratio."""
    got, want = f64(got), f64(want)
    bound = np.broadcast_to(f64(bound), want.shape)
    assert got.shape == want.shape, (got.shape, want.shape)
    if want.size == 0:
        return 0.0, ()
    with np.errstate(invalid="ignore", divide="ignore"):
        err = np.abs(got - want)
        same = (got == want) | (np.isnan(got) & np.isnan(want))
        err = np.where(same, 0.0, err)
        err = np.where(np.isnan(err), np.inf, err)
        ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err == 0, 0.0, np.inf))
    i = int(np.argmax(ratio))
    return float(ratio.flat[i]), np.unravel_index(i, ratio.shape)


def check_within(got, want, bound, what=""):
    """Assert err <= bound everywhere; return the worst err/bound ratio (for reporting)."""
    r, at = worst_ratio(got, want, bound)
    if not r <= 1.0:
        g, w = f64(got)[at], f64(want)[at]
        b = np.broadcast_to(f64(bound), f64(want).shape)[at]
        raise AssertionError(f"{what}: err/bound = {r:.3g} at {tuple(int(i) for i in at)}: "
                             f"got {g!r}, want {w!r}, bound {b:.3g}")
    return r


# ---------------------------------------------------------------------------------------------- activations
def act(x, kind):
    x = f64(x)
    if kind == ACT_RELU:
        return np.maximum(x, 0.0)
    if kind == ACT_SIGMOID:
        with np.errstate(over="ignore"):
            return 1.0 / (1.0 + np.exp(-x))
    return x


def act_grad(y, kind):
    """act'(.) expressed through the activation's OUTPUT y (what the kernels receive)."""
    y = f64(y)
    if kind == ACT_RELU:
        return (y > 0).astype(np.float64)
    if kind == ACT_SIGMOID:
        return (1.0 - y) * y
    return np.ones_like(y)


def act_fwd_bound(pre, pre_bound, kind):
    """Bound on act(fl(pre)) computed in fp32, given |fl(pre) - pre| <= pre_bound.  Sigmoid is
    1 / (1 + expf(-z)): expf <= 2 ulp (relative 4u), the add and the division one rounding each, and the argument
    error scaled by sigma' = p (1 - p); below 2^-126 the result may flush to 0 (expf overflows first)."""
    if kind == ACT_SIGMOID:
        p = act(pre, ACT_SIGMOID)
        return p * (1.0 - p) * pre_bound + gamma(6) * p + TINY
    return f64(pre_bound)                                           # relu and identity add no rounding


def mask_bound(acc_bound, acc_ref, m, kind):
    """Bound on fl(acc * act'(y)): relu multiplies by an exact 0 / 1; sigmoid by fl(fl(1 - y) y) then rounds the
    product (three roundings)."""
    if kind == ACT_SIGMOID:
        return f64(acc_bound) * np.abs(m) * (1.0 + gamma(3)) + gamma(3) * np.abs(f64(acc_ref) * m)
    return f64(acc_bound) * np.abs(m)


# ---------------------------------------------------------------------------------------------- interaction
def tril_pairs(F, itself):
    """(i, j) of the flattened interactions: row-major lower triangle, strict unless itself."""
    return np.tril_indices(F, 0 if itself else -1)


def interact_fwd(T, itself):
    """T [B, F, D] -> (R [B, D + npairs], bound).  Each pair is one fp32 dot product over D (gamma_D); x is copied."""
    T = f64(T)
    B, F, D = T.shape
    li, lj = tril_pairs(F, itself)
    Z = np.matmul(T, T.transpose(0, 2, 1))
    A = np.matmul(np.abs(T), np.abs(T).transpose(0, 2, 1))
    R = np.concatenate([T[:, 0, :], Z[:, li, lj]], axis=1)
    bound = np.concatenate([np.zeros((B, D)), gamma(D) * A[:, li, lj]], axis=1)
    return R, bound


def interact_S(dR, F, D, itself):
    """S = dZ + dZ^T, dZ scattered from dR[:, D:] (the diagonal, when itself, appears twice)."""
    dR = f64(dR)
    B = dR.shape[0]
    li, lj = tril_pairs(F, itself)
    dZ = np.zeros((B, F, F))
    dZ[:, li, lj] = dR[:, D:]
    return dZ + dZ.transpose(0, 2, 1)


def interact_bwd(T, dR, itself, mask0):
    """-> (dT [B, F, D], bound).  Row i of dT is one fp32 chain of F fmas (+ dR on feature 0): gamma_{F+1} times
    |dR| + sum_j |S_ij T_j|; feature 0 then goes through mask_bound."""
    T, dR = f64(T), f64(dR)
    B, F, D = T.shape
    S = interact_S(dR, F, D, itself)
    dT = np.matmul(S, T)
    A = np.matmul(np.abs(S), np.abs(T))
    dT[:, 0, :] += dR[:, :D]
    A[:, 0, :] += np.abs(dR[:, :D])
    bound = gamma(F + 1) * A
    if mask0 != ACT_NONE:
        m = act_grad(T[:, 0, :], mask0)
        bound[:, 0, :] = mask_bound(bound[:, 0, :], dT[:, 0, :], m, mask0)
        dT[:, 0, :] *= m
    return dT, bound


# ---------------------------------------------------------------------------------------------- loss and head
def clamp_limits(thr):
    """(clamped?, lo, hi) exactly as the kernels form them in fp32: lo = thr, hi = 1.0f - thr."""
    thr = np.float32(thr)
    clampd = bool(0.0 < thr < 1.0)
    return clampd, float(thr), float(np.float32(np.float32(1.0) - thr))


def loss_terms(p, t, ws, kind, thr, last_act, n=None):
    """Per-sample loss and gradient from the fp32 activation output p (float64 arithmetic, ATen semantics).
    Returns (per, g, per_bound, g_bound): bounds on the fp32 evaluation of per and of the final gz (loss, clamp
    mask, act')."""
    p, t = f64(p), f64(t)
    n = p.size if n is None else n
    inv_n = 1.0 / n
    clampd, lo, hi = clamp_limits(thr)
    z = np.clip(p, lo, hi) if clampd else p
    if kind == LOSS_MSE:
        d = z - t
        per = d * d
        g = 2.0 * d * inv_n
        per_b = gamma(3) * per                                      # z - t, square
        k = 3                                                       # z - t, 1/n, * inv_n
    else:
        with np.errstate(divide="ignore", invalid="ignore"):
            lz = np.maximum(np.log(z), -100.0)
            l1z = np.maximum(np.log(1.0 - z), -100.0)
        per = (t - 1.0) * l1z - t * lz
        # logf <= 1 ulp (relative 2u); 1.0f - z rounds (relative u), which moves log(1 - z) by <= 2u absolute
        e_l1z = 2.0 * U + 2.0 * U * np.abs(l1z)
        e_lz = 2.0 * U * np.abs(lz)
        per_b = np.abs(t - 1.0) * e_l1z + np.abs(t) * e_lz + gamma(4) * (np.abs(t - 1.0) * np.abs(l1z) +
                                                                           np.abs(t) * np.abs(lz))
        g = (z - t) / np.maximum((1.0 - z) * z, float(np.float32(1e-12)))
        k = 6                                                       # z - t, 1 - z, * z, /, 1/n, * inv_n
        if kind == LOSS_WBCE:
            w = f64(ws)[t.astype(np.int64)]
            per, per_b, g = per * w, (per_b + U * np.abs(per)) * w * (1 + U), g * w
            k += 1
        g = g * inv_n
    if clampd:
        g = np.where((p >= lo) & (p <= hi), g, 0.0)                 # inclusive: torch.clamp's backward
    if last_act == ACT_SIGMOID:
        g = g * (1.0 - p) * p
        k += 3
    elif last_act == ACT_RELU:
        g = np.where(p > 0, g, 0.0)
    return per, g, per_b, gamma(k) * np.abs(g)


def loss_reduce_bound(per, per_b, depth, n):
    """Bound on fl(fl(sum per) * fl(1/n)) when the sum is a tree / chain of the given depth."""
    per, per_b = f64(per), f64(per_b)
    loss = per.sum() / n
    s = np.abs(per).sum() + per_b.sum()
    return loss, (per_b.sum() + gamma(depth) * s) / n + gamma(2) * abs(loss)


def loss_depth(n):
    """loss_kernel: 1024 threads each sum ceil(n/1024) terms, then two 32-lane butterflies (5 levels each)."""
    return -(-n // 1024) + 10


def head_depth(B, rows):
    """head_kernel: thread 0 of each CTA sums its `rows` samples, the last CTA sums the CTA partials in order."""
    return rows + -(-B // rows)


def head_p(h, w, bias, act_last):
    """p = act(h . w + b) and its bound: per lane an fma chain over ceil(K/32) columns, a 5-level butterfly and the
    bias add: gamma_{ceil(K/32) + 6} (sum |h w| + |b|), then act_fwd_bound."""
    h, w = f64(h), f64(w)
    b = float(f64(bias).reshape(-1)[0])
    K = h.shape[1]
    zpre = h @ w + b
    zb = gamma(-(-K // 32) + 6) * (np.abs(h) @ np.abs(w) + abs(b))
    return act(zpre, act_last), act_fwd_bound(zpre, zb, act_last)


def head_backward(h, w, gz, act_prev, depth):
    """From the kernel's own gz: dW = sum_b gz h, db = sum_b gz (chains of the given depth), and
    gprev = gz w act_prev'(h) (one product, then mask_bound).  Returns dict of (value, bound)."""
    h, w, gz = f64(h), f64(w), f64(gz)
    dW = gz @ h
    dWb = gamma(depth) * (np.abs(gz) @ np.abs(h))
    db = gz.sum()
    dbb = gamma(depth) * np.abs(gz).sum()
    gp = gz[:, None] * w[None, :]
    gpb = U * np.abs(gp)
    m = act_grad(h, act_prev)
    return dict(dW=(dW, dWb), db=(db, dbb), gprev=(gp * m, mask_bound(gpb, gp, m, act_prev)))


def act_bwd(gy, y, act_kind, thr):
    """gz = gy * clamp mask * act'(y): exact except the sigmoid product (three roundings)."""
    gy, y = f64(gy), f64(y)
    clampd, lo, hi = clamp_limits(thr)
    g = np.where((y >= lo) & (y <= hi), gy, 0.0) if clampd else gy.copy()
    m = act_grad(y, act_kind)
    return g * m, mask_bound(np.zeros_like(g), g, m, act_kind)


# ---------------------------------------------------------------------------------------------- dense optimizer
def fold_slabs_f32(slabs):
    """Sequential fp32 sum of the split-K slabs in slab order (what the kernel does, reproducible bit for bit)."""
    g = np.array(slabs[0], dtype=np.float32, copy=True)
    for s in slabs[1:]:
        g = (g + np.asarray(s, np.float32)).astype(np.float32)
    return g


def _fma_f32(a, b, c):
    """fmaf(a, b, c): exact product and sum in float64, one rounding to fp32 (the sum's float64 rounding can make
    this differ from a true fmaf by one ulp in rare double-rounding cases)."""
    return (f64(a) * f64(b) + f64(c)).astype(np.float32)


def dense_step_f32(p, g, s, opt, lr, eps):
    """The dense step in the kernels' fp32 operation order: returns (p', s')."""
    p, g = np.asarray(p, np.float32), np.asarray(g, np.float32)
    lr, eps = np.float32(lr), np.float32(eps)
    if opt == OPT_RWSADAGRAD:
        s2 = _fma_f32(g, g, s)
        q = (g / (np.sqrt(s2) + eps)).astype(np.float32)
        return _fma_f32(-lr, q, p), s2
    return _fma_f32(-lr, g, p), s


def dense_step(p, g, s, opt, lr, eps):
    """The same step in float64 (the definition)."""
    p, g = f64(p), f64(g)
    lr, eps = float(np.float32(lr)), float(np.float32(eps))
    if opt == OPT_RWSADAGRAD:
        s2 = f64(s) + g * g
        return p - lr * g / (np.sqrt(s2) + eps), s2
    return p - lr * g, s


def ulp_diff(a, b):
    """|a - b| in units in the last place of fp32 (ordered integer distance; +0 and -0 are 0 apart)."""
    def key(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(a) - key(b))


def pack_layer(W, b):
    """[N, K + 1] = [W | b] (fp32)."""
    W, b = np.asarray(W, np.float32), np.asarray(b, np.float32)
    return np.concatenate([W, b.reshape(-1, 1)], axis=1)


# ---------------------------------------------------------------------------------------------- bf16 split
def split_bf16(x):
    """(hi, lo) as uint16 bit patterns: hi = x.bfloat16(), lo = (x - hi.float()).bfloat16() on the torch CPU."""
    import torch

    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
    hi = t.bfloat16()
    lo = (t - hi.float()).bfloat16()
    return hi.view(torch.int16).numpy().view(np.uint16), lo.view(torch.int16).numpy().view(np.uint16)


# ---------------------------------------------------------------------------------------------- fp32 linear
def linear_fwd(X, W, b, act_kind):
    """Y = act(X W^T + b): one fma chain of K per output (+ the bias add)."""
    X, W = f64(X), f64(W)
    K = X.shape[1]
    pre = X @ W.T
    pb = np.abs(X) @ np.abs(W).T
    if b is not None:
        pre = pre + f64(b)[None, :]
        pb = pb + np.abs(f64(b))[None, :]
        K += 1
    return act(pre, act_kind), act_fwd_bound(pre, gamma(max(K, 1)) * pb, act_kind)


def linear_dgrad(dY, W, Xact, act_prev):
    """dX = (dY W) * act'(Xact): one fma chain of N per output, then mask_bound."""
    dY, W = f64(dY), f64(W)
    N = dY.shape[1]
    v = dY @ W
    vb = gamma(max(N, 1)) * (np.abs(dY) @ np.abs(W))
    if act_prev == ACT_NONE:
        return v, vb
    m = act_grad(Xact, act_prev)
    return v * m, mask_bound(vb, v, m, act_prev)


def linear_wgrad(dY, X):
    """dW = dY^T X (one fma chain of M), db = sum_m dY (8 strided chains of ceil(M/8), then 8 summed in order)."""
    dY, X = f64(dY), f64(X)
    M = dY.shape[0]
    dW = dY.T @ X
    dWb = gamma(max(M, 1)) * (np.abs(dY).T @ np.abs(X))
    db = dY.sum(axis=0)
    dbb = gamma(-(-M // 8) + 8) * np.abs(dY).sum(axis=0)
    return (dW, dWb), (db, dbb)


def ceil_div(a, b):
    return -(-a // b)

