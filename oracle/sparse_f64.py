"""Float64 restatements of the sparse-path kernels, written from the ABI comments of include/dlrm_b200.h and the
semantics of optim/rwsadagrad.py, and the bounds or bitwise orders their tests compare against.  Independent of the
product: nothing here imports dlrm_b200.

Operations (inputs are fp32 values):
  gather       out[b] = sum_{j in bag b} rw[idx[j]] * W[idx[j]]; bag b = [off[b], off[b + 1]), the last bag runs to nnz
               unless include_last; a row-split shard [row_lo, row_lo + row_n) skips the other rows and reads local
               row idx - row_lo.  fp32 order: acc = 0, then acc + W[r] (unweighted) or fmaf(rw[r], W[r], acc) in index
               order -- promised bit for bit.
  coalesce     the occurrences of every touched row, ascending position; their dY rows summed exactly (the
               definition), in fp32 ascending position (lists of up to 32: the list kernels), or per 128-sample chunk
               then chunk partials in chunk order (the tiny-table kernels).  Lists longer than 32 take a fixed-point
               sum whose result depends only on the set of members: within one fp32 ulp of RN(exact), after the
               stated truncation of n * 2^(L + E - 62) per column (|value| < 2^E, n < 2^L).
  row step     SGD w -= lr g;  RWSAdagrad m += mean_D(g^2), w -= lr g / (sqrt(m) + eps).  fp32 orders: the general
               kernels fmaf(-lr, g / (sqrtf(m) + eps), w), the lean kernel fmaf(-lr / (sqrtf(m) + eps), g, w); the
               mean is sq * (1 / D) with sq an fmaf chain per lane, then a butterfly over the lanes.

Bounds follow oracle/dense_f64.py: fl(a op b) = (a op b)(1 + d), |d| <= u = 2^-24, gamma_n = n u / (1 - n u).
"""
from __future__ import annotations

import math

import numpy as np

from .dense_f64 import U, _fma_f32, check_within, f64, gamma, ulp_diff, worst_ratio  # noqa: F401  (re-exported)

OPT_SGD, OPT_RWSADAGRAD = 0, 1
SMALL_CHUNK = 128               # samples per accumulate chunk of the tiny-table update (csrc/emb_small.cu)
LIST_SORTED_MAX = 32            # longest list summed in ascending position; longer lists take the fixed-point sum
SUBNORMAL_HALF = 2.0 ** -150    # largest rounding error of an fp32 result in the subnormal range


def gammas(n):
    """gamma_n for an integer array n."""
    nu = np.asarray(n, np.float64) * U
    assert np.all(nu < 1.0)
    return nu / (1.0 - nu)


# ---------------------------------------------------------------------------------------------- bags and occurrences
def bag_bounds(off, nnz, include_last=False):
    """[start, end) of every bag: offsets has batch + 1 entries when include_last, else the last bag ends at nnz."""
    off = np.asarray(off, np.int64)
    if include_last:
        return off[:-1], off[1:]
    return off, np.append(off[1:], np.int64(nnz))


def occurrences(idx, off, nnz, include_last=False, row_lo=0, row_n=None):
    """(pos, bag, local row) of the occurrences that belong to this table (or shard), ascending position.  Without a
    shard every index in [0, row_n) belongs (row_n None: any non-negative index)."""
    start, end = bag_bounds(off, nnz, include_last)
    lens = np.maximum(end - start, 0)
    bag = np.repeat(np.arange(start.size), lens)
    first = np.repeat(np.cumsum(lens) - lens, lens)
    pos = start[bag] + (np.arange(bag.size) - first)
    r = np.asarray(idx)[pos].astype(np.int64) - row_lo
    keep = r >= 0 if row_n is None else (r >= 0) & (r < row_n)
    return pos[keep], bag[keep], r[keep]


def _rank_in_group(key):
    """For entries already in the order of summation: (stable order by key, rank of each entry inside its key)."""
    order = np.argsort(key, kind="stable")
    k = key[order]
    first = np.searchsorted(k, k, side="left")
    return order, np.arange(k.size) - first


# ---------------------------------------------------------------------------------------------- gather
def gather_f64(W, idx, off, nnz, include_last=False, rw=None, row_lo=0, row_n=None):
    """(out [batch, D] float64, bound): the bound of an fp32 sequential evaluation of a bag of L terms is
    gamma_L * sum |terms| (unweighted: L - 1 roundings; weighted: one fmaf rounding per term)."""
    start, _ = bag_bounds(off, nnz, include_last)
    B, D = start.size, W.shape[1]
    pos, bag, r = occurrences(idx, off, nnz, include_last, row_lo, row_n)
    terms = f64(W)[r] * (f64(rw)[r][:, None] if rw is not None else 1.0)
    out, mag = np.zeros((B, D)), np.zeros((B, D))
    np.add.at(out, bag, terms)
    np.add.at(mag, bag, np.abs(terms))
    return out, gammas(np.bincount(bag, minlength=B))[:, None] * mag


def fma_may_double_round(a, b, c):
    """Where _fma_f32(a, b, c) may differ from fmaf by one ulp: the float64 sum of the exact product and c lies on an
    fp32 rounding midpoint although the exact result does not."""
    p, c = f64(a) * f64(b), f64(c)
    s = p + c
    bv = s - p
    err = (p - (s - bv)) + (c - bv)                     # TwoSum: s + err == p + c exactly
    s32 = s.astype(np.float32)
    t = f64(s32)
    toward = np.where(s > t, np.float32(np.inf), np.float32(-np.inf))
    nb = f64(np.nextafter(s32, toward))
    return (s != t) & (np.abs(nb - s) == np.abs(s - t)) & (err != 0)


def gather_f32(W, idx, off, nnz, include_last=False, rw=None, row_lo=0, row_n=None, fused=True):
    """The kernels' fp32 order: (out [batch, D] fp32, flag) -- flag marks the outputs whose chain contains an fma step
    that _fma_f32 may have double-rounded (then only the bound of gather_f64 holds).  fused=False evaluates the
    weighted term with two roundings (w * x, then the add): not what the kernels do."""
    start, _ = bag_bounds(off, nnz, include_last)
    B, D = start.size, W.shape[1]
    W = np.asarray(W, np.float32)
    pos, bag, r = occurrences(idx, off, nnz, include_last, row_lo, row_n)
    acc = np.zeros((B, D), np.float32)
    flag = np.zeros((B, D), bool)
    order, rank = _rank_in_group(bag)
    for t in range(int(rank.max()) + 1 if rank.size else 0):
        sel = order[rank == t]
        b, x = bag[sel], W[r[sel]]
        if rw is None:
            acc[b] = acc[b] + x
        else:
            wt = np.asarray(rw, np.float32)[r[sel]][:, None]
            if fused:
                flag[b] |= fma_may_double_round(wt, x, acc[b])
                acc[b] = _fma_f32(wt, x, acc[b])
            else:
                acc[b] = wt * x + acc[b]
    return acc, flag


# ---------------------------------------------------------------------------------------------- coalesce
def coalesce(r):
    """(rows: the touched rows ascending, grp: the row index of every occurrence) -- grad.coalesce()'s order."""
    rows, grp = np.unique(np.asarray(r, np.int64), return_inverse=True)
    return rows, grp.reshape(-1)


def sum_exact(G, grp, nrows):
    """float64 [nrows, D]: exact (math.fsum per column) for rows with more than LIST_SORTED_MAX occurrences, a
    float64 sum (relative error ~ 32 * 2^-53, far below fp32) otherwise."""
    G = np.asarray(G, np.float32)
    out = np.zeros((nrows, G.shape[1]))
    np.add.at(out, grp, f64(G))
    cnt = np.bincount(grp, minlength=nrows)
    for i in np.nonzero(cnt > LIST_SORTED_MAX)[0]:
        out[i] = [math.fsum(col) for col in f64(G[grp == i]).T]
    return out


def _seq_f32(G, key, nkeys):
    """fp32 sum per key, from 0, in the order of the entries."""
    G = np.asarray(G, np.float32)
    acc = np.zeros((nkeys, G.shape[1]), np.float32)
    order, rank = _rank_in_group(key)
    for t in range(int(rank.max()) + 1 if rank.size else 0):
        sel = order[rank == t]
        acc[key[sel]] = acc[key[sel]] + G[sel]
    return acc


def sum_f32_ascending(G, grp, nrows):
    """The list kernels' sum of a row with up to 32 occurrences: 0 + g_p0 + g_p1 + ... in ascending position (G in
    ascending position)."""
    return _seq_f32(G, np.asarray(grp, np.int64), nrows)


def sum_f32_chunked(G, grp, nrows, bag, chunk=SMALL_CHUNK):
    """The tiny-table kernels' sum: a sequential fp32 sum per (chunk of `chunk` samples, row) in ascending position,
    then the chunk partials (0 for a chunk without the row) added in chunk order from 0."""
    c = np.asarray(bag, np.int64) // chunk
    nch = int(c.max()) + 1 if c.size else 0
    D = np.asarray(G).shape[1]
    part = _seq_f32(G, c * nrows + np.asarray(grp, np.int64), nch * nrows).reshape(nch, nrows, D)
    g = np.zeros((nrows, D), np.float32)
    for p in part:
        g = g + p
    return g


def sum_f32_chunked_bound(G, grp, nrows, bag, chunk=SMALL_CHUNK):
    """Bound of sum_f32_chunked against the exact sum: a chain of (members in the chunk) + (chunks) additions."""
    c = np.asarray(bag, np.int64) // chunk
    nch = int(c.max()) + 1 if c.size else 0
    per = np.bincount(c * nrows + grp, minlength=nch * nrows).reshape(nch, nrows).max(axis=0, initial=0)
    mag = np.zeros((nrows, np.asarray(G).shape[1]))
    np.add.at(mag, grp, np.abs(f64(G)))
    return gammas(per + nch)[:, None] * mag


def long_sum_ulps(got, members):
    """Distance in fp32 ulps of `got` [D] from [RN(s - T), RN(s + T)]: s = the exact column sums of `members` [n, D],
    T = n * 2^(L + E - 62) the fixed-point truncation (|value| < 2^E per column, n < 2^L).  The long-list sum
    promises <= 1 (the 62 -> 53 -> 24-bit double rounding of (float)((double)s / scale))."""
    members = f64(members)
    n = members.shape[0]
    exact = np.array([math.fsum(col) for col in members.T])
    _, E = np.frexp(np.abs(members).max(axis=0))
    T = n * np.ldexp(1.0, (n.bit_length() + E - 62).astype(np.int64))
    lo, hi = (exact - T).astype(np.float32), (exact + T).astype(np.float32)
    got = np.asarray(got, np.float32)
    return np.where(got < lo, ulp_diff(got, lo), np.where(got > hi, ulp_diff(got, hi), 0))


# ---------------------------------------------------------------------------------------------- row step
def row_step(w, m, g, opt, lr, eps):
    """The float64 definition on rows [n, D]: (w', m').  lr and eps are the fp32 values the kernels receive."""
    lr, eps = float(np.float32(lr)), float(np.float32(eps))
    w, g = f64(w), f64(g)
    if opt == OPT_RWSADAGRAD:
        m2 = f64(m) + (g * g).mean(axis=-1)
        return w - lr * g / (np.sqrt(m2) + eps)[..., None], m2
    return w - lr * g, None if m is None else f64(m)


def sq_f32(g, lanes=32, width=4):
    """sum of g^2 over a row in a kernel's order: lane (c / width) % lanes holds column c, an fmaf chain per lane
    over its columns in ascending order, then a butterfly (xor 16, 8, ...) over the lanes."""
    g = np.asarray(g, np.float32)
    n, D = g.shape
    lane_of = (np.arange(D) // width) % lanes
    part = np.zeros((n, lanes), np.float32)
    for c in range(D):
        part[:, lane_of[c]] = _fma_f32(g[:, c], g[:, c], part[:, lane_of[c]])
    o = lanes // 2
    while o:
        part = part + part[:, np.arange(lanes) ^ o]
        o //= 2
    return part[:, 0]


def row_step_f32(w, m, g, opt, lr, eps, kernel="general"):
    """The step in fp32 in a kernel's order: (w', m').  kernel = "general" (emb_update_kernel, the tiny-table apply
    kernel): fmaf(-lr, g / std, w); "lean" (emb_update_lean_kernel): fmaf(-lr / std, g, w)."""
    w, g = np.asarray(w, np.float32), np.asarray(g, np.float32)
    lr, eps = np.float32(lr), np.float32(eps)
    if opt != OPT_RWSADAGRAD:
        return _fma_f32(-lr, g, w), m
    D = g.shape[1]
    lanes, width = (16, 8) if kernel == "lean" else (32, 4)
    m2 = np.asarray(m, np.float32) + sq_f32(g, lanes, width) * (np.float32(1) / np.float32(D))
    std = (np.sqrt(m2) + eps)[:, None]
    if kernel == "lean":
        return _fma_f32(-lr / std, g, w), m2
    return _fma_f32(-lr, g / std, w), m2


def row_step_bound(w2, m2, g, opt, lr, eps, g_rel=0.0):
    """Bounds (on w', on m') of an fp32 step in either order against row_step's (w2, m2), for the gradient g (fp32)
    that the kernel summed; g_rel = the relative error g may already carry (2u for a long list: one ulp).
      m':  sq has a depth of at most max(4, ceil(D / 16)) fmaf plus 5 tree levels, then * fl(1 / D) and + m: three
           more roundings (or fewer when contracted), plus subnormal rounding of tiny squares;
      std: sqrtf + the eps add (2 roundings), and the m' error through sqrt: min(sqrt(dm), dm / (2 sqrt(m')));
      w':  g / std (or -lr / std) and the fmaf: 2 roundings on the update, 1 on w'."""
    lr, eps = float(np.float32(lr)), float(np.float32(eps))
    g = f64(g)
    if opt != OPT_RWSADAGRAD:
        return gamma(1) * np.abs(f64(w2)) + lr * np.abs(g) * g_rel * 1.01 + SUBNORMAL_HALF, None
    D = g.shape[-1]
    depth = max(4, -(-D // 16)) + 5
    s = (g * g).mean(axis=-1)
    bm = gamma(depth + 3) * s + gamma(1) * np.abs(m2) + 2.02 * g_rel * s + (depth + 3) * SUBNORMAL_HALF
    rm = np.sqrt(m2)
    e_root = np.minimum(np.sqrt(bm), np.where(rm > 0, bm / (2 * np.where(rm > 0, rm, 1.0)), np.inf))
    std = rm + eps
    rel_std = e_root / std + gamma(2)
    upd = lr * np.abs(g) / std[..., None]
    bw = gamma(1) * np.abs(f64(w2)) + upd * (1.01 * (rel_std[..., None] + g_rel) + gamma(3)) + SUBNORMAL_HALF
    return bw, bm
