"""oracle/sparse_f64.py on the CPU: every restatement against torch float64, the fp32 evaluations in the kernels'
orders within their bounds, and negative controls -- plausible kernel mistakes that the checks of
tests/test_gpu_sparse_kernels.py (bitwise comparisons, bounds, the long-list property) must reject."""
import math

import numpy as np
import pytest
import torch

from oracle import dlrm_numpy as N
from oracle import sparse_f64 as S


def _bags(rng, B, rows, lmax, nnz_extra=0):
    lens = rng.integers(0, lmax + 1, B)
    off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    idx = rng.integers(0, rows, int(lens.sum()) + nnz_extra).astype(np.int64)
    return off, idx


def _torch_bag(W, idx, off, psw=None, include_last=False):
    return torch.nn.functional.embedding_bag(torch.from_numpy(idx), torch.from_numpy(W.astype(np.float64)),
                                             torch.from_numpy(off), mode="sum", include_last_offset=include_last,
                                             per_sample_weights=None if psw is None else
                                             torch.from_numpy(psw.astype(np.float64))).numpy()


def _wide(rng, shape):
    """fp32 values over 2^-12 .. 2^12 with random signs: their fp32 sums depend on the order of the terms."""
    return (rng.choice([-1.0, 1.0], shape) * np.exp2(rng.uniform(-12, 12, shape))).astype(np.float32)


# ---------------------------------------------------------------------------------------------- gather
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("include_last", [False, True])
def test_gather_f64_is_embedding_bag(weighted, include_last):
    rng = np.random.default_rng(1)
    W = rng.standard_normal((300, 12)).astype(np.float32)
    rw = rng.uniform(0.5, 1.5, 300).astype(np.float32) if weighted else None
    off, idx = _bags(rng, 57, 300, 9)
    o = np.append(off, idx.size) if include_last else off
    got, bound = S.gather_f64(W, idx, o, idx.size, include_last, rw)
    want = _torch_bag(W, idx, o, None if rw is None else rw[idx], include_last)
    np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-13)
    assert np.all(bound >= 0)


def test_gather_f64_row_split_skips_other_shards():
    rng = np.random.default_rng(2)
    W = rng.standard_normal((400, 8)).astype(np.float32)
    rw = rng.uniform(0.5, 1.5, 400).astype(np.float32)
    off, idx = _bags(rng, 40, 400, 12)
    lo, n = 120, 150
    got, _ = S.gather_f64(W[lo:lo + n], idx, off, idx.size, rw=rw[lo:lo + n], row_lo=lo, row_n=n)
    mine = ((idx >= lo) & (idx < lo + n)).astype(np.float64)
    want = _torch_bag(W, idx, off, rw[idx] * mine)
    np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("include_last", [False, True])
def test_gather_f32_unweighted_is_the_sequential_sum_bitwise(include_last):
    rng = np.random.default_rng(3)
    W = _wide(rng, (200, 16))
    off, idx = _bags(rng, 80, 200, 20)
    o = np.append(off, idx.size) if include_last else off
    got, flag = S.gather_f32(W, idx, o, idx.size, include_last)
    assert np.array_equal(got, N.emb_bag_sum(W, idx, off)) and not flag.any()


@pytest.mark.parametrize("weighted", [False, True])
def test_gather_f32_within_bound(weighted):
    rng = np.random.default_rng(4)
    W = _wide(rng, (500, 32))
    rw = rng.uniform(-2, 2, 500).astype(np.float32) if weighted else None
    off, idx = _bags(rng, 300, 500, 40)
    got, _ = S.gather_f32(W, idx, off, idx.size, rw=rw)
    want, bound = S.gather_f64(W, idx, off, idx.size, rw=rw)
    S.check_within(got, want, bound, "gather_f32")


def test_fma_double_rounding_flag():
    # (1 + 2^-23)(2^-24 - 2^-47) + (1 + 2^-23) = 1 + 2^-23 + 2^-24 - 2^-70: just below an fp32 midpoint, so fmaf gives
    # 1 + 2^-23; the float64 sum rounds onto the midpoint and the second rounding goes to even, 1 + 2^-22
    a, b, c = np.float32(1 + 2.0 ** -23), np.float32(2.0 ** -24 - 2.0 ** -47), np.float32(1 + 2.0 ** -23)
    assert S.fma_may_double_round(a, b, c)
    assert S._fma_f32(a, b, c) == np.float32(1 + 2.0 ** -22)
    assert not S.fma_may_double_round(np.float32(2.0 ** -24), np.float32(1 + 2.0 ** -23), np.float32(1.0))
    assert not S.fma_may_double_round(np.float32(0.1), np.float32(3.0), np.float32(1.0))


# ---------------------------------------------------------------------------------------------- coalesce
def test_coalesce_is_torch_sparse_coalesce():
    rng = np.random.default_rng(5)
    D, rows = 6, 40
    off, idx = _bags(rng, 300, rows, 6)
    dY = _wide(rng, (300, D))
    pos, bag, r = S.occurrences(idx, off, idx.size)
    G = dY[bag]
    uniq, grp = S.coalesce(r)
    got = S.sum_exact(G, grp, uniq.size)
    t = torch.sparse_coo_tensor(torch.from_numpy(r)[None], torch.from_numpy(G.astype(np.float64)), (rows, D)).coalesce()
    assert np.array_equal(t.indices()[0].numpy(), uniq)
    np.testing.assert_allclose(got, t.values().numpy(), rtol=1e-12, atol=1e-9)
    # rows with more than 32 occurrences are exact
    cnt = np.bincount(grp)
    for i in np.nonzero(cnt > 32)[0]:
        assert np.array_equal(got[i], [math.fsum(c) for c in G[grp == i].astype(np.float64).T])


def test_fp32_sums_within_bound():
    rng = np.random.default_rng(6)
    B, D, rows = 700, 8, 5
    off, idx = _bags(rng, B, rows, 3)
    dY = _wide(rng, (B, D))
    pos, bag, r = S.occurrences(idx, off, idx.size)
    uniq, grp = S.coalesce(r)
    exact = S.sum_exact(dY[bag], grp, uniq.size)
    mag = np.zeros_like(exact)
    np.add.at(mag, grp, np.abs(dY[bag].astype(np.float64)))
    asc = S.sum_f32_ascending(dY[bag], grp, uniq.size)
    S.check_within(asc, exact, S.gammas(np.bincount(grp))[:, None] * mag, "ascending")
    ch = S.sum_f32_chunked(dY[bag], grp, uniq.size, bag)
    S.check_within(ch, exact, S.sum_f32_chunked_bound(dY[bag], grp, uniq.size, bag), "chunked")
    # one chunk: the chunked sum is the ascending sum
    one = bag < S.SMALL_CHUNK
    _, g1 = S.coalesce(r[one])
    assert np.array_equal(S.sum_f32_chunked(dY[bag[one]], g1, g1.max() + 1, bag[one]),
                          S.sum_f32_ascending(dY[bag[one]], g1, g1.max() + 1))


def _fixed_point_sum(vals):
    """The long-list kernel's arithmetic (list_sum_exact, csrc/emb_bwd.cu) per column, in an arbitrary member order."""
    vals = np.asarray(vals, np.float32)
    n = vals.shape[0]
    L = n.bit_length()
    out = []
    for col in vals.T:
        _, E = math.frexp(float(np.abs(col).max()))
        sc = math.ldexp(1.0, 62 - L - E)
        s = sum(int(float(v) * sc) for v in col)            # (long long) truncates toward zero; exact int sum
        out.append(np.float32(float(s) / sc))
    return np.array(out, np.float32)


@pytest.mark.parametrize("n", [33, 128, 129, 1000])
def test_long_list_property_holds_for_the_fixed_point_sum(n):
    rng = np.random.default_rng(n)
    vals = _wide(rng, (n, 24))
    for perm in (np.arange(n), rng.permutation(n)):
        got = _fixed_point_sum(vals[perm])
        assert np.all(S.long_sum_ulps(got, vals) <= 1)
    assert np.array_equal(_fixed_point_sum(vals), _fixed_point_sum(vals[::-1]))


# ---------------------------------------------------------------------------------------------- row step
def _torch_step(w, m, g, opt, lr, eps):
    w, g = torch.from_numpy(w.astype(np.float64)), torch.from_numpy(g.astype(np.float64))
    lr, eps = float(np.float32(lr)), float(np.float32(eps))
    if opt == S.OPT_RWSADAGRAD:                                 # optim/rwsadagrad.py: sparse branch
        m = torch.from_numpy(m.astype(np.float64)) + g.pow(2).mean(dim=1)
        return w.addcdiv(g, m.sqrt().add(eps)[:, None], value=-lr).numpy(), m.numpy()
    return w.add(g, alpha=-lr).numpy(), None


@pytest.mark.parametrize("opt", [S.OPT_SGD, S.OPT_RWSADAGRAD])
def test_row_step_is_the_torch_step(opt):
    rng = np.random.default_rng(7)
    w = rng.standard_normal((50, 20)).astype(np.float32)
    g = rng.standard_normal((50, 20)).astype(np.float32) * 0.01
    m = rng.uniform(0, 1e-3, 50).astype(np.float32)
    got, gm = S.row_step(w, m, g, opt, 0.05, 1e-8)
    want, wm = _torch_step(w, m, g, opt, 0.05, 1e-8)
    np.testing.assert_allclose(got, want, rtol=1e-14, atol=1e-15)
    if opt == S.OPT_RWSADAGRAD:
        np.testing.assert_allclose(gm, wm, rtol=1e-14)


@pytest.mark.parametrize("kernel", ["general", "lean"])
@pytest.mark.parametrize("D", [4, 6, 100, 128, 260, 1023])
@pytest.mark.parametrize("opt", [S.OPT_SGD, S.OPT_RWSADAGRAD])
def test_row_step_f32_within_bound(opt, D, kernel):
    rng = np.random.default_rng(D)
    n = 64
    w = rng.standard_normal((n, D)).astype(np.float32) * 0.1
    g = _wide(rng, (n, D)) * np.float32(2.0 ** -14)
    g[:4] *= np.float32(2.0 ** -100)                           # squares underflow in fp32
    w[:4] = 0.0
    m = rng.uniform(0, 1e-4, n).astype(np.float32)
    m[:2] = 0.0
    for eps in (1e-10, 1e-4):
        w2, m2 = S.row_step(w, m, g, opt, 0.05, eps)
        bw, bm = S.row_step_bound(w2, m2, g, opt, 0.05, eps)
        gw, gm = S.row_step_f32(w, m, g, opt, 0.05, eps, kernel)
        S.check_within(gw, w2, bw, "w")
        if opt == S.OPT_RWSADAGRAD:
            S.check_within(gm, m2, bm, "m")
            assert np.all(gw[:4] != 0)                          # the underflowed rows are still updated


# ---------------------------------------------------------------------------------------------- negative controls
def test_control_descending_order_is_rejected():
    rng = np.random.default_rng(10)
    G = _wide(rng, (31, 64))
    grp = np.zeros(31, np.int64)
    asc = S.sum_f32_ascending(G, grp, 1)
    desc = S.sum_f32_ascending(G[::-1], grp, 1)
    assert not np.array_equal(asc, desc)


def test_control_33_member_list_losing_a_member_is_rejected():
    rng = np.random.default_rng(11)
    vals = _wide(rng, (33, 64))
    assert np.all(S.long_sum_ulps(_fixed_point_sum(vals), vals) <= 1)
    assert np.any(S.long_sum_ulps(_fixed_point_sum(vals[:-1]), vals) > 1)
    # and an fp32 sum in list order (not order-independent) misses the property somewhere
    naive = np.zeros(64, np.float32)
    for v in vals[rng.permutation(33)]:
        naive = naive + v
    assert np.any(S.long_sum_ulps(naive, vals) > 1)


def _step_variant(w, m, g, lr, eps, cols=None, eps_inside=False):
    """RWSAdagrad in fp32 with a mistake: the mean over `cols` columns instead of dim, or eps inside the sqrt."""
    w, g = np.asarray(w, np.float32), np.asarray(g, np.float32)
    cols = g.shape[1] if cols is None else cols
    m2 = m + (g.astype(np.float64) ** 2).sum(axis=1).astype(np.float32) * (np.float32(1) / np.float32(cols))
    std = np.sqrt(m2 + np.float32(eps)) if eps_inside else np.sqrt(m2) + np.float32(eps)
    return S._fma_f32(-np.float32(lr), g / std[:, None], w), m2


@pytest.mark.parametrize("mistake", ["mean_over_ld", "eps_inside_sqrt"])
def test_control_wrong_step_is_rejected(mistake):
    rng = np.random.default_rng(12)
    D, ld, eps = 128, 132, 1e-4
    w = rng.standard_normal((64, D)).astype(np.float32) * 0.1
    g = rng.standard_normal((64, D)).astype(np.float32) * 0.01
    m = rng.uniform(0, 1e-4, 64).astype(np.float32)
    w2, m2 = S.row_step(w, m, g, S.OPT_RWSADAGRAD, 0.05, eps)
    bw, bm = S.row_step_bound(w2, m2, g, S.OPT_RWSADAGRAD, 0.05, eps)
    kw = dict(cols=ld) if mistake == "mean_over_ld" else dict(eps_inside=True)
    gw, gm = _step_variant(w, m, g, 0.05, eps, **kw)
    assert S.worst_ratio(gw, w2, bw)[0] > 1.0
    if mistake == "mean_over_ld":
        assert S.worst_ratio(gm, m2, bm)[0] > 1.0
    ok_w, _ = _step_variant(w, m, g, 0.05, eps)                # the correct variant passes the same check
    S.check_within(ok_w, w2, bw, "correct variant")


def test_control_row_lo_not_subtracted_is_rejected():
    rng = np.random.default_rng(13)
    W = rng.standard_normal((400, 16)).astype(np.float32)
    off, idx = _bags(rng, 50, 400, 8)
    lo, n = 100, 200
    right, _ = S.gather_f32(W[lo:lo + n], idx, off, idx.size, row_lo=lo, row_n=n)
    # the shard's indices read as W_shard[idx] = W[lo + idx] (the rows behind the shard exist in the whole table)
    wrong = np.zeros_like(right)
    pos, bag, r = S.occurrences(idx, off, idx.size, row_lo=lo, row_n=n)
    for b, j in zip(bag, pos):
        wrong[b] = wrong[b] + W[lo + idx[j]]
    assert not np.array_equal(right, wrong)


def test_control_last_bag_cut_short_is_rejected():
    rng = np.random.default_rng(14)
    W = rng.standard_normal((100, 16)).astype(np.float32)
    off, idx = _bags(rng, 20, 100, 6, nnz_extra=5)              # the last bag runs 5 positions past its length
    right, _ = S.gather_f32(W, idx, off, idx.size)
    cut, _ = S.gather_f32(W, idx, off, idx.size - 1)
    assert not np.array_equal(right, cut)
    assert np.array_equal(right[:-1], cut[:-1])


def test_control_127_sample_chunks_are_rejected():
    rng = np.random.default_rng(15)
    B, D = 1000, 16
    off = np.arange(B, dtype=np.int64)
    idx = np.zeros(B, np.int64)                                 # a 1-row table hit by every sample
    dY = _wide(rng, (B, D))
    pos, bag, r = S.occurrences(idx, off, B)
    _, grp = S.coalesce(r)
    assert not np.array_equal(S.sum_f32_chunked(dY[bag], grp, 1, bag, 128),
                              S.sum_f32_chunked(dY[bag], grp, 1, bag, 127))


def test_control_weighted_gather_with_two_roundings_is_rejected():
    rng = np.random.default_rng(16)
    W = _wide(rng, (300, 32))
    rw = rng.uniform(0.3, 3, 300).astype(np.float32)
    off, idx = _bags(rng, 100, 300, 10)
    fused, flag = S.gather_f32(W, idx, off, idx.size, rw=rw)
    unfused, _ = S.gather_f32(W, idx, off, idx.size, rw=rw, fused=False)
    assert not np.array_equal(fused[~flag], unfused[~flag])


def test_control_tiny_table_step_skipping_underflowed_rows_is_rejected():
    D, lr, eps = 128, 0.05, 1e-10
    g = np.full((1, D), 1e-24, np.float32)                     # g^2 underflows to 0 in fp32
    w = np.zeros((1, D), np.float32)
    m = np.zeros(1, np.float32)
    w2, m2 = S.row_step(w, m, g, S.OPT_RWSADAGRAD, lr, eps)
    bw, _ = S.row_step_bound(w2, m2, g, S.OPT_RWSADAGRAD, lr, eps)
    assert S.sq_f32(g)[0] == 0.0
    gw, _ = S.row_step_f32(w, m, g, S.OPT_RWSADAGRAD, lr, eps)
    S.check_within(gw, w2, bw, "the step of a row whose sum of squares underflowed")
    assert S.worst_ratio(w, w2, bw)[0] > 1.0                    # skipping the row (w unchanged) is rejected
