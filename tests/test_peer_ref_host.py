"""oracle/peer_f64.py on the CPU: the routes, the fp32 all-reduce against the float64 mean, the barrier's expected
state, and negative controls -- plausible kernel mistakes that the bitwise checks of tests/test_gpu_peer_kernels.py
must reject: routing by b % W, summing the ranks in reverse order, dividing by W instead of multiplying by fp32(1 / W),
and a barrier that writes slot t instead of slot rank."""
import numpy as np
import pytest

from oracle import peer_f64 as P


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("W,bl", [(1, 5), (2, 1), (3, 37), (8, 4)])
def test_route_split_join(W, bl):
    b = np.arange(W * bl)
    r, row = P.route(b, bl)
    assert np.array_equal(r, b // bl) and np.array_equal(row, b % bl)
    assert r.min() == 0 and r.max() == W - 1 and row.max() == bl - 1
    g = np.random.default_rng(W).standard_normal((W * bl, 3)).astype(np.float32)
    slabs = P.split(g, W)
    for k in range(W):
        assert np.array_equal(slabs[k], g[r == k][np.argsort(row[r == k])])
    assert _same(P.join(slabs), g)


@pytest.mark.parametrize("W", [1, 2, 3, 5, 8])
def test_allreduce_f32_within_the_f64_bound(W):
    rng = np.random.default_rng(W)
    bufs = [(rng.choice([-1.0, 1.0], 4000) * np.exp2(rng.uniform(-20, 20, 4000))).astype(np.float32)
            for _ in range(W)]
    got = P.allreduce_mean_f32(bufs)
    want, bound = P.allreduce_mean_f64(bufs)
    err = np.abs(got.astype(np.float64) - want)
    assert np.all(err <= bound)
    assert got.dtype == np.float32
    if W == 1:
        assert _same(got, bufs[0])


def test_control_routing_by_modulo_is_rejected():
    """A gather that routed bag b to rank b % W would fill peer buffer r with other bags than split() expects."""
    W, bl = 3, 5
    g = np.arange(W * bl * 2, dtype=np.float32).reshape(W * bl, 2)
    b = np.arange(W * bl)
    bad = [g[b % W == r] for r in range(W)]
    want = P.split(g, W)
    assert not all(_same(x, y) for x, y in zip(bad, want))


def test_control_reverse_rank_order_is_rejected():
    """fp32 addition is not associative: 1 + 2^-24 + 2^-24 summed from rank 0 gives 1, from rank 2 gives 1 + 2^-23."""
    bufs = [np.array([1.0], np.float32), np.array([2.0 ** -24], np.float32), np.array([2.0 ** -24], np.float32)]
    rev = P.allreduce_mean_f32(bufs[::-1])
    assert not _same(rev, P.allreduce_mean_f32(bufs))
    want, bound = P.allreduce_mean_f64(bufs)            # both orders are within the bound: only bits tell them apart
    assert np.all(np.abs(rev - want) <= bound)


def test_control_division_by_world_is_rejected():
    """At W = 3, s * fp32(1/3) and s / 3 differ for some fp32 s; a kernel that divides fails the bitwise check."""
    s = np.arange(1, 4097, dtype=np.float32)
    bufs = [s, np.zeros_like(s), np.zeros_like(s)]
    mul = P.allreduce_mean_f32(bufs)
    div = s / np.float32(3)
    differ = mul != div
    assert differ.any() and not _same(div, mul)
    want, bound = P.allreduce_mean_f64(bufs)
    assert np.all(np.abs(div - want) <= bound)         # the division is accurate too: only bits tell them apart


@pytest.mark.parametrize("W", [1, 2, 4, 8])
def test_barrier_expected_state(W):
    sent = -5
    sig = np.full((W, 16), sent, np.int64)
    for rank in range(W):
        e, after = P.barrier_after(sig, 41, rank)
        assert e == 42
        assert np.all(after[:, rank] == 42)
        rest = np.ones_like(after, bool)
        rest[:, rank] = False
        assert np.all(after[rest] == sent)
        # control: a barrier that stores into slot t of rank t's array (sig[t][t]) instead of slot rank
        bad = sig.copy()
        for t in range(W):
            bad[t, t] = e
        assert W == 1 or not np.array_equal(bad, after)
