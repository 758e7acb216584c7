"""The peer-memory exchange kernels of a sharded step at world sizes 1 to 8 on ONE GPU.  Every one of them takes its
peers as an array of plain device pointers, so W allocations on cuda:0 are W virtual ranks: the routed gather
(`emb_bag_fwd_p2p` with `train`), the peer-sourced list update (`emb_bwd_update_p2p`), the tiny-table update with
`peer_dY`, the remote-read gather, the routed interaction backward, the dense all-reduce, the barrier and
`block_copy`.

Each routed call is compared bit for bit with the same entry point without peers over the whole batch (same dtype,
alignment and kernel selection), and that result with the restatements of oracle/sparse_f64.py / dense_f64.py /
peer_f64.py.  Outputs are prefilled with NaN; what a kernel must not write (pad columns, the row past batch_local in
every peer buffer, other slots and slabs, untouched rows and accumulators) holds a sentinel that is compared bit for
bit afterwards; list heads and marks must be zero again and the device error word clear.  The worst err/bound ratio
of every family is printed at the end of the module (`pytest -s`).

The barrier cases never wait: before every call each slot it polls already holds at least the epoch it reaches."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from dlrm_b200 import _lib
from dlrm_b200 import placement as PL
from dlrm_b200 import sharding as SH
from oracle import dense_f64 as DF
from oracle import peer_f64 as P
from oracle import sparse_f64 as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = -7.75e33                 # fp32 sentinel of regions that must stay untouched
SENT_BITS = np.float32(SENT).view(np.uint32)
SGD, RWS, ADA = _lib.OPT_SGD, _lib.OPT_RWSADAGRAD, _lib.OPT_ADAGRAD
F16_PAD = np.float16(-7.5)
WORST = {}


def _record(family, r):
    WORST[family] = max(WORST.get(family, 0.0), float(r))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst err/bound per kernel family: " + json.dumps({k: float("%.3g" % v) for k, v in sorted(WORST.items())}))


def L():
    return _lib.lib()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _no_device_errors():
    assert L().dlrm_b200_check_device_errors(_st()) == 0, "an index was reported outside its table"


def _same_bits(a, b, what):
    a = a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    b = b.cpu().numpy() if torch.is_tensor(b) else np.asarray(b)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), what


def _all_sent(a, what):
    a = np.asarray(a, np.float32)
    assert np.all(a.view(np.uint32) == SENT_BITS), what


def _ceil4(n):
    return (n + 3) // 4 * 4


def _wide(rng, shape, lo=-8, hi=2):
    """fp32 values of both signs over 2^lo .. 2^hi: their fp32 sums depend on the order of the terms."""
    return (rng.choice([-1.0, 1.0], shape) * np.exp2(rng.uniform(lo, hi, shape))).astype(np.float32)


def _offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)


def _vp(ptrs):
    return (C.c_void_p * len(ptrs))(*ptrs)


def _rows_table(rng, R, D, f16, lo=-4, hi=0):
    """(fp32 values [R, D] the kernels see, host storage [R, ld] with a sentinel pad, ld): fp16 rows are stored as
    halves and widened exactly."""
    if f16:
        ld = D + 8
        Wh = np.full((R, ld), F16_PAD, np.float16)
        Wh[:, :D] = _wide(rng, (R, D), lo, hi).astype(np.float16)
        return Wh[:, :D].astype(np.float32), Wh, ld
    ld = _ceil4(D) + 4
    Wf = np.full((R, ld), SENT, np.float32)
    Wf[:, :D] = _wide(rng, (R, D), lo, hi)
    return Wf[:, :D].copy(), Wf, ld


def _dev_table(host):
    return _cuda(host.view(np.int16)).view(torch.float16) if host.dtype == np.float16 else _cuda(host)


def _host(t):
    return t.view(torch.int16).cpu().numpy().view(np.float16) if t.dtype == torch.float16 else t.cpu().numpy()


def _bags(rng, B, R, il, lens=(0, 1, 3, 4, 5, 9, 7, 8, 17), tail=5):
    """(idx, off, nnz) of B bags over R rows; include_last: offsets [B + 1] and a capacity tail of out-of-range
    indices past offsets[B]."""
    n = rng.permutation(np.resize(np.asarray(lens), B))
    idx = rng.integers(0, R, int(n.sum())).astype(np.int64)
    off = _offsets(n)
    if il:
        off = np.append(off, idx.size)
        idx = np.append(idx, np.full(tail, R + 11, np.int64))
    return idx, off, (int(off[-1]) if il else idx.size)


# ---------------------------------------------------------------------------------------------- F. all-reduce
@pytest.mark.parametrize("W", [1, 2, 3, 5, 8])
def test_allreduce_mean(W):
    """Every virtual rank reduces its slice; called in rank order and in reverse (the slices are disjoint, so both give
    the same bits).  n from 0 to 2^20 + 7 (the grid-stride loop past 592 CTAs at W <= 5).  Every rank's buffer equals
    the fp32 restatement (sum from 0 in rank order, times fp32(1 / W)) and is within the float64 bound; elements past
    n keep the sentinel.  The reverse-order run keeps all ranks' buffers in one allocation."""
    rng = np.random.default_rng(100 + W)
    pad = 40
    for n in sorted({0, 1, max(W - 1, 0), W, W + 1, 1000003, 2 ** 20 + 7}):
        host = np.full((W, n + pad), SENT, np.float32)
        host[:, :n] = _wide(rng, (W, n), -20, 20)
        want = P.allreduce_mean_f32(list(host[:, :n]))
        ref, bound = P.allreduce_mean_f64(list(host[:, :n]))
        runs = []
        for order, shared in ((range(W), False), (range(W - 1, -1, -1), True)):
            if shared:
                big = _cuda(host)
                bufs = [big[r] for r in range(W)]
            else:
                bufs = [_cuda(host[r]) for r in range(W)]
            peers = _vp([b.data_ptr() for b in bufs])
            for r in order:
                _lib.check(L().dlrm_b200_p2p_allreduce_mean(peers, r, W, n, _st()), "p2p_allreduce_mean")
            got = np.stack([b.cpu().numpy() for b in bufs])
            for r in range(W):
                _same_bits(got[r, :n], want, f"n={n} rank {r}: not the fp32 rank-order mean")
                _all_sent(got[r, n:], f"n={n} rank {r}: wrote past n")
            runs.append(got)
        _same_bits(runs[0], runs[1], f"n={n}: rank order changed the result")
        _record("allreduce", DF.check_within(runs[0][0, :n], ref, bound, f"n={n}"))


def test_allreduce_argument_errors_launch_nothing():
    rng = np.random.default_rng(1)
    host = _wide(rng, (9, 64))
    bufs = [_cuda(h) for h in host]
    p2, p9 = _vp([b.data_ptr() for b in bufs[:2]]), _vp([b.data_ptr() for b in bufs])
    bad = [(p2, 0, 0, 64), (p9, 0, 9, 64), (p2, 2, 2, 64), (p2, -1, 2, 64), (_vp([bufs[0].data_ptr(), None]), 0, 2, 64),
           (p2, 0, 2, -1), (None, 0, 2, 64)]
    for peers, rank, world, n in bad:
        rc = L().dlrm_b200_p2p_allreduce_mean(peers, rank, world, n, _st())
        assert rc != 0 and b"p2p_allreduce_mean" in L().dlrm_b200_last_error(), (rank, world, n)
    torch.cuda.synchronize()
    for b, h in zip(bufs, host):
        _same_bits(b, h, "a refused all-reduce wrote a buffer")


# ---------------------------------------------------------------------------------------------- G. barrier
SIG_SENT = -123456


@pytest.mark.parametrize("W", [1, 2, 4, 8])
def test_barrier_epoch_and_slots(W):
    """Two rounds on both 16-slot channels at the 64-byte offset of the engine's signal array.  Before each call the
    slots it polls, sig[rank][0..W), hold at least the epoch it reaches, so the wait ends on its first read.  After it:
    the epoch word advanced by 1, sig[t][rank] == the new epoch for every t, every other slot unchanged."""
    sig = [torch.full((32,), SIG_SENT, dtype=torch.int32, device=DEV) for _ in range(W)]
    ep = np.array([[5 + 3 * r, 900 + r] for r in range(W)], np.int64)
    epoch = [_cuda(e.astype(np.int32)) for e in ep]
    state = np.full((W, 32), SIG_SENT, np.int64)
    for rnd in range(2):
        for ch in range(2):
            peers = _vp([s.data_ptr() + 64 * ch for s in sig])
            cols = slice(16 * ch, 16 * ch + 16)
            for rank in range(W):
                ready = int(ep[rank, ch]) + 1 + 1000 * (rnd + 1) + rank      # >= the epoch this call reaches
                sig[rank][16 * ch:16 * ch + W] = ready
                state[rank, 16 * ch:16 * ch + W] = ready
                _lib.check(L().dlrm_b200_p2p_barrier(peers, rank, W, epoch[rank].data_ptr() + 4 * ch, _st()),
                           "p2p_barrier")
                e, after = P.barrier_after(state[:, cols], ep[rank, ch], rank)
                state[:, cols], ep[rank, ch] = after, e
                got = np.stack([s.cpu().numpy() for s in sig]).astype(np.int64)
                assert np.array_equal(got, state), f"round {rnd} channel {ch} rank {rank}: signal slots"
                got_ep = np.stack([x.cpu().numpy() for x in epoch]).astype(np.int64)
                assert np.array_equal(got_ep, ep), f"round {rnd} channel {ch} rank {rank}: epoch words"


def test_barrier_argument_errors_launch_nothing():
    sig = [torch.full((16,), SIG_SENT, dtype=torch.int32, device=DEV) for _ in range(9)]
    epoch = torch.zeros(1, dtype=torch.int32, device=DEV)
    p2, p9 = _vp([s.data_ptr() for s in sig[:2]]), _vp([s.data_ptr() for s in sig])
    e = epoch.data_ptr()
    bad = [(p2, 0, 0, e), (p9, 0, 9, e), (p2, 2, 2, e), (p2, -1, 2, e), (p2, 0, 2, None),
           (_vp([sig[0].data_ptr(), None]), 0, 2, e), (None, 0, 2, e)]
    for peers, rank, world, ep in bad:
        rc = L().dlrm_b200_p2p_barrier(peers, rank, world, ep, _st())
        assert rc != 0 and b"p2p_barrier" in L().dlrm_b200_last_error(), (rank, world)
    torch.cuda.synchronize()
    assert int(epoch.item()) == 0
    for s in sig:
        assert np.all(s.cpu().numpy() == SIG_SENT), "a refused barrier wrote a slot"


# ---------------------------------------------------------------------------------------------- H. block_copy
def test_block_copy_64_blocks_into_shared_allocations():
    """64 blocks of 0 to 1 MiB pushed to offsets of four shared allocations with gaps between them (the index exchange
    of a sharded step); every byte around a destination keeps its sentinel."""
    rng = np.random.default_rng(3)
    sizes = [0, 16, 1 << 20] + [int(s) * 16 for s in rng.integers(0, 4096, 61)]
    srcs_h = [rng.integers(0, 256, max(s, 16), dtype=np.uint8) for s in sizes]
    srcs = [_cuda(h) for h in srcs_h]
    cursor, where = [0] * 4, []
    for k, s in enumerate(sizes):
        a = k % 4
        cursor[a] += 16 * int(rng.integers(1, 4))
        where.append((a, cursor[a]))
        cursor[a] += s
    dst_h = [np.full(c + 48, 0xA5, np.uint8) for c in cursor]
    dsts = [_cuda(h) for h in dst_h]
    n = len(sizes)
    _lib.check(L().dlrm_b200_block_copy(_vp([s.data_ptr() for s in srcs]),
                                        _vp([dsts[a].data_ptr() + o for a, o in where]),
                                        (C.c_int64 * n)(*sizes), n, _st()), "block_copy")
    for k, (a, o) in enumerate(where):
        dst_h[a][o:o + sizes[k]] = srcs_h[k][:sizes[k]]
    for d, h in zip(dsts, dst_h):
        _same_bits(d, h, "block_copy: destination bytes")


def test_block_copy_errors_launch_nothing():
    src = [_cuda(np.arange(64, dtype=np.uint8)) for _ in range(65)]
    dst = _cuda(np.full(65 * 64 + 32, 0xA5, np.uint8))
    dp = [dst.data_ptr() + 64 * k for k in range(65)]
    sp = [s.data_ptr() for s in src]
    cases = [(sp, dp, [64] * 65, 65, "n=65"),
             (sp[:1], dp[:1], [8], 1, "16-byte"),
             (sp[:2], dp[:2], [64, 24], 2, "16-byte"),
             ([sp[0], sp[1] + 4], dp[:2], [32, 32], 2, "16-byte"),
             (sp[:2], [dp[0], dp[1] + 4], [32, 32], 2, "16-byte")]
    for s, d, nb, n, msg in cases:
        rc = L().dlrm_b200_block_copy(_vp(s), _vp(d), (C.c_int64 * n)(*nb), n, _st())
        assert rc != 0 and msg.encode() in L().dlrm_b200_last_error(), msg
    torch.cuda.synchronize()
    assert np.all(dst.cpu().numpy() == 0xA5), "a refused block_copy wrote its destination"


# ---------------------------------------------------------------------------------------------- D. remote-read gather
REMOTE_ROWS = 1003              # not divisible by 2, 3, 5 or 8: the last shard is short
REMOTE_CASES = [(D, f16) for D in (8, 12, 16, 32, 64, 100, 128, 256, 512) for f16 in (False, True) if not f16 or D % 8 == 0]


def _remote_tables(rng, D, f16, counts, B, il, itype):
    """Tables of REMOTE_ROWS rows, table k cut into counts[k] shards of ceil(rows / n) rows, each shard in its own
    allocation with ld > dim."""
    tabs = []
    for ns in counts:
        Wv, Wh, ld = _rows_table(rng, REMOTE_ROWS, D, f16, -8, 2)
        rps = -(-REMOTE_ROWS // ns)
        shards = [_dev_table(Wh[s * rps:min((s + 1) * rps, REMOTE_ROWS)]) for s in range(ns)]
        idx, off, nnz = _bags(rng, B, REMOTE_ROWS, il)
        tabs.append(dict(W=Wv, shards=shards, rps=rps, ld=ld, idx=idx, off=off, nnz=nnz,
                         didx=_cuda(idx.astype(itype)), doff=_cuda(off.astype(itype))))
    return tabs


def _remote_desc(tabs, ldo, f16, il):
    d = (_lib.EmbRemoteTable * len(tabs))()
    for k, t in enumerate(tabs):
        for s, w in enumerate(t["shards"]):
            d[k].shard_weight[s] = w.data_ptr()
        d[k].num_shards, d[k].rows_per_shard, d[k].rows, d[k].ld = len(t["shards"]), t["rps"], REMOTE_ROWS, t["ld"]
        d[k].indices, d[k].offsets, d[k].nnz = t["didx"].data_ptr(), t["doff"].data_ptr(), 0 if il else t["nnz"]
        d[k].out_off, d[k].out_stride = k * ldo, len(tabs) * ldo
        d[k].weight_dtype = _lib.DTYPE_F16 if f16 else _lib.DTYPE_F32
    return d


@pytest.mark.parametrize("D,f16", REMOTE_CASES)
def test_remote_gather(D, f16):
    """1, 2, 3, 5 and 8 shards per table (up to 4 tables per call), int32 / int64, with and without include_last,
    bags of 0, 1, U-1, U, U+1, 2U+1 for U = 4 and 8: the output equals the sequential fp32 gather over the joined table
    bit for bit and is within the float64 bound; pad columns keep the sentinel."""
    rng = np.random.default_rng(D * 2 + f16)
    B = 150
    ldo = _ceil4(D) + 4
    for itype, il in ((np.int32, False), (np.int64, False), (np.int32, True), (np.int64, True)):
        for counts in ((1, 3, 5, 8), (2,)):
            tabs = _remote_tables(rng, D, f16, counts, B, il, itype)
            T = len(tabs)
            out = torch.full((B, T, ldo), SENT, dtype=torch.float32, device=DEV)
            out[:, :, :D] = float("nan")
            _lib.check(L().dlrm_b200_emb_bag_fwd_remote(_remote_desc(tabs, ldo, f16, il), T, D, B,
                                                        np.dtype(itype).itemsize, int(il), out.data_ptr(), _st()),
                       "emb_bag_fwd_remote")
            _no_device_errors()
            got = out.cpu().numpy()
            _all_sent(got[:, :, D:], "remote gather wrote pad columns")
            for k, t in enumerate(tabs):
                want, _ = S.gather_f32(t["W"], t["idx"], t["off"], t["nnz"], il)
                _same_bits(got[:, k, :D], want, f"{counts} table {k}: not the fp32 sequential sum")
                ref, bound = S.gather_f64(t["W"], t["idx"], t["off"], t["nnz"], il)
                _record("remote_gather", S.check_within(got[:, k, :D], ref, bound, f"table {k}"))


def test_remote_gather_bad_index_sets_the_error_word():
    """An index equal to rows and a negative one: the error word is set (and clears when read); the other bags are
    exact."""
    rng = np.random.default_rng(11)
    D, B, ldo = 64, 60, 68
    tabs = _remote_tables(rng, D, False, (3,), B, False, np.int64)
    t = tabs[0]
    bags = np.searchsorted(t["off"], np.arange(t["idx"].size), side="right") - 1
    j1, j2 = 0, t["idx"].size - 1
    t["idx"][j1], t["idx"][j2] = REMOTE_ROWS, -3
    t["didx"] = _cuda(t["idx"])
    out = torch.full((B, 1, ldo), SENT, dtype=torch.float32, device=DEV)
    _no_device_errors()
    _lib.check(L().dlrm_b200_emb_bag_fwd_remote(_remote_desc(tabs, ldo, False, False), 1, D, B, 8, 0, out.data_ptr(),
                                                _st()), "emb_bag_fwd_remote")
    assert L().dlrm_b200_check_device_errors(_st()) != 0, "a bad index was not reported"
    assert L().dlrm_b200_check_device_errors(_st()) == 0, "the error word did not clear when read"
    ok = np.setdiff1d(np.arange(B), bags[[j1, j2]])
    good = t["idx"].copy()
    good[[j1, j2]] = 0
    want, _ = S.gather_f32(t["W"], good, t["off"], t["nnz"])
    _same_bits(out.cpu().numpy()[ok, 0, :D], want[ok], "bags without a bad index")


def test_remote_gather_argument_errors_launch_nothing():
    rng = np.random.default_rng(12)
    D, B, ldo = 32, 20, 36
    tabs = _remote_tables(rng, D, False, (2, 2, 2, 2, 2), B, False, np.int64)
    out = torch.full((B, 5, ldo), SENT, dtype=torch.float32, device=DEV)
    rc = L().dlrm_b200_emb_bag_fwd_remote(_remote_desc(tabs, ldo, False, False), 5, D, B, 8, 0, out.data_ptr(), _st())
    assert rc != 0 and b"num_tables" in L().dlrm_b200_last_error()
    d = _remote_desc(tabs[:1], ldo, False, False)
    d[0].rows_per_shard = REMOTE_ROWS // 2            # 2 * 501 < 1003
    rc = L().dlrm_b200_emb_bag_fwd_remote(d, 1, D, B, 8, 0, out.data_ptr(), _st())
    assert rc != 0 and b"shards" in L().dlrm_b200_last_error()
    torch.cuda.synchronize()
    _all_sent(out.cpu().numpy(), "a refused remote gather wrote its output")


# ---------------------------------------------------------------------------------------------- E. routed interact bwd
@pytest.mark.parametrize("one_col", [False, True])
@pytest.mark.parametrize("F,D,itself", [(5, 16, 0), (27, 64, 0), (40, 32, 1)])     # MAXF 8, 32, 64
def test_interact_bwd_routed_and_scaled(F, D, itself, one_col):
    """emb_grad_scale 1, 1/2, 1/3, 1/8: every destination row of a feature >= 1 is fp32(unrouted value * scale) bit for
    bit, feature 0 is never scaled, the routed bf16 g0 pair equals interact_bwd_ex's.  Features 1..F-1 go to two
    'owner' receive buffers (one of them at an offset inside a shared allocation) and the last one also to a third;
    one_col gives that third destination an odd ld, which makes the whole call take the one-column kernel."""
    rng = np.random.default_rng(F * 7 + D + one_col)
    B, mask0 = 300, _lib.ACT_RELU
    npairs = F * (F + 1) // 2 if itself else F * (F - 1) // 2
    ldr = (D + npairs + 1) // 2 * 2                       # even: the unrouted call takes the two-column kernel
    Th = _wide(rng, (B, F * D), -3, 1)
    dRh = _wide(rng, (B, ldr), -3, 1)
    T, dR = _cuda(Th), _cuda(dRh)
    dT = torch.full((B, F * D), float("nan"), device=DEV)
    g0 = [torch.zeros((B, D), dtype=torch.int16, device=DEV) for _ in range(2)]
    _lib.check(L().dlrm_b200_interact_bwd_ex(T.data_ptr(), F * D, dR.data_ptr(), ldr, dT.data_ptr(), F * D, B, F,
                                             D, itself, mask0, g0[0].data_ptr(), g0[1].data_ptr(), D, _st()),
               "interact_bwd_ex")
    ref = dT.cpu().numpy().reshape(B, F, D)
    want, bound = DF.interact_bwd(Th.reshape(B, F, D), dRh[:, :D + npairs], itself, mask0)
    _record("interact_bwd", DF.check_within(ref, want, bound, "unrouted interact_bwd"))
    h = (F - 1) // 2
    for scale in (1.0, 0.5, 1.0 / 3.0, 0.125):
        f0 = torch.full((B + 1, D), SENT, device=DEV)
        shared = torch.full((2, B + 1, h, D), SENT, device=DEV)             # owner A's buffer is slab 1 of 2
        ownB = torch.full((B + 1, F - 1 - h, D), SENT, device=DEV)
        ld3 = D + 3 if one_col else D + 4                   # the row sits at column 2 (8-byte aligned)
        third = torch.full((B + 1, ld3), SENT, device=DEV)
        dst, ld, first = [f0.data_ptr()], [D], [0, 1]
        for i in range(1, F):
            if i - 1 < h:
                dst.append(shared[1].data_ptr() + (i - 1) * D * 4), ld.append(h * D)
            else:
                dst.append(ownB.data_ptr() + (i - 1 - h) * D * 4), ld.append((F - 1 - h) * D)
            if i == F - 1:
                dst.append(third.data_ptr() + 8), ld.append(ld3)
            first.append(len(dst))
        gr = [torch.zeros((B, D), dtype=torch.int16, device=DEV) for _ in range(2)]
        n = len(dst)
        _lib.check(L().dlrm_b200_interact_bwd_p2p(T.data_ptr(), F * D, dR.data_ptr(), ldr, _vp(dst),
                                                  (C.c_int64 * n)(*ld), (C.c_int * (F + 1))(*first), scale, B, F, D,
                                                  itself, mask0, gr[0].data_ptr(), gr[1].data_ptr(), D, _st()),
                   "interact_bwd_p2p")
        sc = np.float32(scale)
        scaled = ref[:, 1:] * sc
        got_f0, got_sh, got_B, got_3 = f0.cpu().numpy(), shared.cpu().numpy(), ownB.cpu().numpy(), third.cpu().numpy()
        _same_bits(got_f0[:B], ref[:, 0], f"scale {scale}: feature 0")
        _same_bits(got_sh[1, :B], scaled[:, :h], f"scale {scale}: owner A")
        _same_bits(got_B[:B], scaled[:, h:], f"scale {scale}: owner B")
        _same_bits(got_3[:B, 2:2 + D], scaled[:, -1], f"scale {scale}: second destination of the last feature")
        _all_sent(got_f0[B], "wrote past the batch")
        _all_sent(got_sh[0], "wrote the other slab of the shared allocation")
        _all_sent(got_sh[1, B], "wrote past the batch")
        _all_sent(got_B[B], "wrote past the batch")
        _all_sent(got_3[B], "wrote past the batch")
        _all_sent(got_3[:, :2], "wrote before the destination")
        _all_sent(got_3[:, 2 + D:], "wrote past the row")
        for a, b in zip(gr, g0):
            _same_bits(a, b, f"scale {scale}: routed bf16 g0 pair")


def test_interact_bwd_128_destinations_accepted_129_refused():
    rng = np.random.default_rng(21)
    B, F, D, itself = 64, 40, 16, 0
    npairs = F * (F - 1) // 2
    T, dR = _cuda(_wide(rng, (B, F * D))), _cuda(_wide(rng, (B, D + npairs)))
    dT = torch.full((B, F * D), float("nan"), device=DEV)
    _lib.check(L().dlrm_b200_interact_bwd(T.data_ptr(), F * D, dR.data_ptr(), D + npairs, dT.data_ptr(), F * D, B, F, D,
                                          itself, 0, _st()), "interact_bwd")
    ref = dT.cpu().numpy().reshape(B, F, D)
    for ndst in (128, 129):                               # feature F - 1 gets every destination past F - 1
        buf = torch.full((ndst, B, D), SENT, device=DEV)
        dst = [buf[q].data_ptr() for q in range(ndst)]
        first = list(range(F)) + [ndst]
        rc = L().dlrm_b200_interact_bwd_p2p(T.data_ptr(), F * D, dR.data_ptr(), D + npairs, _vp(dst),
                                            (C.c_int64 * ndst)(*[D] * ndst), (C.c_int * (F + 1))(*first), 1.0, B, F, D,
                                            itself, 0, None, None, 0, _st())
        got = buf.cpu().numpy()
        if ndst == 128:
            assert rc == 0, L().dlrm_b200_last_error()
            for i in range(F - 1):
                _same_bits(got[i], ref[:, i], f"feature {i}")
            for q in range(F - 1, ndst):
                _same_bits(got[q], ref[:, F - 1], f"destination {q}")
        else:
            assert rc != 0 and b"destinations" in L().dlrm_b200_last_error()
            _all_sent(got, "a refused interact_bwd_p2p wrote a destination")


# ---------------------------------------------------------------------------------------------- C. tiny tables
SMALL_ROWS = [3, 10, 155]
SMALL_SPLIT = (300, 100, 120)   # a row-split shard: rows [100, 220) of a 300-row table
SMALL_CASES = [(W, bl) for W in (2, 3, 4, 8) for bl in (1, 100, 128, 300)]


class Small:
    """Four tiny-table descriptors of one call (3, 10 and 155 rows and a row-split shard, capped at the rows that fit
    shared memory at this dim) over a global batch of
    W * batch_local bags, and the gradient rows in the engine's receive-buffer layout: dY [B][Tl][D], dy_off = j * D,
    dy_stride = Tl * D.  peers() gives rank r's slab [batch_local][Tl][D]: its own allocation, or (shared) slab r of
    one allocation."""

    def __init__(self, rng, W, bl, D, itype, il, f16):
        self.W, self.bl, self.D, self.itype, self.il, self.f16 = W, bl, D, itype, il, f16
        self.B = B = W * bl
        most = 200 * 1024 // (4 * D)                      # rows whose accumulator fits 200 KB of shared memory
        full = [min(R, most) for R in SMALL_ROWS] + [SMALL_SPLIT[0]]
        self.lo = [0, 0, 0, SMALL_SPLIT[1]]
        self.n = full[:3] + [min(SMALL_SPLIT[2], most)]
        self.full = full
        self.Tl = len(full)
        self.idx, self.off, self.nnz, self.didx, self.doff = [], [], [], [], []
        for R in full:
            idx, off, nnz = _bags(rng, B, R, il, lens=(0, 1, 2, 3), tail=9)
            self.idx.append(idx), self.off.append(off), self.nnz.append(nnz)
            self.didx.append(_cuda(idx.astype(itype))), self.doff.append(_cuda(off.astype(itype)))
        self.dY = _wide(rng, (B, self.Tl, D))
        self.W0, self.Wh, self.ld = [], [], 0
        for n in self.n:
            v, h, self.ld = _rows_table(rng, n, D, f16)
            self.W0.append(v), self.Wh.append(h)
        self.m_rws = [rng.uniform(0, 1e-3, n).astype(np.float32) for n in self.n]
        self.m_ada = [rng.uniform(0, 1e-3, (n, D)).astype(np.float32) for n in self.n]
        self.keys = [0x1234 + 77 * k for k in range(self.Tl)]
        self.nbytes = L().dlrm_b200_emb_bwd_small_scratch_bytes(sum(self.n), D, B)

    def peers(self, shared):
        slabs = P.split(self.dY, self.W)
        if shared:
            big = _cuda(np.stack(slabs))
            return [big], [big.data_ptr() + r * big[0].numel() * 4 for r in range(self.W)]
        keep = []
        for s in slabs:                                   # one row past batch_local in every slab
            x = np.full((self.bl + 1, self.Tl, self.D), SENT, np.float32)
            x[:self.bl] = s
            keep.append(_cuda(x))
        return keep, [k.data_ptr() for k in keep]

    def run(self, opt, lr, eps, dy_ptr=None, peers=None, zero=False, expect_error=None):
        """(tables, accumulators) after one call; zero: fp32 zero rows."""
        Wh = [np.where(np.arange(self.ld) < self.D, 0, h).astype(h.dtype) for h in self.Wh] if zero else self.Wh
        dW = [_dev_table(h) for h in Wh]
        mom = self.m_ada if opt == ADA else self.m_rws
        dm = [_cuda(m) for m in mom]
        d = (_lib.EmbBwdTable * self.Tl)()
        for k in range(self.Tl):
            d[k].weight, d[k].momentum, d[k].indices, d[k].offsets = dW[k].data_ptr(), dm[k].data_ptr(), \
                self.didx[k].data_ptr(), self.doff[k].data_ptr()
            d[k].nnz, d[k].rows, d[k].ld = 0 if self.il else self.nnz[k], self.full[k], self.ld
            d[k].use_dy_off, d[k].dy_off = 1, k * self.D
            if self.lo[k]:
                d[k].row_lo, d[k].row_n = self.lo[k], self.n[k]
            if self.f16:
                d[k].weight_dtype, d[k].round_key = _lib.DTYPE_F16, self.keys[k]
        scratch = torch.full((self.nbytes // 4,), float("nan"), device=DEV)
        pv = _vp(peers) if peers is not None else None
        rc = L().dlrm_b200_emb_bwd_small_update(d, self.Tl, self.D, self.B, np.dtype(self.itype).itemsize, int(self.il),
                                                dy_ptr, pv, self.W if peers is not None else 0,
                                                self.bl if peers is not None else 0, self.Tl * self.D, opt, lr, eps,
                                                scratch.data_ptr(), self.nbytes, _st())
        if expect_error:
            assert rc != 0 and expect_error.encode() in L().dlrm_b200_last_error(), L().dlrm_b200_last_error()
            torch.cuda.synchronize()
            for w, h in zip(dW, Wh):
                _same_bits(_host(w).view(np.uint8), h.view(np.uint8), "a refused update wrote a table")
            for x, m in zip(dm, mom):
                _same_bits(x, m, "a refused update wrote an accumulator")
            assert np.all(np.isnan(scratch.cpu().numpy())), "a refused update wrote its scratch"
            _no_device_errors()
            return None
        _lib.check(rc, "emb_bwd_small_update")
        _no_device_errors()
        return [_host(w) for w in dW], [x.cpu().numpy() for x in dm]

    def occ(self, k):
        pos, bag, r = S.occurrences(self.idx[k], self.off[k], self.nnz[k], self.il, self.lo[k], self.n[k])
        rows, grp = S.coalesce(r)
        return rows, grp, bag, self.dY[bag, k]


@pytest.mark.parametrize("W,bl", SMALL_CASES)
def test_tiny_table_update_from_peers(W, bl):
    """emb_bwd_small_update with peer_dY equals the call over the joined dY bit for bit -- SGD, RWSAdagrad and Adagrad,
    fp32 and (dim % 8 == 0) fp16 with its rounding keys; batch_local 1, 100, 128, 300, so that 128-sample chunks start
    and end inside a rank.  D rotates over 16, 128, 260, 512 (NV = 1, 2, 4), int32 / int64 and include_last with the
    case.  The gradient (SGD, lr = 1, zero rows) is the per-chunk fp32 sum; RWSAdagrad is within the float64 bound."""
    i = SMALL_CASES.index((W, bl))
    D = (16, 128, 260, 512)[(i // 4 + i) % 4]          # every batch_local meets every D across the four W
    itype = np.int64 if (i // 2) % 2 else np.int32
    il = i % 3 == 0
    rng = np.random.default_rng(500 + i)
    for f16 in (False, True) if D % 8 == 0 else (False,):
        s = Small(rng, W, bl, D, itype, il, f16)
        dY = _cuda(s.dY)
        keep, peers = s.peers(shared=(i + f16) % 2 == 1)
        for opt, lr, eps in ((SGD, 0.05, 0.0), (RWS, 0.05, 1e-10), (ADA, 0.05, 1e-8)):
            loc = s.run(opt, lr, eps, dy_ptr=dY.data_ptr())
            rem = s.run(opt, lr, eps, peers=peers)
            for k in range(s.Tl):
                _same_bits(rem[0][k].view(np.uint8), loc[0][k].view(np.uint8), f"f16={f16} opt={opt} table {k}: rows")
                _same_bits(rem[1][k], loc[1][k], f"f16={f16} opt={opt} table {k}: accumulators")
            if f16:
                continue
            if opt == RWS:
                for k in range(s.Tl):
                    rows, grp, bag, G = s.occ(k)
                    g = S.sum_f32_chunked(G, grp, rows.size, bag)
                    w2, m2 = S.row_step(s.W0[k][rows], s.m_rws[k][rows], g, RWS, lr, eps)
                    bw, bm = S.row_step_bound(w2, m2, g, RWS, lr, eps)
                    _record("small_p2p_w", S.check_within(rem[0][k][rows, :D], w2, bw, f"table {k} rows"))
                    _record("small_p2p_m", S.check_within(rem[1][k][rows], m2, bm, f"table {k} accumulators"))
            for k in range(s.Tl):
                rows, _, _, _ = s.occ(k)
                rest = np.setdiff1d(np.arange(s.n[k]), rows)
                _same_bits(rem[0][k][rest], s.Wh[k][rest], "untouched rows")
                _same_bits(rem[0][k][:, D:], s.Wh[k][:, D:], "pad columns")
                m0 = s.m_ada if opt == ADA else s.m_rws
                _same_bits(rem[1][k][rest], m0[k][rest], "accumulators of untouched rows")
        if not f16:
            gz = s.run(SGD, 1.0, 0.0, peers=peers, zero=True)[0]
            for k in range(s.Tl):
                rows, grp, bag, G = s.occ(k)
                want = S.sum_f32_chunked(G, grp, rows.size, bag)
                _same_bits(-gz[k][rows, :D], want, f"table {k}: not the chunked fp32 sum")
                _record("small_p2p_g", S.check_within(want, S.sum_exact(G, grp, rows.size),
                                                      S.sum_f32_chunked_bound(G, grp, rows.size, bag), "chunked sum"))
        del keep


@pytest.mark.parametrize("which", ["dY", "peer"])
def test_tiny_table_update_refuses_unaligned_dy(which):
    """dY, or one peer_dY[d], 4 bytes past a 16-byte boundary: the accumulate kernel reads rows with 16-byte loads, so
    the call returns an error with a message and launches nothing -- tables, accumulators, scratch and the error word
    are unchanged."""
    rng = np.random.default_rng(77)
    s = Small(rng, 3, 100, 128, np.int64, False, False)
    _no_device_errors()
    if which == "dY":
        buf = torch.full((s.B * s.Tl * s.D + 4,), SENT, device=DEV)
        buf[1:1 + s.dY.size] = _cuda(s.dY.reshape(-1))
        s.run(SGD, 0.05, 0.0, dy_ptr=buf.data_ptr() + 4, expect_error="small_update: dY must be 16-byte aligned")
    else:
        keep, peers = s.peers(shared=False)
        slab = torch.full((s.bl * s.Tl * s.D + 4,), SENT, device=DEV)
        peers[2] = slab.data_ptr() + 4
        s.run(RWS, 0.05, 1e-10, peers=peers, expect_error="peer 2 dY must be 16-byte aligned")


# ---------------------------------------------------------------------------------------------- B. peer list update
COUNTS = [1, 2, 31, 32, 33, 127, 128, 129, 1000]


class PeerUpdate:
    """The data shape of the list-update tests: three tables, table 0 with rows of exactly COUNTS occurrences (two in
    one bag) plus 300 singles, table 1 without occurrences, table 2 with short random bags; the batch padded with
    empty bags to a multiple of W.  Gradient rows in the engine's receive-buffer layout (dy_off = j * D, dy_stride =
    3 * D).  layout "tables" / "packed" (one shared index array, include_last) / "shard" (table 0 holds rows
    [500, 1500) of 2000)."""

    def __init__(self, rng, D, itype, layout, W, f16=False):
        self.D, self.itype, self.layout, self.W, self.f16 = D, itype, layout, W, f16
        self.il = layout == "packed"
        self.rows = [2000, 64, 700]
        lo, n = (500, 1000) if layout == "shard" else (0, 2000)
        self.shard = (lo, n)
        special = rng.choice(np.arange(lo, lo + n), len(COUNTS), replace=False)
        occ = np.concatenate([np.full(c, r) for c, r in zip(COUNTS, special)] + [rng.integers(0, 2000, 300)])
        occ = occ[rng.permutation(occ.size)]
        lens0 = []
        left = occ.size
        while left:
            lens0.append(min(left, int(rng.integers(1, 9))))
            left -= lens0[-1]
        i2 = np.nonzero(occ == special[1])[0]
        occ = np.delete(occ, i2[1])
        occ = np.insert(occ, i2[0], special[1])
        B = -(-len(lens0) // W) * W
        self.B, self.bl = B, B // W
        lens0 = np.append(lens0, np.zeros(B - len(lens0), np.int64))
        lens2 = rng.integers(0, 4, B)
        idx = [occ.astype(np.int64), np.zeros(0, np.int64), rng.integers(0, 700, int(lens2.sum()))]
        offs = [_offsets(lens0), np.zeros(B, np.int64), _offsets(lens2)]
        self.idx, self.off = idx, offs
        self.dY = _wide(rng, (B, 3, D))
        self.W0, self.Wh, self.ld = [], [], 0
        for R in self.rows:
            v, h, self.ld = _rows_table(rng, R, D, f16)
            self.W0.append(v), self.Wh.append(h)
        self.m_rws = [rng.uniform(0, 1e-3, R).astype(np.float32) for R in self.rows]
        self.m_ada = [rng.uniform(0, 1e-3, (R, D)).astype(np.float32) for R in self.rows]
        self.nnz = [i.size for i in idx]
        self.base = np.concatenate([[0], np.cumsum(self.nnz)[:-1]]).astype(np.int64)
        self.cap = int(sum(self.nnz)) + (37 if self.il else 0)
        if self.il:
            shared = np.concatenate(idx + [np.full(37, 10 ** 6, np.int64)])
            self.didx = [_cuda(shared.astype(itype))] * 3
            self.doff = [_cuda(np.append(o + b, b + i.size).astype(itype)) for o, b, i in zip(offs, self.base, idx)]
        else:
            self.didx = [_cuda(i.astype(itype)) for i in idx]
            self.doff = [_cuda(o.astype(itype)) for o in offs]

    def peers(self, shared, misalign=None):
        """Slab r of the receive buffers: own allocations with a row past batch_local, or one shared allocation.
        misalign = r: slab r starts 4 bytes past a 16-byte boundary."""
        slabs = P.split(self.dY, self.W)
        keep, ptrs = [], []
        if shared:
            big = _cuda(np.stack(slabs))
            keep, ptrs = [big], [big.data_ptr() + r * big[0].numel() * 4 for r in range(self.W)]
        else:
            for s in slabs:
                x = np.full((self.bl + 1, 3, self.D), SENT, np.float32)
                x[:self.bl] = s
                keep.append(_cuda(x))
                ptrs.append(keep[-1].data_ptr())
        if misalign is not None:
            x = torch.full((self.bl * 3 * self.D + 4,), SENT, device=DEV)
            x[1:1 + self.bl * 3 * self.D] = _cuda(slabs[misalign].reshape(-1))
            keep.append(x)
            ptrs[misalign] = x.data_ptr() + 4
        return keep, ptrs

    def run(self, opt, lr, eps, dy_ptr=None, peers=None, zero=False, expect_error=None):
        lo, n = self.shard
        Wh = [np.where(np.arange(self.ld) < self.D, 0, h).astype(h.dtype) for h in self.Wh] if zero else self.Wh
        dW = [_dev_table(h) for h in Wh]
        mom = self.m_ada if opt == ADA else self.m_rws
        dm = [_cuda(m) for m in mom]
        head = [torch.zeros(R, dtype=torch.int32, device=DEV) for R in self.rows]
        mark = torch.zeros(self.cap, dtype=torch.uint8, device=DEV)
        link = torch.zeros(2 * self.cap, dtype=torch.int32, device=DEV)
        esz = 2 if self.f16 else 4
        d = (_lib.EmbBwdTable * 3)()
        for k in range(3):
            d[k].weight, d[k].momentum, d[k].head = dW[k].data_ptr(), dm[k].data_ptr(), head[k].data_ptr()
            d[k].indices = self.didx[k].data_ptr() if (self.il or self.nnz[k]) else None
            d[k].offsets, d[k].rows, d[k].ld, d[k].mark = self.doff[k].data_ptr(), self.rows[k], self.ld, mark.data_ptr()
            d[k].nnz = self.cap if self.il else self.nnz[k]
            d[k].pair_base = 0 if self.il else int(self.base[k])
            d[k].use_dy_off, d[k].dy_off = 1, k * self.D
            if self.f16:
                d[k].weight_dtype, d[k].round_key = _lib.DTYPE_F16, 0xABCDEF + k
        if self.layout == "shard":
            d[0].weight += lo * self.ld * esz
            d[0].momentum += lo * 4 * (self.D if opt == ADA else 1)
            d[0].head += lo * 4
            d[0].row_lo, d[0].row_n = lo, n
        ib, il = np.dtype(self.itype).itemsize, int(self.il)
        _lib.check(L().dlrm_b200_emb_bwd_link(d, 3, self.B, ib, il, link.data_ptr(), _st()), "link")
        if peers is None:
            rc = L().dlrm_b200_emb_bwd_update(d, 3, self.D, self.B, ib, il, link.data_ptr(), dy_ptr, 3 * self.D, 0, opt,
                                              lr, eps, None, _st())
        else:
            rc = L().dlrm_b200_emb_bwd_update_p2p(d, 3, self.D, self.B, ib, il, link.data_ptr(), _vp(peers), self.W,
                                                  self.bl, 3 * self.D, 0, opt, lr, eps, None, _st())
        if expect_error:
            assert rc != 0 and expect_error.encode() in L().dlrm_b200_last_error(), L().dlrm_b200_last_error()
            torch.cuda.synchronize()
            for w, h in zip(dW, Wh):
                _same_bits(_host(w).view(np.uint8), h.view(np.uint8), "a refused update wrote a table")
            return None
        _lib.check(rc, "emb_bwd_update")
        assert all(int(h.abs().sum().item()) == 0 for h in head), "list heads not cleared"
        assert int(mark.sum().item()) == 0, "marks not cleared"
        _no_device_errors()
        return [_host(w) for w in dW], [x.cpu().numpy() for x in dm]

    def local_rows(self, k):
        """(first row, rows) the descriptor of table k covers."""
        return self.shard if k == 0 else (0, self.rows[k])

    def occ(self, k):
        pos, bag, r = S.occurrences(self.idx[k], self.off[k], self.nnz[k], False, *self.local_rows(k))
        rows, grp = S.coalesce(r)
        return rows, grp, self.dY[bag, k]


# lean: 16, 128; general vec NV = 2, 4 (260: masked), 4, 8; scalar: 6, 33, 1023
UPD_P2P_CASES = [(16, "tables", 2), (128, "packed", 3), (256, "shard", 4), (260, "tables", 8), (512, "packed", 2),
                 (1024, "shard", 3), (6, "tables", 4), (33, "packed", 8), (1023, "shard", 2), (16, "shard", 8),
                 (128, "tables", 4), (260, "packed", 3)]


@pytest.mark.parametrize("D,layout,W", UPD_P2P_CASES)
def test_update_from_peers(D, layout, W):
    """emb_bwd_update_p2p over W receive-buffer slabs equals emb_bwd_update over the joined dY bit for bit (rows and
    accumulators) for SGD, RWSAdagrad and element-wise Adagrad, fp32 and (dim % 8 == 0) fp16; lists of <= 32 and > 32
    members span rank boundaries.  The gradient each row got (SGD, lr = 1, zero rows) is the ascending-position fp32
    sum (<= 32 members) or within one ulp of the exact sum (> 32)."""
    i = UPD_P2P_CASES.index((D, layout, W))
    itype = np.int64 if i % 2 else np.int32
    rng = np.random.default_rng(900 + i)
    for f16 in (False, True) if D % 8 == 0 else (False,):
        u = PeerUpdate(rng, D, itype, layout, W, f16)
        dY = _cuda(u.dY)
        keep, peers = u.peers(shared=i % 2 == 1)
        for opt, lr, eps in ((SGD, 0.05, 0.0), (RWS, 0.05, 1e-4 if D % 2 else 1e-10), (ADA, 0.05, 1e-8)):
            loc = u.run(opt, lr, eps, dy_ptr=dY.data_ptr())
            rem = u.run(opt, lr, eps, peers=peers)
            for k in range(3):
                _same_bits(rem[0][k].view(np.uint8), loc[0][k].view(np.uint8), f"f16={f16} opt={opt} table {k}: rows")
                _same_bits(rem[1][k], loc[1][k], f"f16={f16} opt={opt} table {k}: accumulators")
                lo, n = u.local_rows(k)
                rows, _, _ = u.occ(k)
                rest = np.setdiff1d(np.arange(n), rows) + lo
                _same_bits(rem[0][k][rest].view(np.uint8), u.Wh[k][rest].view(np.uint8), "untouched rows")
                m0 = u.m_ada if opt == ADA else u.m_rws
                _same_bits(rem[1][k][rest], m0[k][rest], "accumulators of untouched rows")
        if f16:
            continue
        gz = u.run(SGD, 1.0, 0.0, peers=peers, zero=True)[0]
        for k in range(3):
            lo, n = u.local_rows(k)
            rows, grp, G = u.occ(k)
            gk = -gz[k][rows + lo, :D]
            cnt = np.bincount(grp, minlength=rows.size)
            short = cnt <= S.LIST_SORTED_MAX
            asc = S.sum_f32_ascending(G, grp, rows.size)
            assert np.array_equal(gk[short], asc[short]), f"table {k}: not the ascending-position fp32 sum"
            for j in np.nonzero(~short)[0]:
                ulps = S.long_sum_ulps(gk[j], G[grp == j])
                assert ulps.max() <= 1, f"table {k} row {rows[j]} ({cnt[j]} occurrences): {ulps.max()} ulps"
                _record("update_p2p_long_list_ulps", ulps.max())
        del keep


def test_update_from_a_misaligned_peer_slab():
    """One slab 4 bytes off a 16-byte boundary: fp32 takes the scalar kernel and equals the local call whose dY is
    offset the same way; fp16 (no scalar kernel) is an error without a launch."""
    rng = np.random.default_rng(31)
    u = PeerUpdate(rng, 128, np.int64, "tables", 3)
    keep, peers = u.peers(shared=False, misalign=1)
    buf = torch.full((u.dY.size + 4,), SENT, device=DEV)
    buf[1:1 + u.dY.size] = _cuda(u.dY.reshape(-1))
    for opt in (SGD, RWS):
        loc = u.run(opt, 0.05, 1e-10, dy_ptr=buf.data_ptr() + 4)
        rem = u.run(opt, 0.05, 1e-10, peers=peers)
        for k in range(3):
            _same_bits(rem[0][k], loc[0][k], f"opt={opt} table {k}: rows")
            _same_bits(rem[1][k], loc[1][k], f"opt={opt} table {k}: accumulators")
    f = PeerUpdate(np.random.default_rng(32), 128, np.int64, "tables", 3, f16=True)
    keep16, peers16 = f.peers(shared=False, misalign=2)
    f.run(SGD, 0.05, 0.0, peers=peers16, expect_error="16-byte aligned gradient rows")
    del keep, keep16


# ---------------------------------------------------------------------------------------------- A. routed training gather
# W, batch_local, D, fp16, index type, weighted, include_last, row-split shard
GATHER_P2P_CASES = [
    (3, 1, 16, False, np.int32, False, False, False),
    (3, 37, 64, True, np.int64, True, True, True),
    (4, 37, 128, False, np.int64, False, True, True),
    (4, 1, 256, True, np.int32, False, False, True),
    (8, 37, 512, False, np.int32, True, False, False),
    (8, 1, 6, False, np.int64, False, True, True),
    (8, 37, 16, True, np.int64, True, False, True),
    (3, 37, 6, False, np.int32, True, True, False),
    (4, 37, 512, True, np.int64, False, True, True),
    (3, 37, 256, False, np.int64, True, False, True),
    (4, 1, 64, False, np.int32, True, True, False),
    (8, 37, 128, True, np.int32, False, False, False),
]


class RoutedGather:
    """Three local shards of a rank: whole table 0 (500 rows), table 1 (2000 rows; with `split`, part 1 of 3 = rows
    [700, 1400)), whole table 2 (50 rows).  Pooled rows are routed as sharding.out_routes lays out TP = T [cap, F, D]
    followed by the partial-sum area [slab][cap][D].  include_last uses the packed layout of a training batch: one
    index array with global offsets and a capacity tail, every table's list pairs indexed by position."""

    def __init__(self, rng, W, bl, D, f16, itype, weighted, il, split):
        self.W, self.bl, self.D, self.f16, self.itype, self.il, self.split = W, bl, D, f16, itype, il, split
        self.B = B = W * bl
        self.full = [500, 2000, 50]
        self.lo = [0, 700 if split else 0, 0]
        self.n = [500, 700 if split else 2000, 50]
        self.F = 4
        self.shards = [dict(table=0, nparts=1, part=0), dict(table=1, nparts=3 if split else 1, part=1 if split else 0),
                       dict(table=2, nparts=1, part=0)]
        self.slots = [(1, 3)] if split else []
        self.nslab = 3 if split else 0
        self.idx, self.off, self.nnz = [], [], []          # per table, positions local to the table
        for R in self.full:
            i, o, z = _bags(rng, B, R, False)
            self.idx.append(i), self.off.append(o), self.nnz.append(z)
        self.base = np.concatenate([[0], np.cumsum(self.nnz)[:-1]]).astype(np.int64)
        self.cap = int(sum(self.nnz)) + (37 if il else 0)
        if il:        # the packed layout: one index array, global offsets [B + 1] per table, a capacity tail
            shared = np.concatenate(self.idx + [np.full(37, 10 ** 6, np.int64)])
            self.didx = [_cuda(shared.astype(itype))] * 3
            self.doff = [_cuda(np.append(o + b, b + i.size).astype(itype))
                         for o, b, i in zip(self.off, self.base, self.idx)]
        else:
            self.didx = [_cuda(i.astype(itype)) for i in self.idx]
            self.doff = [_cuda(o.astype(itype)) for o in self.off]
        self.W0, self.Wh, self.ld = [], [], 0
        for n in self.n:
            v, h, self.ld = _rows_table(rng, n, D, f16)
            self.W0.append(v), self.Wh.append(h)
        self.rw = [rng.uniform(-2, 2, n).astype(np.float32) if weighted else None for n in self.n]
        self.drw = [_cuda(r) if r is not None else None for r in self.rw]
        self.m0 = [rng.uniform(0, 1e-3, n).astype(np.float32) for n in self.n]
        self.dY = _wide(rng, (B, 3, D))

    def tp(self, cap, nrows):
        """(TP buffer for `cap` samples with the sentinel everywhere and NaN where the pooled rows of samples
        [0, nrows) go, their positions [3][nrows][D], the routes)."""
        routes, _ = SH.out_routes(self.shards, self.slots, cap, self.F, self.D)
        routes = [(int(o), int(s)) for o, s in routes]
        pos = np.stack([o + np.arange(nrows)[:, None] * s + np.arange(self.D)[None, :] for o, s in routes])
        buf = np.full(cap * self.F * self.D + self.nslab * cap * self.D, SENT, np.float32)
        buf[pos.reshape(-1)] = np.nan
        return buf, pos, routes

    def state(self):
        return dict(W=[_dev_table(h) for h in self.Wh], m=[_cuda(m) for m in self.m0],
                    head=[torch.zeros(n, dtype=torch.int32, device=DEV) for n in self.n],
                    mark=torch.zeros(self.cap, dtype=torch.uint8, device=DEV),
                    link=torch.zeros(2 * self.cap, dtype=torch.int32, device=DEV))

    def desc(self, st, routes):
        f = (_lib.EmbFwdTable * 3)()
        b = (_lib.EmbBwdTable * 3)()
        for k in range(3):
            f[k].weight, f[k].indices, f[k].offsets = st["W"][k].data_ptr(), self.didx[k].data_ptr(), self.doff[k].data_ptr()
            f[k].row_weights = self.drw[k].data_ptr() if self.drw[k] is not None else None
            f[k].nnz, f[k].rows, f[k].ld = 0 if self.il else self.nnz[k], self.full[k], self.ld
            f[k].out_off, f[k].out_stride = routes[k]
            b[k].weight, b[k].momentum, b[k].head = st["W"][k].data_ptr(), st["m"][k].data_ptr(), st["head"][k].data_ptr()
            b[k].indices, b[k].offsets = self.didx[k].data_ptr(), self.doff[k].data_ptr()
            b[k].nnz, b[k].pair_base = (self.cap, 0) if self.il else (self.nnz[k], int(self.base[k]))
            b[k].rows, b[k].ld, b[k].mark = self.full[k], self.ld, st["mark"].data_ptr()
            b[k].use_dy_off, b[k].dy_off = 1, k * self.D
            if self.lo[k] or self.n[k] != self.full[k]:
                f[k].row_lo, f[k].row_n = self.lo[k], self.n[k]
                b[k].row_lo, b[k].row_n = self.lo[k], self.n[k]
            if self.f16:
                f[k].weight_dtype = b[k].weight_dtype = _lib.DTYPE_F16
                b[k].round_key = 0x5EED + k
        return f, b

    def dedup(self):
        filt = torch.zeros((1 << 12) + 1, dtype=torch.int32, device=DEV)
        flags = torch.zeros(self.cap, dtype=torch.uint8, device=DEV)
        susp = torch.zeros(self.cap, dtype=torch.int32, device=DEV)
        return (filt, flags, susp), _lib.EmbDedup(filt.data_ptr(), 12, flags.data_ptr(), susp.data_ptr())

    def step(self, peer, dedup=False):
        """Training gather (local over the whole batch, or routed to W peer TPs) + the list update from the global
        dY: (pooled rows [B, 3, D] in global bag order, TP buffers, positions, bag halves of next[], tables, acc.)"""
        st = self.state()
        ib, il = np.dtype(self.itype).itemsize, int(self.il)
        keep, dd = self.dedup() if dedup else (None, None)
        if peer:
            buf0, pos, routes = self.tp(self.bl + 1, self.bl)
            bufs = [_cuda(buf0) for _ in range(self.W)]
            f, b = self.desc(st, routes)
            _lib.check(L().dlrm_b200_emb_bag_fwd_p2p(f, b, 3, self.D, self.B, ib, il, st["link"].data_ptr(),
                                                     _vp([x.data_ptr() for x in bufs]), self.W, self.bl,
                                                     self.F * self.D, self.D, C.byref(dd) if dd else None, _st()),
                       "emb_bag_fwd_p2p")
        else:
            buf0, pos, routes = self.tp(self.B, self.B)
            bufs = [_cuda(buf0)]
            f, b = self.desc(st, routes)
            _lib.check(L().dlrm_b200_emb_bag_fwd_train(f, b, 3, self.D, self.B, ib, il, st["link"].data_ptr(),
                                                       bufs[0].data_ptr(), self.F * self.D, self.D,
                                                       C.byref(dd) if dd else None, _st()), "emb_bag_fwd_train")
        if dd:
            _lib.check(L().dlrm_b200_emb_bwd_classify(b, 3, self.B, ib, il, st["link"].data_ptr(), C.byref(dd), _st()),
                       "classify")
        got = [x.cpu().numpy() for x in bufs]
        bags = st["link"].view(-1, 2)[:, 1].cpu().numpy()
        dY = _cuda(self.dY)
        _lib.check(L().dlrm_b200_emb_bwd_update(b, 3, self.D, self.B, ib, il, st["link"].data_ptr(), dY.data_ptr(),
                                                3 * self.D, 0, RWS, 0.05, 1e-10, C.byref(dd) if dd else None, _st()),
                   "emb_bwd_update")
        assert all(int(h.abs().sum().item()) == 0 for h in st["head"]), "list heads not cleared"
        assert int(st["mark"].sum().item()) == 0, "marks not cleared"
        _no_device_errors()
        pooled = np.concatenate([g[pos].transpose(1, 0, 2) for g in got])       # [B, 3, D] in global bag order
        return pooled, got, pos, bags, [_host(w) for w in st["W"]], [m.cpu().numpy() for m in st["m"]]


@pytest.mark.parametrize("case", range(len(GATHER_P2P_CASES)))
def test_routed_training_gather(case):
    """emb_bag_fwd_p2p with train descriptors: peer buffer r holds rows [r bl, (r + 1) bl) of the local training
    gather bit for bit, in feature slot 1 + t (whole tables) or the shard's slab of the partial-sum area; the row
    past batch_local and every other slot keep the sentinel; the bag half of every next[] pair equals the local
    call's, and the following update gives the same tables and accumulators."""
    W, bl, D, f16, itype, weighted, il, split = GATHER_P2P_CASES[case]
    g = RoutedGather(np.random.default_rng(1300 + case), W, bl, D, f16, itype, weighted, il, split)
    ref = g.step(peer=False)
    rem = g.step(peer=True)
    _same_bits(rem[0], ref[0], "routed pooled rows differ from the local training gather")
    written = np.zeros(rem[1][0].size, bool)
    written[rem[2].reshape(-1)] = True
    for r, buf in enumerate(rem[1]):
        _all_sent(buf[~written], f"rank {r}: wrote outside its routed rows")
    assert np.array_equal(rem[3], ref[3]), "bag halves of next[] differ"
    for k in range(3):
        _same_bits(rem[4][k].view(np.uint8), ref[4][k].view(np.uint8), f"table {k} after the update")
        _same_bits(rem[5][k], ref[5][k], f"accumulators {k} after the update")
    for k in range(3):
        kw = dict(rw=g.rw[k], row_lo=g.lo[k], row_n=g.n[k])
        want, flag = S.gather_f32(g.W0[k], g.idx[k], g.off[k], g.nnz[k], **kw)      # the per-table view of the batch
        assert np.array_equal(ref[0][:, k][~flag], want[~flag]), f"table {k}: not the fp32 sequential sum"
        r64, bound = S.gather_f64(g.W0[k], g.idx[k], g.off[k], g.nnz[k], **kw)
        _record("gather_p2p_train", S.check_within(ref[0][:, k], r64, bound, f"table {k}"))


def test_routed_training_gather_with_the_duplicate_filter():
    """The same with the duplicate filter (training gather + emb_bwd_classify): pooled rows, next[] bag halves and the
    updated tables equal the local call's."""
    g = RoutedGather(np.random.default_rng(1400), 4, 37, 256, False, np.int64, False, False, True)
    ref = g.step(peer=False, dedup=True)
    rem = g.step(peer=True, dedup=True)
    _same_bits(rem[0], ref[0], "routed pooled rows")
    assert np.array_equal(rem[3], ref[3]), "bag halves of next[] differ"
    for k in range(3):
        _same_bits(rem[4][k], ref[4][k], f"table {k} after the update")
        _same_bits(rem[5][k], ref[5][k], f"accumulators {k} after the update")


# ---------------------------------------------------------------------------------------------- I. one sharded step
STEP_ROWS = [3000, 777, 10, 1501, 155, 3, 900, 420]      # tables 1 and 3 row-split; 2, 4 and 5 tiny
STEP_SPLIT = [1, 3]
STEP_SMALL_MAX = 256            # the engine's default small_rows_max: whole tables up to this many rows are tiny
GUARD = 64                      # sentinel floats after every buffer


def _shard_dicts(shards):
    return [dict(table=s.table, rows=s.rows, row_lo=s.row_lo, row_n=s.local_rows, part=s.part, nparts=s.nparts)
            for s in shards]


class StepRank:
    """The embedding state of one (virtual) rank: its shards' rows (ld = D + 4, sentinel pad) and row-wise
    accumulators, list heads for the shards that are linked (tiny whole tables are not), one mark / next[] array."""

    def __init__(self, shards, Wt, m0, nnz, D):
        self.shards, self.D, self.ld = shards, D, D + 4
        self.W, self.m, self.head, self.pb = [], [], [], []
        base = 0
        for sh in shards:
            t, lo, n = sh["table"], sh["row_lo"], sh["row_n"]
            w = np.full((n, self.ld), SENT, np.float32)
            w[:, :D] = Wt[t][lo:lo + n]
            self.W.append(_cuda(w))
            self.m.append(_cuda(m0[t][lo:lo + n]))
            self.head.append(None if self.small(sh) else torch.zeros(n, dtype=torch.int32, device=DEV))
            self.pb.append(base)
            base += 0 if self.small(sh) else nnz[t]
        self.cap = max(base, 1)
        self.mark = torch.zeros(self.cap, dtype=torch.uint8, device=DEV)
        self.link = torch.zeros(2 * self.cap, dtype=torch.int32, device=DEV)

    @staticmethod
    def small(sh):
        return sh["nparts"] == 1 and sh["rows"] <= STEP_SMALL_MAX

    def desc(self, ks, didx, doff, nnz, routes=None, dy_off=None):
        f, b = (_lib.EmbFwdTable * len(ks))(), (_lib.EmbBwdTable * len(ks))()
        for j, k in enumerate(ks):
            sh = self.shards[k]
            t = sh["table"]
            for d in (f[j], b[j]):
                d.weight, d.indices, d.offsets = self.W[k].data_ptr(), didx[t].data_ptr(), doff[t].data_ptr()
                d.nnz, d.rows, d.ld = nnz[t], sh["rows"], self.ld
                if sh["nparts"] > 1:
                    d.row_lo, d.row_n = sh["row_lo"], sh["row_n"]
            if routes is not None:
                f[j].out_off, f[j].out_stride = routes[k]
            b[j].momentum, b[j].pair_base, b[j].mark = self.m[k].data_ptr(), self.pb[k], self.mark.data_ptr()
            b[j].head = self.head[k].data_ptr() if self.head[k] is not None else None
            b[j].use_dy_off, b[j].dy_off = 1, dy_off[k] if dy_off is not None else 0
        return f, b

    def update(self, didx, doff, nnz, batch, dy_ptr, peers, world, batch_local, dy_off, dy_stride, lr, eps):
        """The list update of the linked shards and the tiny-table update of the others, as the engine runs them."""
        big = [k for k, sh in enumerate(self.shards) if not self.small(sh)]
        small = [k for k, sh in enumerate(self.shards) if self.small(sh)]
        if big:
            _, b = self.desc(big, didx, doff, nnz, dy_off=dy_off)
            if peers is None:
                _lib.check(L().dlrm_b200_emb_bwd_update(b, len(big), self.D, batch, 8, 0, self.link.data_ptr(), dy_ptr,
                                                        dy_stride, 0, RWS, lr, eps, None, _st()), "emb_bwd_update")
            else:
                _lib.check(L().dlrm_b200_emb_bwd_update_p2p(b, len(big), self.D, batch, 8, 0, self.link.data_ptr(),
                                                            _vp(peers), world, batch_local, dy_stride, 0, RWS, lr, eps,
                                                            None, _st()), "emb_bwd_update_p2p")
        if small:
            _, b = self.desc(small, didx, doff, nnz, dy_off=dy_off)
            nb = L().dlrm_b200_emb_bwd_small_scratch_bytes(sum(self.shards[k]["row_n"] for k in small), self.D, batch)
            scratch = torch.full((nb // 4,), float("nan"), device=DEV)
            _lib.check(L().dlrm_b200_emb_bwd_small_update(b, len(small), self.D, batch, 8, 0, dy_ptr,
                                                          _vp(peers) if peers is not None else None,
                                                          world if peers is not None else 0,
                                                          batch_local if peers is not None else 0, dy_stride, RWS, lr,
                                                          eps, scratch.data_ptr(), nb, _st()), "emb_bwd_small_update")
        assert all(h is None or int(h.abs().sum().item()) == 0 for h in self.head), "list heads not cleared"
        assert int(self.mark.sum().item()) == 0, "marks not cleared"
        _no_device_errors()


@pytest.mark.parametrize("W", [2, 4, 8])
def test_sharded_step_exchange(W):
    """One sharded step's exchange at world W, every virtual rank's buffers laid out by the product's own routes
    (placement.plan with two row-split tables, whole and tiny tables; sharding.engine_kwargs / out_routes /
    grad_routes):
      1. per rank, emb_bag_fwd_p2p (training) into every rank's TP, then emb_reduce_partials;
      2. per rank, interact_bwd_p2p (scale 1) into the owners' receive buffers;
      3. per rank, emb_bwd_update_p2p and emb_bwd_small_update from the slabs of its own receive buffer.
    Compared bit for bit with the same kernels on one rank over the global batch: the T rows and partial slabs of
    every rank (a split table = the slab-order sum of the per-shard sequential sums), every receive slab against the
    unrouted interaction backward, every shard's rows and accumulators against the whole-table update."""
    rng = np.random.default_rng(2000 + W)
    D, bl, T = 64, 100, len(STEP_ROWS)
    F, Bg = T + 1, W * bl
    npairs = F * (F - 1) // 2
    ldr = (D + npairs + 1) // 2 * 2
    lr, eps = 0.05, 1e-10
    pl = PL.plan(STEP_ROWS, [1.0] * T, W, force_split=STEP_SPLIT, split_above=float("inf"), max_extra_splits=0)
    assert pl.split_tables() == STEP_SPLIT
    slots = SH.split_slots(pl)
    nslab = sum(n for _, n in slots)
    Wt = [_wide(rng, (R, D), -4, 0) for R in STEP_ROWS]
    m0 = [rng.uniform(0, 1e-3, R).astype(np.float32) for R in STEP_ROWS]
    idx, off, nnz = [], [], []
    for R in STEP_ROWS:
        i, o, z = _bags(rng, Bg, R, False, lens=(0, 1, 2, 3, 5))
        idx.append(i), off.append(o), nnz.append(z)
    didx, doff = [_cuda(i) for i in idx], [_cuda(o) for o in off]

    def tp(cap):
        return torch.full((cap * F * D + nslab * cap * D + GUARD,), SENT, device=DEV)

    def reduce(buf, cap):
        n = len(slots)
        first = np.concatenate([[0], np.cumsum([c for _, c in slots])])
        _lib.check(L().dlrm_b200_emb_reduce_partials(buf.data_ptr() + cap * F * D * 4, buf.data_ptr(), F * D, cap, D,
                                                     (C.c_int * n)(*[1 + t for t, _ in slots]),
                                                     (C.c_int * (n + 1))(*[int(v) for v in first]), n, _st()),
                   "emb_reduce_partials")

    def views(buf, cap):
        x = buf.cpu().numpy()
        return (x[:cap * F * D].reshape(cap, F, D), x[cap * F * D:cap * F * D + nslab * cap * D].reshape(nslab, cap, D),
                x[-GUARD:])

    # ---- 1. forward: one rank over the global batch, then W ranks pushing into each other's TP
    all_sh = _shard_dicts(sorted(pl.shards, key=lambda s: (s.table, s.part)))
    ref = StepRank(all_sh, Wt, m0, nnz, D)
    routes, _ = SH.out_routes(all_sh, slots, Bg, F, D)
    f, _ = ref.desc(range(len(all_sh)), didx, doff, nnz, routes=routes)
    TPref = tp(Bg)
    _lib.check(L().dlrm_b200_emb_bag_fwd(f, len(all_sh), D, Bg, 8, 0, TPref.data_ptr(), F * D, D, _st()), "emb_bag_fwd")
    reduce(TPref, Bg)
    Tref, Pref, gref = views(TPref, Bg)
    _all_sent(gref, "reference TP guard")
    ranks, TPs = [], [tp(bl) for _ in range(W)]
    for r in range(W):
        kw = SH.engine_kwargs(pl, r, T)
        assert kw["n_features"] == F and kw["split_slots"] == slots
        assert kw["ln_emb"] == [s["row_n"] for s in kw["shards"]]
        st = StepRank(kw["shards"], Wt, m0, nnz, D)
        ranks.append(st)
        routes_r, _ = SH.out_routes(kw["shards"], kw["split_slots"], bl, F, D)
        f, b = st.desc(range(len(st.shards)), didx, doff, nnz, routes=routes_r)
        _lib.check(L().dlrm_b200_emb_bag_fwd_p2p(f, b, len(st.shards), D, Bg, 8, 0, st.link.data_ptr(),
                                                 _vp([x.data_ptr() for x in TPs]), W, bl, F * D, D, None, _st()),
                   "emb_bag_fwd_p2p")
    for r in range(W):
        reduce(TPs[r], bl)
    _no_device_errors()
    for r in range(W):
        Tr, Pr, gr = views(TPs[r], bl)
        rows = slice(r * bl, (r + 1) * bl)
        _same_bits(Tr[:, 1:], Tref[rows, 1:], f"rank {r}: T differs from the one-rank forward")
        _same_bits(Pr, Pref[:, rows], f"rank {r}: partial slabs differ from the one-rank forward")
        _all_sent(Tr[:, 0], f"rank {r}: wrote feature 0")
        _all_sent(gr, f"rank {r}: wrote past its TP")
    for t in range(T):
        if t in STEP_SPLIT:
            acc = np.zeros((Bg, D), np.float32)
            for s in pl.of_table(t):
                acc = acc + S.gather_f32(Wt[t][s.row_lo:s.row_hi], idx[t], off[t], nnz[t], row_lo=s.row_lo,
                                         row_n=s.local_rows)[0]
            _same_bits(Tref[:, 1 + t], acc, f"table {t}: not the slab-order sum of the shard sums")
        else:
            _same_bits(Tref[:, 1 + t], S.gather_f32(Wt[t], idx[t], off[t], nnz[t])[0], f"table {t}: not the fp32 sum")
            g64, bound = S.gather_f64(Wt[t], idx[t], off[t], nnz[t])
            _record("sharded_step_gather", S.check_within(Tref[:, 1 + t], g64, bound, f"table {t}"))

    # ---- 2. interaction backward: feature 0 stays local, feature 1 + t goes to every rank storing rows of t
    xs = [_wide(rng, (bl, D), -3, 1) for _ in range(W)]
    dRs = [_wide(rng, (bl, ldr), -3, 1) for _ in range(W)]
    for r in range(W):
        TPs[r][:bl * F * D].view(bl, F, D)[:, 0] = _cuda(xs[r])
    Tg = torch.cat([x[:bl * F * D].view(bl, F * D) for x in TPs])
    dRg = _cuda(np.concatenate(dRs))
    dTg = torch.full((Bg, F * D), float("nan"), device=DEV)
    _lib.check(L().dlrm_b200_interact_bwd(Tg.data_ptr(), F * D, dRg.data_ptr(), ldr, dTg.data_ptr(), F * D, Bg, F, D, 0,
                                          _lib.ACT_RELU, _st()), "interact_bwd")
    dT_ref = dTg.cpu().numpy().reshape(Bg, F, D)
    want, bound = DF.interact_bwd(Tg.cpu().numpy().reshape(Bg, F, D), dRg.cpu().numpy()[:, :D + npairs], 0,
                                  _lib.ACT_RELU)
    _record("sharded_step_interact_bwd", DF.check_within(dT_ref, want, bound, "unrouted interact_bwd"))
    Tl = [len(st.shards) for st in ranks]
    recv = []
    for r in range(W):
        x = torch.full((W * bl * Tl[r] * D + GUARD,), SENT, device=DEV)
        x[:W * bl * Tl[r] * D] = float("nan")
        recv.append(x)
    dT0 = [torch.full((bl, F * D), SENT, device=DEV) for _ in range(W)]
    for r in range(W):
        gr_, first = SH.grad_routes(pl, r, bl, D, F)
        dst = [dT0[r].data_ptr() if rk < 0 else recv[rk].data_ptr() + o * 4 for rk, o, _ in gr_]
        n = len(dst)
        _lib.check(L().dlrm_b200_interact_bwd_p2p(TPs[r].data_ptr(), F * D, _cuda(dRs[r]).data_ptr(), ldr, _vp(dst),
                                                  (C.c_int64 * n)(*[s for _, _, s in gr_]), (C.c_int * (F + 1))(*first),
                                                  1.0, bl, F, D, 0, _lib.ACT_RELU, None, None, 0, _st()),
                   "interact_bwd_p2p")
    for r in range(W):
        g0 = dT0[r].cpu().numpy()
        _same_bits(g0[:, :D], dT_ref[r * bl:(r + 1) * bl, 0], f"rank {r}: feature 0")
        _all_sent(g0[:, D:], f"rank {r}: wrote the embedding columns of its own dT")
        x = recv[r].cpu().numpy()
        R_ = x[:W * bl * Tl[r] * D].reshape(W, bl, Tl[r], D)
        for j, sh in enumerate(ranks[r].shards):
            _same_bits(R_[:, :, j].reshape(Bg, D), dT_ref[:, 1 + sh["table"]],
                       f"rank {r} shard {j} (table {sh['table']}): receive slabs")
        _all_sent(x[-GUARD:], f"rank {r}: wrote past its receive buffer")

    # ---- 3. update: W ranks from their receive slabs against whole tables updated on one rank from dT
    whole = _shard_dicts(PL.plan(STEP_ROWS, [1.0] * T, 1).of_rank(0))
    one = StepRank(whole, Wt, m0, nnz, D)
    big = [k for k, sh in enumerate(whole) if not one.small(sh)]
    _, b = one.desc(big, didx, doff, nnz)
    _lib.check(L().dlrm_b200_emb_bwd_link(b, len(big), Bg, 8, 0, one.link.data_ptr(), _st()), "emb_bwd_link")
    one.update(didx, doff, nnz, Bg, dTg.data_ptr(), None, 0, 0, [(1 + sh["table"]) * D for sh in whole], F * D, lr, eps)
    for r, st in enumerate(ranks):
        slab = bl * Tl[r] * D * 4
        st.update(didx, doff, nnz, Bg, None, [recv[r].data_ptr() + s * slab for s in range(W)], W, bl,
                  [j * D for j in range(Tl[r])], Tl[r] * D, lr, eps)
    Wone = [w.cpu().numpy() for w in one.W]
    mone = [m.cpu().numpy() for m in one.m]
    for r, st in enumerate(ranks):
        for j, sh in enumerate(st.shards):
            t, lo, n = sh["table"], sh["row_lo"], sh["row_n"]
            _same_bits(st.W[j], Wone[t][lo:lo + n],
                       f"rank {r} shard {j} (table {t}): rows differ from the whole-table update")
            _same_bits(st.m[j], mone[t][lo:lo + n], f"rank {r} shard {j} (table {t}): accumulators differ")
    touched = sum(int((Wone[t][:, :D] != Wt[t]).any(axis=1).sum()) for t in range(T))
    assert touched > 0
