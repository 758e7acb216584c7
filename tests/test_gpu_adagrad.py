"""Element-wise Adagrad (DLRM_OPT_ADAGRAD) on the GPU.

Kernels through the C ABI, compared with oracle/adagrad_f64.py: the lean kernel (D <= 128, D % 4 == 0), the general
vec and scalar kernels (the scalar one also takes accumulator rows whose stride is not a multiple of 4), int32 and
int64 indices, include_last, a row-split shard, lists of <= 32 and > 32 members, the tiny-table path, the p2p entry
with world 1 and fp16 rows.  Accumulators of rows with <= 32 members equal the fp32 restatement bit for bit (their
gradient is promised bit for bit); weights are held to the bound of oracle/adagrad_f64.step_bound.  What a kernel
must not write (pad columns of the weight and of the accumulator rows, rows and accumulators not in the batch, a
table without occurrences) keeps a sentinel, compared bit for bit; list heads and marks are zero again and the device
error word clear.  Bad momentum / mom_stride are errors without a launch.

Engine and module level against torch.optim.Adagrad on the CPU port of the model (oracle/torch_cpu_port.py), the CLI
against the reference CLI's recorded run (tests/golden/cli_cfg0_D.*) and a graphed step against an eager one.  The worst err/bound ratio of every kernel family is printed at the end
(`pytest -s`)."""
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from dlrm_b200 import _lib
from oracle import adagrad_f64 as A
from oracle import sparse_f64 as S
from oracle import sr_numpy as SR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENT = -7.75e33
ADA = _lib.OPT_ADAGRAD
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


def _same_bits(a, b, what):
    a = a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    b = b.cpu().numpy() if torch.is_tensor(b) else np.asarray(b)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), what


def _no_device_errors():
    assert L().dlrm_b200_check_device_errors(_st()) == 0, "an index was reported outside its table"


def _wide(rng, shape, lo=-8, hi=2):
    return (rng.choice([-1.0, 1.0], shape) * np.exp2(rng.uniform(lo, hi, shape))).astype(np.float32)


def _offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)


def _ceil4(n):
    return (n + 3) // 4 * 4


@pytest.fixture
def tunable():
    prev = {}

    def set_(name, value):
        prev.setdefault(name, 0)
        _lib.set_tunable(name, value)

    try:
        yield set_
    finally:
        for name, value in prev.items():
            _lib.set_tunable(name, value)


# ---------------------------------------------------------------------------------------------- list update
COUNTS = [1, 2, 31, 32, 33, 100]


class Tables:
    """Three tables of one call: table 0 with rows of COUNTS occurrences plus 200 random ones, table 1 without
    occurrences, table 2 with short random bags.  Weight rows [rows, ld] and accumulator rows [rows, ms] carry the
    sentinel in their pad columns.  layout: "tables" (per-table index arrays), "packed" (one shared index array,
    include_last, a capacity tail), "shard" (table 0 holds rows [300, 1100) of 1500)."""

    def __init__(self, rng, D, itype, layout, ms):
        self.D, self.itype, self.layout, self.ms = D, itype, layout, ms
        self.il = layout == "packed"
        self.rows = [1500, 40, 500]
        self.shard = (300, 800) if layout == "shard" else (0, 1500)
        lo, n = self.shard
        special = rng.choice(np.arange(lo, lo + n), len(COUNTS), replace=False)
        occ = np.concatenate([np.full(c, r) for c, r in zip(COUNTS, special)] + [rng.integers(0, 1500, 200)])
        occ = occ[rng.permutation(occ.size)]
        lens0, left = [], occ.size
        while left:
            lens0.append(min(left, int(rng.integers(1, 9))))
            left -= lens0[-1]
        self.B = B = len(lens0)
        lens2 = rng.integers(0, 4, B)
        idx = [occ.astype(np.int64), np.zeros(0, np.int64), rng.integers(0, 500, int(lens2.sum()))]
        offs = [_offsets(lens0), np.zeros(B, np.int64), _offsets(lens2)]
        self.idx, self.off = idx, offs
        self.ld, self.ldy = _ceil4(D) + 4, _ceil4(D)
        self.dY = _wide(rng, (B, 3, self.ldy))
        self.dY[:, :, D:] = SENT
        self.W0 = [np.full((R, self.ld), SENT, np.float32) for R in self.rows]
        self.S0 = [np.full((R, ms), SENT, np.float32) for R in self.rows]
        for w, s in zip(self.W0, self.S0):
            w[:, :D] = _wide(rng, (w.shape[0], D), -4, 0)
            s[:, :D] = np.abs(_wide(rng, (s.shape[0], D), -12, -2))
        self.nnz = [i.size for i in idx]
        self.base = np.concatenate([[0], np.cumsum(self.nnz)[:-1]]).astype(np.int64)
        self.cap = int(sum(self.nnz)) + (23 if self.il else 0)
        if self.il:
            shared = np.concatenate(idx + [np.full(23, 10 ** 6, np.int64)])
            self.didx = [_cuda(shared.astype(itype))] * 3
            self.doff = [_cuda(np.append(o + b, b + i.size).astype(itype)) for o, b, i in zip(offs, self.base, idx)]
        else:
            self.didx = [_cuda(i.astype(itype)) for i in idx]
            self.doff = [_cuda(o.astype(itype)) for o in offs]
        self.ddY = _cuda(self.dY)
        self.link = torch.zeros(2 * self.cap, dtype=torch.int32, device=DEV)
        self.mark = torch.zeros(self.cap, dtype=torch.uint8, device=DEV)
        self.head = [torch.zeros(R, dtype=torch.int32, device=DEV) for R in self.rows]

    def reset(self):
        self.dW = [_cuda(w) for w in self.W0]
        self.dS = [_cuda(s) for s in self.S0]

    def desc(self, mom_stride=None):
        d = (_lib.EmbBwdTable * 3)()
        lo, n = self.shard
        for k in range(3):
            d[k].weight, d[k].momentum, d[k].head = self.dW[k].data_ptr(), self.dS[k].data_ptr(), self.head[k].data_ptr()
            d[k].mom_stride = self.ms if mom_stride is None else mom_stride
            d[k].indices = self.didx[k].data_ptr() if (self.il or self.nnz[k]) else None
            d[k].offsets, d[k].rows, d[k].ld, d[k].mark = self.doff[k].data_ptr(), self.rows[k], self.ld, self.mark.data_ptr()
            d[k].nnz = self.cap if self.il else self.nnz[k]
            d[k].pair_base = 0 if self.il else int(self.base[k])
        if self.layout == "shard":
            d[0].weight += lo * self.ld * 4
            d[0].momentum += lo * self.ms * 4
            d[0].head += lo * 4
            d[0].row_lo, d[0].row_n = lo, n
        return d

    def run(self, lr, eps, p2p=False):
        ib, il = np.dtype(self.itype).itemsize, int(self.il)
        _lib.check(L().dlrm_b200_emb_bwd_link(self.desc(), 3, self.B, ib, il, self.link.data_ptr(), _st()), "link")
        if p2p:
            peer = (C.c_void_p * 1)(self.ddY.data_ptr())
            _lib.check(L().dlrm_b200_emb_bwd_update_p2p(self.desc(), 3, self.D, self.B, ib, il, self.link.data_ptr(),
                                                        peer, 1, self.B, 3 * self.ldy, self.ldy, ADA, lr, eps, None,
                                                        _st()), "update_p2p")
        else:
            _lib.check(L().dlrm_b200_emb_bwd_update(self.desc(), 3, self.D, self.B, ib, il, self.link.data_ptr(),
                                                    self.ddY.data_ptr(), 3 * self.ldy, self.ldy, ADA, lr, eps, None,
                                                    _st()), "update")
        assert all(int(h.abs().sum().item()) == 0 for h in self.head), "list heads not cleared"
        assert int(self.mark.sum().item()) == 0, "marks not cleared"
        _no_device_errors()

    def check(self, family, lr, eps):
        D = self.D
        for k in range(3):
            lo, n = self.shard if k == 0 else (0, self.rows[k])
            pos, bag, r = S.occurrences(self.idx[k], self.off[k], self.nnz[k], False, lo, n)
            rows, grp = S.coalesce(r)
            G = self.dY[bag, k, :D]
            cnt = np.bincount(grp, minlength=rows.size)
            short = cnt <= S.LIST_SORTED_MAX
            g = S.sum_f32_ascending(G, grp, rows.size)
            gx = S.sum_exact(G, grp, rows.size).astype(np.float32)          # long lists: within one ulp of this
            g = np.where(short[:, None], g, gx)
            W0, S0 = self.W0[k][lo:lo + n], self.S0[k][lo:lo + n]
            w, s = self.dW[k][lo:lo + n].cpu().numpy(), self.dS[k][lo:lo + n].cpu().numpy()
            w32, s32 = A.step_f32(W0[rows, :D], S0[rows, :D], g, lr, eps)
            assert np.array_equal(s[rows, :D][short], s32[short]), f"table {k}: accumulators of short lists"
            w64, s64 = A.step_f64(W0[rows, :D], S0[rows, :D], g, lr, eps)
            g_rel = np.where(short, 0.0, 2.0 ** -23)[:, None]
            bw, bs = A.step_bound(w64, s64, g, lr, eps, g_rel=g_rel)
            _record(family + "_w", S.check_within(w[rows, :D], w64, bw, f"table {k} rows"))
            _record(family + "_s", S.check_within(s[rows, :D], s64, bs, f"table {k} accumulators"))
            rest = np.setdiff1d(np.arange(n), rows)
            _same_bits(w[rest], W0[rest], "rows not in the batch")
            _same_bits(s[rest], S0[rest], "accumulators of rows not in the batch")
            _same_bits(w[:, D:], W0[:, D:], "weight pad columns")
            _same_bits(s[:, D:], S0[:, D:], "accumulator pad columns")
        if self.layout == "shard":
            for part in (slice(0, 300), slice(1100, 1500)):
                _same_bits(self.dW[0][part], self.W0[0][part], "rows of another shard")
                _same_bits(self.dS[0][part], self.S0[0][part], "accumulators of another shard")


ADA_D = [1, 3, 16, 64, 128, 132, 256, 1000]
CASES = ([(D, it, "tables", acc) for D in ADA_D for it in (np.int32, np.int64) for acc in ("vec", "scalar")] +
         [(D, it, lay, "vec") for D in (16, 128, 132) for it, lay in ((np.int32, "packed"), (np.int64, "shard"))])


@pytest.mark.parametrize("D,itype,layout,acc", CASES)
def test_adagrad_list_update(D, itype, layout, acc, tunable):
    """acc = "vec": accumulator rows of stride ceil4(D) + 4 (the lean kernel at D % 4 == 0 and D <= 128, the general
    vec kernel above, the scalar kernel at D % 4 != 0); "scalar": stride D + 1 forces the scalar kernel.  At lean
    shapes the general vec kernel runs too (tunable upd_lean = 2) and must give the same bits."""
    ms = _ceil4(D) + 4 if acc == "vec" else D + 1
    rng = np.random.default_rng(D * 11 + len(layout) + ms)
    t = Tables(rng, D, itype, layout, ms)
    lr, eps = 0.05, (1e-4 if D % 2 else 1e-10)
    lean = acc == "vec" and D % 4 == 0 and D <= 128
    vec = acc == "vec" and D % 4 == 0
    family = "lean" if lean else ("general_vec" if vec else "general_scalar")
    t.reset()
    t.run(lr, eps)
    t.check(family, lr, eps)
    if lean:
        first = ([w.clone() for w in t.dW], [s.clone() for s in t.dS])
        tunable("upd_lean", 2)
        t.reset()
        t.run(lr, eps)
        t.check("general_vec", lr, eps)
        for a, b in zip(first[0] + first[1], t.dW + t.dS):
            _same_bits(a, b, "lean and general kernels differ")


@pytest.mark.parametrize("D", [16, 100, 128])
def test_adagrad_p2p_world_1_equals_the_local_update(D):
    rng = np.random.default_rng(D)
    t = Tables(rng, D, np.int64, "tables", _ceil4(D) + 4)
    t.reset()
    t.run(0.05, 1e-10)
    ref = [x.clone() for x in t.dW + t.dS]
    t.reset()
    t.run(0.05, 1e-10, p2p=True)
    for a, b in zip(ref, t.dW + t.dS):
        _same_bits(a, b, "p2p update differs from the local one")
    t.check("p2p", 0.05, 1e-10)


def test_adagrad_bad_accumulators_are_errors_without_launch():
    rng = np.random.default_rng(1)
    D = 16
    t = Tables(rng, D, np.int64, "tables", _ceil4(D) + 4)
    t.reset()
    _lib.check(L().dlrm_b200_emb_bwd_link(t.desc(), 3, t.B, 8, 0, t.link.data_ptr(), _st()), "link")
    for bad in ("null", "stride"):
        d = t.desc(mom_stride=D - 1 if bad == "stride" else None)
        if bad == "null":
            d[2].momentum = None
        rc = L().dlrm_b200_emb_bwd_update(d, 3, D, t.B, 8, 0, t.link.data_ptr(), t.ddY.data_ptr(), 3 * t.ldy, t.ldy,
                                          ADA, 0.05, 1e-10, None, _st())
        err = L().dlrm_b200_last_error()
        assert rc != 0 and (b"momentum" in err or b"mom_stride" in err), err
        for k in range(3):
            d[k].use_dy_off, d[k].dy_off = 1, k * t.ldy
        rc = L().dlrm_b200_emb_bwd_small_update(d, 3, D, t.B, 8, 0, t.ddY.data_ptr(), None, 0, 0, 3 * t.ldy, ADA,
                                                0.05, 1e-10, t.ddY.data_ptr(), 0, _st())
        err = L().dlrm_b200_last_error()
        assert rc != 0 and (b"momentum" in err or b"mom_stride" in err), err
    torch.cuda.synchronize()
    for k in range(3):
        _same_bits(t.dW[k], t.W0[k], "a refused update wrote its table")
        _same_bits(t.dS[k], t.S0[k], "a refused update wrote its accumulators")
    # the lists linked above are still pending: the valid update consumes them (heads and marks back to zero)
    _lib.check(L().dlrm_b200_emb_bwd_update(t.desc(), 3, D, t.B, 8, 0, t.link.data_ptr(), t.ddY.data_ptr(), 3 * t.ldy,
                                            t.ldy, ADA, 0.05, 1e-10, None, _st()), "update")
    assert all(int(h.abs().sum().item()) == 0 for h in t.head) and int(t.mark.sum().item()) == 0
    _no_device_errors()
    t.check("general_vec_errors", 0.05, 1e-10)


# ---------------------------------------------------------------------------------------------- tiny tables
@pytest.mark.parametrize("itype", [np.int32, np.int64])
@pytest.mark.parametrize("D", [4, 16, 128, 132, 256])
def test_adagrad_tiny_table_update(D, itype):
    """Tables of 1, 3 and 155 rows in one call; batches 1, 129 and 1000; include_last on odd batches.  One row of
    table 2 occurs only with an all-zero gradient row: it is not stepped (torch: s + 0, w + 0)."""
    rng = np.random.default_rng(D)
    rows = [1, 3, 155]
    T, ld, ms = len(rows), _ceil4(D) + 4, _ceil4(D) + 8
    for B in (1, 129, 1000):
        il = B % 2 == 1
        idx, off, didx, doff, nnz = [], [], [], [], []
        for R in rows:
            lens = rng.integers(0, 4, B)
            i = rng.integers(0, R, int(lens.sum())).astype(np.int64)
            if R == 155:
                i[i == 7] = 8                                    # row 7 only through the zero sample below
            o = _offsets(lens)
            if il:
                o = np.append(o, i.size)
                i = np.append(i, np.full(9, R + 3, np.int64))
            idx.append(i), off.append(o), nnz.append(int(o[-1]) if il else i.size)
        ldy = T * _ceil4(D)
        dY = _wide(rng, (B, ldy))
        if B > 1:                                                # sample 0 of table 2: one occurrence of row 7, g = 0
            dY[0, 2 * _ceil4(D):2 * _ceil4(D) + D] = 0
            st, en = S.bag_bounds(off[2], nnz[2], il)
            idx[2] = np.concatenate([idx[2][:st[0]], [7], idx[2][st[0]:]])
            off[2] = np.concatenate([[0], off[2][1:] + 1]) if not il else np.concatenate([[0], off[2][1:] + 1])
            nnz[2] += 1
        for k in range(T):
            didx.append(_cuda(idx[k].astype(itype))), doff.append(_cuda(off[k].astype(itype)))
        nbytes = L().dlrm_b200_emb_bwd_small_scratch_bytes(sum(rows), D, B)
        scratch = torch.full((nbytes // 4,), float("nan"), dtype=torch.float32, device=DEV)
        W0 = [np.full((R, ld), SENT, np.float32) for R in rows]
        S0 = [np.full((R, ms), SENT, np.float32) for R in rows]
        for w, s in zip(W0, S0):
            w[:, :D] = _wide(rng, (w.shape[0], D), -4, 0)
            s[:, :D] = np.abs(_wide(rng, (s.shape[0], D), -12, -2))
        dW, dS = [_cuda(w) for w in W0], [_cuda(s) for s in S0]
        d = (_lib.EmbBwdTable * T)()
        for k in range(T):
            d[k].weight, d[k].momentum, d[k].mom_stride = dW[k].data_ptr(), dS[k].data_ptr(), ms
            d[k].indices, d[k].offsets = didx[k].data_ptr(), doff[k].data_ptr()
            d[k].nnz, d[k].rows, d[k].ld, d[k].use_dy_off, d[k].dy_off = (0 if il else nnz[k]), rows[k], ld, 1, \
                k * _ceil4(D)
        lr, eps = 0.05, 1e-10
        _lib.check(L().dlrm_b200_emb_bwd_small_update(d, T, D, B, np.dtype(itype).itemsize, int(il), _cuda(dY).data_ptr(),
                                                      None, 0, 0, ldy, ADA, lr, eps, scratch.data_ptr(), nbytes,
                                                      _st()), "small_update")
        _no_device_errors()
        for k, R in enumerate(rows):
            pos, bag, r = S.occurrences(idx[k], off[k], nnz[k], il, 0, R)
            G = dY[bag, k * _ceil4(D):k * _ceil4(D) + D]
            tr, grp = S.coalesce(r)
            g = S.sum_f32_chunked(G, grp, tr.size, bag)
            moved = np.any(g != 0, axis=1)
            w, s = dW[k].cpu().numpy(), dS[k].cpu().numpy()
            w32, s32 = A.step_f32(W0[k][tr, :D], S0[k][tr, :D], g, lr, eps)
            assert np.array_equal(s[tr, :D][moved], s32[moved]), f"B={B} table {k}: accumulators"
            w64, s64 = A.step_f64(W0[k][tr, :D], S0[k][tr, :D], g, lr, eps)
            bw, _ = A.step_bound(w64, s64, g, lr, eps)
            _record("small_w", S.check_within(w[tr, :D][moved], w64[moved], bw[moved], f"B={B} table {k} rows"))
            rest = np.union1d(np.setdiff1d(np.arange(R), tr), tr[~moved])
            _same_bits(w[rest], W0[k][rest], "untouched rows or rows with an all-zero gradient")
            _same_bits(s[rest], S0[k][rest], "their accumulators")
            _same_bits(w[:, D:], W0[k][:, D:], "weight pad columns")
            _same_bits(s[:, D:], S0[k][:, D:], "accumulator pad columns")
            if k == 2 and B > 1:
                assert 7 in tr[~moved]


# ---------------------------------------------------------------------------------------------- fp16 rows
@pytest.mark.parametrize("D", [64, 256])
def test_adagrad_fp16_rows_are_sr_of_the_fp32_step(D):
    """fp16 rows (the lean kernel at 64, the general one at 256): rows == sr(fmaf(-lr, g / d, w)) bit for bit for rows
    with up to 32 occurrences (except where the emulated fma may double-round), accumulators fp32 bit for bit."""
    rng = np.random.default_rng(D)
    R, B, lr, eps, key = 600, 300, 0.05, 1e-10, 0x0123456789ABCDEF
    lens = rng.integers(0, 5, B)
    idx = rng.integers(0, R, int(lens.sum())).astype(np.int64)
    off = _offsets(lens)
    ld, ms = D + 8, D + 4
    W = np.zeros((R, ld), np.float16)
    W[:, :D] = (rng.standard_normal((R, D)) * 0.1).astype(np.float16)
    S0 = np.full((R, ms), SENT, np.float32)
    S0[:, :D] = np.abs(rng.standard_normal((R, D)).astype(np.float32)) * 1e-3
    dW, dS = _cuda(W.view(np.int16)).view(torch.float16), _cuda(S0)
    dY = (rng.standard_normal((B, D)) * 0.1).astype(np.float32)
    head = torch.zeros(R, dtype=torch.int32, device=DEV)
    mark = torch.zeros(idx.size, dtype=torch.uint8, device=DEV)
    link = torch.zeros(2 * idx.size, dtype=torch.int32, device=DEV)
    di, do, ddY = _cuda(idx), _cuda(off), _cuda(dY)
    d = _lib.EmbBwdTable()
    d.weight, d.momentum, d.mom_stride, d.head, d.mark = dW.data_ptr(), dS.data_ptr(), ms, head.data_ptr(), mark.data_ptr()
    d.indices, d.offsets, d.nnz, d.rows, d.ld = di.data_ptr(), do.data_ptr(), idx.size, R, ld
    d.weight_dtype, d.round_key = _lib.DTYPE_F16, key
    _lib.check(L().dlrm_b200_emb_bwd_link(C.byref(d), 1, B, 8, 0, link.data_ptr(), _st()), "link")
    _lib.check(L().dlrm_b200_emb_bwd_update(C.byref(d), 1, D, B, 8, 0, link.data_ptr(), ddY.data_ptr(), D, 0, ADA, lr,
                                            eps, None, _st()), "update")
    _no_device_errors()
    assert int(head.abs().sum().item()) == 0 and int(mark.sum().item()) == 0
    got, s = dW.cpu().numpy(), dS.cpu().numpy()
    pos, bag, r = S.occurrences(idx, off, idx.size)
    rows, grp = S.coalesce(r)
    g = S.sum_f32_ascending(dY[bag], grp, rows.size)
    w32 = W[rows, :D].astype(np.float32)
    s2 = (S0[rows, :D] + g * g).astype(np.float32)
    q = (g / (np.sqrt(s2) + np.float32(eps))).astype(np.float32)
    x = S._fma_f32(-np.float32(lr), q, w32)
    flag = S.fma_may_double_round(-np.float32(lr), q, w32)
    want = SR.sr_f16(x, SR.sr_bits(key, rows[:, None], np.arange(D)[None, :]))
    assert np.array_equal(got[rows, :D].view(np.uint16)[~flag], want.view(np.uint16)[~flag])
    assert np.array_equal(s[rows, :D], s2)
    rest = np.setdiff1d(np.arange(R), rows)
    _same_bits(got[rest].view(np.uint16), W[rest].view(np.uint16), "untouched fp16 rows")
    _same_bits(s[rest], S0[rest], "untouched accumulators")
    _same_bits(s[:, D:], S0[:, D:], "accumulator pad columns")


# ---------------------------------------------------------------------------------------------- engine and module
def _torch_reference(g, steps, lr, lr_decay=0.0):
    """torch.optim.Adagrad on the CPU port of the model (the reference's ATen ops): losses and final parameters."""
    from oracle.torch_cpu_port import CpuDLRM

    m = CpuDLRM(g.m_spa, g.ln_emb, g.ln_bot, g.ln_top, op=g.op, itself=g.itself, loss=g.loss, loss_threshold=g.thr)
    m.load(g.params())
    opt = torch.optim.Adagrad(m.parameters(), lr=lr, lr_decay=lr_decay)
    losses = []
    for s in range(steps):
        X, off, idx, T = g.batch(s)
        E = m.loss_fn(m(torch.from_numpy(X), [torch.from_numpy(o) for o in off], [torch.from_numpy(i) for i in idx]),
                      torch.from_numpy(T))
        losses.append(float(E.item()))
        opt.zero_grad()
        E.backward()
        opt.step()
    return losses, m, opt


def _mostly_close(got, want, rtol, atol, cap, frac=1e-3, what=""):
    """All but a fraction `frac` of the elements (or two) within rtol / atol, and none further than `cap`.  Adagrad's first step
    on an element is +-lr whatever the gradient's size, so an element whose summed gradient is nearly zero can take
    the opposite sign in two correct fp32 evaluations; such elements are rare and move by at most 2 lr per step."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    err = np.abs(got - want)
    bad = err > atol + rtol * np.abs(want)
    assert bad.sum() <= max(2, frac * bad.size), f"{what}: {int(bad.sum())} of {bad.size} elements outside the tolerance"
    assert err.max(initial=0) <= cap, f"{what}: max |diff| {err.max():.3g} > {cap}"


def _engine(g, gemm="simt", **kw):
    from dlrm_b200.engine import Engine

    e = Engine(g.m_spa, g.ln_emb, g.ln_bot, g.ln_top, op=g.op, itself=g.itself, sigmoid_bot=-1,
               sigmoid_top=len(g.ln_top) - 2, loss=g.loss, loss_threshold=g.thr, device=DEV, max_batch=g.B, gemm=gemm,
               **kw)
    e.load_params(g.params())
    return e


def _dev_batch(g, s):
    from dlrm_b200.engine import sparse_from_reference

    X, off, idx, T = g.batch(s)
    sp = sparse_from_reference([torch.from_numpy(o) for o in off], [torch.from_numpy(i) for i in idx], DEV)
    return torch.from_numpy(X).to(DEV), sp, torch.from_numpy(T).to(DEV)


@pytest.mark.parametrize("gemm", ["simt", "tc"])
@pytest.mark.parametrize("name", ["cfg0", "mini_cfg1"])
def test_engine_matches_torch_adagrad(name, gemm):
    from golden_util import Golden

    g = Golden(name)
    steps, lr, lr_decay = g.nsteps, 0.05, 0.1
    want, m, opt = _torch_reference(g, steps, lr, lr_decay)
    e = _engine(g, gemm)
    got = []
    for s in range(steps):
        X, sp, T = _dev_batch(g, s)
        got.append(float(e.train_step(X, sp, T, lr, "adagrad", lr_decay=lr_decay).item()))
    torch.cuda.synchronize()
    np.testing.assert_allclose(got, want, rtol=0, atol=3e-5 if gemm == "simt" else 3e-4)
    tol = dict(rtol=2e-3, atol=2e-5) if gemm == "simt" else dict(rtol=2e-2, atol=2e-4)
    for k in range(g.T):
        Wt = m.emb_l[k].weight.detach().numpy()
        st = opt.state[m.emb_l[k].weight]["sum"].numpy()
        _mostly_close(e.table(k).cpu().numpy(), Wt, cap=2 * lr * steps, what=f"table {k}", **tol)
        _mostly_close(e.accumulator_ew(k).cpu().numpy(), st, cap=np.abs(st).max(), what=f"sum {k}", **tol)
        touched = np.any(st != 0, axis=1)
        assert np.all(e.accumulator_ew(k).cpu().numpy()[~touched] == 0), "accumulators of never-touched rows"


def test_dlrm_net_with_fused_adagrad_and_checkpoint_loads_into_torch():
    from golden_util import Golden

    from dlrm_b200 import optim as fused
    from dlrm_b200.dlrm_net import DLRM_Net

    g = Golden("cfg0")
    lr = 0.05
    want, _, ref_opt = _torch_reference(g, g.nsteps, lr)
    net = DLRM_Net(g.m_spa, np.array(g.ln_emb), np.array(g.ln_bot), np.array(g.ln_top), arch_interaction_op=g.op,
                   arch_interaction_itself=g.itself, sigmoid_bot=-1, sigmoid_top=len(g.ln_top) - 2,
                   loss_threshold=g.thr, loss_function=g.loss, device=DEV, max_batch=g.B)
    net._engine.load_params(g.params())
    opt = fused.Adagrad(net.parameters(), lr=lr)
    got = []
    for s in range(g.nsteps):
        X, off, idx, T = g.batch(s)
        lS_o = torch.from_numpy(np.stack(off)).to(DEV)
        E = net.loss_fn(net(torch.from_numpy(X).to(DEV), lS_o, [torch.from_numpy(i).to(DEV) for i in idx]),
                        torch.from_numpy(T).to(DEV))
        got.append(float(E.item()))
        opt.zero_grad()
        E.backward()
        opt.step()
    np.testing.assert_allclose(got, want, rtol=0, atol=3e-4)
    sd = opt.state_dict()
    cpu = torch.optim.Adagrad([torch.nn.Parameter(p.detach().float().cpu().clone()) for p in net.parameters()], lr=lr)
    cpu.load_state_dict(sd)
    rs = ref_opt.state_dict()["state"]
    for i, st in cpu.state_dict()["state"].items():
        assert float(st["step"]) == g.nsteps
        _mostly_close(st["sum"].cpu().numpy(), rs[i]["sum"].numpy(), 2e-2, 2e-5, cap=float(rs[i]["sum"].abs().max()),
                      what=f"sum {i}")


@pytest.mark.parametrize("gemm", ["simt", "tc"])
def test_graphed_adagrad_step_is_bit_identical_to_eager(gemm):
    """GraphedTrainStep with fp32 Adagrad (packed static batch, the whole step in one CUDA graph) == eager steps, bit
    for bit: losses, dense parameters, tables and accumulators."""
    from oracle import dlrm_numpy as O

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
            gs = GraphedTrainStep(e, st, 0.01, "adagrad", warmup=0)
            for hb in hbs:
                st.load(hb, non_blocking=False)
                losses.append(float(gs.replay().item()))
        else:
            for hb in hbs:
                st.load(hb, non_blocking=False)
                losses.append(float(e.train_step(st.X, st.sparse, st.target, 0.01, "adagrad").item()))
        torch.cuda.synchronize()
        res.append((losses, e.dense.clone(), e.tables.clone(), e.acc_ew.clone(), e.dense_state.clone()))
    assert res[0][0] == res[1][0]
    for a, b in zip(res[0][1:], res[1][1:]):
        _same_bits(a, b, "graphed step differs from the eager one")
    assert float(res[0][3].abs().sum()) > 0


# ---------------------------------------------------------------------------------------------- CLI
_CLI_BASE = ["--arch-sparse-feature-size=16", "--arch-embedding-size=1000-1000-1000", "--arch-mlp-bot=13-512-256-64-16",
             "--arch-mlp-top=512-256-1", "--mini-batch-size=128", "--data-generation=random", "--num-batches=6",
             "--print-freq=1", "--learning-rate=0.1", "--numpy-rand-seed=727", "--use-gpu"]


def _flags_D():
    return open(os.path.join(ROOT, "tests", "golden", "cli_cfg0_D.flags")).read().split()


def test_cli_adagrad_follows_the_reference_cli(tmp_path):
    """--optimizer=adagrad: the loss curve, test pass and checkpoint of the reference CLI's run (cli_cfg0_D.txt,
    cli_cfg0_D_ref.pt), and the checkpoint written here loads into torch.optim.Adagrad on the CPU."""
    want = [ln for ln in open(os.path.join(ROOT, "tests", "golden", "cli_cfg0_D.txt")).read().splitlines()]
    ck = str(tmp_path / "ours.pt")
    cmd = [sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py")] + _CLI_BASE + _flags_D() + ["--save-model=" + ck]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    got = [ln for ln in r.stdout.splitlines() if re.match(r"Finished| accuracy|Testing at|Saving model", ln)]
    assert len(got) == len(want), r.stdout
    for a, b in zip(got, want):
        if a.startswith("Finished"):
            la, lb = float(a.rsplit(" ", 1)[1]), float(b.rsplit(" ", 1)[1])
            assert a.rsplit(" ", 1)[0] == b.rsplit(" ", 1)[0] and abs(la - lb) < 2e-5, (a, b)
        elif a.startswith("Saving model"):
            assert b.startswith("Saving model")
        elif a.startswith(" accuracy"):      # 768 test samples: at most two of them on the other side of 0.5
            assert abs(float(a.split()[1]) - float(b.split()[1])) <= 0.27, (a, b)
        else:
            assert a == b
    ref = torch.load(os.path.join(ROOT, "tests", "golden", "cli_cfg0_D_ref.pt"), map_location="cpu", weights_only=False)
    ours = torch.load(ck, map_location="cpu", weights_only=False)
    assert set(ours) == set(ref)
    ro, oo = ref["opt_state_dict"], ours["opt_state_dict"]
    assert sorted(oo["state"]) == sorted(ro["state"])
    for i, st in ro["state"].items():
        assert set(oo["state"][i]) == set(st) == {"step", "sum"}
        assert float(oo["state"][i]["step"]) == float(st["step"])
        _mostly_close(oo["state"][i]["sum"].numpy(), st["sum"].numpy(), 1e-2, 1e-6, cap=float(st["sum"].abs().max()),
                      what=f"sum {i}")
    # lr = 0.01, 6 steps.  Every Adagrad step moves an element by up to lr whatever its gradient's size, so an MLP
    # weight whose gradient sums to nearly zero follows the rounding of the GEMMs: the MLPs are held to that cap only,
    # the tables (whose gradients are the pooled dY rows) also to the element count.
    for k, v in ref["state_dict"].items():
        _mostly_close(ours["state_dict"][k].numpy(), v.numpy(), 0, 1e-4, cap=2 * 0.01 * 6,
                      frac=1e-2 if k.startswith("emb_l") else 1.0, what=k)
    params = [torch.nn.Parameter(v.clone()) for v in ours["state_dict"].values()]
    cpu = torch.optim.Adagrad(params, lr=0.01)
    cpu.load_state_dict(oo)
    assert float(cpu.state[params[0]]["step"]) == float(ro["state"][0]["step"])


def test_cli_adagrad_resumes_from_a_reference_checkpoint():
    """--load-model of the reference CLI's Adagrad checkpoint: the engine takes its sums and step count."""
    from dlrm_b200 import cli

    ck = os.path.join(ROOT, "tests", "golden", "cli_cfg0_D_ref.pt")
    flags = [f for f in _flags_D() if not f.startswith("--test-freq")]
    net = cli.run(_CLI_BASE + flags + ["--load-model=" + ck])      # every batch was trained: all are skipped
    ref = torch.load(ck, map_location="cpu", weights_only=False)
    st = ref["opt_state_dict"]["state"]
    assert net._engine.opt_step == int(float(st[0]["step"]))
    for k in range(3):
        np.testing.assert_array_equal(net._engine.accumulator_ew(k).cpu().numpy(), st[k]["sum"].numpy())
    # and a resumed run of more batches keeps training from there
    net2 = cli.run([a for a in _CLI_BASE if not a.startswith("--num-batches")] + flags +
                   ["--num-batches=8", "--load-model=" + ck])
    assert net2._engine.opt_step == int(float(st[0]["step"])) + 2


# ---------------------------------------------------------------------------------------------- row-split shards
@pytest.mark.parametrize("gemm", ["simt", "tc"])
def test_row_split_engine_trains_like_the_unsplit_one(gemm):
    """Tables 1 and 3 stored as two row-range shards each (placement.plan(force_split=...) at world 1, the engine a
    sharded run builds on every rank; table 2 has 40 rows and takes the tiny-table path): the accumulator arena covers
    exactly the stored rows, and three Adagrad steps give the losses, rows and accumulators of the unsplit engine."""
    from oracle import dlrm_numpy as O

    from dlrm_b200 import placement as P, sharding as SH
    from dlrm_b200.engine import Engine, sparse_from_reference

    rng = np.random.default_rng(5)
    D, ln_emb, ln_bot, tail, B, lr = 64, [3000, 777, 40, 1501], [13, 64, 64], [64, 32, 1], 200, 0.05
    F = len(ln_emb) + 1
    ln_top = [D + F * (F - 1) // 2] + tail
    params = O.random_params(rng, D, ln_emb, ln_bot, ln_top)
    X, off, idx = O.random_batch(rng, ln_emb, B, ln_bot[0], 9)
    tgt = np.round(rng.random((B, 1))).astype(np.float32)
    Xd, Td = torch.from_numpy(X).to(DEV), torch.from_numpy(tgt).to(DEV)
    pl = P.plan(ln_emb, [5.0] * 4, 1, force_split=[1, 3])
    assert pl.split_tables() == [1, 3]
    kw = SH.engine_kwargs(pl, 0, len(ln_emb))
    es = Engine(D, kw["ln_emb"], ln_bot, ln_top, loss="bce", sigmoid_top=len(ln_top) - 2, device=DEV, max_batch=B,
                gemm=gemm, shards=kw["shards"], split_slots=kw["split_slots"], n_features=kw["n_features"])
    es.load_params(SH.slice_params(params, pl, 0))
    streams = SH.local_streams(list(zip(off, idx)), pl, 0)
    sps = sparse_from_reference([torch.from_numpy(o) for o, _ in streams], [torch.from_numpy(i) for _, i in streams], DEV)
    eu = Engine(D, ln_emb, ln_bot, ln_top, loss="bce", sigmoid_top=len(ln_top) - 2, device=DEV, max_batch=B, gemm=gemm)
    eu.load_params(params)
    spu = sparse_from_reference([torch.from_numpy(o) for o in off], [torch.from_numpy(i) for i in idx], DEV)
    for step in range(3):
        ls = float(es.train_step(Xd, sps, Td, lr, "adagrad", lr_decay=0.1).item())
        lu = float(eu.train_step(Xd, spu, Td, lr, "adagrad", lr_decay=0.1).item())
        assert abs(ls - lu) < 2e-5, (step, ls, lu)
    torch.cuda.synchronize()
    assert es.acc_ew.shape == (es.total_rows, D) and es.total_rows == sum(ln_emb)
    assert es.lib.dlrm_b200_check_device_errors(None) == 0
    assert int(es.head.abs().sum().item()) == 0
    for j, s in enumerate(pl.of_rank(0)):
        w_ref = eu.table(s.table)[s.row_lo:s.row_hi].cpu().numpy()
        a_ref = eu.accumulator_ew(s.table)[s.row_lo:s.row_hi].cpu().numpy()
        _mostly_close(es.table(j).cpu().numpy(), w_ref, 2e-4, 2e-6, cap=2 * lr * 3, what=f"shard {j} rows")
        _mostly_close(es.accumulator_ew(j).cpu().numpy(), a_ref, 2e-3, 1e-9, cap=max(float(np.abs(a_ref).max()), 1e-30),
                      what=f"shard {j} accumulators")
        _same_bits(es.accumulator_ew(j).cpu().numpy() == 0, a_ref == 0, f"shard {j}: touched rows")
