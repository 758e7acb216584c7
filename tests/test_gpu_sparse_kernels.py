"""The sparse-path kernels called one by one through the C ABI and compared with the restatements of
oracle/sparse_f64.py: the gather (vec kernel G = 4..32 x NV = 1/2/4, scalar kernel, row-split shard kernel, the
training gather, the peer-routed gather), the link / update kernels (lean, general vec NV = 1..8, general scalar
NV = 1..32, the sorted short-list sum and the fixed-point long-list sum, the duplicate filter) and the tiny-table
update.

Outputs are prefilled with NaN; what a kernel must not write (pad columns, other rows, other output slots, the
accumulators of untouched rows, the other peer buffer) is compared bit for bit afterwards, the list heads and marks
must be zero again, and the device error word must stay clear (every descriptor passes `rows`).  Results the
kernels promise bit for bit are compared bit for bit: the gather against the sequential fp32 sum (fmaf per term
when weighted), the gradient of a row with up to 32 occurrences against the fp32 ascending-position sum, the
tiny-table gradient against the per-chunk restatement, SGD rows against fmaf(-lr, g, w).  The gradient a kernel
used is read back exactly from an SGD step with lr = 1 over zero rows (w' = -g).  RWSAdagrad rows and accumulators
are compared with the float64 step within the bound of oracle/sparse_f64.row_step_bound; longer lists with the
long-list property (one fp32 ulp of the exact sum).  The worst err/bound ratio of every kernel family is printed at
the end of the module (`pytest -s`)."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from dlrm_b200 import _lib
from oracle import sparse_f64 as S
from oracle import sr_numpy as SR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = -7.75e33                 # fp32 sentinel of regions that must stay untouched
SGD, ADA = _lib.OPT_SGD, _lib.OPT_RWSADAGRAD
WORST = {}


def _record(family, r):
    WORST[family] = max(WORST.get(family, 0.0), float(r))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst err/bound per kernel family: " + json.dumps({k: float("%.3g" % v) for k, v in sorted(WORST.items())}))


@pytest.fixture
def tunable():
    """Set process-wide kernel knobs for one test; the previous values (DLRM_TUNE or the default 0) come back after."""
    env = {k.strip(): int(v) for k, v in (kv.split("=") for kv in filter(None, os.environ.get("DLRM_TUNE", "").split(",")))}
    prev = {}

    def set_(name, value):
        prev.setdefault(name, env.get(name, 0))
        _lib.set_tunable(name, value)

    try:
        yield set_
    finally:
        for name, value in prev.items():
            _lib.set_tunable(name, value)


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


def _ceil4(n):
    return (n + 3) // 4 * 4


def _wide(rng, shape, lo=-8, hi=2):
    """fp32 values of both signs over 2^lo .. 2^hi: their fp32 sums depend on the order of the terms."""
    return (rng.choice([-1.0, 1.0], shape) * np.exp2(rng.uniform(lo, hi, shape))).astype(np.float32)


def _offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)


# ---------------------------------------------------------------------------------------------- gather
LENS = [0, 1, 3, 4, 5, 9, 7, 8, 17]        # 0, 1, U-1, U, U+1, 2U+1 for U = 4 and 8


class Gather:
    """T tables of one call in the reference layout (per-table index arrays), their rows with pad columns, and an
    output [batch, T, ldo] whose pad columns hold the sentinel."""

    def __init__(self, rng, D, itype, weighted, include_last, B, rows=(40, 3000), lens=LENS, tail=5):
        self.D, self.itype, self.il, self.B, self.T = D, itype, include_last, B, len(rows)
        self.ld, self.ldo = _ceil4(D) + 4, _ceil4(D) + 4
        self.rows = rows
        self.W, self.rw, self.idx, self.off, self.nnz = [], [], [], [], []
        for R in rows:
            W = np.full((R, self.ld), SENT, np.float32)
            W[:, :D] = _wide(rng, (R, D))
            n = rng.permutation(np.resize(lens, B))
            idx = rng.integers(0, R, int(n.sum())).astype(np.int64)
            off = _offsets(n)
            if include_last:                       # offsets [B + 1]; a capacity tail of out-of-range indices
                off = np.append(off, idx.size)
                idx = np.append(idx, np.full(tail, R + 11, np.int64))
            self.W.append(W)
            self.rw.append(rng.uniform(-2, 2, R).astype(np.float32) if weighted else None)
            self.idx.append(idx)
            self.off.append(off)
            self.nnz.append(int(off[-1]) if include_last else idx.size)
        self.dW = [_cuda(w) for w in self.W]
        self.drw = [_cuda(r) if r is not None else None for r in self.rw]
        self.didx = [_cuda(i.astype(itype)) for i in self.idx]
        self.doff = [_cuda(o.astype(itype)) for o in self.off]

    def desc(self, **per_table):
        d = (_lib.EmbFwdTable * self.T)()
        for k in range(self.T):
            d[k].weight, d[k].indices, d[k].offsets = self.dW[k].data_ptr(), self.didx[k].data_ptr(), self.doff[k].data_ptr()
            d[k].row_weights = self.drw[k].data_ptr() if self.drw[k] is not None else None
            d[k].nnz = 0 if self.il else self.nnz[k]       # ignored with include_last
            d[k].rows, d[k].ld = self.rows[k], self.ld
            for name, vals in per_table.items():
                setattr(d[k], name, vals[k])
        return d

    def out(self):
        o = torch.full((self.B, self.T, self.ldo), SENT, dtype=torch.float32, device=DEV)
        o[:, :, :self.D] = float("nan")
        return o

    def run(self, out=None):
        out = self.out() if out is None else out
        _lib.check(L().dlrm_b200_emb_bag_fwd(self.desc(), self.T, self.D, self.B, np.dtype(self.itype).itemsize,
                                             int(self.il), out.data_ptr(), self.T * self.ldo, self.ldo, _st()),
                   "emb_bag_fwd")
        return out

    def check(self, out, family):
        got = out.cpu().numpy()
        assert np.all(got[:, :, self.D:].view(np.uint32) == np.float32(SENT).view(np.uint32)), "wrote pad columns"
        for k in range(self.T):
            W = self.W[k][:, :self.D]
            want, flag = S.gather_f32(W, self.idx[k], self.off[k], self.nnz[k], self.il, self.rw[k])
            ref, bound = S.gather_f64(W, self.idx[k], self.off[k], self.nnz[k], self.il, self.rw[k])
            g = got[:, k, :self.D]
            assert np.array_equal(g[~flag], want[~flag]), f"table {k}: not the fp32 sequential sum"
            _record(family, S.check_within(g, ref, bound, f"{family} table {k}"))
            _same_bits(self.dW[k], self.W[k], "the gather wrote its table")


GATHER_D = [4, 8, 12, 16, 32, 48, 64, 100, 128, 132, 256, 260, 512, 516, 1000]


@pytest.mark.parametrize("include_last", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("itype", [np.int32, np.int64])
@pytest.mark.parametrize("D", GATHER_D)
def test_gather(D, itype, weighted, include_last):
    """Every vec instantiation (G = 4/8/16/32, NV = 1/2/4, masked columns at 100 / 132 / 260 / 516) and the scalar
    kernel (4, 8, 12, 48, 1000): bags of 0, 1, U-1, U, U+1, 2U+1 indices."""
    g = Gather(np.random.default_rng(D), D, itype, weighted, include_last, B=203)
    g.check(g.run(), "gather_weighted" if weighted else "gather")
    _no_device_errors()


@pytest.mark.parametrize("unroll", [4, 0])
@pytest.mark.parametrize("S_", [1, 2, 3, 0])
@pytest.mark.parametrize("D", [16, 32, 64, 128, 256, 512])
def test_gather_tunables(D, S_, unroll, tunable):
    """bags per lane group S in {1, 2, 3, default 4} (capped at G - 1) and U in {4, default 8}; batches 1, S - 1, S,
    S + 1 and odd, so that the last group of a CTA holds fewer than S bags."""
    tunable("emb_bags_per_group", S_)
    tunable("emb_unroll", unroll)
    G = {16: 4, 32: 8, 64: 16}.get(D, 32)
    s = min(S_ or 4, G - 1)
    rng = np.random.default_rng(D + S_)
    for B in sorted({1, max(s - 1, 1), s, s + 1, 97}):
        for weighted in (False, True):
            g = Gather(rng, D, np.int64, weighted, False, B=B)
            g.check(g.run(), "gather_weighted" if weighted else "gather")
    _no_device_errors()


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("D", [16, 100, 256, 6])
def test_gather_row_split_and_routing(D, weighted):
    """A row-split shard [row_lo, row_lo + row_n) sums only its rows, read at local index row - row_lo (the shard
    kernel; the scalar kernel at D = 6), and out_off / out_stride route table k into slot 1 + k of a [B, F, ldo]
    operand; slot 0 and the pad columns keep the sentinel."""
    rng = np.random.default_rng(D)
    B, R, lo, n, F = 150, 900, 300, 400, 4
    ld = _ceil4(D) + 4
    W = _wide(rng, (R, D))
    Wfull = np.full((R, ld), SENT, np.float32)
    Wfull[:, :D] = W
    rw = rng.uniform(-2, 2, n).astype(np.float32) if weighted else None
    lens = rng.permutation(np.resize(LENS, B))
    idx = rng.integers(0, R, int(lens.sum())).astype(np.int64)
    off = _offsets(lens)
    dW, di, do = _cuda(Wfull), _cuda(idx), _cuda(off)
    drw = _cuda(rw) if weighted else None
    out = torch.full((B, F, ld), SENT, dtype=torch.float32, device=DEV)
    slots = [1, 3]                                          # the shard and the whole table
    for s in slots:
        out[:, s, :D] = float("nan")
    d = (_lib.EmbFwdTable * 2)()
    for k, s in enumerate(slots):
        d[k].indices, d[k].offsets, d[k].nnz, d[k].rows, d[k].ld = di.data_ptr(), do.data_ptr(), idx.size, R, ld
        d[k].out_off, d[k].out_stride = s * ld, F * ld
    d[0].weight, d[0].row_lo, d[0].row_n = dW.data_ptr() + lo * ld * 4, lo, n
    d[0].row_weights = drw.data_ptr() if weighted else None
    d[1].weight = dW.data_ptr()
    rw_full = None
    if weighted:
        rw_full = rng.uniform(-2, 2, R).astype(np.float32)
        drw_full = _cuda(rw_full)
        d[1].row_weights = drw_full.data_ptr()
    _lib.check(L().dlrm_b200_emb_bag_fwd(d, 2, D, B, 8, 0, out.data_ptr(), 0, 0, _st()), "emb_bag_fwd")
    got = out.cpu().numpy()
    for k, s in enumerate(slots):
        kw = dict(rw=rw, row_lo=lo, row_n=n) if k == 0 else dict(rw=rw_full)
        Wk = W[lo:lo + n] if k == 0 else W
        want, flag = S.gather_f32(Wk, idx, off, idx.size, **kw)
        ref, bound = S.gather_f64(Wk, idx, off, idx.size, **kw)
        assert np.array_equal(got[:, s, :D][~flag], want[~flag]), f"slot {s}"
        _record("gather_shard", S.check_within(got[:, s, :D], ref, bound, f"slot {s}"))
    rest = np.ones(got.shape, bool)
    for s in slots:
        rest[:, s, :D] = False
    assert np.all(got[rest].view(np.uint32) == np.float32(SENT).view(np.uint32)), "wrote outside the routed slots"
    _no_device_errors()


@pytest.mark.parametrize("D", [128, 6])
def test_gather_p2p_routes_every_bag_to_its_rank(D):
    """emb_bag_fwd_p2p with world = 2 and both 'peer' buffers on this GPU: bag b lands in buffer b / batch_local,
    row b % batch_local; everything else of both buffers keeps the sentinel."""
    rng = np.random.default_rng(7)
    g = Gather(rng, D, np.int64, False, False, B=2 * 37)
    bl = g.B // 2
    bufs = []
    for _ in range(2):
        b = torch.full((bl + 1, g.T, g.ldo), SENT, dtype=torch.float32, device=DEV)
        b[:bl, :, :D] = float("nan")
        bufs.append(b)
    peer = (C.c_void_p * 2)(*[b.data_ptr() for b in bufs])
    _lib.check(L().dlrm_b200_emb_bag_fwd_p2p(g.desc(), None, g.T, D, g.B, 8, 0, None, peer, 2, bl, g.T * g.ldo, g.ldo,
                                             None, _st()), "emb_bag_fwd_p2p")
    ref = g.run()
    _same_bits(torch.cat([bufs[0][:bl], bufs[1][:bl]]), ref, "p2p routing")
    for b in bufs:
        assert np.all(b[bl].cpu().numpy().view(np.uint32) == np.float32(SENT).view(np.uint32)), "wrote past batch_local"
    g.check(ref, "gather")
    _no_device_errors()


# ---------------------------------------------------------------------------------------------- link + update
COUNTS = [1, 2, 31, 32, 33, 127, 128, 129, 1000]


class Update:
    """Three tables of one call: table 0 with rows of exactly COUNTS occurrences (two in one bag) plus 300 singles,
    table 1 without occurrences, table 2 with short random bags.  layout "tables": per-table index arrays
    (pair_base = earlier nnz, windows of 32 positions straddle the table boundaries); "packed": one shared index
    array with global offsets and include_last, followed by a capacity tail of out-of-range indices; "shard": table 0
    holds rows [500, 1500) of 2000 only."""

    def __init__(self, rng, D, itype, layout):
        self.D, self.itype, self.layout = D, itype, layout
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
        self.B = B = len(lens0)
        # a duplicate inside one bag: the second member of a 2-occurrence row joins the first one's bag
        i2 = np.nonzero(occ == special[1])[0]
        occ = np.delete(occ, i2[1])
        occ = np.insert(occ, i2[0], special[1])
        lens2 = rng.integers(0, 4, B)
        idx = [occ.astype(np.int64), np.zeros(0, np.int64), rng.integers(0, 700, int(lens2.sum()))]
        offs = [_offsets(lens0), np.zeros(B, np.int64), _offsets(lens2)]
        self.idx, self.off = idx, offs                      # per table, positions local to the table
        self.ld = _ceil4(D) + 4
        self.ldy = _ceil4(D)
        self.dY = _wide(rng, (B, 3, self.ldy))
        self.dY[:, :, D:] = SENT
        self.W0 = [np.full((R, self.ld), SENT, np.float32) for R in self.rows]
        for w in self.W0:
            w[:, :D] = _wide(rng, (w.shape[0], D), -4, 0)
        self.m0 = [rng.uniform(0, 1e-3, R).astype(np.float32) for R in self.rows]
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
        self.ddY = _cuda(self.dY)
        self.link = torch.zeros(2 * self.cap, dtype=torch.int32, device=DEV)
        self.mark = torch.zeros(self.cap, dtype=torch.uint8, device=DEV)
        self.head = [torch.zeros(R, dtype=torch.int32, device=DEV) for R in self.rows]

    def reset(self, W=None, m=None):
        self.dW = [_cuda(w) for w in (W or self.W0)]
        self.dm = [_cuda(x) for x in (m or self.m0)]

    def bwd_desc(self):
        d = (_lib.EmbBwdTable * 3)()
        lo, n = self.shard
        for k in range(3):
            d[k].weight, d[k].momentum, d[k].head = self.dW[k].data_ptr(), self.dm[k].data_ptr(), self.head[k].data_ptr()
            d[k].indices = self.didx[k].data_ptr() if (self.il or self.nnz[k]) else None
            d[k].offsets, d[k].rows, d[k].ld, d[k].mark = self.doff[k].data_ptr(), self.rows[k], self.ld, self.mark.data_ptr()
            d[k].nnz = self.cap if self.il else self.nnz[k]
            d[k].pair_base = 0 if self.il else int(self.base[k])
        if self.layout == "shard":
            d[0].weight += lo * self.ld * 4
            d[0].momentum += lo * 4
            d[0].head += lo * 4
            d[0].row_lo, d[0].row_n = lo, n
        return d

    def fwd_desc(self):
        d = (_lib.EmbFwdTable * 3)()
        lo, n = self.shard
        for k in range(3):
            d[k].weight, d[k].offsets, d[k].rows, d[k].ld = self.dW[k].data_ptr(), self.doff[k].data_ptr(), self.rows[k], self.ld
            d[k].indices = self.didx[k].data_ptr() if (self.il or self.nnz[k]) else None
            d[k].nnz = 0 if self.il else self.nnz[k]
        if self.layout == "shard":
            d[0].weight += lo * self.ld * 4
            d[0].row_lo, d[0].row_n = lo, n
        return d

    def build_lists(self, how):
        ib, il = np.dtype(self.itype).itemsize, int(self.il)
        if how == "link":
            _lib.check(L().dlrm_b200_emb_bwd_link(self.bwd_desc(), 3, self.B, ib, il, self.link.data_ptr(), _st()), "link")
            return None
        out = torch.full((self.B, 3, self.ld), float("nan"), dtype=torch.float32, device=DEV)
        dd = None
        if how.startswith("filter"):
            log2 = int(how[6:])
            self._filt = torch.zeros((1 << log2) + 1, dtype=torch.int32, device=DEV)
            self._flags = torch.zeros(self.cap, dtype=torch.uint8, device=DEV)
            self._susp = torch.zeros(self.cap, dtype=torch.int32, device=DEV)
            dd = _lib.EmbDedup(self._filt.data_ptr(), log2, self._flags.data_ptr(), self._susp.data_ptr())
        ref = torch.full_like(out, float("nan"))
        _lib.check(L().dlrm_b200_emb_bag_fwd(self.fwd_desc(), 3, self.D, self.B, ib, il, ref.data_ptr(), 3 * self.ld,
                                             self.ld, _st()), "emb_bag_fwd")
        _lib.check(L().dlrm_b200_emb_bag_fwd_train(self.fwd_desc(), self.bwd_desc(), 3, self.D, self.B, ib, il,
                                                   self.link.data_ptr(), out.data_ptr(), 3 * self.ld, self.ld,
                                                   C.byref(dd) if dd else None, _st()), "emb_bag_fwd_train")
        # the training gather pools like the inference gather, bit for bit
        _same_bits(out[:, :, :self.D], ref[:, :, :self.D], "training gather vs inference gather")
        if dd:
            _lib.check(L().dlrm_b200_emb_bwd_classify(self.bwd_desc(), 3, self.B, ib, il, self.link.data_ptr(),
                                                      C.byref(dd), _st()), "classify")
        return out, dd

    def update(self, opt, lr, eps, how="link"):
        r = self.build_lists(how)
        dd = r[1] if r else None
        _lib.check(L().dlrm_b200_emb_bwd_update(self.bwd_desc(), 3, self.D, self.B, np.dtype(self.itype).itemsize,
                                                int(self.il), self.link.data_ptr(), self.ddY.data_ptr(), 3 * self.ldy,
                                                self.ldy, opt, lr, eps, C.byref(dd) if dd else None, _st()), "update")
        assert all(int(h.abs().sum().item()) == 0 for h in self.head), "list heads not cleared"
        assert int(self.mark.sum().item()) == 0, "marks not cleared"
        _no_device_errors()
        return r[0] if r else None

    def coalesced(self, k):
        """(local rows, per-occurrence row index, per-occurrence gradient rows) of table k."""
        lo, n = self.shard if k == 0 else (0, self.rows[k])
        pos, bag, r = S.occurrences(self.idx[k], self.off[k], self.nnz[k], False, lo, n)
        rows, grp = S.coalesce(r)
        return rows, grp, self.dY[bag, k, :self.D], r

    def table(self, k):
        """(rows, accumulators) this table's descriptor covers (the shard's rows for table 0 of "shard")."""
        lo, n = self.shard if k == 0 else (0, self.rows[k])
        return self.dW[k][lo:lo + n].cpu().numpy(), self.dm[k][lo:lo + n].cpu().numpy()


UPD_D = [4, 16, 100, 128, 256, 260, 512, 516, 1024, 6, 33, 66, 130, 258, 514, 1023]
UPD_CASES = ([(D, it, "tables") for D in UPD_D for it in (np.int32, np.int64)] +
             [(D, it, lay) for D in (16, 128, 260, 33) for it, lay in ((np.int32, "packed"), (np.int64, "shard"))])


@pytest.mark.parametrize("opt", [SGD, ADA])
@pytest.mark.parametrize("D,itype,layout", UPD_CASES)
def test_update_lists(D, itype, layout, opt, tunable):
    rng = np.random.default_rng(D * 7 + len(layout))
    u = Update(rng, D, itype, layout)
    lo, n = u.shard
    lean = D % 4 == 0 and D <= 128
    # 1) the gradient each row was updated with: SGD, lr = 1, zero rows -> w' = -g exactly
    zero = [np.where(np.arange(u.ld) < D, np.float32(0), w) for w in u.W0]
    u.reset(W=zero)
    u.update(SGD, 1.0, 0.0)
    g_kernel = []
    for k in range(3):
        rows, grp, G, r = u.coalesced(k)
        w, _ = u.table(k)
        gk = -w[rows, :D]
        g_kernel.append((rows, gk))
        cnt = np.bincount(grp, minlength=rows.size)
        short = cnt <= S.LIST_SORTED_MAX
        asc = S.sum_f32_ascending(G, grp, rows.size)
        assert np.array_equal(gk[short], asc[short]), f"table {k}: not the ascending-position fp32 sum"
        for i in np.nonzero(~short)[0]:
            ulps = S.long_sum_ulps(gk[i], G[grp == i])
            assert ulps.max() <= 1, f"table {k} row {rows[i]} ({cnt[i]} occurrences): {ulps.max()} ulps"
            _record("long_list_ulps", ulps.max())
        z = zero[k][lo:lo + n] if k == 0 else zero[k]
        untouched = np.setdiff1d(np.arange(w.shape[0]), rows)
        _same_bits(w[untouched], z[untouched], "untouched rows")
        _same_bits(w[:, D:], z[:, D:], "pad columns")
    # 2) the step itself, through every way of building the lists
    lr, eps = 0.05, 1e-4 if D % 2 else 1e-10
    hows = ["link", "train", "link"] + ([] if lean else ["filter10", "filter20"])
    results = {}
    for how in hows:
        u.reset()
        u.update(opt, lr, eps, how)
        results.setdefault(how, []).append([u.table(k) for k in range(3)])
    if lean:                                                 # the general kernel at D <= 128, and the filter
        tunable("upd_lean", 2)
        for how in ("link", "filter10", "filter20"):
            u.reset()
            u.update(opt, lr, eps, how)
            results.setdefault("general_" + how, []).append([u.table(k) for k in range(3)])
    ref = results["link"][0]
    for how, runs in results.items():
        same = not (how.startswith("general") or how.startswith("filter")) or not lean
        for res in runs:
            for k in range(3):
                if same or opt == SGD:
                    _same_bits(res[k][0], ref[k][0], f"{how}: rows differ from the link-kernel lists")
                    _same_bits(res[k][1], ref[k][1], f"{how}: accumulators differ")
    general = results.get("general_link", [ref])[0]
    for label, res in (("lean" if lean else "general", ref), ("general", general)):
        for k in range(3):
            rows, gk = g_kernel[k]
            w, m = res[k]
            W0 = u.W0[k][lo:lo + n] if k == 0 else u.W0[k]
            m0 = u.m0[k][lo:lo + n] if k == 0 else u.m0[k]
            if opt == SGD:
                want = S._fma_f32(-np.float32(lr), gk, W0[rows, :D])
                flag = S.fma_may_double_round(-np.float32(lr), gk, W0[rows, :D])
                assert np.array_equal(w[rows, :D][~flag], want[~flag]), f"table {k}: SGD rows"
                assert S.ulp_diff(w[rows, :D], want).max(initial=0) <= 1
            else:
                w2, m2 = S.row_step(W0[rows, :D], m0[rows], gk, opt, lr, eps)
                bw, bm = S.row_step_bound(w2, m2, gk, opt, lr, eps)
                _record(f"update_{label}_w", S.check_within(w[rows, :D], w2, bw, f"table {k} rows"))
                _record(f"update_{label}_m", S.check_within(m[rows], m2, bm, f"table {k} accumulators"))
            untouched = np.setdiff1d(np.arange(w.shape[0]), rows)
            _same_bits(w[untouched], W0[untouched], "rows not in the batch")
            _same_bits(m[untouched], m0[untouched], "accumulators of untouched rows")
            _same_bits(w[:, D:], W0[:, D:], "columns dim..ld")


def test_update_dim_1025_is_an_error_without_launch():
    u = Update(np.random.default_rng(0), 1024, np.int64, "tables")
    u.reset()
    u.build_lists("link")
    rc = L().dlrm_b200_emb_bwd_update(u.bwd_desc(), 3, 1025, u.B, 8, 0, u.link.data_ptr(), u.ddY.data_ptr(), 3 * u.ldy,
                                      u.ldy, SGD, 0.05, 0.0, None, _st())
    assert rc != 0 and b"dim" in L().dlrm_b200_last_error()
    torch.cuda.synchronize()
    for k in range(3):
        _same_bits(u.dW[k], u.W0[k], "a refused update wrote its table")


@pytest.mark.parametrize("path", ["list", "small"])
def test_update_of_a_row_whose_sum_of_squares_underflows(path):
    """A touched row with |g| ~ 1e-24: g^2 underflows to 0 in fp32, but RWSAdagrad still moves the row by
    -lr g / (sqrt(m) + eps) (optim/rwsadagrad.py has no such exception).  Rows of zeros make the step visible."""
    D, R, B, lr, eps = 128, 5, 4, 0.05, 1e-10
    idx = np.array([1, 2, 2, 3], np.int64)                   # row 2: two occurrences; row 3: an ordinary row
    g = np.zeros((B, D), np.float32)
    g[0], g[1], g[2], g[3] = 1e-24, 3e-24, 2e-24, 0.5
    off = np.arange(B, dtype=np.int64)
    W = np.zeros((R, D), np.float32)
    m = np.zeros(R, np.float32)
    dW, dm, dY = _cuda(W), _cuda(m), _cuda(g)
    di, do = _cuda(idx), _cuda(off)
    d = _lib.EmbBwdTable()
    d.weight, d.momentum, d.indices, d.offsets, d.nnz, d.rows = dW.data_ptr(), dm.data_ptr(), di.data_ptr(), \
        do.data_ptr(), B, R
    if path == "list":
        head = torch.zeros(R, dtype=torch.int32, device=DEV)
        mark = torch.zeros(B, dtype=torch.uint8, device=DEV)
        link = torch.zeros(2 * B, dtype=torch.int32, device=DEV)
        d.head, d.mark = head.data_ptr(), mark.data_ptr()
        _lib.check(L().dlrm_b200_emb_bwd_link(C.byref(d), 1, B, 8, 0, link.data_ptr(), _st()), "link")
        _lib.check(L().dlrm_b200_emb_bwd_update(C.byref(d), 1, D, B, 8, 0, link.data_ptr(), dY.data_ptr(), D, 0, ADA,
                                                lr, eps, None, _st()), "update")
    else:
        d.use_dy_off, d.dy_off = 1, 0
        nbytes = L().dlrm_b200_emb_bwd_small_scratch_bytes(R, D, B)
        scratch = torch.zeros(nbytes // 4, dtype=torch.float32, device=DEV)
        _lib.check(L().dlrm_b200_emb_bwd_small_update(C.byref(d), 1, D, B, 8, 0, dY.data_ptr(), None, 0, 0, D, ADA, lr,
                                                      eps, scratch.data_ptr(), nbytes, _st()), "small_update")
    _no_device_errors()
    rows, grp = S.coalesce(idx)
    gs = S.sum_f32_ascending(g, grp, rows.size)
    w2, m2 = S.row_step(W[rows], m[rows], gs, ADA, lr, eps)
    bw, bm = S.row_step_bound(w2, m2, gs, ADA, lr, eps)
    got_w, got_m = dW.cpu().numpy(), dm.cpu().numpy()
    _record("underflow_" + path, S.check_within(got_w[rows], w2, bw, f"{path}: rows"))
    S.check_within(got_m[rows], m2, bm, f"{path}: accumulators")
    assert np.all(got_w[1] != 0) and np.all(got_w[2] != 0)
    _same_bits(got_w[[0, 4]], W[[0, 4]], "untouched rows")


# ---------------------------------------------------------------------------------------------- tiny tables
def _small_rows_max(D):
    return min(4096, 200 * 1024 // (4 * D))


@pytest.mark.parametrize("itype", [np.int32, np.int64])
@pytest.mark.parametrize("D", [4, 100, 128, 132, 256, 512])
def test_tiny_table_update(D, itype):
    """Tables of 1, 3, 155 and the most rows that fit 200 KB of shared memory, in one call; batches 1, 127, 128, 129
    and 4097 (a partial last chunk of 128 samples); include_last on the odd batches.  The gradient is bitwise the
    per-chunk restatement (read back from SGD, lr = 1, zero rows), SGD rows bitwise, RWSAdagrad within bound."""
    rng = np.random.default_rng(D)
    rows = sorted({min(r, _small_rows_max(D)) for r in (1, 3, 155)} | {_small_rows_max(D)})
    T = len(rows)
    ld = _ceil4(D) + 4
    for B in (1, 127, 128, 129, 4097):
        il = B % 2 == 1
        idx, off, didx, doff, nnz = [], [], [], [], []
        for R in rows:
            lens = rng.integers(0, 4, B)
            i = rng.integers(0, R, int(lens.sum())).astype(np.int64)
            o = _offsets(lens)
            if il:
                o = np.append(o, i.size)
                i = np.append(i, np.full(9, R + 3, np.int64))      # a capacity tail past offsets[batch]
            idx.append(i), off.append(o), nnz.append(int(o[-1]) if il else i.size)
            didx.append(_cuda(i.astype(itype))), doff.append(_cuda(o.astype(itype)))
        ldy = T * _ceil4(D)
        dY = _wide(rng, (B, ldy))
        ddY = _cuda(dY)
        nbytes = L().dlrm_b200_emb_bwd_small_scratch_bytes(sum(rows), D, B)
        scratch = torch.full((nbytes // 4,), float("nan"), dtype=torch.float32, device=DEV)

        def run(opt, lr, eps, W, m):
            dW, dm = [_cuda(w) for w in W], [_cuda(x) for x in m]
            d = (_lib.EmbBwdTable * T)()
            for k in range(T):
                d[k].weight, d[k].momentum, d[k].indices, d[k].offsets = dW[k].data_ptr(), dm[k].data_ptr(), \
                    didx[k].data_ptr(), doff[k].data_ptr()
                d[k].nnz, d[k].rows, d[k].ld, d[k].use_dy_off, d[k].dy_off = (0 if il else nnz[k]), rows[k], ld, 1, \
                    k * _ceil4(D)
            _lib.check(L().dlrm_b200_emb_bwd_small_update(d, T, D, B, np.dtype(itype).itemsize, int(il), ddY.data_ptr(),
                                                          None, 0, 0, ldy, opt, lr, eps, scratch.data_ptr(), nbytes,
                                                          _st()), "small_update")
            _no_device_errors()
            return [w.cpu().numpy() for w in dW], [x.cpu().numpy() for x in dm]

        W0 = [np.full((R, ld), SENT, np.float32) for R in rows]
        for w in W0:
            w[:, :D] = _wide(rng, (w.shape[0], D), -4, 0)
        m0 = [rng.uniform(0, 1e-3, R).astype(np.float32) for R in rows]
        zero = [np.where(np.arange(ld) < D, np.float32(0), w) for w in W0]
        gz, _ = run(SGD, 1.0, 0.0, zero, m0)
        ws, _ = run(SGD, 0.05, 0.0, W0, m0)
        wa, ma = run(ADA, 0.05, 1e-10, W0, m0)
        for k, R in enumerate(rows):
            pos, bag, r = S.occurrences(idx[k], off[k], nnz[k], il, 0, R)
            G = dY[bag, k * _ceil4(D):k * _ceil4(D) + D]
            tr, grp = S.coalesce(r)
            want_g = S.sum_f32_chunked(G, grp, tr.size, bag)
            assert np.array_equal(-gz[k][tr, :D], want_g), f"B={B} table {k}: not the chunked fp32 sum"
            want = S._fma_f32(-np.float32(0.05), want_g, W0[k][tr, :D])
            flag = S.fma_may_double_round(-np.float32(0.05), want_g, W0[k][tr, :D])
            assert np.array_equal(ws[k][tr, :D][~flag], want[~flag]), f"B={B} table {k}: SGD rows"
            w2, m2 = S.row_step(W0[k][tr, :D], m0[k][tr], want_g, ADA, 0.05, 1e-10)
            bw, bm = S.row_step_bound(w2, m2, want_g, ADA, 0.05, 1e-10)
            _record("small_w", S.check_within(wa[k][tr, :D], w2, bw, f"B={B} table {k} rows"))
            _record("small_m", S.check_within(ma[k][tr], m2, bm, f"B={B} table {k} accumulators"))
            _record("small_g", S.check_within(want_g, S.sum_exact(G, grp, tr.size),
                                              S.sum_f32_chunked_bound(G, grp, tr.size, bag), "chunked sum"))
            rest = np.setdiff1d(np.arange(R), tr)
            for res in (ws[k], wa[k]):
                _same_bits(res[rest], W0[k][rest], "untouched rows")
                _same_bits(res[:, D:], W0[k][:, D:], "columns dim..ld")
            _same_bits(ma[k][rest], m0[k][rest], "accumulators of untouched rows")


def test_tiny_table_too_large_for_shared_memory_is_refused():
    D = 128
    R = _small_rows_max(D) + 1
    W = torch.zeros((R, D), device=DEV)
    i = torch.zeros(4, dtype=torch.int64, device=DEV)
    o = torch.arange(4, dtype=torch.int64, device=DEV)
    dY = torch.ones((4, D), device=DEV)
    d = _lib.EmbBwdTable()
    d.weight, d.indices, d.offsets, d.nnz, d.rows, d.use_dy_off = W.data_ptr(), i.data_ptr(), o.data_ptr(), 4, R, 1
    nbytes = L().dlrm_b200_emb_bwd_small_scratch_bytes(R, D, 4)
    scratch = torch.zeros(nbytes // 4, device=DEV)
    rc = L().dlrm_b200_emb_bwd_small_update(C.byref(d), 1, D, 4, 8, 0, dY.data_ptr(), None, 0, 0, D, SGD, 1.0, 0.0,
                                            scratch.data_ptr(), nbytes, _st())
    assert rc != 0 and b"shared memory" in L().dlrm_b200_last_error()
    torch.cuda.synchronize()
    assert int(W.abs().sum().item()) == 0


# ---------------------------------------------------------------------------------------------- fp16 rows
@pytest.mark.parametrize("D", [512, 1024])
def test_fp16_general_update_is_sr_of_the_fp32_step(D):
    """fp16 rows at D 512 / 1024 (the general kernel, NV = 4 / 8): SGD rows == sr_table(fmaf(-lr, g, w)) bit for bit
    for rows with up to 32 occurrences; untouched rows are not rewritten."""
    rng = np.random.default_rng(D)
    R, B, lr, key = 600, 300, 0.05, 0x0123456789ABCDEF
    lens = rng.integers(0, 5, B)
    idx = rng.integers(0, R, int(lens.sum())).astype(np.int64)
    off = _offsets(lens)
    ld = D + 8
    W = np.zeros((R, ld), np.float16)
    W[:, :D] = (rng.standard_normal((R, D)) * 0.1).astype(np.float16)
    dW = _cuda(W.view(np.int16)).view(torch.float16)
    dY = (rng.standard_normal((B, D)) * 0.1).astype(np.float32)
    head = torch.zeros(R, dtype=torch.int32, device=DEV)
    mark = torch.zeros(idx.size, dtype=torch.uint8, device=DEV)
    link = torch.zeros(2 * idx.size, dtype=torch.int32, device=DEV)
    di, do, ddY = _cuda(idx), _cuda(off), _cuda(dY)
    d = _lib.EmbBwdTable()
    d.weight, d.head, d.mark, d.indices, d.offsets, d.nnz, d.rows, d.ld = dW.data_ptr(), head.data_ptr(), \
        mark.data_ptr(), di.data_ptr(), do.data_ptr(), idx.size, R, ld
    d.weight_dtype, d.round_key = _lib.DTYPE_F16, key
    _lib.check(L().dlrm_b200_emb_bwd_link(C.byref(d), 1, B, 8, 0, link.data_ptr(), _st()), "link")
    _lib.check(L().dlrm_b200_emb_bwd_update(C.byref(d), 1, D, B, 8, 0, link.data_ptr(), ddY.data_ptr(), D, 0, SGD, lr,
                                            0.0, None, _st()), "update")
    _no_device_errors()
    assert int(head.abs().sum().item()) == 0 and int(mark.sum().item()) == 0
    got = dW.cpu().numpy()
    pos, bag, r = S.occurrences(idx, off, idx.size)
    rows, grp = S.coalesce(r)
    g = S.sum_f32_ascending(dY[bag], grp, rows.size)
    w32 = W[rows, :D].astype(np.float32)
    x = S._fma_f32(-np.float32(lr), g, w32)
    flag = S.fma_may_double_round(-np.float32(lr), g, w32)
    want = SR.sr_f16(x, SR.sr_bits(key, rows[:, None], np.arange(D)[None, :]))
    assert np.array_equal(got[rows, :D].view(np.uint16)[~flag], want.view(np.uint16)[~flag])
    rest = np.setdiff1d(np.arange(R), rows)
    _same_bits(got[rest].view(np.uint16), W[rest].view(np.uint16), "untouched fp16 rows")
    _same_bits(got[:, D:].view(np.uint16), W[:, D:].view(np.uint16), "fp16 pad columns")
