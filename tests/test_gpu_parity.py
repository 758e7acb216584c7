"""GPU parity tests proper: the CUDA path (through the C ABI) against the oracle and the
live-reference goldens.  Run with `pytest -m gpu` on an H100."""
import ctypes as C

import numpy as np
import pytest
import torch

from golden_util import ALL_CASES, Golden, O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _engine(g: Golden, max_batch=None):
    from dlrm_b200.engine import Engine

    e = Engine(g.m_spa, g.ln_emb, g.ln_bot, g.ln_top, op=g.op, itself=g.itself, sigmoid_bot=-1,
               sigmoid_top=len(g.ln_top) - 2, loss=g.loss, loss_threshold=g.thr, device=DEV,
               max_batch=max_batch or g.B)
    e.load_params(g.params())
    return e


def _dev_batch(g: Golden, s):
    from dlrm_b200.engine import sparse_from_reference

    X, off, idx, T = g.batch(s)
    sp = sparse_from_reference([torch.from_numpy(o) for o in off], [torch.from_numpy(i) for i in idx], DEV)
    return torch.from_numpy(X).to(DEV), sp, torch.from_numpy(T).to(DEV)


# ----------------------------------------------------------------------------- gather kernel
@pytest.mark.parametrize("D", [2, 4, 8, 16, 32, 64, 100, 128, 256, 384])
@pytest.mark.parametrize("itype", [np.int64, np.int32])
def test_emb_bag_fwd_bitexact(D, itype):
    from dlrm_b200 import _lib

    rng = np.random.default_rng(D)
    T, B = 5, 203
    rows = [1, 7, 1000, 50000, 300]
    Ws = [rng.standard_normal((r, D)).astype(np.float32) for r in rows]
    X, off, idx = O.random_batch(rng, rows, B, lmax=37)
    # ragged extras: empty bags in table 1, a very long bag in table 2
    off[1] = np.zeros(B, dtype=np.int64)
    off[1][B // 2:] = idx[1].size  # first half empty except bag B//2-1 which holds everything
    lib = _lib.lib()
    desc = (_lib.EmbFwdTable * T)()
    keep = []
    for k in range(T):
        w = torch.from_numpy(Ws[k]).to(DEV)
        i = torch.from_numpy(idx[k].astype(itype)).to(DEV)
        o = torch.from_numpy(off[k].astype(itype)).to(DEV)
        keep += [w, i, o]
        desc[k].weight, desc[k].indices, desc[k].offsets = w.data_ptr(), i.data_ptr(), o.data_ptr()
        desc[k].row_weights, desc[k].nnz, desc[k].rows = None, idx[k].size, rows[k]
    out = torch.full((B, T, D), float("nan"), device=DEV)
    _lib.check(lib.dlrm_b200_emb_bag_fwd(desc, T, D, B, np.dtype(itype).itemsize, 0, out.data_ptr(), T * D, D,
                                         torch.cuda.current_stream().cuda_stream))
    got = out.cpu().numpy()
    for k in range(T):
        want = O.emb_bag_sum(Ws[k], idx[k], off[k])
        assert np.array_equal(got[:, k, :], want), f"table {k} D={D} not bit-exact"


def test_emb_bag_fwd_weighted_and_include_last():
    from dlrm_b200 import _lib

    rng = np.random.default_rng(3)
    D, B, rows = 128, 64, 500
    W = rng.standard_normal((rows, D)).astype(np.float32)
    rw = rng.uniform(0.5, 1.5, rows).astype(np.float32)
    X, off, idx = O.random_batch(rng, [rows], B, lmax=12)
    offl = np.concatenate([off[0], [idx[0].size]]).astype(np.int64)
    lib = _lib.lib()
    w, r = torch.from_numpy(W).to(DEV), torch.from_numpy(rw).to(DEV)
    i, o = torch.from_numpy(idx[0]).to(DEV), torch.from_numpy(offl).to(DEV)
    desc = (_lib.EmbFwdTable * 1)()
    desc[0].weight, desc[0].indices, desc[0].offsets = w.data_ptr(), i.data_ptr(), o.data_ptr()
    desc[0].row_weights, desc[0].nnz, desc[0].rows = r.data_ptr(), 0, rows  # nnz ignored w/ include_last
    out = torch.zeros((B, D), device=DEV)
    _lib.check(lib.dlrm_b200_emb_bag_fwd(desc, 1, D, B, 8, 1, out.data_ptr(), D, B * D,
                                         torch.cuda.current_stream().cuda_stream))
    want = O.emb_bag_sum(W, idx[0], off[0], psw=rw[idx[0]])
    np.testing.assert_allclose(out.cpu().numpy(), want, rtol=1e-6, atol=1e-7)


# ----------------------------------------------------------------------------- forward vs reference
@pytest.mark.parametrize("name", ALL_CASES)
def test_forward_vs_reference_golden(name):
    g = Golden(name)
    e = _engine(g)
    X, sp, T = _dev_batch(g, 0)
    out = e.forward(X, sp).cpu().numpy()
    # north_star: logits within 1e-5 of the reference CPU forward
    np.testing.assert_allclose(out, g["f_out"], rtol=0, atol=1e-5)
    Tb = e.Tbuf[:g.B].cpu().numpy()
    np.testing.assert_allclose(Tb[:, 0, :], g["f_x"], rtol=2e-5, atol=2e-6)
    for k in range(g.T):
        if g.has(f"f_ly{k}"):
            if g.weighted:
                np.testing.assert_allclose(Tb[:, 1 + k, :], g[f"f_ly{k}"], rtol=1e-6, atol=1e-7)
            else:
                assert np.array_equal(Tb[:, 1 + k, :], g[f"f_ly{k}"]), f"ly[{k}] not bit-exact vs reference"
    if g.op == "dot":
        R = e.Rbuf[:g.B, :e.num_int].cpu().numpy()
        np.testing.assert_allclose(R, g["f_R"], rtol=2e-5, atol=5e-6)


@pytest.mark.parametrize("name", ALL_CASES)
def test_backward_vs_reference_golden(name):
    g = Golden(name)
    if g.weighted:
        pytest.skip("weighted pooling: forward only (SURVEY §8f-3)")
    e = _engine(g)
    X, sp, T = _dev_batch(g, 0)
    e.forward(X, sp)
    e.backward(X, sp, T)
    assert abs(float(e.loss_buf.item()) - float(g["f_loss"])) < 5e-6
    for nm in ("bot", "top"):
        for i in range(len(e.W[nm])):
            np.testing.assert_allclose(*g.dense_grad(f"g_{nm}W{i}", e.dW[nm][i].cpu().numpy()), rtol=5e-4, atol=5e-7)
            np.testing.assert_allclose(e.db[nm][i].cpu().numpy(), g[f"g_{nm}b{i}"], rtol=5e-4, atol=5e-7)
    dT = e.dT[:g.B].cpu().numpy()
    _, off, idx, _ = g.batch(0)
    for k in range(g.T):
        if not g.has(f"g_emb{k}_rows"):
            continue
        rows, vals = O.coalesce(*O.sparse_grad(idx[k], off[k], dT[:, 1 + k, :]))
        assert np.array_equal(rows, g[f"g_emb{k}_rows"])
        np.testing.assert_allclose(vals, g[f"g_emb{k}_vals"], rtol=5e-4, atol=5e-7)


def _robust_close(a, b, atol_med, atol_max, what):
    err = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).ravel()
    assert np.median(err) <= atol_med, f"{what}: median err {np.median(err)}"
    assert np.quantile(err, 0.999) <= atol_max, f"{what}: p99.9 err {np.quantile(err, 0.999)}"


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad"])
@pytest.mark.parametrize("name", [c for c in ALL_CASES if c != "cfg0_weighted"])
def test_train_steps_vs_reference_golden(name, opt):
    g = Golden(name)
    e = _engine(g)
    lr = float(g[f"{opt}_lr"])
    losses = []
    for s in range(g.nsteps):
        X, sp, T = _dev_batch(g, s)
        losses.append(float(e.train_step(X, sp, T, lr, optimizer=opt).item()))
        if s == 0:  # after ONE step everything is a well-conditioned function of the batch-0 grads
            for k in range(g.T):
                if g.has(f"{opt}1_emb{k}_rows"):
                    rows = g[f"{opt}1_emb{k}_rows"]
                    np.testing.assert_allclose(e.table(k)[torch.from_numpy(rows).to(DEV)].cpu().numpy(),
                                               g[f"{opt}1_emb{k}_vals"], rtol=2e-4, atol=2e-6)
                assert abs(float(e.table(k).double().sum().item()) - float(g[f"{opt}1_emb{k}_sum"])) < 1e-3
                if opt == "rwsadagrad":
                    m = e.momentum[int(e.row_base[k]):int(e.row_base[k + 1])].cpu().numpy()
                    np.testing.assert_allclose(m, g[f"{opt}1_mom{k}"], rtol=1e-3, atol=1e-10)
    assert int(e.head.abs().sum().item()) == 0, "row-list heads not reset"
    tight = opt == "sgd"
    np.testing.assert_allclose(losses, g[f"{opt}_losses"], rtol=0, atol=1e-5 if tight else 2e-4)
    X, sp, T = _dev_batch(g, g.nsteps)
    pa = e.forward(X, sp).cpu().numpy()
    _robust_close(pa, g[f"{opt}_p_after"], 2e-5 if tight else 5e-4, 1e-4 if tight else 5e-3, "p_after")
    for k in range(g.T):
        if g.has(f"{opt}_emb{k}_rows"):
            rows = torch.from_numpy(g[f"{opt}_emb{k}_rows"]).to(DEV)
            _robust_close(e.table(k)[rows].cpu().numpy(), g[f"{opt}_emb{k}_vals"], 1e-6 if tight else 2e-5,
                          1e-5 if tight else 2.5 * lr, f"emb{k}")
    for nm in ("bot", "top"):
        for i in range(len(e.W[nm])):
            _robust_close(e.b[nm][i].cpu().numpy(), g[f"{opt}_{nm}b{i}"], 1e-6 if tight else 2e-5,
                          1e-5 if tight else 2.5 * lr, f"{nm}b{i}")
            if g.has(f"{opt}_{nm}W{i}"):
                _robust_close(e.W[nm][i].cpu().numpy(), g[f"{opt}_{nm}W{i}"], 1e-6 if tight else 2e-5,
                              1e-5 if tight else 2.5 * lr, f"{nm}W{i}")


# ----------------------------------------------------------------------------- sparse update kernel

@pytest.mark.parametrize("D", [128, 256])          # the lean update kernel (dim <= 128) / the general one
def test_emb_update_long_lists_give_the_same_result_every_time(D):
    """Rows with far more than 32 occurrences (lists that outgrow the kept chunks too): the per-row lists are built
    by atomicExch in arrival order, yet repeating the same link + update from the same state must give bit-identical
    rows and accumulators -- otherwise every later training step differs from run to run."""
    from dlrm_b200.engine import Engine, sparse_from_reference

    rng = np.random.default_rng(5)
    ln_emb, B = [20, 300], 1024
    e = Engine(D, ln_emb, [4, D], [D + 3, 1], device=DEV, max_batch=B, small_rows_max=0)
    W0 = [rng.standard_normal((r, D)).astype(np.float32) for r in ln_emb]
    X, off, idx = O.random_batch(rng, ln_emb, B, m_den=4, lmax=10)
    sp = sparse_from_reference([torch.from_numpy(o) for o in off], [torch.from_numpy(i) for i in idx], DEV)
    assert max(np.bincount(idx[0]).max(), np.bincount(idx[1]).max()) > 4 * 32
    e.dT.copy_(torch.from_numpy(rng.standard_normal((B, 3, D)).astype(np.float32)))
    e.ensure_optimizer_state("rwsadagrad")
    results = []
    for _ in range(4):
        for k in range(2):
            e.table(k).copy_(torch.from_numpy(W0[k]))
        e.momentum.zero_()
        e.emb_link(sp)
        e.emb_update(sp, e.dT.view(-1)[D:], 3 * D, D, "rwsadagrad", 0.05)
        torch.cuda.synchronize()
        results.append((e.tables.clone(), e.momentum.clone()))
    for t, m in results[1:]:
        assert torch.equal(t, results[0][0]) and torch.equal(m, results[0][1])


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad"])
@pytest.mark.parametrize("D,rows,B,lmax", [(128, 50, 300, 10), (128, 3, 400, 3), (16, 40, 100, 8),
                                            (6, 10, 50, 4), (256, 1000, 64, 20), (128, 200000, 256, 10)])
def test_emb_update_with_duplicates(opt, D, rows, B, lmax, filtered):
    """Heavy duplication (few rows, many bags): coalesce + optimizer vs the oracle
    (optim/rwsadagrad.py:117-143 restated).  Lists longer than 32 exercise the order-independent long-list sum."""
    from dlrm_b200.engine import Engine, sparse_from_reference

    rng = np.random.default_rng(D + rows)
    ln_emb = [rows, rows * 2 + 1]
    # filtered: the per-row list machinery for every table (tiny tables would otherwise take the dense path)
    e = Engine(D, ln_emb, [4, D], [D + 3, 1], device=DEV, max_batch=B, small_rows_max=0 if filtered else 256)
    Ws = [rng.standard_normal((r, D)).astype(np.float32) for r in ln_emb]
    for k in range(2):
        e.table(k).copy_(torch.from_numpy(Ws[k]))
    X, off, idx = O.random_batch(rng, ln_emb, B, m_den=4, lmax=lmax)
    sp = sparse_from_reference([torch.from_numpy(o) for o in off], [torch.from_numpy(i) for i in idx], DEV)
    dY = rng.standard_normal((B, 3, D)).astype(np.float32)
    e.dT.copy_(torch.from_numpy(dY))
    e.ensure_optimizer_state(opt)
    mom = [rng.uniform(0, 1, r).astype(np.float32) for r in ln_emb]
    if opt == "rwsadagrad":
        for k in range(2):
            e.momentum[int(e.row_base[k]):int(e.row_base[k + 1])].copy_(torch.from_numpy(mom[k]))
    if filtered:   # training gather with the duplicate filter + classify (suspects only are linked)
        e.use_filter = True
        scratch = torch.empty((B, 3, D), device=DEV)
        e.emb_forward(sp, scratch.view(-1)[D:], 3 * D, D, link=True)
        assert e._filtered
    else:          # every occurrence linked (stand-alone link kernel)
        e.emb_link(sp)
    e.emb_update(sp, e.dT.view(-1)[D:], 3 * D, D, opt, 0.05)
    torch.cuda.synchronize()
    assert int(e.head.abs().sum().item()) == 0
    for k in range(2):
        ind, val = O.sparse_grad(idx[k], off[k], dY[:, 1 + k, :])
        Wk = Ws[k].copy()
        if opt == "sgd":
            O.sgd_sparse(Wk, ind, val, 0.05)
        else:
            mk = mom[k].copy()
            O.rwsadagrad_sparse(Wk, mk, ind, val, 0.05)
            got_m = e.momentum[int(e.row_base[k]):int(e.row_base[k + 1])].cpu().numpy()
            np.testing.assert_allclose(got_m, mk, rtol=2e-5, atol=1e-7)
        np.testing.assert_allclose(e.table(k).cpu().numpy(), Wk, rtol=2e-5, atol=2e-5)


# ----------------------------------------------------------------------------- full-size properties
def test_cfg1_full_size_gather_properties():
    """BASELINE.json configs[1] at full size: 26 x 1e6 x 128 tables, B=2048.  The oracle cannot
    hold 13 GB comfortably in a unit test, so check (a) a sample of bags against the oracle on the
    rows they touch, bit-exact, (b) linearity: gather(2W) == 2*gather(W) bit-exact, (c) a checksum
    of checksums equal to the sum over touched rows."""
    from dlrm_b200.engine import Engine, SparseInput
    from dlrm_b200.data import make_batch, to_device_packed

    T, R, D, B = 26, 1_000_000, 128, 2048
    ln_top0 = D + (T + 1) * T // 2
    e = Engine(D, [R] * T, [13, 512, 256, D], [ln_top0, 1024, 512, 256, 1], device=DEV, max_batch=B)
    e.init_params(1)
    hb = make_batch(np.random.default_rng(5), [R] * T, B, 13, lmax=10)
    db = to_device_packed(hb, DEV)
    sp = db.sparse
    out = torch.empty((B, T, D), device=DEV)
    e.emb_forward(sp, out.view(-1), T * D, D)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    offs = hb.offsets  # [T, B+1] global positions
    idx = hb.indices
    rng = np.random.default_rng(0)
    for k in rng.choice(T, 6, replace=False):
        for b in rng.choice(B, 40, replace=False):
            rows = idx[offs[k, b]:offs[k, b + 1]]
            Wr = e.table(int(k))[torch.from_numpy(rows).to(DEV)].cpu().numpy()
            want = O.emb_bag_sum(Wr, np.arange(rows.size), np.array([0]))
            assert np.array_equal(got[b, k], want[0])
    # linearity
    e.tables.mul_(2.0)
    out2 = torch.empty_like(out)
    e.emb_forward(sp, out2.view(-1), T * D, D)
    assert torch.equal(out2, out * 2.0)
    e.tables.mul_(0.5)
    # checksum of checksums (float64): sum of all pooled outputs == sum over every touched row
    tot = 0.0
    for k in range(T):
        rows = torch.from_numpy(idx[offs[k, 0]:offs[k, B]]).to(DEV)
        tot += float(e.table(k)[rows].double().sum().item())
    assert abs(float(out.double().sum().item()) - tot) < 1e-6 * max(1.0, abs(tot)) + 1e-3


# ----------------------------------------------------------------------------- routed interaction backward
@pytest.mark.parametrize("F,D,itself", [(4, 16, 0), (27, 128, 0), (9, 64, 1), (40, 32, 0)])
def test_interact_bwd_routed_equals_plain(F, D, itself):
    """interact_bwd_p2p (per-feature destinations, the sharded gradient exchange) writes exactly the
    values interact_bwd writes, into an arbitrary per-feature layout (here: two 'owner' slabs)."""
    from dlrm_b200 import _lib

    lib = _lib.lib()
    B = 300
    torch.manual_seed(F * 131 + D)
    npairs = F * (F + 1) // 2 if itself else F * (F - 1) // 2
    T = torch.randn(B, F * D, device=DEV)
    dR = torch.randn(B, D + npairs, device=DEV)
    dT = torch.zeros(B, F * D, device=DEV)
    s = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.dlrm_b200_interact_bwd(T.data_ptr(), F * D, dR.data_ptr(), D + npairs, dT.data_ptr(), F * D,
                                          B, F, D, itself, 1, s), "interact_bwd")
    # features 1..h -> slab A [B, h, D] (at an offset, like slab `rank` of a peer); the rest -> slab B
    h = (F - 1) // 2
    f0 = torch.zeros(B, D, device=DEV)
    slabA = torch.zeros(2, B, max(h, 1), D, device=DEV)
    slabB = torch.zeros(B, max(F - 1 - h, 1), D, device=DEV)
    dst, ld, first = [f0.data_ptr()], [D], [0, 1]
    extra = torch.zeros(B, 3, D, device=DEV)       # the LAST feature has a second destination (a row-split table)
    for i in range(1, F):
        if i - 1 < h:
            dst.append(slabA[1].data_ptr() + (i - 1) * D * 4); ld.append(h * D)
        else:
            dst.append(slabB.data_ptr() + (i - 1 - h) * D * 4); ld.append((F - 1 - h) * D)
        if i == F - 1:
            dst.append(extra.data_ptr() + 2 * D * 4); ld.append(3 * D)
        first.append(len(dst))
    n = len(dst)
    _lib.check(lib.dlrm_b200_interact_bwd_p2p(T.data_ptr(), F * D, dR.data_ptr(), D + npairs,
                                              (C.c_void_p * n)(*dst), (C.c_int64 * n)(*ld), (C.c_int * (F + 1))(*first),
                                              1.0, B, F, D, itself, 1, None, None, 0, s), "interact_bwd_p2p")
    torch.cuda.synchronize()
    ref = dT.view(B, F, D)
    assert torch.equal(extra[:, 2], ref[:, F - 1]) and float(extra[:, :2].abs().sum()) == 0.0
    assert torch.equal(f0, ref[:, 0])
    assert torch.equal(slabA[1][:, :h], ref[:, 1:1 + h])
    assert torch.equal(slabB[:, :F - 1 - h], ref[:, 1 + h:])
    assert float(slabA[0].abs().sum()) == 0.0
