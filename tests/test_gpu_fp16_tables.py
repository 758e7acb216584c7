"""fp16 embedding tables on the GPU: gather parity with the widened table, stochastic rounding of the fused update
bit for bit against the numpy restatement (oracle/sr_numpy.py), fp16 vs fp32 engines, duplicates, determinism,
checkpoints, end-to-end training and refusals.  Run with `pytest -m gpu` on an H100."""
import numpy as np
import pytest
import torch

from golden_util import Golden, O
from oracle import sr_numpy as SR

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _f16(a):
    return np.asarray(a, dtype=np.float32).astype(np.float16)


def _engine(D, ln_emb, B, ntab=None, **kw):
    from dlrm_b200.engine import Engine

    T = ntab or len(ln_emb)          # global tables (row-split shards count once)
    return Engine(D, ln_emb, [4, D], [D + (T + 1) * T // 2, 1], device=DEV, max_batch=B, **kw)


def _sp(off, idx):
    from dlrm_b200.engine import sparse_from_reference

    return sparse_from_reference([torch.from_numpy(o) for o in off], [torch.from_numpy(i) for i in idx], DEV)


# ----------------------------------------------------------------------------- gather
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("itype", [np.int64, np.int32])
@pytest.mark.parametrize("D", [16, 128])
def test_fp16_gather_equals_oracle_over_widened_table(D, itype, weighted):
    rng = np.random.default_rng(D + (itype == np.int32) + 2 * weighted)
    ln_emb, B = [300, 5000], 200
    e = _engine(D, ln_emb, B, emb_dtype="fp16")
    Ws = [_f16(rng.standard_normal((r, D))) for r in ln_emb]
    rw = [rng.uniform(0.5, 1.5, r).astype(np.float32) for r in ln_emb] if weighted else None
    e.load_params(dict(emb=Ws, bot=[(np.zeros((D, 4), np.float32), np.zeros(D, np.float32))],
                       top=[(np.zeros((1, D + 3), np.float32), np.zeros(1, np.float32))], v_W_l=rw))
    for k in range(2):
        assert np.array_equal(e.table(k).cpu().numpy().view(np.uint16), Ws[k].view(np.uint16))
    X, off, idx = O.random_batch(rng, ln_emb, B, m_den=4, lmax=12)
    off = [o.astype(itype) for o in off]
    idx = [i.astype(itype) for i in idx]
    out = torch.full((B, 2, D), float("nan"), device=DEV)
    e.emb_forward(_sp(off, idx), out, 2 * D, D)
    for k in range(2):
        want = O.emb_bag_sum(Ws[k].astype(np.float32), idx[k], off[k], None if rw is None else rw[k][idx[k]])
        assert np.array_equal(out[:, k, :].cpu().numpy(), want)
    # include_last: offsets with B + 1 entries (the packed convention)
    from dlrm_b200.engine import SparseInput

    offl = [np.concatenate([o, [len(i)]]).astype(itype) for o, i in zip(off, idx)]
    spl = SparseInput([torch.from_numpy(i).to(DEV) for i in idx], [torch.from_numpy(o).to(DEV) for o in offl], B,
                      True, sum(len(i) for i in idx))
    out2 = torch.full((B, 2, D), float("nan"), device=DEV)
    e.emb_forward(spl, out2, 2 * D, D)
    assert torch.equal(out2, out)


@pytest.mark.parametrize("D", [16, 128])
def test_fp16_row_split_gather_equals_fp32_over_widened_table(D):
    """Table 0 held as two row-split shards: fp16 partial sums + reduction == the fp32 engine's, bit for bit."""
    rng = np.random.default_rng(7)
    R, B = 4000, 256
    shards = [dict(table=0, rows=R, row_lo=0, row_n=R // 2, part=0, nparts=2),
              dict(table=0, rows=R, row_lo=R // 2, row_n=R // 2, part=1, nparts=2),
              dict(table=1, rows=500, row_lo=0, row_n=500, part=0, nparts=1)]
    W0, W1 = _f16(rng.standard_normal((R, D))), _f16(rng.standard_normal((500, D)))
    X, off, idx = O.random_batch(rng, [R, 500], B, m_den=4, lmax=10)
    outs = []
    for dt in ("fp16", "fp32"):
        e = _engine(D, [R // 2, R // 2, 500], B, ntab=2, emb_dtype=dt, shards=shards)
        e.table(0).copy_(torch.from_numpy(W0[:R // 2].astype(np.float32)))
        e.table(1).copy_(torch.from_numpy(W0[R // 2:].astype(np.float32)))
        e.table(2).copy_(torch.from_numpy(W1.astype(np.float32)))
        sp = _sp([off[0], off[0], off[1]], [idx[0], idx[0], idx[1]])
        e.emb_forward(sp)
        e.reduce_partials(B)
        outs.append(e.Tbuf[:B, 1:3, :].clone())
    assert torch.equal(outs[0], outs[1])
    want = O.emb_bag_sum(W1.astype(np.float32), idx[1], off[1])
    assert np.array_equal(outs[0][:, 1, :].cpu().numpy(), want)


# ----------------------------------------------------------------------------- stochastic rounding, bit for bit
@pytest.mark.parametrize("D,rows", [(128, 5000), (16, 3000), (256, 4000), (128, 100)])
def test_sr_update_matches_numpy_restatement(D, rows):
    """SGD with lr = 2^-4, every touched row hit once: the pre-rounding value w - lr g is exact in float64, so the
    stored fp16 rows must equal SR(w - lr g) of the restatement bit for bit.  D = 128: lean kernel; D = 256: general
    kernel; 100 rows: the small-table kernel.  Untouched rows keep their bits."""
    rng = np.random.default_rng(D + rows)
    B, lr, seed, step = 512, 2.0 ** -4, 12345, 9
    e = _engine(D, [rows], B, emb_dtype="fp16", round_seed=seed)
    W = _f16(rng.standard_normal((rows, D)) * 0.1)
    e.table(0).copy_(torch.from_numpy(W.astype(np.float32)))
    n = min(B, rows)
    idx = rng.permutation(rows)[:n].astype(np.int64)
    off = np.arange(n, dtype=np.int64)
    g = _f16(rng.standard_normal((n, D))).astype(np.float32)
    dY = np.zeros((n, 1, D), np.float32)
    dY[:, 0, :] = g
    sp = _sp([off], [idx])
    e.opt_step = step
    e.ensure_optimizer_state("sgd")
    e.emb_link(sp)
    e.emb_update(sp, torch.from_numpy(dY).to(DEV), D, D, "sgd", lr)
    torch.cuda.synchronize()
    got = e.table(0).cpu().numpy()
    x = (W[idx].astype(np.float64) - lr * g.astype(np.float64)).astype(np.float32)
    want = SR.sr_f16(x, SR.sr_bits(SR.round_key(seed, step, 0), idx[:, None], np.arange(D)[None, :]))
    assert np.array_equal(got[idx].view(np.uint16), want.view(np.uint16))
    untouched = np.setdiff1d(np.arange(rows), idx)
    assert np.array_equal(got[untouched].view(np.uint16), W[untouched].view(np.uint16))
    # both neighbours occur (the rounding is stochastic, not nearest)
    rn = x.astype(np.float16)
    assert (want != rn).any() and (want == rn).any()
    assert int(e.head.abs().sum().item()) == 0


# ----------------------------------------------------------------------------- fp16 vs fp32 engine
@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad"])
@pytest.mark.parametrize("name", ["cfg0", "mini_cfg1"])
def test_fp16_engine_one_step_equals_sr_of_fp32_engine(name, opt):
    from dlrm_b200.engine import Engine, round_key

    g = Golden(name)
    p = g.params()
    p["emb"] = [_f16(W).astype(np.float32) for W in p["emb"]]      # fp16-representable start
    X, off, idx, T = g.batch(0)
    res = {}
    for dt in ("fp32", "fp16"):
        e = Engine(g.m_spa, g.ln_emb, g.ln_bot, g.ln_top, op=g.op, itself=g.itself, sigmoid_bot=-1,
                   sigmoid_top=len(g.ln_top) - 2, loss=g.loss, loss_threshold=g.thr, device=DEV, max_batch=g.B,
                   emb_dtype=dt, round_seed=3)
        e.load_params(p)
        e.ensure_optimizer_state(opt)
        loss = e.train_step(torch.from_numpy(X).to(DEV), _sp(off, idx), torch.from_numpy(T).to(DEV), 0.05, opt)
        torch.cuda.synchronize()
        res[dt] = (float(loss.item()), [e.table(k).float().cpu().numpy() for k in range(g.T)],
                   e.momentum.cpu().numpy() if opt == "rwsadagrad" else None, e)
    assert res["fp16"][0] == res["fp32"][0]
    if opt == "rwsadagrad":
        assert np.array_equal(res["fp16"][2], res["fp32"][2])
    for k in range(g.T):
        rows = np.unique(idx[k])
        x = res["fp32"][1][k]
        want = SR.sr_f16(x[rows], SR.sr_bits(round_key(3, 1, k), rows[:, None], np.arange(g.m_spa)[None, :]))
        got = res["fp16"][1][k]
        assert np.array_equal(got[rows].astype(np.float16).view(np.uint16), want.view(np.uint16)), k
        rest = np.setdiff1d(np.arange(g.ln_emb[k]), rows)
        assert np.array_equal(got[rest], p["emb"][k][rest])


# ----------------------------------------------------------------------------- duplicates
@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad"])
@pytest.mark.parametrize("D,rows,B,lmax", [(128, 50, 300, 10), (128, 3, 400, 3), (16, 40, 100, 8),
                                            (6, 10, 50, 4), (256, 1000, 64, 20), (128, 200000, 256, 10)])
def test_fp16_update_with_duplicates(opt, D, rows, B, lmax):
    """The duplicate grid of the fp32 update test with fp16 tables: every stored value is an fp16 neighbour of the
    oracle's fp32 result (allowing the fp32 kernel's tolerance), heads and marks are zero afterwards."""
    rng = np.random.default_rng(D + rows)
    ln_emb = [rows, rows * 2 + 1]
    if D % 8:
        with pytest.raises(ValueError, match="divisible by 8"):
            _engine(D, ln_emb, B, emb_dtype="fp16")
        return
    e = _engine(D, ln_emb, B, emb_dtype="fp16")
    Ws = [_f16(rng.standard_normal((r, D))).astype(np.float32) for r in ln_emb]
    for k in range(2):
        e.table(k).copy_(torch.from_numpy(Ws[k]))
    X, off, idx = O.random_batch(rng, ln_emb, B, m_den=4, lmax=lmax)
    sp = _sp(off, idx)
    dY = rng.standard_normal((B, 3, D)).astype(np.float32)
    e.dT.copy_(torch.from_numpy(dY))
    e.ensure_optimizer_state(opt)
    mom = [rng.uniform(0, 1, r).astype(np.float32) for r in ln_emb]
    if opt == "rwsadagrad":
        for k in range(2):
            e.momentum[int(e.row_base[k]):int(e.row_base[k + 1])].copy_(torch.from_numpy(mom[k]))
    e.emb_link(sp)
    e.emb_update(sp, e.dT.view(-1)[D:], 3 * D, D, opt, 0.05)
    torch.cuda.synchronize()
    assert int(e.head.abs().sum().item()) == 0 and int(e.mark.sum().item()) == 0
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
        got = e.table(k).float().cpu().numpy().astype(np.float64)
        tol = 2e-5 * (1.0 + np.abs(Wk))
        lo_a, hi_a = SR.neighbours((Wk - tol).astype(np.float32))
        lo_b, hi_b = SR.neighbours((Wk + tol).astype(np.float32))
        lo = np.minimum.reduce([lo_a, hi_a, lo_b, hi_b]).astype(np.float64)
        hi = np.maximum.reduce([lo_a, hi_a, lo_b, hi_b]).astype(np.float64)
        assert np.all((got >= lo) & (got <= hi)), k
        touched = np.zeros(ln_emb[k], bool)
        touched[np.unique(idx[k])] = True
        assert np.array_equal(got[~touched], Ws[k][~touched])


# ----------------------------------------------------------------------------- determinism
def _dup_case(rng_seed=5, D=128, rows=300, B=256):
    rng = np.random.default_rng(rng_seed)
    W = _f16(rng.standard_normal((rows, D))).astype(np.float32)
    X, off, idx = O.random_batch(rng, [rows], B, m_den=4, lmax=40)
    dY = rng.standard_normal((B, 1, D)).astype(np.float32)
    return W, off, idx, dY


def test_fp16_update_is_deterministic_and_split_invariant():
    D, rows, B = 128, 3000, 256
    W, off, idx, dY = _dup_case(D=D, rows=rows, B=B)
    dYt = torch.from_numpy(dY).to(DEV)
    outs = []
    for _ in range(2):
        e = _engine(D, [rows], B, emb_dtype="fp16", small_rows_max=0)
        e.table(0).copy_(torch.from_numpy(W))
        e.ensure_optimizer_state("rwsadagrad")
        e.opt_step = 4
        sp = _sp(off, idx)
        e.emb_link(sp)
        e.emb_update(sp, dYt, D, D, "rwsadagrad", 0.05)
        torch.cuda.synchronize()
        outs.append((e.table(0).clone(), e.momentum.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    # the same table held as two row-split shards (global rows key the rounding)
    shards = [dict(table=0, rows=rows, row_lo=0, row_n=rows // 2, part=0, nparts=2),
              dict(table=0, rows=rows, row_lo=rows // 2, row_n=rows - rows // 2, part=1, nparts=2)]
    e = _engine(D, [rows // 2, rows - rows // 2], B, ntab=1, emb_dtype="fp16", shards=shards, small_rows_max=0)
    e.table(0).copy_(torch.from_numpy(W[:rows // 2]))
    e.table(1).copy_(torch.from_numpy(W[rows // 2:]))
    e.ensure_optimizer_state("rwsadagrad")
    e.opt_step = 4
    sp = _sp([off[0], off[0]], [idx[0], idx[0]])
    e.emb_link(sp)
    dY2 = torch.cat([dYt, dYt], dim=1).contiguous()
    e.emb_update(sp, dY2, 2 * D, D, "rwsadagrad", 0.05)
    torch.cuda.synchronize()
    split = torch.cat([e.table(0), e.table(1)])
    assert torch.equal(split, outs[0][0])
    assert torch.equal(e.momentum, outs[0][1])


def _net(g, **kw):
    from dlrm_b200.dlrm_net import DLRM_Net

    np.random.seed(1)
    net = DLRM_Net(g.m_spa, np.array(g.ln_emb), np.array(g.ln_bot), np.array(g.ln_top),
                   arch_interaction_op=g.op, arch_interaction_itself=g.itself, sigmoid_bot=-1,
                   sigmoid_top=len(g.ln_top) - 2, loss_threshold=g.thr, loss_function=g.loss, device=DEV, gemm="tc",
                   max_batch=g.B, **kw)
    p = g.params()
    sd = {f"emb_l.{k}.weight": torch.from_numpy(W) for k, W in enumerate(p["emb"])}
    for nm in ("bot", "top"):
        for i, (W, b) in enumerate(p[nm]):
            sd[f"{nm}_l.{2 * i}.weight"] = torch.from_numpy(W)
            sd[f"{nm}_l.{2 * i}.bias"] = torch.from_numpy(b)
    net.load_state_dict(sd)            # an fp32 (reference) checkpoint: round to nearest
    return net, p


def _batch(g, s):
    X, off, idx, T = g.batch(s % g.nsteps)
    return (torch.from_numpy(X), torch.from_numpy(np.stack(off)), [torch.from_numpy(i) for i in idx],
            torch.from_numpy(T))


def _steps(net, opt, g, s0, n):
    losses = []
    for s in range(s0, s0 + n):
        X, lS_o, lS_i, T = _batch(g, s)
        E = net.loss_fn(net(X, lS_o, lS_i), T.to(DEV))
        losses.append(float(E.item()))
        opt.zero_grad()
        E.backward()
        opt.step()
    return losses


def test_fp16_checkpoint_resume_is_bit_identical():
    """4 straight steps == 2 steps + state_dict save / load into a fresh model + 2 steps (opt_step round-trips, so
    the resumed run draws the same rounding bits)."""
    import io

    from dlrm_b200 import optim as fused

    g = Golden("cfg0")
    net, p = _net(g, emb_dtype=torch.float16)
    assert net.emb_l[0].weight.dtype == torch.float16
    assert np.array_equal(net.emb_l[0].weight.detach().cpu().numpy(), p["emb"][0].astype(np.float16))
    opt = fused.RWSAdagrad(net.parameters(), lr=float(g["rwsadagrad_lr"]))
    straight = _steps(net, opt, g, 0, 4)
    ref_tables = [net.emb_l[k].weight.detach().clone() for k in range(g.T)]

    net1, _ = _net(g, emb_dtype=torch.float16)
    opt1 = fused.RWSAdagrad(net1.parameters(), lr=float(g["rwsadagrad_lr"]))
    first = _steps(net1, opt1, g, 0, 2)
    buf = io.BytesIO()
    torch.save({"model": net1.state_dict(), "opt": opt1.state_dict()}, buf)
    buf.seek(0)
    ck = torch.load(buf, weights_only=False)
    assert ck["model"]["emb_l.0.weight"].dtype == torch.float16
    net2, _ = _net(g, emb_dtype=torch.float16)
    opt2 = fused.RWSAdagrad(net2.parameters(), lr=float(g["rwsadagrad_lr"]))
    net2.load_state_dict(ck["model"])
    opt2.load_state_dict(ck["opt"])
    second = _steps(net2, opt2, g, 2, 2)
    assert first + second == straight
    for k in range(g.T):
        assert torch.equal(net2.emb_l[k].weight.detach(), ref_tables[k])
    # an fp16 checkpoint loads into an fp32 model exactly
    net3, _ = _net(g)
    net3.load_state_dict(ck["model"])
    assert torch.equal(net3.emb_l[0].weight.detach(), ck["model"]["emb_l.0.weight"].float().to(DEV))


# ----------------------------------------------------------------------------- end to end
def test_fp16_training_tracks_the_reference_golden():
    """DLRM_Net + RWSAdagrad on cfg0 with fp16 tables: losses within 1e-3 of the live-reference golden, p_after
    within a median of 5e-4 (observed errors are printed)."""
    from dlrm_b200 import optim as fused

    g = Golden("cfg0")
    net, _ = _net(g, emb_dtype=torch.float16)
    opt = fused.RWSAdagrad(net.parameters(), lr=float(g["rwsadagrad_lr"]))
    losses = _steps(net, opt, g, 0, g.nsteps)
    X, lS_o, lS_i, T = _batch(g, 0)
    Xa, offa, idxa, _ = g.batch(g.nsteps) if g.has("b%d_X" % g.nsteps) else g.batch(0)
    with torch.no_grad():
        pa = net(torch.from_numpy(Xa), torch.from_numpy(np.stack(offa)), [torch.from_numpy(i) for i in idxa])
    lerr = np.abs(np.array(losses) - g["rwsadagrad_losses"]).max()
    perr = np.median(np.abs(pa.cpu().numpy() - g["rwsadagrad_p_after"]))
    print("fp16 tables vs reference golden: max |loss err| %.3g, median |p_after err| %.3g" % (lerr, perr))
    assert lerr <= 1e-3 and perr <= 5e-4


# ----------------------------------------------------------------------------- refusals
def test_fp16_refusals():
    from dlrm_b200 import _lib

    with pytest.raises(ValueError, match="divisible by 8"):
        _engine(12, [10], 8, emb_dtype="fp16")
    with pytest.raises(SystemExit, match="divisible by 8"):
        from dlrm_b200.dlrm_net import DLRM_Net

        DLRM_Net(12, np.array([10]), np.array([4, 12]), np.array([13, 1]), arch_interaction_op="dot",
                 device=DEV, emb_dtype=torch.float16)
    # the C ABI refuses an fp16 descriptor with dim % 8 != 0
    e = _engine(16, [10], 8, emb_dtype="fp16")
    sp = _sp([np.arange(8, dtype=np.int64)], [np.arange(8, dtype=np.int64)])
    desc = e._fwd_desc(sp)
    out = torch.zeros((8, 12), device=DEV)
    rc = e.lib.dlrm_b200_emb_bag_fwd(desc, 1, 12, 8, 8, 0, out.data_ptr(), 12, 0, 0)
    assert rc < 0 and b"dim % 8" in _lib.lib().dlrm_b200_last_error()
    # backward without a fused optimizer
    g = Golden("cfg0")
    net, _ = _net(g, emb_dtype=torch.float16)
    X, lS_o, lS_i, T = _batch(g, 0)
    E = net.loss_fn(net(X, lS_o, lS_i), T.to(DEV))
    with pytest.raises(RuntimeError, match="fused optimizers"):
        E.backward()
    # a captured training step would replay one step's rounding bits
    from dlrm_b200.engine import GraphedTrainStep

    with pytest.raises(RuntimeError, match="eager"):
        GraphedTrainStep(net._engine, None, 0.01)


# ----------------------------------------------------------------------------- C ABI: 8-byte aligned fp16 rows
@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad"])
def test_fp16_unpadded_rows_through_the_c_abi(opt):
    """dim 128 with ld = dim + 4 halves -- the unpadded [128 halves | fp32 accumulator | int32 head] row, so odd rows
    start on 8-byte boundaries only.  The gather and the update must handle it (the update through its 8-byte-access
    kernel): gather == oracle over the widened rows, SGD rows == SR(w - lr g) bit for bit, RWSAdagrad rows within an
    fp16 neighbour of the fp32 result, accumulator exact for single occurrences."""
    import ctypes as C

    from dlrm_b200 import _lib

    lib = _lib.lib()
    D, ld, rows, n, lr, key = 128, 132, 3001, 700, 2.0 ** -4, 0x1234567890ABCDEF
    rng = np.random.default_rng(11)
    W = _f16(rng.standard_normal((rows, D)) * 0.1)
    buf = torch.zeros((rows, ld), dtype=torch.float16, device=DEV)
    buf[:, :D].copy_(torch.from_numpy(W).to(DEV))
    mom0 = rng.uniform(0.5, 1.0, rows).astype(np.float32)
    buf.view(torch.int32)[:, D // 2].view(torch.float32).copy_(torch.from_numpy(mom0))   # accumulator word
    idx = torch.from_numpy(rng.permutation(rows)[:n].astype(np.int64)).to(DEV)
    off = torch.arange(n, dtype=torch.int64, device=DEV)
    g = _f16(rng.standard_normal((n, D))).astype(np.float32)
    dY = torch.from_numpy(g).to(DEV)
    base = buf.data_ptr()
    # forward over the unpadded rows
    fd = _lib.EmbFwdTable()
    fd.weight, fd.indices, fd.offsets, fd.nnz, fd.rows, fd.ld, fd.weight_dtype = base, idx.data_ptr(), off.data_ptr(), \
        n, rows, ld, _lib.DTYPE_F16
    out = torch.full((n, D), float("nan"), device=DEV)
    _lib.check(lib.dlrm_b200_emb_bag_fwd(C.byref(fd), 1, D, n, 8, 0, out.data_ptr(), D, 0, 0), "emb_bag_fwd")
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), W[idx.cpu().numpy()].astype(np.float32))
    # link + update
    bd = _lib.EmbBwdTable()
    bd.weight, bd.ld, bd.weight_dtype, bd.round_key = base, ld, _lib.DTYPE_F16, key
    bd.momentum, bd.mom_stride = base + 2 * D, ld // 2
    bd.head, bd.head_stride = base + 2 * D + 4, ld // 2
    mark = torch.zeros(n, dtype=torch.uint8, device=DEV)
    link = torch.zeros(2 * n, dtype=torch.int32, device=DEV)
    bd.mark, bd.indices, bd.offsets, bd.nnz, bd.rows = mark.data_ptr(), idx.data_ptr(), off.data_ptr(), n, rows
    _lib.check(lib.dlrm_b200_emb_bwd_link(C.byref(bd), 1, n, 8, 0, link.data_ptr(), 0), "emb_bwd_link")
    code = _lib.OPT_SGD if opt == "sgd" else _lib.OPT_RWSADAGRAD
    _lib.check(lib.dlrm_b200_emb_bwd_update(C.byref(bd), 1, D, n, 8, 0, link.data_ptr(), dY.data_ptr(), D, 0, code,
                                            lr, 1e-10, None, 0), "emb_bwd_update")
    torch.cuda.synchronize()
    got = buf[:, :D].cpu().numpy()
    i = idx.cpu().numpy()
    gd = g.astype(np.float64)
    if opt == "sgd":
        x = (W[i].astype(np.float64) - lr * gd).astype(np.float32)
        want = SR.sr_f16(x, SR.sr_bits(key, i[:, None], np.arange(D)[None, :]))
        assert np.array_equal(got[i].view(np.uint16), want.view(np.uint16))
    else:
        m_new = mom0[i].astype(np.float64) + (gd * gd).mean(axis=1)
        got_m = buf.view(torch.int32)[:, D // 2].view(torch.float32).cpu().numpy()
        np.testing.assert_allclose(got_m[i], m_new, rtol=1e-6)
        x = W[i].astype(np.float64) - lr * gd / (np.sqrt(m_new)[:, None] + 1e-10)
        tol = 1e-5 * np.abs(x) + 1e-7           # the kernel's fp32 arithmetic vs this float64 restatement
        lo, hi = SR.neighbours((x - tol).astype(np.float32)), SR.neighbours((x + tol).astype(np.float32))
        lo_b = np.minimum.reduce([lo[0], lo[1], hi[0], hi[1]]).astype(np.float64)
        hi_b = np.maximum.reduce([lo[0], lo[1], hi[0], hi[1]]).astype(np.float64)
        gv = got[i].astype(np.float64)
        assert np.all((gv >= lo_b) & (gv <= hi_b))
    rest = np.setdiff1d(np.arange(rows), i)
    assert np.array_equal(got[rest].view(np.uint16), W[rest].view(np.uint16))
    assert int(buf.view(torch.int32)[:, D // 2 + 1].abs().sum().item()) == 0 and int(mark.sum().item()) == 0


# ----------------------------------------------------------------------------- initialisation
def test_fp16_init_is_round_to_nearest_of_the_fp32_init():
    """init_params(seed): the fp16 tables equal RN(fp32 engine's tables) element for element, including a table of
    more than 2^24 rows (two draw chunks; the first spans more than 2^31 elements of the row-strided view)."""
    ln_emb, D = [17_000_000, 1000, 5], 128
    e32 = _engine(D, ln_emb, 64)
    e32.init_params(5)
    e16 = _engine(D, ln_emb, 64, emb_dtype="fp16")
    e16.init_params(5)
    for k, n in enumerate(ln_emb):
        for r0 in range(0, n, 1 << 22):
            a = e16.table(k)[r0:r0 + (1 << 22)]
            b = e32.table(k)[r0:r0 + (1 << 22)].half()
            assert torch.equal(a, b), (k, r0)
    assert torch.equal(e16.dense, e32.dense)
