"""Host row cache on the H100: the cache kernels (csrc/host_tables.cu) step by step against the policy model
(oracle/host_cache_model.py) and a torch oracle of the rows, engines with a cache against engines with every table on
the device (bit for bit), the CLI against the recorded reference runs, checkpoints both ways, and the device memory."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle.host_cache_model import HostCacheModel

from test_gpu_host_tables import (_CLI_BASE, _LOSS, GOLD, LN, Pinned, _batches, _losses, _run, _state, _st, L,
                                  DEV)

pytestmark = pytest.mark.gpu


def _ids(rng, dist, R, n, hot=400):
    if dist == "uniform":
        return rng.integers(0, min(R, hot), n)
    return (rng.zipf(1.3, n) - 1) % R


def _batch(rng, rows, B, idx_bytes, packed, dist):
    offs, idxs = [], []
    for R in rows:
        lens = rng.integers(0, 5, B)
        idxs.append(_ids(rng, dist, R, int(lens.sum())).astype(np.int64))
        offs.append(np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64))
    dt = torch.int64 if idx_bytes == 8 else torch.int32
    if packed:
        flat = np.concatenate(idxs)
        base = np.concatenate([[0], np.cumsum([i.size for i in idxs])])
        off = [np.concatenate([o, [len(i)]]) + b for o, i, b in zip(offs, idxs, base[:-1])]
        I = torch.from_numpy(flat).to(dt).to(DEV)
        return [I] * len(rows), [torch.from_numpy(o).to(dt).to(DEV) for o in off], idxs
    return ([torch.from_numpy(i).to(dt).to(DEV) for i in idxs], [torch.from_numpy(o).to(dt).to(DEV) for o in offs],
            idxs)


@pytest.mark.parametrize("N", [64, 1024, 4096])
@pytest.mark.parametrize("idx_bytes", [4, 8])
@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("dist", ["uniform", "zipf"])
@pytest.mark.parametrize("layout", ["interleaved", "separate_adagrad"])
def test_cache_kernels_against_the_model(N, idx_bytes, packed, dist, layout):
    """Seeded steps, training and forward-only: after each, the map, tags, last uses, step and counters equal the
    model's, every resident row equals the oracle's row and every other host row its host copy."""
    from dlrm_b200 import _lib

    if layout != "interleaved" and (N != 64 or idx_bytes != 8):
        pytest.skip("the separate layout runs at one size and index type")
    rng = np.random.default_rng(N + idx_bytes * 3 + packed * 7 + len(dist))
    D, B, rows = 16, 96, [1500, 600]         # N = 4096 holds every row
    inter = layout == "interleaved"
    ld = D + 4 if inter else D
    head_col = D + 1 if inter else -1
    W = [torch.randn(R, ld) for R in rows]
    if inter:
        for w in W:
            w[:, D + 1:].zero_()
    M = [torch.rand(R) for R in rows] if not inter else None
    A = [torch.rand(R, D) for R in rows] if not inter else None
    truth_w = [w.clone() for w in W]
    truth_m = [m.clone() for m in M] if M else None
    truth_a = [a.clone() for a in A] if A else None
    pins = [Pinned(t) for t in W + (M or []) + (A or [])]
    try:
        cap = B * 4 * len(rows)
        maps = [torch.zeros(R, dtype=torch.int32, device=DEV) for R in rows]
        sw = torch.zeros((N + cap, ld), device=DEV)
        smom = torch.zeros(N + cap, device=DEV) if M else None
        shead = torch.zeros(N + cap, dtype=torch.int32, device=DEV) if not inter else None
        sacc = torch.zeros(N + cap, D, device=DEV) if A else None
        sidx = torch.zeros(cap, dtype=torch.int64 if idx_bytes == 8 else torch.int32, device=DEV)
        lst = torch.zeros(cap, dtype=torch.int32, device=DEV)
        key = torch.zeros(cap, dtype=torch.int64, device=DEV)
        cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
        tag = torch.full((N,), -1, dtype=torch.int64, device=DEV)
        used = torch.zeros(N, dtype=torch.int32, device=DEV)
        step = torch.zeros(1, dtype=torch.int32, device=DEV)
        shd = torch.zeros(N // 32, dtype=torch.int32, device=DEV)
        snx = torch.zeros(cap, dtype=torch.int32, device=DEV)
        sets = torch.zeros(N // 32, dtype=torch.int32, device=DEV)
        nsets = torch.zeros(1, dtype=torch.int32, device=DEV)
        stats = torch.zeros(4, dtype=torch.int64, device=DEV)
        st = _lib.HostStage(weight=sw.data_ptr(), momentum=smom.data_ptr() if M else None,
                            head=shead.data_ptr() if shead is not None else None,
                            acc_ew=sacc.data_ptr() if A else None, slot_idx=sidx.data_ptr(), list=lst.data_ptr(),
                            key=key.data_ptr(), count=cnt.data_ptr(), capacity=cap, ld=ld, head_col=head_col,
                            cache_rows=N, cache_tag=tag.data_ptr(), cache_used=used.data_ptr(), step=step.data_ptr(),
                            set_head=shd.data_ptr(), set_next=snx.data_ptr(), sets=sets.data_ptr(),
                            num_sets=nsets.data_ptr(), stats=stats.data_ptr())
        model = HostCacheModel(N)
        for s in range(12):
            train = s % 4 != 2
            idx, off, raw = _batch(rng, rows, B, idx_bytes, packed, dist)
            arr = (_lib.HostTable * 2)()
            base = 0
            for k in range(2):
                d = arr[k]
                d.weight, d.rows, d.map = W[k].data_ptr(), rows[k], maps[k].data_ptr()
                d.momentum = M[k].data_ptr() if M else None
                d.acc_ew = A[k].data_ptr() if A else None
                d.indices, d.offsets, d.nnz = idx[k].data_ptr(), off[k].data_ptr(), idx[k].numel()
                d.pos_base = 0 if packed else base
                base += raw[k].size
            st.forward_only = int(not train)
            assert L().dlrm_b200_host_stage_in(arr, 2, C.byref(st), D, B, idx_bytes, int(packed), _st()) == 0, \
                L().dlrm_b200_last_error()
            torch.cuda.synchronize()
            slots = sidx.cpu().numpy().astype(np.int64)
            pairs = [(k, int(r)) for k in range(2) for r in raw[k]]
            arena = sw.cpu()
            touched = {}
            for p, (k, r) in enumerate(pairs):
                sl = int(slots[p])
                assert touched.setdefault((k, r), sl) == sl
                if (k, r) in model.where:
                    assert sl == model.where[(k, r)], "a resident row must be read from its slot"
                else:
                    assert sl >= N
                want = truth_w[k][r].clone()
                if inter:
                    want[head_col] = 0
                assert torch.equal(arena[sl], want), (s, k, r)
                if A:
                    assert torch.equal(sacc[sl].cpu(), truth_a[k][r]) and smom[sl].item() == truth_m[k][r].item()
            if train:
                # the update: every touched row and its words change (the list head stays zero)
                sl = torch.tensor(sorted(set(touched.values())), device=DEV)
                c = 0.25 * (s + 1)
                sw[sl, :D + (1 if inter else 0)] += c
                if M:
                    smom[sl] += c
                    sacc[sl] *= 1.5
                for (k, r) in touched:
                    truth_w[k][r, :D + (1 if inter else 0)] += c
                    if M:
                        truth_m[k][r] += c
                        truth_a[k][r] *= 1.5
                assert L().dlrm_b200_host_write_back(arr, 2, C.byref(st), D, _st()) == 0, L().dlrm_b200_last_error()
                model.train_step(pairs)
            else:
                assert L().dlrm_b200_host_release(arr, 2, C.byref(st), D, _st()) == 0
                model.forward_pass(pairs)
            torch.cuda.synchronize()
            assert L().dlrm_b200_check_device_errors(_st()) == 0
            for k in range(2):
                assert maps[k].cpu().tolist() == model.device_map(k, rows[k]), (s, k)
            assert tag.cpu().tolist() == model.tag and used.cpu().tolist() == model.used
            assert int(step.item()) == model.step
            assert stats.cpu().tolist() == [model.hits, model.inserts, model.evictions, model.staged]
            arena = sw.cpu()
            for (k, r), sl in model.where.items():
                want = truth_w[k][r].clone()
                if inter:
                    want[head_col] = 0
                assert torch.equal(arena[sl], want)
                if M:
                    assert smom[sl].item() == truth_m[k][r].item() and torch.equal(sacc[sl].cpu(), truth_a[k][r])
                if shead is not None:
                    assert int(shead[sl].item()) == 0
            for k in range(2):
                out = torch.ones(rows[k], dtype=torch.bool)
                out[[r for (t, r) in model.where if t == k]] = False
                assert torch.equal(W[k][out], truth_w[k][out])
                if M:
                    assert torch.equal(M[k][out], truth_m[k][out]) and torch.equal(A[k][out], truth_a[k][out])
        assert model.hits > 0 and model.inserts > 0
        if N == 64:
            assert model.evictions > 0 and model.staged > 0
        if N == 4096:
            assert model.evictions == 0
        # flush: every row home, the cache empty, the counters kept
        assert L().dlrm_b200_host_cache_flush(arr, 2, C.byref(st), D, _st()) == 0
        torch.cuda.synchronize()
        model.flush()
        for k in range(2):
            assert torch.equal(W[k], truth_w[k])
            if M:
                assert torch.equal(M[k], truth_m[k]) and torch.equal(A[k], truth_a[k])
            assert int(maps[k].abs().sum().item()) == 0
        assert tag.cpu().tolist() == [-1] * N and used.cpu().tolist() == [0] * N
        assert stats.cpu().tolist() == [model.hits, model.inserts, model.evictions, model.staged]
    finally:
        torch.cuda.synchronize()
        for p in pins:
            p.close()


# ---------------------------------------------------------------------------------------------------------- engines
def _engine(host, gemm, cache=0, interleave=None, D=32):
    from dlrm_b200.engine import Engine

    F = len(LN) + 1
    top = [D + F * (F - 1) // 2, 64, 1]
    e = Engine(D, LN, [13, 64, D], top, sigmoid_top=len(top) - 2, device=DEV, max_batch=256, gemm=gemm,
               interleave_momentum=interleave, host_tables=host, host_cache_rows=cache)
    e.init_params(seed=3)
    return e


def _host_pairs(e, b):
    """(host table index, row) of every host-table occurrence of a packed batch."""
    out = []
    idx = b.sparse.indices[0].cpu().numpy()
    for n, k in enumerate(e.host):
        o = b.sparse.offsets[k].cpu().numpy()
        out += [(n, int(r)) for r in idx[int(o[0]):int(o[-1])]]
    return out


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad", "adagrad"])
@pytest.mark.parametrize("gemm", ["simt", "tc"])
@pytest.mark.parametrize("mode", ["eager", "graphed"])
@pytest.mark.parametrize("layout", [None, False])
@pytest.mark.parametrize("cache", [64, 4096])
def test_engine_steps_with_a_cache_are_bit_identical_to_device_tables(opt, gemm, mode, layout, cache):
    """Losses every step; mid-run a forward-only pass and a table read (which writes the cache back); tables and
    accumulators at the end.  The counters follow the model, and only the table read flushes."""
    from dlrm_b200.engine import GraphedTrainStep

    if layout is False and gemm == "tc":
        pytest.skip("the separate layout runs on one GEMM path")
    bs = _batches(10, seed=4)
    res = []
    for h, c in (([], 0), ([0, 2, 4], cache)):
        e = _engine(h, gemm, cache=c, interleave=layout)
        losses, mids = [], []
        model = HostCacheModel(cache) if h else None
        for b in bs[:9]:
            e.prepare(b.sparse, True)           # the largest staging arena first: a graph keeps its addresses
        if mode == "graphed":
            st = bs[9]
            st.buf.copy_(bs[0].buf)
            g = GraphedTrainStep(e, st, 0.05, opt, warmup=0)
        for i, b in enumerate(bs[:8]):
            if mode == "eager":
                losses.append(e.train_step(b.X, b.sparse, b.target, 0.05, opt).clone())
            else:
                st.buf.copy_(b.buf)
                g.replay()
                losses.append(e.loss_buf.clone())
            if h:
                model.train_step(_host_pairs(e, b))
            if i == 3:
                mids.append(e.forward(bs[8].X, bs[8].sparse).clone())      # forward only
                if h:
                    model.forward_pass(_host_pairs(e, bs[8]))
                    s = e.host_cache_stats()
                    assert s["flushes"] == 0
                    assert [s[k] for k in ("hits", "inserts", "evictions", "staged")] == \
                        [model.hits, model.inserts, model.evictions, model.staged]
                    assert s["steps"] == model.step == 4
                mids.append(e.table(0)[:50].clone())                         # a read: flush + invalidate
                if h:
                    model.flush()
                    assert e.host_cache_stats()["flushes"] == 1
                    assert int(e.slot_map.abs().sum().item()) == 0
        p = e.forward(bs[8].X, bs[8].sparse).clone()
        if h:
            s = e.host_cache_stats()
            assert [s[k] for k in ("hits", "inserts", "evictions", "staged")] == \
                [model.hits, model.inserts, model.evictions, model.staged]
            assert s["hits"] > 0
        torch.cuda.synchronize()
        res.append((torch.stack(losses), mids + [p], _state(e, opt)))
        assert L().dlrm_b200_check_device_errors(_st()) == 0
    (l0, m0, s0), (l1, m1, s1) = res
    assert torch.equal(l0, l1)
    for a, b in zip(m0 + s0, m1 + s1):
        assert torch.equal(a.cpu(), b.cpu())


def test_bad_index_mid_run_is_reported_and_the_cache_stays_consistent():
    """The step with the bad index reports it and the next step reports nothing.  The steps before it equal the
    all-device run.  (The gather reads a bad index as row 0 of its descriptor, which for a host table is arena row 0,
    so the bad step itself depends on the arena layout, with or without a cache.)  The bad occurrence touches no
    cache state: the counters follow the model fed the valid rows only, and a flush leaves the map empty."""
    bs = _batches(4, seed=5)
    bad = bs[1]
    bad.indices[int(bad.offsets[0][0].item())] = LN[0] + 5
    res = []
    for h, c in (([], 0), ([0, 2, 4], 64)):
        e = _engine(h, "tc", cache=c)
        model = HostCacheModel(64)
        losses = []
        for i, b in enumerate(bs):
            losses.append(e.train_step(b.X, b.sparse, b.target, 0.05, "rwsadagrad").clone())
            torch.cuda.synchronize()
            assert (L().dlrm_b200_check_device_errors(_st()) != 0) == (i == 1)
            if h:
                model.train_step([(t, r) for t, r in _host_pairs(e, b) if not (t == 0 and r >= LN[0])])
        if h:
            s = e.host_cache_stats()
            assert [s[k] for k in ("hits", "inserts", "evictions", "staged")] == \
                [model.hits, model.inserts, model.evictions, model.staged]
            e.table(0)
            assert int(e.slot_map.abs().sum().item()) == 0
        res.append(torch.stack(losses))
    assert torch.equal(res[0][:1], res[1][:1])


def test_refusals():
    from dlrm_b200.engine import Engine

    kw = dict(device=DEV, max_batch=64)
    with pytest.raises(ValueError, match="needs host tables"):
        Engine(16, [1000, 1000], [13, 16], [16 + 3, 1], host_cache_rows=64, **kw)
    with pytest.raises(ValueError, match="int32 slot map"):
        Engine(16, [1000, 1000], [13, 16], [16 + 3, 1], host_tables=[0], host_cache_rows=1 << 31, **kw)
    e = Engine(16, [1000, 1000], [13, 16], [16 + 3, 1], host_tables=[0], host_cache_rows=33, **kw)
    assert e.cache_rows == 64


def test_auto_cache_grows_its_staging_without_a_second_copy(monkeypatch):
    """An "auto" cache sized against a given free-bytes figure: a later batch with more index positions grows the
    staging arena.  The cache is written back and its arena released first, so the growth never holds a second copy
    of the cache rows, and the run stays bit-identical to the all-device run."""
    from dlrm_b200.data import make_batch, to_device_packed
    from dlrm_b200.engine import Engine

    rows, N, reserve = 1_000_000, 500_000, 1 << 30
    row = 132 * 4 + 13                                  # interleaved D = 128 row + metadata (sgd)
    rng = np.random.default_rng(7)
    small = [to_device_packed(make_batch(rng, [rows, 1000], 512, lmax=1, fixed=True), DEV) for _ in range(3)]
    large = to_device_packed(make_batch(rng, [rows, 1000], 2048, lmax=1, fixed=True), DEV)
    for b in small[1:] + [large]:                      # re-use rows of the first batch: hits
        n = b.sparse.indices[0].numel() // 4
        b.sparse.indices[0][:n] = small[0].sparse.indices[0][:n]
    seq = small + [large, small[0], large]
    free0 = reserve + N * row + small[0].sparse.nnz_total * (132 * 4 + 4 + 8 + 8)
    res = []
    for h in ([], [0]):
        e = Engine(128, [rows, 1000], [13, 128], [128 + 3, 1], sigmoid_top=0, device=DEV, max_batch=2048,
                   host_tables=h, host_cache_rows="auto" if h else 0, host_cache_reserve=reserve)
        e.init_params(seed=0)
        real = torch.cuda.mem_get_info
        losses, grew = [], None
        for i, b in enumerate(seq):
            if h and i == 0:
                monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a, **k: (free0, real()[1]))
            if h and i == 3:
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
            losses.append(e.train_step(b.X, b.sparse, b.target, 0.05, "sgd").clone())
            if h and i == 0:
                monkeypatch.setattr(torch.cuda, "mem_get_info", real)
                assert e.cache_rows == N
            if h and i == 3:
                torch.cuda.synchronize()
                grew = torch.cuda.max_memory_allocated() - base
                assert e.host_cache_stats()["flushes"] == 1 and e.stage_cap == large.sparse.nnz_total
        if h:
            s = e.host_cache_stats()
            assert s["hits"] > 0 and s["inserts"] > 0
            assert grew < N * row // 4, grew                    # a second copy would be N * row = 270 MB
        torch.cuda.synchronize()
        res.append((torch.stack(losses), e.table(0)[:2000].cpu().clone(), e.dense.cpu().clone()))
        assert L().dlrm_b200_check_device_errors(_st()) == 0
        del e
        torch.cuda.empty_cache()
    for a, b in zip(res[0], res[1]):
        assert bool(torch.isfinite(a).all()) and torch.equal(a.cpu(), b.cpu())


def test_memory_bound_of_a_cache():
    from dlrm_b200.data import make_batch, to_device_packed
    from dlrm_b200.engine import Engine

    torch.cuda.synchronize()
    rows, N = 2_000_000, 1 << 16
    before = torch.cuda.memory_allocated()
    e = Engine(128, [rows, 1000], [13, 128], [128 + 3, 1], device=DEV, max_batch=2048, host_tables=[0],
               host_cache_rows=N)
    e.init_params(seed=0)
    b = to_device_packed(make_batch(np.random.default_rng(0), [rows, 1000], 2048, lmax=1, fixed=True), DEV)
    e.prepare(b.sparse, True)
    e.train_step(b.X, b.sparse, b.target, 0.05, "sgd")
    torch.cuda.synchronize()
    grew = torch.cuda.memory_allocated() - before
    stage = e.stage_cap * (132 * 4 + 8 + 8 + 4)
    cache = N * (132 * 4 + 8 + 4 + 1) + e.stage_cap * 4
    assert e.cache_rows == N and e.host_cache_stats()["inserts"] > 0
    assert grew < 4 * rows + stage + cache + (64 << 20), grew
    del e
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- module / CLI
@pytest.mark.parametrize("tag", ["A", "B", "C", "D"])
def test_cli_cfg0_runs_with_a_host_cache(tag):
    flags = open(os.path.join(GOLD, "cli_cfg0_%s.flags" % tag)).read().split()
    want = open(os.path.join(GOLD, "cli_cfg0_%s.txt" % tag)).read()
    got = _run(_CLI_BASE + flags + ["--gemm=simt", "--emb-host-tables=0-1-2", "--emb-host-cache=64"])
    want_l = [float(m.group(1)) for m in re.finditer(r"Finished training it .* loss ([0-9.]+)", want)]
    assert len(_losses(got)) == len(want_l) > 0
    np.testing.assert_allclose(_losses(got), want_l, rtol=0, atol=2e-5)
    test = re.compile(r"Testing at - .*")
    assert test.findall(got) == test.findall(want)


def test_cli_bin_and_kaggle_runs_with_a_host_cache():
    other = re.compile(r"Sparse fea|Randomized|Defined|Split data|Testing at|accuracy|^recall ")
    flags = open(os.path.join(GOLD, "cli_bin_A.flags")).read().split() + [
        "--raw-data-file=" + os.path.join(GOLD, "bin_day"),
        "--processed-data-file=" + os.path.join(GOLD, "bin_processed.npz"), "--use-gpu", "--gemm=simt"]
    counts = np.minimum(np.load(os.path.join(GOLD, "bin_day_fea_count.npz"))["counts"], 1000)
    lst = "-".join(str(k) for k in np.flatnonzero(counts > 256))
    dev, host = _run(flags), _run(flags + ["--emb-host-tables=" + lst, "--emb-host-cache=64"])
    want = open(os.path.join(GOLD, "cli_bin_A.txt")).read()
    np.testing.assert_allclose(_losses(host), [float(v) for v in re.findall(r"loss ([0-9.]+)", want)], rtol=0, atol=2e-5)
    assert _losses(host) == _losses(dev)
    assert [ln for ln in host.splitlines() if other.search(ln)] == [ln for ln in dev.splitlines() if other.search(ln)]
    flags = open(os.path.join(GOLD, "cli_kaggle_A.flags")).read().split() + [
        "--raw-data-file=" + os.path.join(GOLD, "kaggle.txt"),
        "--processed-data-file=" + os.path.join(GOLD, "kaggle_processed.npz"), "--use-gpu", "--gemm=simt"]
    counts = np.load(os.path.join(GOLD, "kaggle_processed.npz"))["counts"]
    lst = "-".join(str(k) for k in np.flatnonzero(counts > 256))
    # the Kaggle goldens' tables are all tiny (<= 256 rows) unless some count says otherwise: a cache needs a host table
    got = _run(flags + (["--emb-host-tables=" + lst, "--emb-host-cache=64"] if lst else [])).splitlines()
    want = open(os.path.join(GOLD, "cli_kaggle_A.txt")).read().splitlines()
    wl = [float(_LOSS.match(ln).group(1)) for ln in want if _LOSS.match(ln)]
    gl = [float(_LOSS.match(ln).group(1)) for ln in got if _LOSS.match(ln)]
    assert len(gl) == len(wl) > 0
    np.testing.assert_allclose(gl, wl, rtol=0, atol=1e-5)
    assert [ln for ln in got if other.search(ln)] == [ln for ln in want if other.search(ln)]


def test_checkpoints_move_between_cached_host_and_device_runs(tmp_path):
    from dlrm_b200 import cli

    args = [a for a in _CLI_BASE if not a.startswith("--num-batches")] + ["--optimizer=rwsadagrad", "--gemm=simt"]
    cached = ["--emb-host-tables=0-2", "--emb-host-cache=64"]
    nets = {}
    for name, extra in (("dev", []), ("host", cached)):
        ck = str(tmp_path / (name + ".pt"))
        net = cli.run(args + extra + ["--num-batches=3", "--save-model=" + ck])
        if extra:
            s = net._engine.host_cache_stats()
            assert s["inserts"] > 0 and s["hits"] > 0
        nets[name] = ck
    a = torch.load(nets["dev"], map_location="cpu", weights_only=False)
    b = torch.load(nets["host"], map_location="cpu", weights_only=False)
    for k in a["state_dict"]:
        assert torch.equal(a["state_dict"][k].cpu(), b["state_dict"][k].cpu()), k
    for k in a["opt_state_dict"]["state"]:
        for f in a["opt_state_dict"]["state"][k]:
            if torch.is_tensor(a["opt_state_dict"]["state"][k][f]):
                assert torch.equal(a["opt_state_dict"]["state"][k][f].cpu(),
                                   b["opt_state_dict"]["state"][k][f].cpu()), (k, f)
    out = []
    for ck, extra in ((nets["dev"], ["--emb-host-tables=0-1-2", "--emb-host-cache=64"]), (nets["host"], [])):
        net = cli.run(args + extra + ["--num-batches=5", "--load-model=" + ck])
        out.append({k: v.detach().cpu().clone() for k, v in net.state_dict().items()})
    for k in out[0]:
        assert torch.equal(out[0][k], out[1][k]), k
    txt = _run(args + ["--num-batches=3", "--test-freq=3"] + cached)
    assert "Testing at" in txt
    txt = _run(args + ["--num-batches=3", "--inference-only", "--load-model=" + nets["host"]] + cached)
    assert "Testing at" in txt or "Saved at" in txt
