"""Host embedding tables on the H100: the staging kernels (csrc/host_tables.cu) against a torch oracle, engines with
host tables against engines with every table on the device (bit for bit), the module and the CLI against the
recorded reference runs, checkpoints between the two kinds of run, and the device memory a host table costs."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
DEV = "cuda:0"

pytestmark = pytest.mark.gpu


def L():
    from dlrm_b200 import _lib

    return _lib.lib()


def _st():
    return torch.cuda.current_stream().cuda_stream


class Pinned:
    """A registered (mapped, UVA) CPU tensor, unregistered on close."""

    def __init__(self, t):
        self.t = t
        assert L().dlrm_b200_host_register(t.data_ptr(), t.numel() * t.element_size()) == 0, L().dlrm_b200_last_error()

    def close(self):
        assert L().dlrm_b200_host_unregister(self.t.data_ptr()) == 0


def _batch(rng, rows, B, idx_dtype, packed, hot=20):
    """Bags of 0..8 indices drawn from `hot` rows per table (heavy duplicates, empty bags)."""
    offs, idxs = [], []
    for R in rows:
        lens = rng.integers(0, 9, B)
        pool = rng.choice(R, size=min(hot, R), replace=False)
        idxs.append(rng.choice(pool, size=int(lens.sum())).astype(np.int64))
        offs.append(np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64))
    dt = torch.int64 if idx_dtype == 8 else torch.int32
    if packed:
        flat = np.concatenate(idxs)
        base = np.concatenate([[0], np.cumsum([i.size for i in idxs])])
        off = [np.concatenate([o, [len(i)]]) + b for o, i, b in zip(offs, idxs, base[:-1])]
        I = torch.from_numpy(flat).to(dt).to(DEV)
        return [I] * len(rows), [torch.from_numpy(o).to(dt).to(DEV) for o in off], int(flat.size), idxs
    return ([torch.from_numpy(i).to(dt).to(DEV) for i in idxs], [torch.from_numpy(o).to(dt).to(DEV) for o in offs],
            sum(i.size for i in idxs), idxs)


@pytest.mark.parametrize("idx_bytes", [4, 8])
@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("layout", ["interleaved", "separate", "separate_adagrad"])
def test_staging_kernels_against_torch(idx_bytes, packed, layout):
    from dlrm_b200 import _lib

    rng = np.random.default_rng(idx_bytes * 10 + packed + len(layout))
    D, B, rows = 16, 64, [3000, 500]
    inter = layout == "interleaved"
    ld = D + 4 if inter else D
    head_col = D + 1 if inter else -1
    W = [torch.randn(R, ld) for R in rows]
    if inter:
        for w in W:
            w[:, D + 1:].zero_()       # list head and pad: zero between steps
    M = [torch.rand(R) for R in rows] if layout == "separate" else None
    A = [torch.rand(R, D) for R in rows] if layout == "separate_adagrad" else None
    pins = [Pinned(t) for t in W + (M or []) + (A or [])]
    try:
        idx, off, cap, raw = _batch(rng, rows, B, idx_bytes, packed)
        maps = [torch.zeros(R, dtype=torch.int32, device=DEV) for R in rows]
        sw = torch.full((cap, ld), -7.0, device=DEV)
        smom = torch.zeros(cap, device=DEV) if M else None
        shead = torch.full((cap,), 5, dtype=torch.int32, device=DEV) if not inter else None
        sacc = torch.zeros(cap, D, device=DEV) if A else None
        sidx = torch.zeros(cap, dtype=torch.int64 if idx_bytes == 8 else torch.int32, device=DEV)
        lst = torch.zeros(cap, dtype=torch.int32, device=DEV)
        key = torch.zeros(cap, dtype=torch.int64, device=DEV)
        cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
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
        st = _lib.HostStage(weight=sw.data_ptr(), momentum=smom.data_ptr() if M else None,
                            head=shead.data_ptr() if shead is not None else None,
                            acc_ew=sacc.data_ptr() if A else None, slot_idx=sidx.data_ptr(), list=lst.data_ptr(),
                            key=key.data_ptr(), count=cnt.data_ptr(), capacity=cap, ld=ld, head_col=head_col)
        assert L().dlrm_b200_host_stage_in(arr, 2, C.byref(st), D, B, idx_bytes, int(packed), _st()) == 0, \
            L().dlrm_b200_last_error()
        torch.cuda.synchronize()
        assert L().dlrm_b200_check_device_errors(_st()) == 0
        slots = sidx.cpu().numpy().astype(np.int64)
        staged = sw.cpu()
        distinct = 0
        seen = {}
        base = 0
        for k in range(2):
            for j, r in enumerate(raw[k]):
                p = base + j
                s = int(slots[p])
                want = W[k][r].clone()
                if inter:
                    want[head_col] = 0
                assert torch.equal(staged[s], want), (k, j)
                if M:
                    assert smom[s].item() == M[k][r].item()
                if A:
                    assert torch.equal(sacc[s].cpu(), A[k][r])
                if shead is not None:
                    assert shead[s].item() == 0
                assert seen.setdefault((k, int(r)), s) == s          # one slot per row
            distinct += len(set(raw[k].tolist()))
            base += raw[k].size
        assert len(set(seen.values())) == len(seen) == distinct == int(cnt.item())
        # write back modified staged rows: those host rows take them, every other host row is unchanged
        before = [w.clone() for w in W]
        mb = [m.clone() for m in M] if M else None
        ab = [a.clone() for a in A] if A else None
        listed = lst[:distinct].long()
        sw[listed] += 1.5
        if inter:
            sw[listed, head_col] = 3.0                               # a list head left set is written back as zero
        if M:
            smom[listed] += 2.0
        if A:
            sacc[listed] *= 2.0
        assert L().dlrm_b200_host_write_back(arr, 2, C.byref(st), D, _st()) == 0
        torch.cuda.synchronize()
        staged = sw.cpu()
        for k in range(2):
            touched = np.zeros(rows[k], bool)
            touched[raw[k]] = True
            assert torch.equal(W[k][~torch.from_numpy(touched)], before[k][~torch.from_numpy(touched)])
            if M:
                assert torch.equal(M[k][~torch.from_numpy(touched)], mb[k][~torch.from_numpy(touched)])
            if A:
                assert torch.equal(A[k][~torch.from_numpy(touched)], ab[k][~torch.from_numpy(touched)])
            for r in set(raw[k].tolist()):
                s = seen[(k, r)]
                want = staged[s].clone()
                if inter:
                    want[head_col] = 0
                assert torch.equal(W[k][r], want)
                if M:
                    assert M[k][r].item() == smom[s].item()
                if A:
                    assert torch.equal(A[k][r], sacc[s].cpu())
            assert int(maps[k].abs().sum().item()) == 0, "slot map not empty after the write-back"
        # release: the map empties, nothing is written
        after = [w.clone() for w in W]
        assert L().dlrm_b200_host_stage_in(arr, 2, C.byref(st), D, B, idx_bytes, int(packed), _st()) == 0
        sw.fill_(9.0)
        assert L().dlrm_b200_host_release(arr, 2, C.byref(st), D, _st()) == 0
        torch.cuda.synchronize()
        assert all(torch.equal(a, w) for a, w in zip(after, W))
        assert all(int(m.abs().sum().item()) == 0 for m in maps)
        # an index outside its table: reported like the gather's, no host access, slot -1
        bad = idx[0].clone()
        pos = int(off[0][0].item())
        if bad.numel() > pos:
            bad[pos] = rows[0]
            arr[0].indices = bad.data_ptr()
            if packed:
                arr[1].indices = bad.data_ptr()
            assert L().dlrm_b200_host_stage_in(arr, 2, C.byref(st), D, B, idx_bytes, int(packed), _st()) == 0
            torch.cuda.synchronize()
            assert int(sidx[pos].item()) == -1
            assert L().dlrm_b200_check_device_errors(_st()) != 0
            assert L().dlrm_b200_host_release(arr, 2, C.byref(st), D, _st()) == 0
            torch.cuda.synchronize()
            assert all(int(m.abs().sum().item()) == 0 for m in maps)
            assert L().dlrm_b200_check_device_errors(_st()) == 0
    finally:
        torch.cuda.synchronize()
        for p in pins:
            p.close()


# ---------------------------------------------------------------------------------------------------------- engines
LN = [3000, 200, 5000, 40, 2500]


def _engine(host, gemm, interleave=None, D=32):
    from dlrm_b200.engine import Engine

    F = len(LN) + 1
    top = [D + F * (F - 1) // 2, 64, 1]
    e = Engine(D, LN, [13, 64, D], top, sigmoid_top=len(top) - 2, device=DEV, max_batch=256, gemm=gemm,
               interleave_momentum=interleave, host_tables=host)
    e.init_params(seed=3)
    return e


def _batches(n, B=256, seed=0):
    from dlrm_b200.data import make_batch, to_device_packed

    rng = np.random.default_rng(seed)
    return [to_device_packed(make_batch(rng, LN, B, lmax=6), DEV) for _ in range(n)]


def _state(e, opt):
    out = [e.table(k).clone() for k in range(len(LN))]
    if opt == "rwsadagrad":
        out += [e.momentum_of(k).clone() for k in range(len(LN))]
    if opt == "adagrad":
        out += [e.accumulator_ew(k).clone() for k in range(len(LN))]
    return out + [e.dense.clone()]


@pytest.mark.parametrize("opt", ["sgd", "rwsadagrad", "adagrad"])
@pytest.mark.parametrize("gemm", ["simt", "tc"])
@pytest.mark.parametrize("host", [[0, 2], [0, 2, 4]])
@pytest.mark.parametrize("mode", ["eager", "graphed"])
def test_engine_steps_are_bit_identical_to_device_tables(opt, gemm, host, mode):
    from dlrm_b200.engine import GraphedTrainStep

    bs = _batches(7)
    res = []
    for h in ([], host):
        e = _engine(h, gemm)
        losses = []
        if mode == "eager":
            for b in bs[:5]:
                losses.append(e.train_step(b.X, b.sparse, b.target, 0.05, opt).clone())
        else:
            st = bs[6]                                   # the static batch buffer of the graph
            st.buf.copy_(bs[0].buf)
            g = GraphedTrainStep(e, st, 0.05, opt, warmup=0)
            for b in bs[:5]:
                st.buf.copy_(b.buf)
                g.replay()
                losses.append(e.loss_buf.clone())
        p = e.forward(bs[5].X, bs[5].sparse).clone()
        torch.cuda.synchronize()
        res.append((torch.stack(losses), p, _state(e, opt)))
        assert L().dlrm_b200_check_device_errors(_st()) == 0
        if h:
            assert int(e.slot_map.abs().sum().item()) == 0
    (l0, p0, s0), (l1, p1, s1) = res
    assert torch.equal(l0, l1)
    assert torch.equal(p0, p1)
    for a, b in zip(s0, s1):
        assert torch.equal(a.cpu(), b.cpu())


def test_separate_layout_and_forward_only_passes():
    """interleave=False (DLRM_Net's fp32 layout), with forward-only passes between the steps."""
    bs = _batches(4, seed=1)
    res = []
    for h in ([], [0, 2, 4]):
        e = _engine(h, "simt", interleave=False)
        out = []
        for b in bs[:3]:
            out.append(e.forward(bs[3].X, bs[3].sparse).clone())
            out.append(e.train_step(b.X, b.sparse, b.target, 0.05, "rwsadagrad").clone())
        torch.cuda.synchronize()
        res.append((out, _state(e, "rwsadagrad")))
    for a, b in zip(res[0][0] + res[0][1], res[1][0] + res[1][1]):
        assert torch.equal(a.cpu(), b.cpu())


def test_refusals():
    from dlrm_b200.engine import Engine

    kw = dict(device=DEV, max_batch=64)
    with pytest.raises(ValueError, match="fp32"):
        Engine(16, [1000, 1000], [13, 16], [16 + 3, 1], emb_dtype="fp16", host_tables=[0], **kw)
    with pytest.raises(ValueError, match="tiny"):
        Engine(16, [1000, 100], [13, 16], [16 + 3, 1], host_tables=[1], **kw)
    e = Engine(16, [1000, 1000], [13, 16], [16 + 3, 1], host_tables=[0], **kw)
    e.use_filter = True
    from dlrm_b200.engine import sparse_from_reference

    sp = sparse_from_reference([torch.zeros(4, dtype=torch.int64)] * 2, [torch.arange(4)] * 2, DEV)
    with pytest.raises(ValueError, match="duplicate filter"):
        e.emb_forward(sp, out=torch.zeros(4, 2, 16, device=DEV), stride_sample=32, stride_table=16)
    e.use_filter = False
    assert int(e.slot_map.abs().sum().item()) == 0
    with pytest.raises(ValueError, match="weighted pooling"):
        e.load_params(dict(emb=[np.zeros((1000, 16), np.float32)] * 2, bot=[(np.zeros((16, 13), np.float32),
                           np.zeros(16, np.float32))], top=[(np.zeros((1, 19), np.float32), np.zeros(1, np.float32))],
                           v_W_l=[np.ones(1000, np.float32)] * 2))


def test_bad_index_is_reported_and_the_next_step_is_clean():
    """An index outside a host table raises the device error as on a device table; no slot stays claimed, and the
    engine's next step reports nothing."""
    bs = _batches(2, seed=2)
    bad = bs[0]
    bad.indices[int(bad.offsets[0][0].item())] = LN[0] + 5
    for h in ([], [0, 2, 4]):
        e = _engine(h, "tc")
        e.train_step(bad.X, bad.sparse, bad.target, 0.05, "sgd")
        torch.cuda.synchronize()
        assert L().dlrm_b200_check_device_errors(_st()) != 0
        if h:
            assert int(e.slot_map.abs().sum().item()) == 0
        e.train_step(bs[1].X, bs[1].sparse, bs[1].target, 0.05, "sgd")
        torch.cuda.synchronize()
        assert L().dlrm_b200_check_device_errors(_st()) == 0


def test_memory_bound_of_a_multi_gb_host_table():
    from dlrm_b200.engine import Engine

    torch.cuda.synchronize()
    rows = 8_000_000                                   # 8e6 x 132 floats: 4.2 GB of pinned rows
    before = torch.cuda.memory_allocated()
    e = Engine(128, [rows, 1000], [13, 128], [128 + 3, 1], device=DEV, max_batch=2048, host_tables=[0])
    e.init_params(seed=0)
    from dlrm_b200.data import make_batch, to_device_packed

    b = to_device_packed(make_batch(np.random.default_rng(0), [rows, 1000], 2048, lmax=1, fixed=True), DEV)
    e.prepare(b.sparse, True)
    torch.cuda.synchronize()
    grew = torch.cuda.memory_allocated() - before
    table_bytes = rows * 132 * 4
    stage = e.stage_cap * (132 * 4 + 8 + 8 + 4)
    assert e.pinned_bytes >= table_bytes
    assert grew < 4 * rows + stage + (64 << 20), (grew, table_bytes)
    del e
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- module / CLI
_CLI_BASE = ["--arch-sparse-feature-size=16", "--arch-embedding-size=1000-1000-1000", "--arch-mlp-bot=13-512-256-64-16",
             "--arch-mlp-top=512-256-1", "--mini-batch-size=128", "--data-generation=random", "--num-batches=6",
             "--print-freq=1", "--learning-rate=0.1", "--numpy-rand-seed=727", "--use-gpu"]
_LOSS = re.compile(r"Finished training it .* loss ([0-9.]+)")


def _run(args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py")] + args, capture_output=True,
                       text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def _losses(text):
    return [float(m.group(1)) for m in _LOSS.finditer(text)]


@pytest.mark.parametrize("tag", ["A", "B", "C", "D"])
def test_cli_cfg0_runs_with_host_tables(tag):
    flags = open(os.path.join(GOLD, "cli_cfg0_%s.flags" % tag)).read().split()
    want = open(os.path.join(GOLD, "cli_cfg0_%s.txt" % tag)).read()
    got = _run(_CLI_BASE + flags + ["--gemm=simt", "--emb-host-tables=0-1-2"])
    want_l = [float(m.group(1)) for m in re.finditer(r"Finished training it .* loss ([0-9.]+)", want)]
    assert len(_losses(got)) == len(want_l) > 0
    np.testing.assert_allclose(_losses(got), want_l, rtol=0, atol=2e-5)
    test = re.compile(r"Testing at - .*")
    assert test.findall(got) == test.findall(want)


def test_cli_bin_and_kaggle_runs_with_host_tables():
    other = re.compile(r"Sparse fea|Randomized|Defined|Split data|Testing at|accuracy|^recall ")
    flags = open(os.path.join(GOLD, "cli_bin_A.flags")).read().split() + [
        "--raw-data-file=" + os.path.join(GOLD, "bin_day"),
        "--processed-data-file=" + os.path.join(GOLD, "bin_processed.npz"), "--use-gpu", "--gemm=simt"]
    counts = np.minimum(np.load(os.path.join(GOLD, "bin_day_fea_count.npz"))["counts"], 1000)
    lst = "-".join(str(k) for k in np.flatnonzero(counts > 256))
    dev, host = _run(flags), _run(flags + ["--emb-host-tables=" + lst])
    want = open(os.path.join(GOLD, "cli_bin_A.txt")).read()
    np.testing.assert_allclose(_losses(host), [float(v) for v in re.findall(r"loss ([0-9.]+)", want)], rtol=0, atol=2e-5)
    assert _losses(host) == _losses(dev)
    assert [ln for ln in host.splitlines() if other.search(ln)] == [ln for ln in dev.splitlines() if other.search(ln)]
    flags = open(os.path.join(GOLD, "cli_kaggle_A.flags")).read().split() + [
        "--raw-data-file=" + os.path.join(GOLD, "kaggle.txt"),
        "--processed-data-file=" + os.path.join(GOLD, "kaggle_processed.npz"), "--use-gpu", "--gemm=simt"]
    counts = np.load(os.path.join(GOLD, "kaggle_processed.npz"))["counts"]
    lst = "-".join(str(k) for k in np.flatnonzero(counts > 256))
    got = _run(flags + ["--emb-host-tables=" + lst]).splitlines()
    want = open(os.path.join(GOLD, "cli_kaggle_A.txt")).read().splitlines()
    wl = [float(_LOSS.match(ln).group(1)) for ln in want if _LOSS.match(ln)]
    gl = [float(_LOSS.match(ln).group(1)) for ln in got if _LOSS.match(ln)]
    assert len(gl) == len(wl) > 0
    np.testing.assert_allclose(gl, wl, rtol=0, atol=1e-5)
    assert [ln for ln in got if other.search(ln)] == [ln for ln in want if other.search(ln)]


def test_checkpoints_move_between_host_and_device_runs(tmp_path):
    from dlrm_b200 import cli

    args = [a for a in _CLI_BASE if not a.startswith("--num-batches")] + ["--optimizer=rwsadagrad", "--gemm=simt"]
    nets = {}
    for name, extra in (("dev", []), ("host", ["--emb-host-tables=0-2"])):
        ck = str(tmp_path / (name + ".pt"))
        cli.run(args + extra + ["--num-batches=3", "--save-model=" + ck])
        nets[name] = ck
    # the same three steps either way
    a = torch.load(nets["dev"], map_location="cpu", weights_only=False)
    b = torch.load(nets["host"], map_location="cpu", weights_only=False)
    for k in a["state_dict"]:
        assert torch.equal(a["state_dict"][k].cpu(), b["state_dict"][k].cpu()), k
    # cross-load and continue: a host run from the device checkpoint equals a device run from the host one
    out = []
    for ck, extra in ((nets["dev"], ["--emb-host-tables=0-1-2"]), (nets["host"], [])):
        net = cli.run(args + extra + ["--num-batches=5", "--load-model=" + ck])
        out.append({k: v.detach().cpu().clone() for k, v in net.state_dict().items()})
    for k in out[0]:
        assert torch.equal(out[0][k], out[1][k]), k
    # test pass and --inference-only with host tables
    txt = _run(args + ["--num-batches=3", "--test-freq=3", "--emb-host-tables=0-2"])
    assert "Testing at" in txt
    txt = _run(args + ["--num-batches=3", "--inference-only", "--load-model=" + nets["host"], "--emb-host-tables=0-2"])
    assert "Testing at" in txt or "Saved at" in txt
