"""Row-wise 8- / 4-bit quantized embedding tables on the GPU: the quantize kernel against torch's CPU prepack, the
quantized gather against torch's CPU embedding_bag_{byte,4bit}_rowwise_offsets (bit for bit), DLRM_Net's
quantize_embedding and emb_dtype="int8" / "int4" models, checkpoint loads, graph replays, the training refusals and
the command line's inference-only runs."""
import os
import re
import types

import numpy as np
import pytest
import torch

from dlrm_b200 import _lib
from dlrm_b200 import engine as E

import test_gpu_criteo_dataset as kaggle_cli

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OPS = torch.ops.quantized
PREPACK = {8: OPS.embedding_bag_byte_prepack, 4: OPS.embedding_bag_4bit_prepack}
POOL = {8: OPS.embedding_bag_byte_rowwise_offsets, 4: OPS.embedding_bag_4bit_rowwise_offsets}
QDT = {8: _lib.DTYPE_Q8, 4: _lib.DTYPE_Q4}


def L():
    return _lib.lib()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _bits_equal(a, b):
    a = a.detach().cpu().contiguous().numpy().view(np.uint32)
    b = b.detach().cpu().contiguous().numpy().view(np.uint32)
    return a.shape == b.shape and bool(np.all(a == b))


def _float_rows(rng, n, d, extreme=False):
    """Random rows with constant rows and large ranges.  extreme: ranges that overflow the 4-bit format's fp16 scale
    and bias (compared as bytes only: pooling such rows gives NaN, whose bits are not portable)."""
    w = (rng.standard_normal((n, d)) * 0.05).astype(np.float32)
    w[0], w[1] = 0.25, 0.0                       # constant rows
    w[2] *= 1e30 if extreme else 1e4
    w[3] = np.linspace(-1e6, 1e6, d) if extreme else np.linspace(-6e4, 6e4, d)
    return torch.from_numpy(w)


# ------------------------------------------------------------------------------------------ quantize kernel
@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("d", [8, 64, 128, 256])
@pytest.mark.parametrize("src_dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("pad", [0, 4])
def test_quantize_kernel_is_byte_identical_to_torch_prepack(bits, d, src_dtype, pad):
    """pad > 0: the source rows are interleaved with other words (row stride d + pad), like the engine's rows."""
    w = _float_rows(np.random.default_rng(d + pad), 777, d, extreme=src_dtype == torch.float32).to(src_dtype)
    arena = torch.full((777, d + pad), 7.0, dtype=src_dtype, device=DEV)
    arena[:, :d].copy_(w)
    src = arena[:, :d]
    width = E.quant_row_bytes(d, bits)
    out = torch.full((777, width), 0xAB, dtype=torch.uint8, device=DEV)
    _lib.check(L().dlrm_b200_emb_quantize_rows(src.data_ptr(), _lib.DTYPE_F16 if src_dtype == torch.float16 else
                                               _lib.DTYPE_F32, src.stride(0), 777, d, out.data_ptr(), QDT[bits], 0,
                                               _st()), "quantize")
    want = PREPACK[bits](w.float())
    assert torch.equal(out.cpu(), want)


def test_quantize_kernel_refuses_bad_shapes():
    lib = L()
    assert lib.dlrm_b200_emb_quantize_rows(1, 0, 0, 1, 6, 16, _lib.DTYPE_Q8, 0, None) != 0
    assert b"dim" in lib.dlrm_b200_last_error()
    assert lib.dlrm_b200_emb_quantize_rows(1, 0, 0, 1, 12, 16, _lib.DTYPE_Q4, 0, None) != 0
    assert lib.dlrm_b200_emb_quantize_rows(1, 0, 0, 1, 16, 16, _lib.DTYPE_F16, 0, None) != 0


def _engine(ln, d=16, emb_dtype="int8", gemm="simt"):
    F = len(ln) + 1
    top = [d + F * (F - 1) // 2, 32, 1]
    return E.Engine(d, ln, [13, 32, d], top, sigmoid_top=len(top) - 2, device=DEV, max_batch=256, gemm=gemm,
                    emb_dtype=emb_dtype)


@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("src", ["cpu32", "cpu16", "dev32"])
def test_engine_quantizes_tables_larger_than_a_chunk(monkeypatch, bits, src):
    monkeypatch.setattr(E, "QUANT_CHUNK_ROWS", 1000)
    e = _engine([2500, 300], d=64, emb_dtype="int%d" % bits)
    w = _float_rows(np.random.default_rng(5), 2500, 64, extreme=src != "cpu16")
    w = w.half() if src == "cpu16" else w
    e.quantize_rows(0, w.to(DEV) if src == "dev32" else w)
    assert torch.equal(e.table_q(0).cpu(), PREPACK[bits](w.float()))
    # a row range of the second table
    w1 = _float_rows(np.random.default_rng(6), 100, 64)
    e.quantize_rows(1, w1, r0=150)
    assert torch.equal(e.table_q(1)[150:250].cpu(), PREPACK[bits](w1))
    assert int(e.table_q(1)[:150].abs().sum()) == 0
    with pytest.raises(ValueError):
        e.quantize_rows(1, w1, r0=250)


# ------------------------------------------------------------------------------------------ quantized gather
def _gather(packed, bits, d, idx, off, rw=None, include_last=False, idx_dtype=torch.int64):
    """One dlrm_b200_emb_bag_fwd launch over every table: out [B, T, d]."""
    T = len(packed)
    B = off[0].numel() - (1 if include_last else 0)
    dp = [p.to(DEV) for p in packed]
    di = [i.to(DEV, idx_dtype) for i in idx]
    do = [o.to(DEV, idx_dtype) for o in off]
    dw = None if rw is None else [r.to(DEV) for r in rw]
    arr = (_lib.EmbFwdTable * T)()
    for k in range(T):
        a = arr[k]
        a.weight, a.ld, a.weight_dtype = dp[k].data_ptr(), dp[k].stride(0), QDT[bits]
        a.indices = di[k].data_ptr() if di[k].numel() else 0
        a.offsets, a.nnz, a.rows = do[k].data_ptr(), di[k].numel(), dp[k].shape[0]
        a.row_weights = dw[k].data_ptr() if dw is not None else None
    out = torch.full((B, T, d), float("nan"), dtype=torch.float32, device=DEV)
    _lib.check(L().dlrm_b200_emb_bag_fwd(arr, T, d, B, 8 if idx_dtype == torch.int64 else 4, int(include_last),
                                         out.data_ptr(), T * d, d, _st()), "emb_bag_fwd")
    torch.cuda.synchronize()
    return out


def _case(rng, rows, d, bits, B):
    w = _float_rows(rng, rows, d) if rows > 8 else torch.from_numpy(rng.standard_normal((rows, d)).astype(np.float32))
    packed = PREPACK[bits](w)
    sizes = rng.integers(0, 4, B)
    sizes[:6] = [0, 1, 200, 0, 37, 2]                   # empty bags, bags of 1 to 200 rows
    off = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    idx = rng.integers(0, rows, int(sizes.sum())).astype(np.int64)
    return packed, torch.from_numpy(idx), torch.from_numpy(off)


@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("d", [8, 16, 32, 64, 128, 256, 1024])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("idx_dtype", [torch.int64, torch.int32])
def test_gather_is_bit_identical_to_torch(bits, d, weighted, idx_dtype):
    """Three tables in one launch (one tiny); reference-format and include-last offsets.  d = 1024 (> 512) takes the
    one-thread-per-element kernel, the others the lane-group kernel."""
    rng = np.random.default_rng(bits * 100 + d)
    B = 300
    cases = [_case(rng, n, d, bits, B) for n in (5000, 3, 1200)]
    packed, idx, off = [c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases]
    rw = [torch.from_numpy(rng.random(p.shape[0]).astype(np.float32) * 3 - 1) for p in packed] if weighted else None
    want = torch.stack([POOL[bits](packed[k], idx[k], off[k], per_sample_weights=None if rw is None else rw[k][idx[k]])
                        for k in range(3)], dim=1)
    got = _gather(packed, bits, d, idx, off, rw, idx_dtype=idx_dtype)
    assert _bits_equal(got, want)
    off_l = [torch.cat([o, torch.tensor([i.numel()])]) for o, i in zip(off, idx)]
    got_l = _gather(packed, bits, d, idx, off_l, rw, include_last=True, idx_dtype=idx_dtype)
    assert _bits_equal(got_l, want)
    assert L().dlrm_b200_check_device_errors(_st()) == 0


@pytest.mark.parametrize("bits", [8, 4])
def test_gather_bad_index_sets_the_error_word_and_other_bags_match(bits):
    rng = np.random.default_rng(9)
    packed, idx, off = _case(rng, 1000, 64, bits, 100)
    ends = torch.cat([off[1:], torch.tensor([idx.numel()])])
    hit = next(b for b in range(10, 100) if int(ends[b]) > int(off[b]))     # a non-empty bag
    idx_bad = idx.clone()
    idx_bad[int(off[hit])] = 1000 + 5
    got = _gather([packed], bits, 64, [idx_bad], [off])
    assert L().dlrm_b200_check_device_errors(_st()) & 1
    want = POOL[bits](packed, idx, off)
    keep = [b for b in range(100) if b != hit]
    assert _bits_equal(got[keep, 0], want[keep])
    assert L().dlrm_b200_check_device_errors(_st()) == 0


def test_gather_refuses_training_and_row_ranges():
    packed, idx, off = _case(np.random.default_rng(1), 100, 16, 8, 10)
    p, i, o = packed.to(DEV), idx.to(DEV), off.to(DEV)
    arr = (_lib.EmbFwdTable * 1)()
    arr[0].weight, arr[0].weight_dtype, arr[0].indices, arr[0].offsets = p.data_ptr(), _lib.DTYPE_Q8, i.data_ptr(), \
        o.data_ptr()
    arr[0].nnz, arr[0].rows, arr[0].row_lo, arr[0].row_n = i.numel(), 100, 10, 50
    out = torch.zeros((10, 1, 16), device=DEV)
    assert L().dlrm_b200_emb_bag_fwd(arr, 1, 16, 10, 8, 0, out.data_ptr(), 16, 16, _st()) != 0
    assert b"whole tables" in L().dlrm_b200_last_error()
    arr[0].row_lo = arr[0].row_n = 0
    bw = (_lib.EmbBwdTable * 1)()
    link = torch.zeros(2 * i.numel() + 2, dtype=torch.int32, device=DEV)
    assert L().dlrm_b200_emb_bag_fwd_train(arr, bw, 1, 16, 10, 8, 0, link.data_ptr(), out.data_ptr(), 16, 16, None,
                                           _st()) != 0
    assert b"forward-only" in L().dlrm_b200_last_error()


# ------------------------------------------------------------------------------------------ DLRM_Net
LN = [3000, 200, 4000, 17]
D = 16


def _net(emb_dtype=torch.float32, seed=11, ln=LN, d=D, weighted=None):
    from dlrm_b200.dlrm_net import DLRM_Net

    np.random.seed(seed)
    F = len(ln) + 1
    top = [d + F * (F - 1) // 2, 32, 1]
    return DLRM_Net(d, ln, [13, 32, d], top, arch_interaction_op="dot", sigmoid_top=len(top) - 2,
                    device=DEV, max_batch=256, gemm="simt", emb_dtype=emb_dtype, weighted_pooling=weighted)


def _batch(rng, ln, B=256, L=3):
    X = torch.from_numpy(rng.random((B, 13)).astype(np.float32)).to(DEV)
    lS_o = torch.arange(0, B * L, L).repeat(len(ln), 1).to(DEV)
    lS_i = [torch.from_numpy(rng.integers(0, n, B * L)).to(DEV) for n in ln]
    return X, lS_o, lS_i


@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("weighted", [None, "fixed", "learned"])
def test_quantize_embedding_pools_the_packed_rows(bits, weighted):
    net = _net(weighted=weighted)
    sd = {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}
    net.quantize_embedding(bits)
    assert net.quantize_emb and net.quantize_bits == bits and len(net.emb_l_q) == len(LN)
    for k in range(len(LN)):
        assert torch.equal(net.emb_l_q[k].cpu(), PREPACK[bits](net.emb_l[k].weight.detach().cpu()))
    assert sd.keys() == net.state_dict().keys()                     # the float tables stay
    rng = np.random.default_rng(2)
    X, lS_o, lS_i = _batch(rng, LN)
    ly = net.apply_emb(lS_o, lS_i)
    for k in range(len(LN)):
        psw = None if weighted is None else torch.ones(lS_i[k].numel())
        want = POOL[bits](net.emb_l_q[k].cpu(), lS_i[k].cpu(), lS_o[k].cpu(), per_sample_weights=psw)
        assert _bits_equal(ly[k], want)
    with torch.no_grad():
        p = net(X, lS_o, lS_i)
    assert torch.isfinite(p).all()
    with pytest.raises(SystemExit):
        net.quantize_embedding(2)


@pytest.mark.parametrize("bits", [8, 4])
def test_quantize_embedding_of_fp16_tables_reads_the_interleaved_rows(bits):
    net = _net(emb_dtype=torch.float16)
    assert net._engine.interleave and net.emb_l[0].weight.stride(0) > D
    net.quantize_embedding(bits)
    rng = np.random.default_rng(3)
    X, lS_o, lS_i = _batch(rng, LN)
    ly = net.apply_emb(lS_o, lS_i)
    for k in range(len(LN)):
        packed = PREPACK[bits](net.emb_l[k].weight.detach().float().cpu())
        assert torch.equal(net.emb_l_q[k].cpu(), packed)
        assert _bits_equal(ly[k], POOL[bits](packed, lS_i[k].cpu(), lS_o[k].cpu()))


@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("ln", [LN, [400_000, 300]])        # numpy draw, and the device draw above 50 M elements
def test_int_model_has_the_rows_of_float_model_plus_quantize_embedding(bits, ln):
    d = 128 if ln[0] > 10_000 else D
    f = _net(ln=ln, d=d)
    assert f.emb_l[0].weight.stride() == (d, 1)          # the fp32 tables the int model's draw reproduces are dense
    f.quantize_embedding(bits)
    q = _net(emb_dtype="int%d" % bits, ln=ln, d=d)
    assert q.quantize_emb and q.quantize_bits == bits and len(q.emb_l) == 0
    for k in range(len(ln)):
        assert torch.equal(q.emb_l_q[k], f.emb_l_q[k])
    for a, b in zip(q.bot_l.parameters(), f.bot_l.parameters()):
        assert torch.equal(a, b)
    rng = np.random.default_rng(4)
    X, lS_o, lS_i = _batch(rng, ln)
    with torch.no_grad():
        assert torch.equal(q(X, lS_o, lS_i), f(X, lS_o, lS_i))
    with pytest.raises(RuntimeError, match="never"):
        q.state_dict()


@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("ck_dtype", [torch.float32, torch.float16])
def test_checkpoint_loads_quantized_within_one_chunk_of_memory(tmp_path, bits, ck_dtype):
    ln, d = [2_500_000, 1000], 128
    src = _net(ln=[10, 10], d=d)      # only the MLP keys are taken from it
    mlp = {k: v.detach().cpu() for k, v in src.state_dict().items() if not k.startswith("emb_l")}
    g = torch.Generator().manual_seed(3)
    tabs = [(torch.rand((n, d), generator=g) * 0.2 - 0.1).to(ck_dtype) for n in ln]
    sd = dict(mlp, **{"emb_l.%d.weight" % k: t for k, t in enumerate(tabs)})
    path = str(tmp_path / "ck.pt")
    torch.save({"state_dict": sd}, path)
    del sd, tabs
    ld = torch.load(path, map_location="cpu", mmap=True, weights_only=False)["state_dict"]
    q = _net(emb_dtype="int%d" % bits, ln=ln, d=d)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    q.load_state_dict(ld)
    torch.cuda.synchronize()
    chunk = E.QUANT_CHUNK_ROWS * d * 4
    slack = 16 << 20
    assert torch.cuda.max_memory_allocated() - base <= chunk + slack
    for k in range(len(ln)):
        want = PREPACK[bits](ld["emb_l.%d.weight" % k].float())
        assert torch.equal(q.emb_l_q[k].cpu(), want)
    for a, b in zip(q.top_l.parameters(), src.top_l.parameters()):
        assert torch.equal(a, b)


@pytest.mark.parametrize("bits", [8, 4])
def test_forward_graph_replay_equals_the_eager_forward(bits):
    from dlrm_b200.engine import GraphedTrainStep, sparse_from_reference

    q = _net(emb_dtype="int%d" % bits)
    eng = q._engine
    rng = np.random.default_rng(8)
    X, lS_o, lS_i = _batch(rng, LN)
    sp = sparse_from_reference(lS_o, lS_i, DEV)
    eager = eng.forward(X, sp).clone()
    stage = types.SimpleNamespace(X=X.clone(), sparse=sp, target=None)
    g = GraphedTrainStep(eng, stage, 0.0, "sgd", warmup=1, train=False)
    X2, lS_o2, lS_i2 = _batch(np.random.default_rng(8), LN)
    stage.X.copy_(X2)
    out = g.replay().clone()
    assert torch.equal(out, eager)


def test_training_is_refused_on_quantized_tables():
    from dlrm_b200 import optim as fused
    from dlrm_b200.engine import sparse_from_reference

    for net in (_net(emb_dtype="int8"), _net()):
        if not net._engine.quant_only:
            net.quantize_embedding(4)
        rng = np.random.default_rng(1)
        X, lS_o, lS_i = _batch(rng, LN)
        T = torch.ones((256, 1), device=DEV)
        p = net(X, lS_o, lS_i)
        with pytest.raises(RuntimeError, match="inference-only"):
            net.loss_fn(p, T).backward()
        for opt in (fused.SGD, fused.RWSAdagrad, fused.Adagrad):
            with pytest.raises(RuntimeError, match="inference-only"):
                opt(net.parameters(), lr=0.1)
        sp = sparse_from_reference(lS_o, lS_i, DEV)
        with pytest.raises(RuntimeError, match="inference-only"):
            net._engine.train_step(X, sp, T, 0.1, "sgd")


# ------------------------------------------------------------------------------------------ command line
@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("graphed", [False, True])
def test_cli_kaggle_mlperf_metrics_match_the_reference_quantized_run(bits, graphed):
    """The reference's quantized test pass with --mlperf-logging on the Kaggle fixture, from its own checkpoint: the
    float, 8-bit and 4-bit runs print different metrics, and the recorded line is reproduced (eagerly and in graph
    replays)."""
    extra = ["--gemm=simt", "--load-model=" + os.path.join(kaggle_cli.GOLD, "cli_kaggle_Q_ref.pt")]
    got = kaggle_cli._cli("Q%d" % bits, extra + (["--cuda-graph-steps"] if graphed else []))
    keep = re.compile(r"Testing state|^recall ")
    want = open(os.path.join(kaggle_cli.GOLD, "cli_kaggle_Q%d.txt" % bits)).read().splitlines()
    assert [ln for ln in got.splitlines() if keep.search(ln)] == want
    assert "quantized emb sizes" not in got
    if graphed:
        assert "test batches replayed" in got


# ------------------------------------------------------------------------------------------ reference goldens
def _golden_net(z, bits, weighted, emb_dtype=torch.float32):
    """DLRM_Net holding the recorded model (reference state_dict keys); quantized as the reference was."""
    from dlrm_b200.dlrm_net import DLRM_Net

    ln_emb, ln_bot, ln_top = (z[k].tolist() for k in ("ln_emb", "ln_bot", "ln_top"))
    net = DLRM_Net(int(z["m_spa"]), ln_emb, ln_bot, ln_top, arch_interaction_op="dot", sigmoid_top=len(ln_top) - 2,
                   device=DEV, max_batch=int(z["B"]), emb_dtype=emb_dtype,
                   weighted_pooling="fixed" if weighted else None)
    sd = {"emb_l.%d.weight" % k: torch.from_numpy(z["emb%d" % k]) for k in range(len(ln_emb))}
    for nm in ("bot", "top"):
        for i in range(len(z["ln_" + nm]) - 1):
            sd["%s_l.%d.weight" % (nm, 2 * i)] = torch.from_numpy(z["%sW%d" % (nm, i)])
            sd["%s_l.%d.bias" % (nm, 2 * i)] = torch.from_numpy(z["%sb%d" % (nm, i)])
    net.load_state_dict(sd)
    if weighted:
        for k in range(len(ln_emb)):
            net.v_W_l[k].copy_(torch.from_numpy(z["vW%d" % k]))
    if emb_dtype == torch.float32:
        net.quantize_embedding(bits)
    return net


@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("path", ["quantize_embedding", "emb_dtype"])
def test_reference_goldens(bits, weighted, path):
    """emb_l_q equals the reference's packed tables byte for byte; the logits are within 1e-5 of the reference's
    (the bf16x3 MLP bound; the pooled rows themselves are bit-identical)."""
    z = dict(np.load(os.path.join(kaggle_cli.GOLD, "cfg0_quant.npz")))
    net = _golden_net(z, bits, weighted, torch.float32 if path == "quantize_embedding" else "int%d" % bits)
    for k in range(len(z["ln_emb"])):
        assert np.array_equal(net.emb_l_q[k].cpu().numpy(), z["q%d_emb%d" % (bits, k)])
    for s in range(int(z["nbatch"])):
        X = torch.from_numpy(z["b%d_X" % s])
        lS_o = torch.from_numpy(z["b%d_off" % s])
        lS_i = [torch.from_numpy(z["b%d_idx%d" % (s, k)]) for k in range(len(z["ln_emb"]))]
        with torch.no_grad():
            p = net(X, lS_o, lS_i).cpu().numpy()
        want = z["q%d_%sp%d" % (bits, "w_" if weighted else "", s)]
        assert np.abs(p - want).max() <= 1e-5


_CLI_BASE = ["--arch-sparse-feature-size=16", "--arch-embedding-size=1000-1000-1000", "--arch-mlp-bot=13-512-256-64-16",
             "--arch-mlp-top=512-256-1", "--mini-batch-size=128", "--data-generation=random", "--num-batches=6",
             "--print-freq=1", "--learning-rate=0.1", "--numpy-rand-seed=727", "--use-gpu"]
_CK = {"Q8": "cli_cfg0_C_ref.pt", "Q4": "cli_cfg0_C_ref.pt", "QW8": "cli_cfg0_W1_ref.pt", "QW4": "cli_cfg0_W1_ref.pt"}


@pytest.mark.parametrize("tag", ["Q8", "Q4", "QW8", "QW4"])
def test_cli_reproduces_the_reference_quantized_inference(tag):
    """The reference CLI's quantized test pass on its own checkpoints (QW: learned v_W_l as per-sample weights)."""
    import subprocess
    import sys

    flags = open(os.path.join(kaggle_cli.GOLD, "cli_cfg0_%s.flags" % tag)).read().split()
    r = subprocess.run([sys.executable, os.path.join(kaggle_cli.ROOT, "dlrm_s_pytorch.py")] + _CLI_BASE + flags
                       + ["--load-model=" + os.path.join(kaggle_cli.GOLD, _CK[tag])], capture_output=True, text=True,
                       timeout=600, cwd=kaggle_cli.ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    keep = re.compile(r"Training state|Testing state|Testing for inference only|^ accuracy")
    want = open(os.path.join(kaggle_cli.GOLD, "cli_cfg0_%s.txt" % tag)).read().splitlines()
    assert [ln for ln in r.stdout.splitlines() if keep.search(ln)] == want


@pytest.mark.parametrize("bits", [8, 4])
def test_cli_bin_records_mlperf_metrics_quantized(tmp_path, bits):
    """The MLPerf binary records with --mlperf-logging: the quantized test pass computes the metrics on the device,
    eagerly and in graph replays, with the same line.  (The reference's quantized branch cannot run this path: its
    binary loader hands non-contiguous index tensors to the quantized ops, which refuse them.)"""
    import test_gpu_bin_records as bin_cli

    ck = str(tmp_path / "ck.pt")
    bin_cli._cli(["--gemm=simt", "--save-model=" + ck])
    flags = ["--gemm=simt", "--load-model=" + ck, "--inference-only", "--quantize-emb-with-bit=%d" % bits]
    eager = bin_cli._cli(flags)
    graphed = bin_cli._cli(flags + ["--cuda-graph-steps"])
    e, g = re.findall(r"^recall .*", eager, re.M), re.findall(r"^recall .*", graphed, re.M)
    assert len(e) == 1 and e == g
    assert float(re.search(r"auc ([0-9.]+)", e[0]).group(1)) > 0.7
