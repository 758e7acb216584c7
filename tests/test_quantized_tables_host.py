"""Row-wise 8- / 4-bit quantized embedding tables, host side: the numpy restatement (oracle/quant_rowwise.py) is
bit-identical to torch's CPU prepack and pooling ops, the command line routes --quantize-emb-with-bit to
DLRM_Net(emb_dtype="int8" | "int4") and refuses what it does not support, and the MLPerf byte counts."""
import os

import numpy as np
import pytest
import torch

from oracle import quant_rowwise as Q

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
OPS = torch.ops.quantized


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all(a.view(np.uint32) == b.view(np.uint32)))


def _tables(rng, n, d):
    w = (rng.standard_normal((n, d)) * 0.05).astype(np.float32)
    w[0] = 0.25                                          # constant row: range 0
    w[1] = 0.0
    w[2] *= 1e30                                         # large range
    w[3] *= 1e-30                                        # tiny range
    w[4] = np.linspace(-6e4, 6e4, d)                     # 4-bit: range / 15 near the fp16 limit
    w[5] = np.linspace(-1e6, 1e6, d)                     # 4-bit: fp16 scale overflows
    w[6, 0], w[7, -1] = np.inf, -np.inf                  # infinite entries
    return w


@pytest.mark.parametrize("d", [4, 8, 64, 128])
def test_prepack_is_bit_identical_to_torch(d):
    w = _tables(np.random.default_rng(d), 300, d)
    t = torch.from_numpy(w)
    assert np.array_equal(Q.prepack8(w), OPS.embedding_bag_byte_prepack(t).numpy())
    assert np.array_equal(Q.prepack4(w), OPS.embedding_bag_4bit_prepack(t).numpy())


def test_prepack_of_fp16_rows_is_the_prepack_of_the_widened_rows():
    w = _tables(np.random.default_rng(1), 200, 64)[8:].astype(np.float16)
    wide = torch.from_numpy(w.astype(np.float32))
    assert np.array_equal(Q.prepack8(w.astype(np.float32)), OPS.embedding_bag_byte_prepack(wide).numpy())
    assert np.array_equal(Q.prepack4(w.astype(np.float32)), OPS.embedding_bag_4bit_prepack(wide).numpy())


@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("d", [4, 8, 64, 128])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("idx_dtype", [torch.int64, torch.int32])
def test_pooling_is_bit_identical_to_torch(bits, d, weighted, idx_dtype):
    rng = np.random.default_rng(bits * 1000 + d)
    w = _tables(rng, 400, d)[8:]
    packed = (OPS.embedding_bag_byte_prepack if bits == 8 else OPS.embedding_bag_4bit_prepack)(torch.from_numpy(w))
    sizes = np.array([0, 1, 2, 0, 37, 200, 5, 0, 64, 1])                # empty bags, bags of 1 to 200 rows
    off = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    idx = rng.integers(0, w.shape[0], int(sizes.sum()))
    psw = (rng.random(idx.size).astype(np.float32) * 4 - 2) if weighted else None
    op = OPS.embedding_bag_byte_rowwise_offsets if bits == 8 else OPS.embedding_bag_4bit_rowwise_offsets
    ref = op(packed, torch.from_numpy(idx).to(idx_dtype), torch.from_numpy(off).to(idx_dtype),
             per_sample_weights=None if psw is None else torch.from_numpy(psw)).numpy()
    assert _bits_equal(Q.pool(packed.numpy(), bits, idx, off, psw), ref)
    # include-last offsets (batch + 1 entries) give the same sums
    off_l = np.append(off, idx.size)
    assert _bits_equal(Q.pool(packed.numpy(), bits, idx, off_l, psw, include_last=True), ref)


def test_fma_rounds_once():
    """a * b = 3 + 3 * 2^-23 lies exactly halfway between the floats 3 + 2^-22 and 3 + 2^-21 (the even one), and c =
    -2^-60 is below half a float64 ulp there: the float64 sum is the midpoint itself, so rounding it to fp32 gives the
    even neighbour, while the fused result -- just below the midpoint -- is 3 + 2^-22.  Only the tie correction finds it."""
    a = np.array([1.0 + 2.0 ** -23], np.float32)
    b = np.array([3.0], np.float32)
    c = np.array([-(2.0 ** -60)], np.float32)
    double_rounded = (a.astype(np.float64) * 3.0 + c.astype(np.float64)).astype(np.float32)
    assert double_rounded[0] == np.float32(3.0 + 2.0 ** -21)
    assert Q._fma(a, b, c)[0] == np.float32(3.0 + 2.0 ** -22)
    assert Q._fma(a, b, -c)[0] == np.float32(3.0 + 2.0 ** -21)


def test_mlperf_table_bytes():
    from dlrm_b200 import mlperf
    from dlrm_b200.engine import quant_row_bytes

    rows = int(np.sum(np.asarray(mlperf.TABLE_ROWS, dtype=np.int64)))
    assert quant_row_bytes(128, 8) == 136 and quant_row_bytes(128, 4) == 68
    assert round(rows * quant_row_bytes(128, 8) / 1e9, 1) == 27.8
    assert round(rows * quant_row_bytes(128, 4) / 1e9, 1) == 13.9
    assert round(rows * 272 / 1e9, 1) == 55.5


# ---------------------------------------------------------------- command line (stand-in model, as tests/test_cli_host.py)
@pytest.fixture
def cli_on_cpu(monkeypatch):
    import dlrm_b200.cli as cli
    import dlrm_b200.dlrm_net as dn
    import dlrm_b200.optim as fo

    built = []

    class StandIn(torch.nn.Module):
        def __init__(self, m_spa, ln_emb, ln_bot, ln_top, **kw):
            super().__init__()
            built.append(kw)
            self.lin = torch.nn.Linear(int(ln_bot[0]), 1)
            self.loss_fn = torch.nn.MSELoss()

        def forward(self, X, lS_o, lS_i):
            return torch.sigmoid(self.lin(X))

    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)
    monkeypatch.setattr(dn, "DLRM_Net", StandIn)
    monkeypatch.setattr(fo, "SGD", torch.optim.SGD)
    monkeypatch.setattr(fo, "RWSAdagrad", torch.optim.SGD)
    return cli, built


BASE = ["--arch-sparse-feature-size=16", "--arch-embedding-size=64-16", "--arch-mlp-bot=5-16", "--arch-mlp-top=8-1",
        "--mini-batch-size=8", "--print-freq=1", "--use-gpu", "--num-batches=2"]


@pytest.mark.parametrize("bits,dtype", [(8, "int8"), (4, "int4")])
def test_cli_inference_only_builds_quantized_tables(cli_on_cpu, capsys, bits, dtype):
    cli, built = cli_on_cpu
    cli.run(BASE + ["--inference-only", "--quantize-emb-with-bit=%d" % bits])
    assert built[-1]["emb_dtype"] == dtype
    out = capsys.readouterr().out
    assert "Testing for inference only" in out and " accuracy " in out
    assert "quantized emb sizes" not in out


def test_cli_without_quantization_keeps_float_tables(cli_on_cpu):
    cli, built = cli_on_cpu
    cli.run(BASE + ["--inference-only"])
    assert built[-1]["emb_dtype"] == torch.float32


@pytest.mark.parametrize("flags,msg", [
    (["--quantize-emb-with-bit=8"], "4 and 8-bit quantization on GPU is not supported"),
    (["--quantize-emb-with-bit=4"], "4 and 8-bit quantization on GPU is not supported"),
    (["--inference-only", "--quantize-mlp-with-bit=8"], "4 and 8-bit quantization on GPU is not supported"),
    (["--inference-only", "--quantize-emb-with-bit=8", "--emb-dtype=fp16"], "replaces the table storage type"),
    (["--inference-only", "--quantize-emb-with-bit=4", "--emb-host-tables=0"], "--emb-host-tables is not supported"),
])
def test_cli_refusals(cli_on_cpu, flags, msg):
    cli, _ = cli_on_cpu
    with pytest.raises(SystemExit) as e:
        cli.run(BASE + flags)
    assert msg in str(e.value)


def test_cli_refuses_sharded_quantized_runs(cli_on_cpu, monkeypatch):
    cli, _ = cli_on_cpu
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit) as e:
        cli.run(BASE + ["--inference-only", "--quantize-emb-with-bit=8"])
    assert "runs on one GPU" in str(e.value)


def test_restatement_reproduces_the_reference_goldens():
    z = np.load(os.path.join(GOLD, "cfg0_quant.npz"))
    for k in range(len(z["ln_emb"])):
        assert np.array_equal(Q.prepack8(z["emb%d" % k]), z["q8_emb%d" % k])
        assert np.array_equal(Q.prepack4(z["emb%d" % k]), z["q4_emb%d" % k])
