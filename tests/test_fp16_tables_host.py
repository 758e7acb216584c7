"""fp16 embedding tables, host side: the stochastic-rounding restatement (oracle/sr_numpy.py), the fp16 row layout,
the placement's bytes per row and the CLI flag.  No GPU needed."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import sr_numpy as SR  # noqa: E402


def _cases():
    rng = np.random.default_rng(0)
    normal = (rng.standard_normal(2000) * 10.0 ** rng.uniform(-4, 4, 2000)).astype(np.float32)
    sub16 = (rng.uniform(-1, 1, 500) * 2.0 ** -14).astype(np.float32)          # fp16 subnormal range
    sub32 = np.array([1e-40, -1e-40, 2.0 ** -149, -(2.0 ** -149)], dtype=np.float32)
    zeros = np.array([0.0, -0.0], dtype=np.float32)
    return np.concatenate([normal, sub16, sub32, zeros])


def test_sr_returns_a_neighbour_and_keeps_representable_values():
    x = _cases()
    r = np.random.default_rng(1).integers(0, 1 << 16, x.size)
    y = SR.sr_f16(x, r)
    lo, hi = SR.neighbours(x)
    assert np.all((y.view(np.uint16) == lo.view(np.uint16)) | (y.view(np.uint16) == hi.view(np.uint16)))
    # lo is toward zero, hi away from it, and they bracket x
    ax = np.abs(x.astype(np.float64))
    assert np.all(np.abs(lo.astype(np.float64)) <= ax) and np.all(np.abs(hi.astype(np.float64)) > ax)
    rep = x.astype(np.float16)                                  # representable inputs are returned unchanged
    for rr in (0, 1 << 15, (1 << 16) - 1):
        out = SR.sr_f16(rep.astype(np.float32), np.full(rep.size, rr))
        assert np.array_equal(out.view(np.uint16), rep.view(np.uint16))
    z = SR.sr_f16(np.array([0.0, -0.0], np.float32), np.array([0, 65535]))
    assert z.view(np.uint16).tolist() == [0x0000, 0x8000]


def test_sr_threshold_is_exact():
    """r < floor(2^16 (|x| - |lo|) / ulp) picks hi: probe both sides of the threshold."""
    lo = np.float16(1.0)
    ulp = 2.0 ** -10
    x = np.float32(1.0 + 0.25 * ulp)                            # threshold floor(0.25 * 2^16) = 16384
    assert SR.sr_f16(x, 16383) == np.float16(1.0 + ulp)
    assert SR.sr_f16(x, 16384) == lo
    xn = np.float32(-x)
    assert SR.sr_f16(xn, 16383) == np.float16(-(1.0 + ulp)) and SR.sr_f16(xn, 16384) == -lo
    # fp32 subnormal input: threshold 0, always rounds to (signed) zero
    assert SR.sr_f16(np.float32(1e-40), 0).view(np.uint16) == 0
    assert SR.sr_f16(np.float32(-1e-40), 0).view(np.uint16) == 0x8000


def test_sr_overflow_and_nan():
    x = np.array([65504.0, 65505.0, -65520.0, 1e30, np.inf, -np.inf, np.nan], dtype=np.float32)
    y = SR.sr_f16(x, np.zeros(x.size, np.int64))
    assert y[0] == np.float16(65504.0)
    assert np.isposinf(y[1]) and np.isneginf(y[2]) and np.isposinf(y[3]) and np.isposinf(y[4]) and np.isneginf(y[5])
    assert np.isnan(y[6])


@pytest.mark.parametrize("x", [1.0001, -3.14159, 1e-3, 7.7e-6, 2.1e-7, 1234.567])
def test_sr_is_unbiased_over_65536_columns(x):
    """A fixed x rounded with the hash bits of 2^16 columns of one row: the mean is within ulp16(x)/64 of x."""
    n = 1 << 16
    key = SR.round_key(7, 3, 11)
    r = SR.sr_bits(key, np.full(n, 12345), np.arange(n))
    y = SR.sr_f16(np.full(n, x, np.float32), r).astype(np.float64)
    lo, hi = SR.neighbours(np.float32(x))
    ulp = abs(float(hi) - float(lo))
    assert abs(y.mean() - float(np.float32(x))) <= ulp / 64


def test_sr_bits_deterministic_and_keyed():
    k1, k2 = SR.round_key(0, 1, 0), SR.round_key(0, 2, 0)
    assert k1 == SR.round_key(0, 1, 0) and k1 != k2 and k1 != SR.round_key(1, 1, 0) and k1 != SR.round_key(0, 1, 1)
    rows, cols = np.arange(64)[:, None], np.arange(128)[None, :]
    a, b = SR.sr_bits(k1, rows, cols), SR.sr_bits(k1, rows, cols)
    assert np.array_equal(a, b) and a.min() >= 0 and a.max() < (1 << 16)
    assert not np.array_equal(a, SR.sr_bits(k2, rows, cols))
    # a row-split shard sees the same bits for the same global rows
    assert np.array_equal(SR.sr_bits(k1, rows[32:], cols), a[32:])
    W = np.random.default_rng(3).standard_normal((64, 128)).astype(np.float32)
    assert np.array_equal(SR.sr_table(W[32:], k1, row0=32).view(np.uint16), SR.sr_table(W, k1)[32:].view(np.uint16))


def test_round_key_matches_the_product():
    """The engine's key (dlrm_b200/engine.py) and the restatement agree (pure Python on both sides)."""
    from dlrm_b200.engine import round_key

    for seed, step, table in [(0, 1, 0), (5, 100, 25), (2 ** 40, 7, 3)]:
        assert round_key(seed, step, table) == SR.round_key(seed, step, table)


def test_fp16_row_layout():
    """[D halves | fp32 accumulator | int32 head | pad]: 16-byte aligned rows, the two words after the halves."""
    from dlrm_b200.engine import fp16_row_stride

    assert fp16_row_stride(128) == 136                        # 272 bytes
    for D in (8, 16, 32, 64, 128, 256, 512):
        ld = fp16_row_stride(D)
        assert (ld * 2) % 16 == 0 and ld * 2 >= 2 * D + 8 and ld * 2 - (2 * D + 8) < 16
        assert (D * 2) % 4 == 0                                 # accumulator word aligned: column D/2 of a 4-byte view
    # uncapped MLPerf tables at dim 128: 204.2 M rows x 272 B = 55.5 GB (fits one 80 GB H100); fp32 rows 104.5 GB
    from dlrm_b200 import mlperf as M

    rows = sum(M.TABLE_ROWS)
    assert abs(rows * fp16_row_stride(128) * 2 / 1e9 - 55.5) < 0.1
    assert rows * 128 * 4 / 1e9 > 80


def test_placement_uses_fp16_bytes_per_row():
    from dlrm_b200 import placement as P

    assert P.row_bytes(128, "fp32") == 512 and P.row_bytes(128, "fp16") == 272
    with pytest.raises(ValueError):
        P.row_bytes(128, "bf16")
    # a 300 M-row table: too big for one 100 GB rank in fp32 rows, fits in fp16 rows
    rows, cost = [300_000_000, 1000], [0.1, 1.0]
    kw = dict(mem_budget_bytes=100e9, target_imbalance=10.0)
    fp32 = P.plan(rows, cost, 2, bytes_per_row=P.row_bytes(128, "fp32"), **kw)
    fp16 = P.plan(rows, cost, 2, bytes_per_row=P.row_bytes(128, "fp16"), **kw)
    assert 0 in fp32.split_tables() and 0 not in fp16.split_tables()


def test_cli_parses_emb_dtype():
    from dlrm_b200 import cli

    p = cli.build_parser()
    assert p.parse_args([]).emb_dtype == "fp32"
    assert p.parse_args(["--emb-dtype", "fp16"]).emb_dtype == "fp16"
    with pytest.raises(SystemExit):
        p.parse_args(["--emb-dtype", "bf16"])
