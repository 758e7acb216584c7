"""Numpy restatement of the fp16 embedding tables' stochastic rounding (include/dlrm_b200.h,
dlrm_emb_bwd_table_t.round_key) -- written from the header's definition, independent of the product.

For finite fp32 x:  x itself when it is an fp16 value; otherwise lo = the fp16 neighbour toward zero,
hi = the one away from zero, and the result is hi iff r < floor(2^16 (|x| - |lo|) / (|hi| - |lo|)).
|x| > 65504 gives +-inf, NaN stays NaN.  r = 16 bits of h = splitmix64(round_key ^ R * K_ROW ^ (c // 4) * K_SLOT)
for global row R and column c, bits [16 (c % 4), 16 (c % 4) + 16); round_key = splitmix64(seed * K_STEP ^
(step + 1) * K_TABLE ^ (table + 1) * K_SLOT).
"""
from __future__ import annotations

import numpy as np

K_TABLE, K_ROW, K_SLOT, K_STEP = 0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0xD6E8FEB86659FD93
_M64 = (1 << 64) - 1


def splitmix64(x):
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def round_key(seed: int, step: int, table: int) -> int:
    base = ((seed * K_STEP) ^ ((step + 1) * K_TABLE) ^ ((table + 1) * K_SLOT)) & _M64
    return int(splitmix64(np.uint64(base)))


def sr_bits(key: int, rows, cols) -> np.ndarray:
    """The 16-bit r of (global row, column) pairs (broadcast together) under `key`."""
    rows = np.asarray(rows, dtype=np.uint64)
    cols = np.asarray(cols, dtype=np.uint64)
    with np.errstate(over="ignore"):
        h = splitmix64(np.uint64(key) ^ (rows * np.uint64(K_ROW)) ^ ((cols // np.uint64(4)) * np.uint64(K_SLOT)))
    return ((h >> (np.uint64(16) * (cols % np.uint64(4)))) & np.uint64(0xFFFF)).astype(np.int64)


def neighbours(x) -> tuple:
    """(lo, hi): the fp16 values next to fp32 x toward and away from zero (lo == x when x is an fp16 value)."""
    x = np.asarray(x, dtype=np.float32)
    ax = np.abs(x.astype(np.float64))
    with np.errstate(over="ignore"):
        rn = x.astype(np.float16)
    bits = rn.view(np.uint16).astype(np.int64)
    over = np.abs(rn.astype(np.float64)) > ax          # rounded away from zero: step back toward zero
    lo_bits = np.where(over, bits - 1, bits)
    lo = lo_bits.astype(np.uint16).view(np.float16)
    hi = (lo_bits + 1).astype(np.uint16).view(np.float16)
    return lo, hi


def sr_f16(x, r) -> np.ndarray:
    """Stochastic rounding of fp32 x to fp16 with the 16-bit integers r (broadcast with x)."""
    x = np.asarray(x, dtype=np.float32)
    r = np.asarray(r, dtype=np.int64)
    ax = np.abs(x.astype(np.float64))
    big = ~(ax <= 65504.0)                              # overflow or NaN
    xs = np.where(big, np.float32(0), x)
    lo, hi = neighbours(xs)
    flo, fhi = np.abs(lo.astype(np.float64)), np.abs(hi.astype(np.float64))
    axs = np.abs(xs.astype(np.float64))
    exact = flo == axs
    with np.errstate(invalid="ignore", divide="ignore"):
        t = np.floor((axs - flo) / np.where(exact, 1.0, fhi - flo) * 65536.0)
    out = np.where(exact, lo, np.where(r < t, hi, lo))
    inf = np.where(np.signbit(x), np.float16(-np.inf), np.float16(np.inf))
    out = np.where(big, np.where(np.isnan(x), np.float16(np.nan), inf), out)
    return out.astype(np.float16)


def sr_table(W32, key: int, row0: int = 0) -> np.ndarray:
    """sr_f16 of a [rows, D] fp32 block whose first row is global row `row0`."""
    W32 = np.asarray(W32, dtype=np.float32)
    rows = np.arange(row0, row0 + W32.shape[0])[:, None]
    cols = np.arange(W32.shape[1])[None, :]
    return sr_f16(W32, sr_bits(key, rows, cols))
