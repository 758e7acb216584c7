"""Row-wise 8- and 4-bit quantized embedding tables in numpy: the packed rows of
torch.ops.quantized.embedding_bag_{byte,4bit}_prepack and the sums of
torch.ops.quantized.embedding_bag_{byte,4bit}_rowwise_offsets, restated operation by operation in fp32 so that
every result is bit-identical to those CPU ops (tests/test_quantized_tables_host.py checks it).

8-bit row: [D uint8 | fp32 scale | fp32 bias], bias = min(row), scale = (max - min) / 255,
           q = rint((x - min) * (255 / ((max - min) + 1e-8))).
4-bit row: [D/2 bytes | fp16 scale | fp16 bias], column 2j in the low nibble of byte j, 2j+1 in the high one;
           bias = fp16(min), scale = fp16((max - float(bias)) / 15) (1 when that is 0 or its inverse is inf),
           q = clamp(rint((x - float(bias)) * (1 / scale)), 0, 15).
Pooling:   every bag in index order, acc = fma(scale * w, q, acc + bias * w), scale * w and bias * w rounded to fp32
           first (w = the per-sample weight, 1 without one).
Rows with infinite entries are covered; rows holding a NaN are not (the CPU op's bytes for them follow its vectorised
min / max, which this restatement and the GPU kernel do not reproduce).
"""
import numpy as np

f32 = np.float32


def prepack8(x):
    x = np.asarray(x, dtype=f32)
    n, d = x.shape
    mn = x.min(axis=1) if d else np.zeros(n, f32)
    mx = x.max(axis=1) if d else np.zeros(n, f32)
    rng = (mx - mn).astype(f32)
    scale = (rng / f32(255)).astype(f32)
    inv = (f32(255) / (rng + f32(1e-8))).astype(f32)
    with np.errstate(invalid="ignore", over="ignore"):
        q = np.rint(((x - mn[:, None]).astype(f32) * inv[:, None]).astype(f32))
        q = np.nan_to_num(q, nan=0.0, posinf=0.0, neginf=0.0)   # NaN / inf products: the conversion's 0 (see tests)
    out = np.zeros((n, d + 8), np.uint8)
    out[:, :d] = np.clip(q, 0, 255).astype(np.uint8)
    out[:, d:d + 4] = scale.view(np.uint8).reshape(n, 4)
    out[:, d + 4:] = mn.astype(f32).view(np.uint8).reshape(n, 4)
    return out


def prepack4(x):
    x = np.asarray(x, dtype=f32)
    n, d = x.shape
    assert d % 2 == 0
    mn = x.min(axis=1)
    mx = x.max(axis=1)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        bias16 = mn.astype(np.float16)
        bias = bias16.astype(f32)
        rng = (mx - bias).astype(f32)
        scale = np.where(rng == 0, f32(1), (rng / f32(15)).astype(f32)).astype(f32)
        scale = scale.astype(np.float16).astype(f32)
        scale = np.where(scale == 0, f32(1), scale).astype(f32)
        inv = (f32(1) / scale).astype(f32)
        bad = np.isinf(inv)
        scale = np.where(bad, f32(1), scale).astype(f32)
        inv = np.where(bad, f32(1), inv).astype(f32)
        q = np.rint(((x - bias[:, None]).astype(f32) * inv[:, None]).astype(f32))
        q = np.nan_to_num(q, nan=0.0, posinf=15.0, neginf=0.0)
    q = np.clip(q, 0, 15).astype(np.uint8)
    out = np.zeros((n, d // 2 + 4), np.uint8)
    out[:, :d // 2] = q[:, 0::2] | (q[:, 1::2] << 4)
    out[:, d // 2:d // 2 + 2] = scale.astype(np.float16).view(np.uint8).reshape(n, 2)
    out[:, d // 2 + 2:] = bias16.view(np.uint8).reshape(n, 2)
    return out


def unpack(packed, bits):
    """(q [n, D] as fp32, scale [n] fp32, bias [n] fp32) of packed rows."""
    p = np.asarray(packed, dtype=np.uint8)
    n = p.shape[0]
    if bits == 8:
        d = p.shape[1] - 8
        q = p[:, :d].astype(f32)
        sb = np.ascontiguousarray(p[:, d:]).view(f32).reshape(n, 2)
        return q, sb[:, 0].copy(), sb[:, 1].copy()
    d = 2 * (p.shape[1] - 4)
    q = np.empty((n, d), f32)
    q[:, 0::2] = p[:, :d // 2] & 15
    q[:, 1::2] = p[:, :d // 2] >> 4
    sb = np.ascontiguousarray(p[:, d // 2:]).view(np.float16).reshape(n, 2).astype(f32)
    return q, sb[:, 0].copy(), sb[:, 1].copy()


def pool(packed, bits, indices, offsets, per_sample_weights=None, include_last=False):
    """[B, D] fp32 sums of the bags (offsets as nn.EmbeddingBag takes them), in index order."""
    q, scale, bias = unpack(packed, bits)
    idx = np.asarray(indices, dtype=np.int64)
    off = np.asarray(offsets, dtype=np.int64)
    B = off.size - 1 if include_last else off.size
    ends = off[1:] if include_last else np.append(off[1:], idx.size)
    w = None if per_sample_weights is None else np.asarray(per_sample_weights, dtype=f32)
    out = np.zeros((B, q.shape[1]), f32)
    for b in range(B):
        acc = np.zeros(q.shape[1], f32)
        for j in range(off[b], ends[b]):
            r = idx[j]
            s, t = scale[r], bias[r]
            if w is not None:
                s, t = f32(s * w[j]), f32(t * w[j])
            acc = _fma(np.full_like(acc, s), q[r], (acc + t).astype(f32))
        out[b] = acc
    return out


def _fma(a, b, c):
    """fp32 fused multiply-add with one rounding.  a * b is exact in float64 (24-bit x 8-bit significands); the sum
    is rounded to float64 and then to fp32, and the one case where that double rounding differs from a single one --
    the float64 sum landing exactly halfway between two floats -- is settled by the sign of the float64 sum's error."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)                     # exact: p + c == s + err
    f = s.astype(f32)
    with np.errstate(over="ignore", invalid="ignore"):
        g = np.nextafter(f, np.where(s > f.astype(np.float64), f32(np.inf), f32(-np.inf)).astype(f32))
        tie = (err != 0) & (f.astype(np.float64) != s) & ((f.astype(np.float64) + g.astype(np.float64)) / 2 == s)
    up = np.where(err > 0, np.maximum(f, g), np.minimum(f, g))
    return np.where(tie, up, f).astype(f32)
