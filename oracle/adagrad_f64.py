"""Float64 restatement of the element-wise Adagrad step (torch.optim.Adagrad, `_single_tensor_adagrad`, on a sparse
gradient coalesced over duplicates), its fp32 evaluation in the order the kernels use (include/dlrm_b200.h, the
embedding backward), and the error bound that order gives.  Independent of the product: nothing here imports
dlrm_b200.

For every touched row r and column j (rows that do not occur are not touched at all):
    s'  = s + g^2
    w'  = w - clr * g / (sqrt(s') + eps),      clr = lr / (1 + (step - 1) * lr_decay)
fp32 order of the kernels:
    s'  = RN(RN(g * g) + s)                    two roundings, as torch's grad.pow(2) then the sparse add
    d   = RN(RN(sqrt(s')) + eps)
    q   = RN(g / d)
    w'  = fmaf(-clr, q, w)                     torch's CPU add_ may round -clr * q first: held to the bound, not bits
Dense parameters take the same algorithm through the dense kernels (oracle/dense_f64.dense_step, RWSAdagrad branch).

Bounds follow oracle/dense_f64.py: fl(a op b) = (a op b)(1 + d), |d| <= u = 2^-24, gamma_n = n u / (1 - n u).
"""
from __future__ import annotations

import numpy as np

from .dense_f64 import _fma_f32, f64, gamma  # noqa: F401  (re-exported)
from .sparse_f64 import SUBNORMAL_HALF, coalesce, occurrences, sum_f32_ascending  # noqa: F401  (re-exported)

OPT_ADAGRAD = 2


def clr(lr, step, lr_decay):
    """The decayed learning rate of optimizer step `step` (1-based), as torch.optim.Adagrad computes it."""
    return lr / (1.0 + (step - 1) * lr_decay)


def step_f64(w, s, g, lr, eps):
    """The definition in float64 on rows [n, D]: (w', s').  lr and eps are the fp32 values the kernels receive."""
    lr, eps = float(np.float32(lr)), float(np.float32(eps))
    w, s, g = f64(w), f64(s), f64(g)
    s2 = s + g * g
    return w - lr * g / (np.sqrt(s2) + eps), s2


def step_f32(w, s, g, lr, eps, *, fma_accumulator=False, eps_in_sqrt=False, row_mean=False):
    """The kernels' fp32 order: (w', s').  The keyword variants are WRONG orders, kept as negative controls for the
    tests: an FMA-contracted accumulator (one rounding), eps inside the square root, and RWSAdagrad's row-wise mean of
    g^2 in place of the per-element accumulator."""
    w, s, g = np.asarray(w, np.float32), np.asarray(s, np.float32), np.asarray(g, np.float32)
    lr, eps = np.float32(lr), np.float32(eps)
    if row_mean:
        s2 = (s + (g * g).mean(axis=-1, keepdims=True, dtype=np.float32)).astype(np.float32)
    elif fma_accumulator:
        s2 = _fma_f32(g, g, s)
    else:
        s2 = (s + g * g).astype(np.float32)              # numpy: RN(g * g), then RN(s + .)
    d = np.sqrt(s2 + eps) if eps_in_sqrt else np.sqrt(s2) + eps
    q = (g / d.astype(np.float32)).astype(np.float32)
    return _fma_f32(-lr, q, w), s2


def step_bound(w2, s2, g, lr, eps, g_rel=0.0):
    """Bounds (on w', on s') of the fp32 order against step_f64's (w2, s2), for the fp32 gradient g the kernel used;
    g_rel = the relative error g may already carry (2u for a long list: one ulp).
      s':  RN(g^2) and the add: gamma_2 (s + g^2), plus 2 g_rel g^2 and the subnormal rounding of a tiny g^2;
      d:   the s' error through sqrt, min(sqrt(ds), ds / (2 sqrt(s'))), then sqrt and + eps: 2 roundings;
      w':  the division and -clr * q (fused, or a separate rounding on the CPU): 2 roundings on the update, 1 on w'."""
    lr, eps = float(np.float32(lr)), float(np.float32(eps))
    g, s2 = f64(g), f64(s2)
    gg = g * g
    bs = gamma(2) * np.abs(s2) + 2.02 * g_rel * gg + 2 * SUBNORMAL_HALF
    rs = np.sqrt(s2)
    e_root = np.minimum(np.sqrt(bs), np.where(rs > 0, bs / (2 * np.where(rs > 0, rs, 1.0)), np.inf))
    d = rs + eps
    rel_d = e_root / d + gamma(2)
    upd = lr * np.abs(g) / d
    bw = gamma(1) * np.abs(f64(w2)) + upd * (1.01 * (rel_d + g_rel) + gamma(2)) + SUBNORMAL_HALF
    return bw, bs


def dense_rows_sparse_grad(rows_n, D, idx, G):
    """The uncoalesced sparse COO gradient of an [rows_n, D] table whose occurrences idx carry the rows G (what
    autograd's embedding_bag backward hands torch.optim): indices [1, nnz], values [nnz, D]."""
    import torch

    return torch.sparse_coo_tensor(torch.as_tensor(np.asarray(idx, np.int64))[None, :],
                                   torch.as_tensor(np.asarray(G, np.float32)), (rows_n, D))
