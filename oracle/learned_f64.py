"""Float64 restatement of the fused embedding update with learned weighted pooling (include/dlrm_b200.h, row_weights
!= NULL), written from the reference's math: EmbeddingBag(mode="sum", per_sample_weights=v[idx]) followed by
optimizer.step() on the tables (sparse) and on v (dense, dlrm_s_pytorch.py:425-428, :1348-1369).  Independent of the
product: nothing here imports dlrm_b200.

For a touched row r with occurrences j (bag b_j) and S_r = sum_j dY[b_j]:
  row gradient     g_r  = v[r] * S_r
  weight gradient  dv_r = <S_r, W_old[r]>
  rows             SGD / RWSAdagrad (oracle.sparse_f64.row_step) or element-wise Adagrad (oracle.adagrad_f64.step_f64)
  v                SGD v -= lr dv;  RWSAdagrad / Adagrad (dense branch): s += dv^2, v -= lr dv / (sqrt(s) + eps)
Rows, accumulators, v and its sum of untouched rows are returned unchanged.
"""
from __future__ import annotations

import numpy as np

from . import adagrad_f64 as AG
from .sparse_f64 import OPT_RWSADAGRAD, OPT_SGD, coalesce, f64, occurrences, row_step, sum_exact

OPT_ADAGRAD = 2


def learned_step_f64(W, acc, v, vsum, idx, off, nnz, dY, opt, lr, eps, include_last=False):
    """One table: (W', acc', v', vsum', rows) in float64.  W [n, D] fp32 rows; acc: None (SGD), [n] (RWSAdagrad) or
    [n, D] (Adagrad); v, vsum [n] (vsum None for SGD); dY [batch, D]: the gradient of this table's pooled rows."""
    pos, bag, r = occurrences(idx, off, nnz, include_last)
    rows, grp = coalesce(r)
    S = sum_exact(np.asarray(dY, np.float32)[bag], grp, rows.size)
    W2, v2 = f64(W).copy(), f64(v).copy()
    acc2 = None if acc is None else f64(acc).copy()
    vs2 = None if vsum is None else f64(vsum).copy()
    w_old = f64(W)[rows]
    dv = (S * w_old).sum(axis=1)
    g = f64(v)[rows][:, None] * S
    lr64, eps64 = float(np.float32(lr)), float(np.float32(eps))
    if opt == OPT_ADAGRAD:
        W2[rows], acc2[rows] = AG.step_f64(w_old, f64(acc)[rows], g, lr, eps)
    else:
        wn, mn = row_step(w_old, None if acc is None else f64(acc)[rows], g, opt, lr, eps)
        W2[rows] = wn
        if opt == OPT_RWSADAGRAD:
            acc2[rows] = mn
    if opt == OPT_SGD:
        v2[rows] = f64(v)[rows] - lr64 * dv
    else:
        s = f64(vsum)[rows] + dv * dv
        vs2[rows] = s
        v2[rows] = f64(v)[rows] - lr64 * dv / (np.sqrt(s) + eps64)
    return W2, acc2, v2, vs2, rows
