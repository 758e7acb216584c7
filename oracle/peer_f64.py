"""Restatements of the peer-memory exchange of a sharded step, written from the ABI comments of include/dlrm_b200.h
("Table-wise sharded runs" and the NCCL-free cross-GPU steps), and the bounds their tests compare against.
Independent of the product: nothing here imports dlrm_b200.

  route        global bag b of a world of W ranks with batch_local samples each lives on rank b / batch_local, local
               row b - rank * batch_local (a division, not b % W).
  all-reduce   every rank ends with the mean over ranks of every element: in fp32 the sum from 0.0f in rank order
               0 .. W-1, then ONE multiply by fp32(1 / W) (not a division by W).
  barrier      one call on `rank` advances its epoch word by 1 and stores the new epoch into slot `rank` of the signal
               array of every rank t < W; no other slot changes.
"""
from __future__ import annotations

import numpy as np

from .dense_f64 import U, f64, gamma  # noqa: F401  (re-exported)

SUBNORMAL_HALF = 2.0 ** -150    # largest rounding error of an fp32 result in the subnormal range


# ---------------------------------------------------------------------------------------------- routes
def route(b, batch_local):
    """(rank, local row) of global bag(s) b."""
    b = np.asarray(b, np.int64)
    r = b // int(batch_local)
    return r, b - r * int(batch_local)


def split(a, world):
    """A global [B, ...] array -> the W per-rank slabs [B / W, ...] (slab r = rows routed to rank r)."""
    a = np.asarray(a)
    assert a.shape[0] % world == 0, (a.shape, world)
    bl = a.shape[0] // world
    return [a[r * bl:(r + 1) * bl] for r in range(world)]


def join(slabs):
    """Inverse of split: the per-rank slabs in rank order -> the global array."""
    return np.concatenate([np.asarray(s) for s in slabs], axis=0)


# ---------------------------------------------------------------------------------------------- all-reduce
def allreduce_mean_f32(bufs):
    """The kernel's fp32 order: acc = 0.0f; acc += buf[r] for r = 0 .. W-1; acc *= fp32(1 / W)."""
    W = len(bufs)
    acc = np.zeros(np.asarray(bufs[0]).shape, np.float32)
    for b in bufs:
        acc = acc + np.asarray(b, np.float32)
    return acc * (np.float32(1.0) / np.float32(W))


def allreduce_mean_f64(bufs):
    """(mean, bound): the float64 mean over ranks and the bound of the fp32 evaluation above against it -- W - 1
    rounded additions, fp32(1 / W) (one rounding) and the multiply (one more): gamma_{W+1} * sum |x| / W, plus the
    subnormal rounding of the product."""
    x = np.stack([f64(b) for b in bufs])
    W = x.shape[0]
    return x.mean(axis=0), gamma(W + 1) * np.abs(x).sum(axis=0) / W + SUBNORMAL_HALF


# ---------------------------------------------------------------------------------------------- barrier
def barrier_after(sig, epoch, rank):
    """(epoch', sig') after one barrier call on `rank`: sig [W][slots] holds every rank's signal array."""
    sig = np.array(sig, copy=True)
    e = int(epoch) + 1
    sig[:, rank] = e
    return e, sig
