"""CUDA-graph steps for the command line (`--cuda-graph-steps`): every full-size training batch is copied into a static
device stage and trained by ONE replay of a captured `engine.GraphedTrainStep`, and every full-size test batch is scored
by a replay of a captured forward.  The learning rate lives in the engine's device scalar (`device_lr=True`), so the
schedule (`LRPolicy`, warm-up and decay) and the `lr_decay` of RWSAdagrad / Adagrad change it from step to step
exactly as the eager optimizer step would.

Batches of any other shape (the short last batch of an epoch or of the test set) return None from `train()` /
`forward()`, and the caller runs its eager step on the same engine and optimizer state.  The graphed step is
`Engine.train_step`: its loss comes from the fused head, not from torch's loss module, so the losses agree with the
eager command line's within rounding but are not bit-identical to them.
"""
from __future__ import annotations

from typing import Optional

import torch

from .data import DeviceBatch, PackedLayout
from .engine import GraphedTrainStep


class _Stage(DeviceBatch):
    """Static packed batch of B samples with one index per table and sample: table k's indices are positions
    [k B, (k + 1) B), so the offsets are copied in as lS_o + k B."""

    def __init__(self, B: int, T: int, m_den: int, device):
        super().__init__(PackedLayout(B, T, m_den, B * T), device)
        self.B, self.T, self.m_den = B, T, m_den
        base = torch.arange(T, dtype=torch.int64, device=device) * B
        self.base = base.view(T, 1)
        self.offsets[:, B].copy_(base + B)
        self.nnz = B * T

    def fits(self, X, lS_o, lS_i) -> bool:
        shape = (self.T, self.B)
        return (isinstance(lS_i, torch.Tensor) and isinstance(lS_o, torch.Tensor) and tuple(lS_i.shape) == shape
                and tuple(lS_o.shape) == shape and tuple(X.shape) == (self.B, self.m_den)
                and lS_i.device == self.buf.device and lS_o.device == self.buf.device
                and X.device == self.buf.device)

    def load_from(self, X, lS_o, lS_i, T=None):
        """Device-to-device copies of one batch in the reference's format (X, lS_o [T, B], lS_i [T, B], T)."""
        self.X.copy_(X)
        if T is not None:
            self.target.copy_(T.view(self.B, 1))
        self.indices.view(self.T, self.B).copy_(lS_i)
        torch.add(lS_o, self.base, out=self.offsets[:, :self.B])


class GraphSteps:
    """The captured training step and test forward of one `DLRM_Net`, with their static stages."""

    def __init__(self, net, optimizer, train_batch: int, test_batch: Optional[int], m_den: int,
                 optimizer_name: str):
        eng = net._engine
        self.net, self.opt, self.eng = net, optimizer, eng
        T, dev = eng.T, eng.device
        self.train_stage = _Stage(train_batch, T, m_den, dev) if optimizer is not None else None
        self.test_stage = _Stage(test_batch, T, m_den, dev) if test_batch else None
        # buffers that only grow (activations, occurrence lists, staging arena, scratch) take their final size before
        # either capture, the test shape first: a later step of another size must not reallocate what a graph uses
        for st, train in ((self.test_stage, False), (self.train_stage, True)):
            if st is not None:
                eng.prepare(st.sparse, train=train, batch=st.B)
        self.train_graph = self.test_graph = None
        if self.train_stage is not None:
            g = optimizer.param_groups[0]
            self.train_graph = GraphedTrainStep(eng, self.train_stage, g["lr"], optimizer_name, warmup=0,
                                                device_lr=True)
        if self.test_stage is not None:
            self.test_graph = GraphedTrainStep(eng, self.test_stage, 0.0, optimizer_name if optimizer else "sgd",
                                               warmup=0, train=False)
        self.counts = {"train_graphed": 0, "train_eager": 0, "test_graphed": 0, "test_eager": 0}

    def train(self, X, lS_o, lS_i, T) -> Optional[torch.Tensor]:
        """One graphed training step on a full-size batch: returns the loss (1-element device tensor), or None (the
        batch has another shape: the caller runs the eager step)."""
        st = self.train_stage
        if st is None or not st.fits(X, lS_o, lS_i):
            self.counts["train_eager"] += 1
            return None
        st.load_from(X, lS_o, lS_i, T)
        g = self.opt.param_groups[0]
        loss = self.train_graph.replay(g["lr"], g.get("lr_decay", 0.0))
        self.counts["train_graphed"] += 1
        return loss

    def forward(self, X, lS_o, lS_i) -> Optional[torch.Tensor]:
        """Scores [B, 1] of a full-size test batch (valid until the next replay), or None (eager)."""
        st = self.test_stage
        if st is None or not st.fits(X, lS_o, lS_i):
            self.counts["test_eager"] += 1
            return None
        st.load_from(X, lS_o, lS_i)
        out = self.test_graph.replay()
        self.counts["test_graphed"] += 1
        return out

    def report(self) -> str:
        c = self.counts
        return ("CUDA-graph steps: {} train steps replayed, {} eager (other batch sizes); {} test batches replayed, "
                "{} eager".format(c["train_graphed"], c["train_eager"], c["test_graphed"], c["test_eager"]))
