#!/usr/bin/env python
"""In-step timeline of one eager CFG2 training step: when every kernel launch FINISHES on its
stream, relative to the start of the step -- shows which launches overlap across the three streams
(main / embedding / weight-gradient) and where a stream sits idle.  ncu serialises kernels and flushes
caches, so it cannot show this; CUDA events on the launching streams can.

    python tools/step_timeline.py [--steps 20] [--pdl 0|1] > timeline.txt

Method: `TimelineEngine` subclasses the product Engine and turns its launch counter (`n_launch`, bumped
after every C-ABI launch) into a property whose setter records a CUDA event on the current stream,
tagged with the Python call site.  Nothing in dlrm_b200/ is modified.  Events cost ~1 us each on the
stream, so absolute times are slightly inflated; the ORDER and OVERLAP are what to read.
"""
import argparse
import os
import sys
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--pdl", type=int, default=1)
    ap.add_argument("--gemm", default="tc")
    args = ap.parse_args()
    os.environ["DLRM_TUNE"] = "pdl=%d" % (1 if args.pdl else 2)

    from dlrm_b200.data import DeviceBatch, make_batch
    from dlrm_b200.engine import Engine

    class TimelineEngine(Engine):
        _rec = None          # list of (tag, stream id, event) while a step is being traced
        _count = 0

        @property
        def n_launch(self):
            return self._count

        @n_launch.setter
        def n_launch(self, v):
            self._count = v
            if self._rec is not None:
                f = sys._getframe(1)
                ev = torch.cuda.Event(enable_timing=True)
                s = torch.cuda.current_stream()
                ev.record(s)
                self._rec.append(("%s:%d" % (f.f_code.co_name, f.f_lineno), s.cuda_stream, ev))

    torch.cuda.set_device(0)
    dev = "cuda:0"
    D, T, R, B = 128, 26, 1_000_000, 2048
    ln_emb, ln_bot = [R] * T, [13, 512, 256, 128]
    ln_top = [D + (T + 1) * T // 2, 1024, 512, 256, 1]
    eng = TimelineEngine(D, ln_emb, ln_bot, ln_top, loss="bce", sigmoid_top=len(ln_top) - 2, device=dev,
                         max_batch=B, gemm=args.gemm)
    eng.init_params(0)
    eng.ensure_optimizer_state("rwsadagrad")
    rng = np.random.default_rng(1234)
    ring = []
    for _ in range(8):
        hb = make_batch(rng, ln_emb, B, 13, 10)
        db = DeviceBatch(hb.layout, dev)
        db.load(hb, non_blocking=False)
        ring.append(db)
    for i in range(args.warmup):
        db = ring[i % len(ring)]
        eng.train_step(db.X, db.sparse, db.target, 0.01, "rwsadagrad")
    torch.cuda.synchronize()

    names = {torch.cuda.current_stream().cuda_stream: "main", eng.s_emb.cuda_stream: "emb", eng.s_wg.cuda_stream: "wgrad"}
    acc = defaultdict(list)          # (order, tag, stream) -> [finish time in us]
    totals = []
    for i in range(args.steps):
        db = ring[(args.warmup + i) % len(ring)]
        torch.cuda.synchronize()
        eng._rec = []
        t0 = torch.cuda.Event(enable_timing=True)
        t0.record()
        eng.train_step(db.X, db.sparse, db.target, 0.01, "rwsadagrad")
        t1 = torch.cuda.Event(enable_timing=True)
        t1.record()
        torch.cuda.synchronize()
        rec, eng._rec = eng._rec, None
        for k, (tag, sid, ev) in enumerate(rec):
            acc[(k, tag, names.get(sid, hex(sid)))].append(t0.elapsed_time(ev) * 1e3)
        totals.append(t0.elapsed_time(t1) * 1e3)
    print("# eager step, pdl=%d: median finish time of every launch group (us from step start), %d steps"
          % (args.pdl, args.steps))
    print("# step total (main stream, incl. joins): median %.1f us" % float(np.median(totals)))
    last = defaultdict(float)
    print("%-4s %-7s %-34s %9s %9s" % ("#", "stream", "call site (engine.py)", "finish", "since prev on stream"))
    for (k, tag, sname), v in sorted(acc.items()):
        t = float(np.median(v))
        print("%-4d %-7s %-34s %9.1f %9.1f" % (k, sname, tag, t, t - last[sname]))
        last[sname] = t


if __name__ == "__main__":
    main()
