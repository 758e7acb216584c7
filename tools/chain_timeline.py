#!/usr/bin/env python
"""Per-task timeline of the persistent MLP-chain kernels (csrc/gemm_chain.cu, dlrm_b200_gemm_chain_set_trace)
inside real CFG2-shaped training steps.  Writes $DLRM_TRACE_DIR (default traces/)/<tag>_chain_trace.npz (one [tasks, 8] array per
chain: claim, deps ready, last TMA issued, first operands landed, last MMA issued, accumulator ready, epilogue
done (ns, relative to the first claim), SM id) and prints a per-problem summary.  Run on the GPU box."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main(tag="trace", B=2048, rows=100_000, T=26):
    from dlrm_b200.data import DeviceBatch, make_batch
    from dlrm_b200.engine import Engine

    dev = "cuda:0"
    D = 128
    ln_emb = [rows] * T
    ln_bot = [13, 512, 256, 128]
    ln_top = [D + (T + 1) * T // 2, 1024, 512, 256, 1]
    eng = Engine(D, ln_emb, ln_bot, ln_top, loss="bce", sigmoid_top=len(ln_top) - 2, device=dev, max_batch=B, gemm="tc")
    eng.init_params(0)
    eng.ensure_optimizer_state("rwsadagrad")
    rng = np.random.default_rng(0)
    hb = make_batch(rng, ln_emb, B, 13, 10)
    db = DeviceBatch(hb.layout, dev)
    db.load(hb, non_blocking=False)
    for _ in range(3):
        eng.train_step(db.X, db.sparse, db.target, 0.01, "rwsadagrad")
    torch.cuda.synchronize()
    traces = {}
    for key, ch in eng.tc_chains.items():
        t = torch.zeros((ch.info()["tasks"], 8), dtype=torch.int64, device=dev)
        ch.set_trace(t)
        traces[key] = t
    for _ in range(2):
        eng.train_step(db.X, db.sparse, db.target, 0.01, "rwsadagrad")
    torch.cuda.synchronize()
    out = {}
    for key, t in traces.items():
        a = t.cpu().numpy().astype(np.int64)
        eng.tc_chains[key].set_trace(None)
        ch = eng.tc_chains[key]
        t0 = a[:, 0].min()
        rel = a.copy()
        rel[:, :7] -= t0
        out["%s_%s" % key] = rel
        # problem boundaries from the plans
        begins, names = [], []
        n = 0
        for p in ch.plans:
            i = p.info()
            begins.append(n)
            n += i["ctas"]
            names.append("M%d N%d K%d bn%d sk%d" % (p.desc.M, p.desc.N, p.desc.K, i["tile_n"], i["splits"]))
        begins.append(n)
        print("== chain %s: %d tasks on %d CTAs, %d stages, span %.1f us" % (
            key, n, ch.info()["ctas"], ch.info()["stages"], (rel[:, 6].max()) / 1e3))
        for j, nm in enumerate(names):
            r = rel[begins[j]:begins[j + 1]]
            print("  %-34s tasks %4d | claim %6.1f..%6.1f | deps +%5.1f | tma-issue +%5.1f | 1st data +%5.1f | mma +%5.1f "
                  "| acc->epi +%5.1f | epi %5.1f | done %6.1f..%6.1f us" % (
                      nm, len(r), r[:, 0].min() / 1e3, r[:, 0].max() / 1e3,
                      np.median(r[:, 1] - r[:, 0]) / 1e3, np.median(r[:, 2] - r[:, 1]) / 1e3,
                      np.median(r[:, 3] - r[:, 1]) / 1e3, np.median(r[:, 4] - r[:, 3]) / 1e3,
                      np.median(r[:, 5] - r[:, 4]) / 1e3, np.median(r[:, 6] - r[:, 5]) / 1e3,
                      r[:, 6].min() / 1e3, r[:, 6].max() / 1e3))
    out_dir = os.environ.get("DLRM_TRACE_DIR", "traces")
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "%s_chain_trace.npz" % tag), **out)


if __name__ == "__main__":
    main(*(sys.argv[1:2] or ["trace"]))
