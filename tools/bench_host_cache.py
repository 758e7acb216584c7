"""The host row cache on one GPU: the cache kernels alone at given hit rates, and the MLPerf training step with a
cache in front of the host tables.

  python tools/bench_host_cache.py [--out DIR] [--steps 100] [--iters 30] [--shares 0,0.02,0.2]

1. Cache kernels: stage-in + write-back (insert or return) of n distinct rows of a pinned fp32 table (528-byte
   interleaved rows), a share h of them drawn from a hot set that earlier steps made resident, the rest uniform over
   the table.  CUDA events per step; the hit rate printed is the one the cache counters measured.  n = 53,248 (the
   one-hot batch of 2048 x 26), cache 262,144 rows, cache 0 as the baseline.
2. Train step of bench/run_and_time.sh's model (MLPerf MLPs, D = 128, one-hot, batch 2048, rwsadagrad, fp32 tables) at
   a 10 M row cap with tables 0, 9, 19, 20, 21 on the host, per cache size (0 and shares of the host rows): the
   all-device engine and the cached host engine timed a, b, a, b, for uniform ids and for Zipf ids (exponent
   ZIPF_A, ranks scattered over the rows by a fixed multiplicative hash).  Each stream first runs WARM steps; every
   step of a stream has its own batch.
Prints one JSON object; the card's name, power limit and max SM clock come first."""
import argparse
import ctypes as C
import gc
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dlrm_b200 import _lib  # noqa: E402
from dlrm_b200.engine import Engine  # noqa: E402
from dlrm_b200.mlperf import TABLE_ROWS  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_host_tables import BIG, DEV, ROW, card, mem_available  # noqa: E402

ZIPF_A = 1.1
WARM = 200


def _stage(n_cache, cap, ld=132):
    t = dict(sw=torch.zeros(n_cache + cap, ld, device=DEV), sidx=torch.zeros(cap, dtype=torch.int64, device=DEV),
             lst=torch.zeros(cap, dtype=torch.int32, device=DEV), key=torch.zeros(cap, dtype=torch.int64, device=DEV),
             cnt=torch.zeros(1, dtype=torch.int32, device=DEV))
    st = _lib.HostStage(weight=t["sw"].data_ptr(), slot_idx=t["sidx"].data_ptr(), list=t["lst"].data_ptr(),
                        key=t["key"].data_ptr(), count=t["cnt"].data_ptr(), capacity=cap, ld=ld, head_col=129)
    if n_cache:
        t.update(tag=torch.full((n_cache,), -1, dtype=torch.int64, device=DEV),
                 used=torch.zeros(n_cache, dtype=torch.int32, device=DEV),
                 step=torch.zeros(1, dtype=torch.int32, device=DEV),
                 shd=torch.zeros(n_cache // 32, dtype=torch.int32, device=DEV),
                 snx=torch.zeros(cap, dtype=torch.int32, device=DEV),
                 sets=torch.zeros(n_cache // 32, dtype=torch.int32, device=DEV),
                 nsets=torch.zeros(1, dtype=torch.int32, device=DEV),
                 stats=torch.zeros(4, dtype=torch.int64, device=DEV))
        st.cache_rows, st.cache_tag, st.cache_used, st.step = (n_cache, t["tag"].data_ptr(), t["used"].data_ptr(),
                                                               t["step"].data_ptr())
        st.set_head, st.set_next, st.sets = t["shd"].data_ptr(), t["snx"].data_ptr(), t["sets"].data_ptr()
        st.num_sets, st.stats = t["nsets"].data_ptr(), t["stats"].data_ptr()
    return t, st


def kernels(rows, n, n_cache, shares, iters):
    lib = _lib.lib()
    table = torch.zeros(rows, 132)
    assert lib.dlrm_b200_host_register(table.data_ptr(), table.numel() * 4) == 0, lib.dlrm_b200_last_error()
    out = []
    try:
        g = torch.Generator(device=DEV)
        g.manual_seed(0)
        smap = torch.zeros(rows, dtype=torch.int32, device=DEV)
        hot = torch.randperm(rows, device=DEV, generator=g)[:max(n_cache // 2, 1)]
        t, st = _stage(n_cache, n)
        idx = torch.zeros(n, dtype=torch.int64, device=DEV)
        off = torch.tensor([0, n], dtype=torch.int64, device=DEV)
        d = (_lib.HostTable * 1)()
        d[0].weight, d[0].indices, d[0].offsets, d[0].nnz = table.data_ptr(), idx.data_ptr(), off.data_ptr(), n
        d[0].rows, d[0].map = rows, smap.data_ptr()
        s = torch.cuda.current_stream().cuda_stream

        def draw(h):
            k = int(round(h * n))
            a = hot[torch.randperm(hot.numel(), device=DEV, generator=g)[:k]] if k else hot[:0]
            b = torch.randint(0, rows, (4 * n,), device=DEV, generator=g)
            b = b[~torch.isin(b, hot)].unique()
            b = b[torch.randperm(b.numel(), device=DEV, generator=g)][:n - a.numel()]
            idx.copy_(torch.cat([a, b]))

        def step():
            _lib.check(lib.dlrm_b200_host_stage_in(d, 1, C.byref(st), 128, 1, 8, 1, s), "stage_in")
            _lib.check(lib.dlrm_b200_host_write_back(d, 1, C.byref(st), 128, s), "write_back")

        if n_cache:      # warm: the hot set, a step at a time
            for c0 in range(0, hot.numel(), n):
                part = hot[c0:c0 + n]
                idx[:part.numel()].copy_(part)
                off[1] = part.numel()
                step()
            off[1] = n
        for h in shares:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ms, hits0 = 0.0, (int(t["stats"][0].item()) if n_cache else 0)
            for _ in range(iters):
                draw(h)
                ev[0].record()
                step()
                ev[1].record()
                torch.cuda.synchronize()
                ms += ev[0].elapsed_time(ev[1])
            hit = (int(t["stats"][0].item()) - hits0) / (iters * n) if n_cache else 0.0
            out.append(dict(cache_rows=n_cache, target_hit=h, measured_hit=round(hit, 4),
                            us_per_step=round(ms / iters * 1e3, 1)))
    finally:
        torch.cuda.synchronize()
        lib.dlrm_b200_host_unregister(table.data_ptr())
    return out


def model(rows, host, cache):
    e = Engine(128, rows, [13, 512, 256, 128], [479, 1024, 1024, 512, 256, 1], sigmoid_top=4, device=DEV,
               max_batch=2048, gemm="tc", host_tables=host, host_cache_rows=cache)
    e.init_params(seed=0)
    torch.cuda.synchronize()
    return e


def batches(rows, n, seed, dist):
    from dlrm_b200.data import make_batch, to_device_packed

    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        b = to_device_packed(make_batch(rng, rows, 2048, lmax=1, fixed=True), DEV)
        if dist == "zipf":
            idx = b.sparse.indices[0]
            for k, R in enumerate(rows):
                o = b.sparse.offsets[k]
                lo, hi = int(o[0].item()), int(o[-1].item())
                z = (rng.zipf(ZIPF_A, hi - lo).astype(np.uint64) - 1) * np.uint64(2654435761) % np.uint64(R)
                idx[lo:hi] = torch.from_numpy(z.astype(np.int64)).to(idx.dtype).to(DEV)
        out.append(b)
    return out


def step_ms(e, bs, steps, warm=0):
    for i in range(warm):
        b = bs[i % len(bs)]
        e.train_step(b.X, b.sparse, b.target, 0.01, "rwsadagrad")
    torch.cuda.synchronize()
    a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        b = bs[i % len(bs)]
        e.train_step(b.X, b.sparse, b.target, 0.01, "rwsadagrad")
    z.record()
    torch.cuda.synchronize()
    return a.elapsed_time(z) / max(steps, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--shares", default="0,0.02,0.2")
    args = ap.parse_args()
    res = dict(card=card(), mem_available=mem_available(), zipf_exponent=ZIPF_A, warm_steps=WARM)
    rows = 4_000_000
    res["kernels"] = [kernels(rows, 53248, n, [0.0, 0.5, 0.9, 0.99], args.iters) for n in (0, 262144)
                      for _ in range(2)]
    rows10 = [min(r, 10_000_000) for r in TABLE_ROWS]
    host_rows = sum(rows10[k] for k in BIG)
    need = host_rows * ROW
    if need + (16 << 30) > mem_available():
        res["train_10M"] = "not run: %d pinned bytes do not fit MemAvailable %d" % (need, mem_available())
    else:
        ea = model(rows10, [], 0)
        # fresh batches for every step of a host engine: warm, then two timed runs; a cache sees no batch twice
        streams = {d: batches(rows10, WARM + 2 * args.steps, 1, d) for d in ("uniform", "zipf")}
        res["train_10M"] = []
        for share in [float(v) for v in args.shares.split(",")]:
            n = int(host_rows * share) // 32 * 32
            eb = model(rows10, BIG, n)
            for dist, bs in streams.items():
                s0 = eb.host_cache_stats()
                step_ms(eb, bs[:WARM], 0, warm=WARM)
                s1 = eb.host_cache_stats()
                t = {"a_device": [], "b_host": []}
                for r in range(2):
                    run = bs[WARM + r * args.steps:WARM + (r + 1) * args.steps]
                    t["a_device"].append(round(step_ms(ea, run, args.steps), 3))
                    t["b_host"].append(round(step_ms(eb, run, args.steps), 3))
                s2 = eb.host_cache_stats()
                seen = sum(s2[k] - s1[k] for k in ("hits", "inserts", "staged"))
                res["train_10M"].append(dict(cache_rows=n, share_of_host_rows=share, ids=dist, ms_per_step=t,
                                             hit_rate=round((s2["hits"] - s1["hits"]) / max(seen, 1), 4),
                                             evictions_per_step=round((s2["evictions"] - s1["evictions"])
                                                                      / (2 * args.steps), 1),
                                             warm_hit_rate=round((s1["hits"] - s0["hits"]) / max(
                                                 sum(s1[k] - s0[k] for k in ("hits", "inserts", "staged")), 1), 4)))
                print(json.dumps(res["train_10M"][-1]), file=sys.stderr)
            del eb
            gc.collect()
            torch.cuda.empty_cache()
    txt = json.dumps(res)
    print(txt)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_host_cache.json"), "w") as fh:
            fh.write(txt + "\n")


if __name__ == "__main__":
    main()
