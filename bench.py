#!/usr/bin/env python
"""bench.py -- samples/s of the DLRM fwd+bwd+optimizer hot path on N H100s.
One "step" = one pass of the hot path (index exchange, forward, loss, backward, fused row-wise-Adagrad embedding
update, dense update) over one synthetic batch.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--workload cfg3|cfg2|cfg1]
                    [--dump-outputs DIR]

Workloads (BASELINE.json configs)
  cfg3 (default, every N): MLPerf-DLRM synthetic -- the config the headline metric is quoted on: 26 tables of the
        Criteo-Terabyte sizes with every table capped at 20 M rows, as the reference's --max-ind-range caps them
        (104.2 M rows x dim 128 = 53.3 GB fp32, 55 GB with the per-row optimizer words: fits one 80 GB H100),
        multi-hot bags of fixed length L_k (214 lookups per sample), bot 13-512-256-128, top
        479-1024-1024-512-256-1, batch 8192 PER GPU (global 65536 at 8 GPUs: weak scaling), fwd+bwd+RWSAdagrad.
        Tables are placed by dlrm_b200/placement.py (cost-balanced, the L=100 / L=27 tables row-split over all
        ranks).
  cfg2: 26 x 1e6 x 128 tables, random bags of <= 10 indices, bot 13-512-256-128, top 479-1024-512-256-1, batch
        2048 per GPU (round 1's headline);  cfg1: cfg2's model, forward only.

Every N (1 included) runs the same sharded engine (one process per GPU; N = 1 is a 1-rank group).  Timing:
a ring of >= 8 distinct pre-generated batches (their touched rows exceed the 50 MB L2 many times over: "inputs
larger than L2"); CUDA events on the launching stream; max over ranks; nvidia-smi clocks sampled during the
timed region.  `value`: the packed batches already sit in HBM.  `e2e`: packed pinned host batches -> one H2D
copy per step (copy stream, double-buffered) -> step -> loss D2H.

--dump-outputs DIR writes what the last device-resident timed step computed (rank 0) as DIR/<name>.npy: the loss,
the predictions, the dense parameters after the update and a fixed, seeded sample of embedding rows and their
accumulators.  Inputs and initial parameters are fixed by seeds, so two builds can be compared output for output.
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import threading
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

CFG3_MAX_ROWS = 20_000_000       # per-table row cap of cfg3 (--max-ind-range): 26 tables fit one 80 GB GPU
DUMP_ROWS = 32768                 # embedding rows in the --dump-outputs sample (16 MB)
CFG2 = dict(m_spa=128, rows=[1_000_000] * 26, ln_bot=[13, 512, 256, 128], top_tail=[1024, 512, 256, 1], B=2048,
            lmax=10, hot=None)


def workload(name, world=1):
    from dlrm_b200 import mlperf as M

    if name == "cfg4":
        # one giant row-split table (8e7 rows x 128 = 42 GB per GPU with the per-row optimizer words, scaled with
        # N: 6.4e8 rows at 8 GPUs) + 25 tables of 1e6 rows, random bags, batch 8192 per GPU (65536 at 8)
        return dict(m_spa=128, rows=[80_000_000 * world] + [1_000_000] * 25, ln_bot=[13, 512, 256, 128],
                    top_tail=[1024, 512, 256, 1], B=8192, lmax=10, hot=None)
    if name == "cfg3":
        return dict(m_spa=M.DIM, rows=[min(r, CFG3_MAX_ROWS) for r in M.TABLE_ROWS], ln_bot=list(M.LN_BOT), top_tail=list(M.TOP_TAIL), B=8192,
                    lmax=None, hot=list(M.MULTI_HOT))
    return dict(CFG2)


def model_dims(W):
    D, T = W["m_spa"], len(W["rows"])
    return D, W["rows"], W["ln_bot"], [D + (T + 1) * T // 2] + W["top_tail"]


def lookups_per_sample(W):
    """Expected embedding rows read per sample and table (the placement cost)."""
    if W["hot"] is not None:
        return [float(h) for h in W["hot"]]
    # round(max(1, u*min(R, lmax))) draws, de-duplicated: ~5.05 at R = 1e6, lmax = 10 (SURVEY 8d)
    return [5.05 if r >= 1000 else min(float(r), 5.0) for r in W["rows"]]


# ------------------------------------------------------------------------------ clocks
class ClockSampler:
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index=0):
        self.rows, self.proc, self.thr, self.gpu = [], None, None, gpu_index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.gpu), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except Exception:
            self.proc = None
            return
        self.thr = threading.Thread(target=self._read, daemon=True)
        self.thr.start()

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), line.strip()))

    def stop(self, t0, t1):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], None, set()
        for ts, line in self.rows:
            f = [x.strip() for x in line.split(",")]
            if len(f) < 9:
                continue
            try:
                clk, mx_ = float(f[1]), float(f[2])
            except ValueError:
                continue
            mx = mx_
            if t0 - 0.05 <= ts <= t1 + 0.15:
                sm.append(clk)
                for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"),
                                     f[5:9]):
                    if val.lower().startswith("active"):
                        reasons.add(name)
        if not sm:  # region shorter than the sampling period: use every sample
            sm = [float(l.split(",")[1]) for _, l in self.rows if len(l.split(",")) >= 9] or [0.0]
        return {"sm_mhz": float(np.median(sm)), "sm_max_mhz": mx, "reasons": sorted(reasons),
                "samples": len(sm)}


# ------------------------------------------------------------------------------ CPU arm
def cpu_arm(args, W, budget_s=20.0, threads=None):
    """The reference's CPU implementation of the path on the host cores, on a bounded sample of the workload:
    the UNMODIFIED reference (oracle/_ref, vendored by build(); kind "reference") when present, else its torch-CPU
    port (oracle/torch_cpu_port.py; kind "port").  Tables larger than `cap` rows are capped (host RAM / init time);
    the bag structure, the MLPs and the optimizer are the workload's."""
    from oracle import live_reference as LR
    from oracle.torch_cpu_port import CpuDLRM, RowWiseAdagradCPU, time_cpu_steps
    from dlrm_b200 import mlperf as M
    from dlrm_b200.data import make_batch

    train = args.workload != "cfg1"
    D, rows, ln_bot, ln_top = model_dims(W)
    cap = 1_000_000
    rows_c = [min(int(r), cap) for r in rows]
    Bc = 2048
    R, where = LR.load()
    kind = "reference" if R is not None else "port"
    if R is not None:
        model, opt = LR.build_model(R, D, rows_c, ln_bot, ln_top, "bce")
    else:
        model = CpuDLRM(D, rows_c, ln_bot, ln_top, loss="bce")
        opt = RowWiseAdagradCPU(model.parameters(), lr=0.01)
    batches = []
    for s in range(4):
        if W["hot"] is not None:
            idx = M.multi_hot_batch(99, s, rows_c, W["hot"], 0, Bc, dtype=np.int64)
            X, T = M.dense_and_targets(99, s, 0, Bc)
            lS_i = [torch.from_numpy(a.reshape(-1)) for a in idx]
            lS_o = [torch.arange(Bc, dtype=torch.int64) * int(h) for h in W["hot"]]
            batches.append((torch.from_numpy(X), lS_o, lS_i, torch.from_numpy(T)))
        else:
            hb = make_batch(np.random.default_rng(99 + s), rows_c, Bc, 13, W["lmax"], pin=False)
            X, lS_o, lS_i, T = hb.reference_format()
            batches.append((X, [o for o in lS_o], lS_i, T))
    if R is not None:      # the reference stacks the offsets (collate_wrapper_random_offset)
        batches = [(X, torch.stack(list(o)), i, T) for X, o, i, T in batches]

    def run(n):
        return time_cpu_steps(model, opt, batches, n, train)

    if threads:
        torch.set_num_threads(threads)
    run(2)  # warm-up
    # "all the host threads it can use": one thread per core is NOT the fastest setting for this sparse,
    # sync-heavy path -- probe a few counts and keep the best
    ncpu = os.cpu_count() or 1
    best = (torch.get_num_threads(), float("inf"))
    if not threads:
        for th in sorted({t for t in (8, 16, 32, 64, ncpu) if t <= ncpu}):
            torch.set_num_threads(th)
            run(1)
            tt = run(2) / 2
            if tt < best[1]:
                best = (th, tt)
        torch.set_num_threads(best[0])
    cores = torch.get_num_threads()
    t1 = run(2) / 2
    n = int(max(3, min(200, budget_s / max(t1, 1e-4))))
    dt = run(n)
    return {"value": n * Bc / dt, "unit": "samples/s", "cores": cores, "kind": kind,
            "sample": "%d steps of batch %d (%s), %s, tables capped at %d rows (host RAM / init time), %s, torch %s "
                      "CPU, %d threads (best of 8/16/32/64/all on a %d-cpu host)" % (
                          n, Bc, args.workload, "fwd+bwd+RWSAdagrad" if train else "fwd only", cap,
                          "unmodified reference dlrm_s_pytorch.DLRM_Net + optim/rwsadagrad.py" if R is not None
                          else "torch-CPU port of the reference path", torch.__version__, cores, ncpu),
            "ms_per_step": 1e3 * dt / n}


def reference_arm(args, W):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    train = args.workload != "cfg1"
    cb = cpu_arm(args, W, budget_s=max(5.0, min(120.0, 1.0 * (args.steps + args.warmup))))
    line = {
        "impl": "reference", "metric": metric_name(train), "value": cb["value"], "unit": "samples/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": cb["ms_per_step"],
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "fp32",
        "data": "synthetic", "config": config_dict(args, W, 1), "cpu_baseline": cb,
        "e2e": {"value": cb["value"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line))


def metric_name(train):
    return "samples/sec (fwd+bwd) MLPerf-DLRM synthetic" if train else "samples/sec (fwd) MLPerf-DLRM synthetic"


def config_dict(args, W, n):
    desc = {"cfg3": "cfg3: MLPerf-DLRM synthetic, 26 Criteo-Terabyte-sized tables capped at 20 M rows (104.18 M rows x 128, "
                    "53.3 GB fp32), "
                    "multi-hot L_k sum 214, bot 13-512-256-128, top 479-1024-1024-512-256-1, batch 8192/GPU, "
                    "fwd+bwd+RWSAdagrad",
            "cfg4": "cfg4: ONE row-split table of 8e7 x N rows x 128 (41 GB fp32 per GPU) + 25 x 1e6 x 128 tables, bot "
                    "13-512-256-128, top 479-1024-512-256-1, batch 8192/GPU, random data Lmax=10, fwd+bwd+RWSAdagrad",
            "cfg2": "cfg2: 26x1e6x128 tables, bot 13-512-256-128, top 479-1024-512-256-1, batch 2048/GPU, random data "
                    "Lmax=10, fwd+bwd+RWSAdagrad",
            "cfg1": "cfg1: cfg2's model, forward only"}[args.workload]
    return {"workload": desc, "global_batch": W["B"] * n,
            "parallelism": ("placement.plan (cost-balanced table-wise + row-split) x%d + dp%d" % (n, n)) if n > 1 else "single",
            "l2_policy": "ring of %d distinct batches (inputs larger than L2)" % args.ring, "gemm": args.gemm}


# ------------------------------------------------------------------------------ our arm
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def parity_check(de_cls, dev, gemm):
    """Two RWSAdagrad steps of tests/golden/cfg0.npz (recorded from the LIVE reference, single process, whole
    batch) through the SAME sharded engine, placement policy and exchange as the timed run: max errors of the loss
    curve, the logits after the steps, the touched table rows and the row-wise accumulators.  The batch (128) is
    split over the ranks; 3 tables on N ranks forces row-split shards for N > 2."""
    import torch.distributed as dist
    from dlrm_b200 import placement as P, sharding as S
    from dlrm_b200.engine import sparse_from_reference

    from oracle import dlrm_numpy as O

    z = dict(np.load(os.path.join(ROOT, "tests", "golden", "cfg0.npz")))
    z.update(np.load(os.path.join(ROOT, "tests", "golden", "cfg0_rwsadagrad.npz")))
    rank, world = dist.get_rank(), dist.get_world_size()
    D, ln_emb = int(z["m_spa"]), [int(v) for v in z["ln_emb"]]
    ln_bot, ln_top = [int(v) for v in z["ln_bot"]], [int(v) for v in z["ln_top"]]
    Bg, T = int(z["B"]), len(ln_emb)
    B = Bg // world
    pl = P.plan(ln_emb, [5.0] * T, world, force_split=[0] if world <= 2 else [])
    de = de_cls(D, ln_emb, ln_bot, ln_top, local_batch=B, device=dev, gemm=gemm, exchange="p2p", placement=pl,
                loss=str(z["loss"]), semantics="single_process")   # the golden is a single-process run of the batch
    params = O.random_params(np.random.default_rng(int(z["seed"])), D, ln_emb, ln_bot, ln_top)   # the golden's weights
    de.eng.load_params(S.slice_params(params, pl, rank))
    lr = float(z["rwsadagrad_lr"])
    nsteps = int(z["nsteps"])
    sl = slice(rank * B, (rank + 1) * B)
    losses = []

    def batch(s):
        per_table = [(torch.from_numpy(z["b%d_off" % s][k]), torch.from_numpy(z["b%d_idx%d" % (s, k)])) for k in range(T)]
        st = S.local_streams(per_table, pl, rank)
        sp = sparse_from_reference([o for o, _ in st], [i for _, i in st], dev)
        X = torch.from_numpy(z["b%d_X" % s][sl].copy()).to(dev)
        Tt = torch.from_numpy(z["b%d_T" % s][sl].copy()).to(dev)
        return X, sp, Tt

    for s in range(nsteps):
        X, sp, Tt = batch(s)
        l = de.train_step(X, sp, Tt, lr, "rwsadagrad").clone()
        if world > 1:
            dist.all_reduce(l, op=dist.ReduceOp.AVG)
        losses.append(float(l.item()))
    X, sp, Tt = batch(nsteps)
    p = de.forward(X, sp).cpu().numpy()
    err = {"loss": float(np.abs(np.array(losses) - z["rwsadagrad_losses"]).max()),
           "p_after": float(np.abs(p - z["rwsadagrad_p_after"][sl]).max()), "rows_p999": 0.0, "momentum": 0.0}
    for j, s_ in enumerate(pl.of_rank(rank)):
        k = s_.table
        rows, vals = z["rwsadagrad_emb%d_rows" % k], z["rwsadagrad_emb%d_vals" % k]
        m = (rows >= s_.row_lo) & (rows < s_.row_hi)
        if m.any():
            got = de.eng.table(j).cpu().numpy()[rows[m] - s_.row_lo]
            err["rows_p999"] = max(err["rows_p999"], float(np.quantile(np.abs(got - vals[m]), 0.999)))
        mom = de.eng.momentum[int(de.eng.row_base[j]):int(de.eng.row_base[j + 1])].cpu().numpy()
        ref = z["rwsadagrad_mom%d" % k][s_.row_lo:s_.row_hi]
        err["momentum"] = max(err["momentum"], float(np.abs(mom - ref).max() / max(float(np.abs(ref).max()), 1e-30)))
    t = torch.tensor([err["loss"], err["p_after"], err["rows_p999"], err["momentum"]], device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    err = dict(zip(("loss", "p_after", "rows_p999", "momentum_rel"), [float(v) for v in t.tolist()]))
    err.update(golden="tests/golden/cfg0.npz (live reference, 2 RWSAdagrad steps, global batch 128)",
               split_tables=pl.split_tables(), ok=bool(err["loss"] < 3e-4 and err["p_after"] < 5e-3))
    return err      # the (tiny) engine stays alive: its buffers are mapped into the peers


class Progress:
    """Stage log + watchdog.  Every stage is announced on stderr (rank 0; all ranks with DLRM_BENCH_VERBOSE=1) with
    the seconds since start, so that a stalled run says WHERE it stalled.  A daemon thread watches the time spent in
    the current stage: past the limit (DLRM_BENCH_STAGE_LIMIT seconds, default 240, once a number has been measured;
    DLRM_BENCH_SETUP_LIMIT, default 1500, before) rank 0 prints the bench line
    with whatever has been measured so far plus an "error" field, and every rank leaves with os._exit -- a stuck
    collective or a spinning kernel would otherwise hold the job until the caller's own timeout with no line at all.
    Optional stages (parity check, kernel rooflines, phase timeline) run AFTER the timed regions for that reason."""

    def __init__(self, rank):
        import threading

        self.rank, self.t0 = rank, time.time()
        self.stage_name, self.stage_t = "start", self.t0
        # before a number exists a stall can only be reported, so the limit is long (cold 8-GPU boxes take minutes
        # to bring NCCL up); after it, the optional stages get DLRM_BENCH_STAGE_LIMIT seconds each
        self.limit = float(os.environ.get("DLRM_BENCH_STAGE_LIMIT", "240"))
        self.limit_before_value = max(self.limit, float(os.environ.get("DLRM_BENCH_SETUP_LIMIT", "1500")))
        self.verbose = rank == 0 or os.environ.get("DLRM_BENCH_VERBOSE") == "1"
        self.line = None              # filled by the main flow as results arrive (rank 0)
        self.extra = {}
        self.printed = False
        self.lock = threading.Lock()
        self.done = False
        threading.Thread(target=self._watch, daemon=True).start()

    def stage(self, name):
        self.stage_name, self.stage_t = name, time.time()
        if self.verbose:
            print("[bench r%d %6.1fs] %s" % (self.rank, self.stage_t - self.t0, name), file=sys.stderr, flush=True)

    def emit(self, error=None):
        """Print the bench line once (rank 0)."""
        with self.lock:
            if self.printed or self.rank != 0 or self.line is None:
                return
            self.printed = True
            line = dict(self.line)
            line.update(self.extra)
            if error:
                line["error"] = error
            print(json.dumps(line), flush=True)

    def _watch(self):
        while not self.done:
            time.sleep(2.0)
            dt = time.time() - self.stage_t
            measured = self.line is not None or (self.rank != 0 and self.stage_name.startswith(("parity", "teardown", "phase")))
            if not self.done and dt > (self.limit if measured else self.limit_before_value):
                msg = "stalled in stage '%s' for %.0f s (rank %d)" % (self.stage_name, dt, self.rank)
                print("[bench r%d] WATCHDOG: %s" % (self.rank, msg), file=sys.stderr, flush=True)
                have_value = self.line is not None and self.line.get("value") is not None
                if self.rank == 0 and self.line is None:
                    self.line = {"metric": None, "value": None}
                self.emit(error=msg)
                # other ranks past the timed regions: rank 0 reports, they just leave
                os._exit(0 if have_value or (self.rank != 0 and measured) else 3)


def ours(args, W):
    import torch.distributed as dist
    from dlrm_b200 import dist as ddist, placement as P
    from dlrm_b200.data import DeviceBatch
    from dlrm_b200.engine import GraphedTrainStep

    if "RANK" not in os.environ:       # N = 1 without a launcher: a 1-rank group
        os.environ.update(RANK="0", WORLD_SIZE="1", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1",
                          MASTER_PORT=str(_free_port()))
    prog = Progress(int(os.environ.get("RANK", "0")))
    prog.stage("process group (NCCL bring-up)")
    # NCCL only brings the job up (handles, scalars, barriers): no NVLS / multicast setup is needed for that
    os.environ.setdefault("NCCL_NVLS_ENABLE", "0")
    rank, world = ddist.init_distributed("nccl")
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    dev = os.environ.get("DLRM_BENCH_TEST_DEVICE") or "cuda:%d" % local     # (tests/test_bench_host.py drives the flow on fakes)
    torch.cuda.set_device(local)
    warm = torch.zeros(1, device=dev)      # create the communicator now: NCCL prints its version line to stdout at
    dist.all_reduce(warm)                  # the first collective, and the JSON line must be the LAST line
    torch.cuda.synchronize()
    train = args.workload != "cfg1"
    D, rows, ln_bot, ln_top = model_dims(W)
    B, T = W["B"], len(rows)
    cost = lookups_per_sample(W)
    prog.stage("engine: placement, tables, peer mappings")
    pl = P.plan(rows, cost, world)
    de = ddist.DistEngine(D, rows, ln_bot, ln_top, local_batch=B, device=dev, gemm=args.gemm, exchange="p2p",
                          placement=pl, split_forward=args.split_forward)
    de.eng.init_params(100 + rank)
    if world > 1:
        de.sync_dense_params_from_rank0()
    de.eng.ensure_optimizer_state("rwsadagrad")
    lr = 0.01
    nsets = 2
    fixed = W["hot"] is not None
    prog.stage("inputs: host batches, device ring, index exchange buffers")
    # ---- inputs: a ring of packed pinned host batches (this rank's share) + their device copies
    if fixed:
        mh = ddist.MultiHotExchange(de, W["hot"], 13, nsets)
        host = [mh.fill_host(mh.host_buffer(), 1234, i, rows) for i in range(args.ring)]
        devr = [h.to(dev) for h in host]
        stages = [types.SimpleNamespace(sparse=mh.sparse[k], X=mh.X[k], target=mh.target[k]) for k in range(nsets)]

        def pre(k):
            return lambda: mh.exchange(k)

        def load_dev(k, i):
            mh.stage[k].copy_(devr[i % args.ring], non_blocking=True)

        def load_host(k, i):
            return mh.upload(k, host[i % args.ring])
    else:
        hostb = [ddist.make_sharded_batch(1000 + i, rows, rank, world, B, 13, W["lmax"], placement=pl)
                 for i in range(args.ring)]
        devb = []
        for hb, X, Tt in hostb:
            db = DeviceBatch(hb.layout, dev)
            db.load(hb, non_blocking=False)
            devb.append((db, X.to(dev), Tt.to(dev)))
        sdb = [DeviceBatch(hostb[0][0].layout, dev) for _ in range(nsets)]
        for s_ in sdb:
            s_.load(hostb[0][0], non_blocking=False)
        stages = [types.SimpleNamespace(sparse=sdb[k].sparse, X=devb[0][1].clone(), target=devb[0][2].clone())
                  for k in range(nsets)]

        def pre(k):
            return None

        def load_dev(k, i):
            db, Xd, Td = devb[i % args.ring]
            n = db.layout.used(db.nnz)
            sdb[k].buf[:n].copy_(db.buf[:n], non_blocking=True)
            stages[k].X.copy_(Xd, non_blocking=True)
            stages[k].target.copy_(Td, non_blocking=True)

        def load_host(k, i):
            hb, Xh, Th = hostb[i % args.ring]
            n = sdb[k].load(hb)
            stages[k].X.copy_(Xh, non_blocking=True)
            stages[k].target.copy_(Th, non_blocking=True)
            return n + Xh.numel() * 4 + Th.numel() * 4
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    graphs = None
    prog.stage("CUDA graph capture (3 eager steps + capture per buffer set)")
    if not args.no_graph:
        graphs = [GraphedTrainStep(de.eng, stages[k], lr, "rwsadagrad", train=train, pre=pre(k)) for k in range(nsets)]

    def run_set(k):
        if graphs is not None:
            return graphs[k].replay()
        p = pre(k)
        if p is not None:
            p()
        if train:
            return de.eng.train_step(stages[k].X, stages[k].sparse, stages[k].target, lr, "rwsadagrad")
        return de.eng.forward(stages[k].X, stages[k].sparse)

    def sync_all():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    def resident_step(i):
        k = i % nsets
        load_dev(k, i)
        return run_set(k)

    prog.stage("warm-up steps")
    for w in range(args.warmup):
        resident_step(w)
    sync_all()
    prog.stage("timed steps (device-resident inputs)")
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
        time.sleep(0.25)
    sync_all()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.time()
    n0 = de.eng.n_launch
    ev0.record()
    for r in range(args.steps):
        out = resident_step(args.warmup + r)
    ev1.record()
    sync_all()
    t1 = time.time()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, de.eng, out, B, train)
    launches = de.eng.n_launch - n0
    ms = torch.tensor([ev0.elapsed_time(ev1) / args.steps], device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms.item())
    if rank == 0:       # from here on a stall still yields a line with the device-resident number
        prog.line = {"metric": metric_name(train), "value": B * world / (ms * 1e-3), "unit": "samples/s", "n_gpus": world,
                     "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True,
                     "scaling": "weak", "vs_baseline": None, "data": "synthetic", "config": config_dict(args, W, world),
                     "gpu_launches": int(launches), "e2e": None}

    prog.stage("timed steps (end to end: H2D + step + loss D2H)")
    # ---- e2e: host buffers; H2D of the packed batch + D2H of the loss inside the timed region
    copy_stream = torch.cuda.Stream()
    loss_host = torch.zeros(1).pin_memory()
    main = torch.cuda.current_stream()
    h2d = 0

    def e2e_loop(nsteps, base):
        nonlocal h2d
        ready = [torch.cuda.Event() for _ in range(nsets)]
        freed = [torch.cuda.Event() for _ in range(nsets)]
        for f in freed:
            f.record(main)
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(freed[0])
            h2d += load_host(0, base)
            ready[0].record(copy_stream)
        for r in range(nsteps):
            cur, nxt = r % nsets, (r + 1) % nsets
            if r + 1 < nsteps:
                with torch.cuda.stream(copy_stream):
                    copy_stream.wait_event(freed[nxt])
                    h2d += load_host(nxt, base + r + 1)
                    ready[nxt].record(copy_stream)
            main.wait_event(ready[cur])
            out = run_set(cur)
            loss_host.copy_(out.view(-1)[-1:], non_blocking=True)
            freed[cur].record(main)
        main.synchronize()

    e2e_loop(max(args.warmup // 2, 2), 0)
    h2d = 0
    sync_all()
    ev0.record()
    e2e_loop(args.steps, 5)
    ev1.record()
    sync_all()
    ms2 = torch.tensor([ev0.elapsed_time(ev1) / args.steps], device=dev)
    if world > 1:
        dist.all_reduce(ms2, op=dist.ReduceOp.MAX)
    ms2 = float(ms2.item())
    # per-rank gather bytes (balance of the placement)
    gb = torch.tensor([de.gather_bytes_per_step(cost)], device=dev, dtype=torch.float64)
    gbs = [torch.zeros_like(gb) for _ in range(world)]
    if world > 1:
        dist.all_gather(gbs, gb)
    else:
        gbs = [gb]
    gbs = [float(g.item()) for g in gbs]

    if rank == 0:
        clocks = sampler.stop(t0, t1)
        Bg = B * world
        prog.line = {
            "metric": metric_name(train), "value": Bg / (ms * 1e-3), "unit": "samples/s", "n_gpus": world,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None,
            "dtype": {"simt": "fp32", "tc": "fp32 (bf16x3 split on wgmma, fp32 accumulate)", "tc_bf16": "bf16"}[args.gemm],
            "data": "synthetic", "config": config_dict(args, W, world),
            "roofline": None, "roofline_update": None, "cpu_baseline": None,
            "e2e": {"value": Bg / (ms2 * 1e-3), "unit": "samples/s", "h2d_bytes_per_step": int(h2d / args.steps),
                    "d2h_bytes_per_step": 4, "ms_per_step": ms2,
                    "note": "per rank: ONE packed pinned buffer with ITS samples (dense, targets, int32 indices of all "
                            "tables) -> one H2D copy on a copy stream (double-buffered) -> index exchange over NVLink + "
                            "step in one CUDA graph -> loss read back" if fixed else
                            "per rank: packed pinned sparse batch (its tables, global batch) + dense slice, H2D every "
                            "step, loss read back"},
            "gpu_launches": int(launches), "exchange": "p2p (peer-mapped stores over NVLink, own barriers)",
            "cuda_graph": graphs is not None,
            "nvlink": de.nvlink_bytes_per_step(ms * 1e-3, mh.nbytes if fixed else 0, cost),
            "split_forward": args.split_forward,
            "placement": {"split_tables": pl.split_tables(), "imbalance": pl.imbalance(),
                          "gather_bytes_per_rank_per_step": gbs,
                          "gather_bytes_max_over_min": max(gbs) / max(min(gbs), 1.0)},
            "parity_check": None, "clocks": clocks,
        }
    # ---- the stages below add fields to the line; if one of them stalls the watchdog prints the line without it
    if not args.no_check and train:
        prog.stage("parity check: golden cfg0 through the same sharded engine / placement policy / exchange")
        try:
            prog.extra["parity_check"] = parity_check(ddist.DistEngine, dev, args.gemm)
        except Exception as exc:      # the measured numbers above are still reported, with the failure next to them
            prog.extra["parity_check"] = {"ok": False, "error": repr(exc)[:400]}
    # Rank 0 ALONE times its gather / update kernels (at N > 1 the other ranks wait in the next collective): the loop
    # refreshes the indices between a link and its update without the step's barriers, which is only safe while no
    # peer is running its own link / update on indices this rank's exchange overwrites.
    if rank == 0:
        prog.stage("kernel rooflines (gather, gather+link, update between CUDA events)")
        peaks = {}
        try:
            with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as fh:
                peaks = json.load(fh)
        except Exception:
            pass
        hbm_peak = float(peaks.get("hbm_gbs", 3350.0))
        peak_src = ("measured (MEASURED_PEAKS.json hbm_gbs)" if "hbm_gbs" in peaks
                    else "H100 SXM data sheet 3350 GB/s (not a measured peak)")
        try:
            roof, roof_upd = measure_rooflines(de, stages, load_dev, pre, args, W, cost, hbm_peak, peak_src, train)
            prog.extra.update(roofline=roof, roofline_update=roof_upd)
        except Exception as exc:
            prog.extra["roofline"] = {"error": repr(exc)[:400]}
        if not args.no_cpu and world == 1:
            prog.stage("cpu baseline (live reference on the host cores)")
            prog.stage_t += 600.0          # building the reference model's 13 GB of tables takes a while
            try:
                prog.extra["cpu_baseline"] = cpu_arm(args, W, budget_s=args.cpu_budget)
            except Exception as exc:
                prog.extra["cpu_baseline"] = {"error": repr(exc)[:400]}
        prog.stage("bench line")
        prog.emit()
    # ---- optional phase timeline (eager launches, timing events on every stream): where the step's time goes
    if args.phases > 0:
        prog.stage("phase timeline (eager steps)")
        acc = {}
        order = []
        for r in range(args.phases + 2):
            k = r % nsets
            load_dev(k, r)
            sync_all()
            de.eng._marks = []
            de.eng._mark("step_begin")
            p = pre(k)
            if p is not None:
                p()
                de.eng._mark("index_exchange")
            if train:
                de.eng.train_step(stages[k].X, stages[k].sparse, stages[k].target, lr, "rwsadagrad")
            else:
                de.eng.forward(stages[k].X, stages[k].sparse)
            de.eng._mark("step_end")
            torch.cuda.synchronize()
            marks, de.eng._marks = de.eng._marks, None
            if r < 2:
                continue
            for name, ev in marks[1:]:
                if name not in acc:
                    acc[name] = []
                    order.append(name)
                acc[name].append(marks[0][1].elapsed_time(ev) * 1e3)
        phases = {"n_gpus": world, "workload": args.workload, "unit": "us after step_begin (event recorded when the named phase finished on its stream; "
                          "'emb:' = embedding stream; eager launches, mean of %d steps)" % args.phases,
                  "marks": [[n, round(float(np.mean(acc[n])), 1)] for n in order]}
        if rank == 0:       # AFTER the bench line (a separate stderr line + file): the bench line stays the one stdout line
            print("phases " + json.dumps(phases), file=sys.stderr, flush=True)
            if args.phases_out:
                with open(args.phases_out, "w") as fh:
                    json.dump(phases, fh)
    prog.stage("teardown")
    try:
        if world > 1:
            dist.barrier()
        prog.done = True
        dist.destroy_process_group()
    except Exception as exc:      # the line is out; a failed optional stage must not turn into a failed run
        prog.done = True
        print("[bench r%d] teardown: %r" % (rank, exc), file=sys.stderr, flush=True)
        sys.stdout.flush()
        os._exit(0)


def dump_outputs(path, eng, out, B, train):
    """The arrays the last timed step computed, as float32 / float64 .npy files under `path` (< 64 MB in all)."""
    os.makedirs(path, exist_ok=True)
    arrays = {"p": out} if not train else {"loss": out.view(-1), "p": eng.top_act[-1][:B], "dense_params": eng.dense}
    if train:
        g = torch.Generator().manual_seed(0)
        idx = torch.randint(0, eng.total_rows, (DUMP_ROWS,), generator=g).sort().values.to(eng.tables.device)
        arrays.update(emb_rows=eng.tables[idx, :eng.D], emb_accumulator=eng.momentum[idx],
                      emb_row_index=idx.double())
    for name, t in arrays.items():
        a = t.detach().cpu().numpy()
        np.save(os.path.join(path, name + ".npy"), a if a.dtype == np.float64 else a.astype(np.float32))


def measure_rooflines(de, stages, load_dev, pre, args, W, cost, hbm_peak, peak_src, train):
    """The HBM-bound kernels timed with CUDA events on the launching stream (N = 1): the forward gather alone
    (back-to-back launches over the batch ring) and, for training, (gather+link, update) pairs."""
    eng = de.eng
    D, B, T = eng.D, de.Bg, len(W["rows"])
    n = max(min(args.steps, 64), 16)
    k = 0
    pk = pre(k)

    def prep(i):
        load_dev(k, i)
        if pk is not None:
            pk()

    for i in range(3):
        prep(i)
        eng.emb_forward(stages[k].sparse)
    torch.cuda.synchronize()
    def hold_gpu():
        # The host needs ~0.1-0.2 ms per iteration to build the launch descriptors; with an empty queue that time would
        # sit between the two events of a short kernel.  A spin kernel first, so that every launch of the loop is
        # already queued when the GPU reaches it.
        if hasattr(torch.cuda, "_sleep"):
            torch.cuda._sleep(int(4e5) * (n + 8))         # ~0.2 ms of spinning per queued iteration

    # gather alone: the index refresh (D2D + exchange) sits between the timed launches, so bracket each launch
    evs = []
    hold_gpu()
    for i in range(n):
        prep(i)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.emb_forward(stages[k].sparse)
        eng.reduce_partials(de.B)
        e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    tg = float(np.median([a.elapsed_time(b) for a, b in evs])) * 1e-3
    # this rank's share: the rows of its shards the global batch touches, all index words of its shards (a shard
    # scans every occurrence of its table), one pooled row per (sample, shard)
    nnz = de.gather_bytes_per_step(cost) / (D * 4)
    scanned = float(sum(cost[s.table] for s in de.mine)) * B
    T = len(de.mine)
    idx_b = 4 if W["hot"] is not None else 8
    by = nnz * D * 4 + scanned * idx_b + T * B * idx_b + T * B * D * 4  # SURVEY 8(d): rows + indices + offsets + pooled out
    ach = by / tg / 1e9
    roof = {"kernel": "emb_fwd_vec_kernel (multi-table EmbeddingBag gather, forward)", "bound": "hbm", "achieved": ach,
            "peak": hbm_peak, "unit": "GB/s", "frac": ach / hbm_peak, "peak_source": peak_src,
            "avg_launch_us": tg * 1e6, "algorithmic_bytes_per_launch": by,
            "how": "CUDA events around each gather launch on the launching stream, median of %d over the batch ring" % n}
    roof_upd = None
    if train:
        eng.dT.normal_()
        eng.head.zero_()
        evs = []
        hold_gpu()
        for i in range(n + 3):
            prep(i)
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e0.record()
            eng.emb_forward(stages[k].sparse, link=True)
            eng.reduce_partials(de.B)
            e1.record()
            eng.emb_update(stages[k].sparse, optimizer="rwsadagrad", lr=1e-6)
            e2.record()
            if i >= 3:
                evs.append((e0, e1, e2))
        torch.cuda.synchronize()
        t_gl = float(np.median([a.elapsed_time(b) for a, b, _ in evs])) * 1e-3
        tu = float(np.median([b.elapsed_time(c) for _, b, c in evs])) * 1e-3
        by_u = nnz * (D * 4 * 2 + 8) + T * B * D * 4 + scanned * idx_b  # SURVEY 8(d) bytes_bwd (unique rows ~ nnz)
        achu = by_u / tu / 1e9
        roof_upd = {"kernel": "emb_update_kernel (+ emb_small_*: coalesce + row-wise Adagrad, in place)", "bound": "hbm",
                    "achieved": achu, "peak": hbm_peak, "unit": "GB/s", "frac": achu / hbm_peak,
                    "avg_launch_us": tu * 1e6, "algorithmic_bytes_per_launch": by_u,
                    "train_gather_plus_link_us": t_gl * 1e6,
                    "train_gather": {"achieved": by / t_gl / 1e9, "frac": by / t_gl / 1e9 / hbm_peak},
                    "how": "CUDA events between the launches of (gather+link, update) pairs, medians"}
    return roof, roof_upd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="cfg3", choices=["cfg3", "cfg2", "cfg1", "cfg4"])
    ap.add_argument("--ring", type=int, default=8)
    ap.add_argument("--gemm", default="tc", choices=["tc", "tc_bf16"])
    ap.add_argument("--split-forward", default="partial", choices=["partial", "remote"],
                    help="row-split tables: every rank pools a partial sum of its rows (partial), or the sample's owner "
                         "reads the rows from their owners over NVLink inside the gather (remote)")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--phases", type=int, default=0, help="also record a per-phase timeline over this many eager steps")
    ap.add_argument("--phases-out", default=None)
    ap.add_argument("--no-check", action="store_true", help="skip the pre-run parity check against the live-reference golden")
    ap.add_argument("--cpu-budget", type=float, default=15.0)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the arrays the last timed step computed to DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if args.dump_outputs and args.impl != "ours":
        ap.error("--dump-outputs writes what the GPU path computed; it needs --impl ours")
    args.warmup = max(args.warmup, 3)
    W = workload(args.workload, max(int(os.environ.get("WORLD_SIZE", "1")), 1))
    if args.impl == "reference":
        return reference_arm(args, W)
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; dlrm_b200 has no CPU path (use --impl reference for the CPU arm)")
    ours(args, W)


if __name__ == "__main__":
    main()
