"""The command line with and without --cuda-graph-steps on bench/run_and_time.sh's model.

  python tools/bench_cli_graph_steps.py [--batches 1000] [--rounds 2] [--out DIR]

Synthetic MLPerf binary records (uniform labels, dense counts and ids; the 26 MLPerf table sizes capped at 10 M rows,
fp32 tables, batch 2048, one test pass over 3 x 16384 records at the end) are written to a temporary directory, and
`dlrm_s_pytorch.py` with run_and_time.sh's flags trains on them, alternating eager (a) and graphed (b) runs: a, b, a, b.
Per run: ms/it of every --print-time window after the first (the first one holds the warm-up), and the wall time of the
test pass, from its "Testing at" line to its metric line.  Prints one JSON object; the card's name, power limit and
max SM clock come first."""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dlrm_b200.binrecords import numpy_to_binary  # noqa: E402
from dlrm_b200.mlperf import TABLE_ROWS  # noqa: E402

B, TEST_B, CAP, PRINT = 2048, 16384, 10_000_000, 100


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def write_records(d, n_train, n_test, seed=0):
    rng = np.random.default_rng(seed)
    for name, n in (("train", n_train), ("test", n_test)):
        y = rng.integers(0, 2, n)
        x_int = rng.integers(0, 1000, (n, 13))
        x_cat = rng.integers(0, np.minimum(np.asarray(TABLE_ROWS), CAP), (n, 26))
        numpy_to_binary(y, x_int, x_cat, os.path.join(d, "terabyte_processed_%s.bin" % name))
    np.savez(os.path.join(d, "day_fea_count.npz"), counts=np.asarray(TABLE_ROWS, dtype=np.int64))


def run(d, batches, graphed):
    flags = ["--arch-sparse-feature-size=128", "--arch-mlp-bot=13-512-256-128", "--arch-mlp-top=1024-1024-512-256-1",
             "--max-ind-range=%d" % CAP, "--data-generation=dataset", "--data-set=terabyte",
             "--raw-data-file=" + os.path.join(d, "day"),
             "--processed-data-file=" + os.path.join(d, "terabyte_processed.npz"), "--loss-function=bce",
             "--round-targets=True", "--learning-rate=1.0", "--mini-batch-size=%d" % B, "--print-freq=%d" % PRINT,
             "--print-time", "--test-freq=%d" % batches, "--test-mini-batch-size=%d" % TEST_B, "--memory-map",
             "--mlperf-logging", "--mlperf-bin-loader", "--mlperf-bin-shuffle", "--use-gpu"]
    if graphed:
        flags.append("--cuda-graph-steps")
    p = subprocess.Popen([sys.executable, "-u", os.path.join(ROOT, "dlrm_s_pytorch.py")] + flags, cwd=d,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    lines = []
    for ln in p.stdout:
        lines.append((time.perf_counter(), ln.rstrip("\n")))
    if p.wait() != 0:
        raise RuntimeError("run failed:\n" + "\n".join(ln for _, ln in lines[-30:]))
    ms = [float(m.group(1)) for _, ln in lines for m in [re.search(r"([0-9.]+) ms/it", ln)] if m]
    t_test = next(t for t, ln in lines if ln.startswith("Testing at"))
    t_done = next(t for t, ln in lines if ln.startswith("recall "))
    report = [ln for _, ln in lines if ln.startswith("CUDA-graph steps")]
    losses = [float(v) for _, ln in lines for v in re.findall(r"Finished training it .* loss ([0-9.]+)", ln)]
    return {"ms_per_it": ms[1:], "ms_per_it_median": float(np.median(ms[1:])), "test_pass_s": t_done - t_test,
            "last_loss": losses[-1], "metrics": next(ln for _, ln in lines if ln.startswith("recall ")),
            "graph_report": report[0] if report else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    d = tempfile.mkdtemp(prefix="cli_graph_steps_")
    try:
        write_records(d, a.batches * B, 3 * TEST_B)
        res = {"card": card(), "batch": B, "test_batch": TEST_B, "row_cap": CAP, "train_batches": a.batches,
               "runs": []}
        for r in range(a.rounds):
            for graphed in (False, True):
                out = run(d, a.batches, graphed)
                out.update(round=r, mode="graphed" if graphed else "eager")
                res["runs"].append(out)
                print(json.dumps(out), file=sys.stderr, flush=True)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    txt = json.dumps(res)
    print(txt)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_cli_graph_steps.json"), "w") as f:
            f.write(txt)


if __name__ == "__main__":
    main()
