"""Regenerate the MLPerf binary-loader fixture and the reference's recorded run on it (tests/test_gpu_bin_records.py):

    python oracle/make_bin_goldens.py [--out DIR]        # default: tests/golden

Writes bin_processed_{train,test}.bin (int32 records [label | 13 dense | 26 ids], from our own generator with a
planted label signal), bin_day_fea_count.npz (table 0 larger than --max-ind-range, so the cap and the modulo act)
and, per run tag, cli_bin_<tag>.flags / cli_bin_<tag>.txt: the reference CLI's 'Finished training', 'Testing at'
and metric lines, recorded through oracle/ref_bin_driver.py.  Test infrastructure: needs the reference checkout."""
import argparse
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(ROOT)
sys.path.insert(0, ROOT)

from dlrm_b200.binrecords import numpy_to_binary  # noqa: E402

COUNTS = np.array([5000, 7, 300, 20, 1500] + [11] * 21)
N_TRAIN, N_TEST = 2000, 1000
RUNS = {
    "A": ["--arch-sparse-feature-size=16", "--arch-mlp-bot=13-64-16", "--arch-mlp-top=64-1", "--max-ind-range=1000",
          "--data-generation=dataset", "--data-set=terabyte", "--loss-function=bce", "--round-targets=True",
          "--learning-rate=0.2", "--nepochs=2", "--mini-batch-size=64", "--print-freq=8", "--test-freq=8",
          "--test-mini-batch-size=256", "--memory-map", "--mlperf-logging", "--mlperf-bin-loader",
          "--numpy-rand-seed=727"],
}
KEEP = re.compile(r"Finished training|Testing at|^recall |reached, stop training")


def data_flags(d):
    return ["--raw-data-file=" + os.path.join(d, "bin_day"),
            "--processed-data-file=" + os.path.join(d, "bin_processed.npz")]


def make_fixture(out):
    rng = np.random.RandomState(2024)

    def split(n, path):
        x_cat = np.stack([rng.randint(0, c, n) for c in COUNTS], 1)
        x_int = rng.randint(0, 300, (n, 13))
        x_int[rng.rand(n, 13) < 0.3] = 0
        z = (x_cat[:, 1] < 3) * 2.0 + (np.log1p(x_int[:, 0]) - 3.0) * 0.8 + (x_cat[:, 0] % 1000 < 300) * 0.5 - 1.0
        y = (rng.rand(n) < 1 / (1 + np.exp(-z))).astype(np.int64)
        numpy_to_binary(y, x_int, x_cat, path)

    split(N_TRAIN, os.path.join(out, "bin_processed_train.bin"))
    split(N_TEST, os.path.join(out, "bin_processed_test.bin"))
    np.savez(os.path.join(out, "bin_day_fea_count.npz"), counts=COUNTS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden"))
    args = ap.parse_args()
    make_fixture(args.out)
    for tag, flags in RUNS.items():
        with open(os.path.join(args.out, "cli_bin_%s.flags" % tag), "w") as fh:
            fh.write(" ".join(flags) + "\n")
        with tempfile.TemporaryDirectory() as tmp:        # the reference writes its TensorBoard run into the cwd
            r = subprocess.run([sys.executable, os.path.join(ROOT, "oracle", "ref_bin_driver.py")] + flags
                               + data_flags(os.path.abspath(args.out)), cwd=tmp, capture_output=True, text=True)
        if r.returncode != 0:
            raise SystemExit("reference CLI failed:\n" + r.stdout[-2000:] + r.stderr[-2000:])
        lines = [ln for ln in r.stdout.splitlines() if KEEP.search(ln)]
        with open(os.path.join(args.out, "cli_bin_%s.txt" % tag), "w") as fh:
            fh.write("\n".join(lines) + "\n")
        print("tag %s: %d lines" % (tag, len(lines)))


if __name__ == "__main__":
    main()
