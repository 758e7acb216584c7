"""Regenerate the processed Criteo Kaggle fixture and the reference's recorded runs on it (tests/test_gpu_criteo_dataset.py,
tests/test_criteo_dataset_host.py):

    python oracle/make_kaggle_goldens.py [--out DIR]        # default: tests/golden

1. Writes a deterministic synthetic Kaggle-format train.txt (label, 13 counts, 26 hex categoricals, tab separated;
   empty fields, negative counts, skewed cardinalities) of N_LINES lines: 7 "days" of 200, so train is 1200 samples
   (a short last batch at 32 and 64) and test / val are 100 each.
2. Runs the UNMODIFIED reference CLI on the CPU once to preprocess it (data_utils.getCriteoAdData), then records
   runs A-C with the processed files in place.  Writes kaggle_processed.npz, kaggle_day_count.npz,
   kaggle_fea_count.npz and, per run, cli_kaggle_<tag>.flags / cli_kaggle_<tag>.txt (the dataset, training, test
   and metric lines of stdout).
3. Dumps the reference CriteoDataset's sample order of every split and randomize mode, numpy's global RNG state
   after the train and test constructors (kaggle_orders.npz), and its __getitem__ + collate_wrapper_criteo_offset
   batches of two splits (kaggle_batches.npz).

Test infrastructure: needs the reference checkout (DLRM_REFERENCE)."""
import argparse
import contextlib
import io
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("DLRM_REFERENCE", "/root/reference")

N_LINES = 1400
CARD = [2, 3, 5, 7, 10, 20, 30, 50, 80, 100, 150, 200, 300, 400, 500, 700, 900, 1100, 4, 6, 12, 25, 60, 250, 1, 40]
COMMON = ["--arch-sparse-feature-size=16", "--arch-mlp-bot=13-64-16", "--arch-mlp-top=64-1", "--data-generation=dataset",
          "--data-set=kaggle", "--loss-function=bce", "--round-targets=True", "--numpy-rand-seed=727"]
RUNS = {
    "A": COMMON + ["--learning-rate=0.1", "--optimizer=sgd", "--data-randomize=total", "--mini-batch-size=32",
                   "--nepochs=2", "--print-freq=8", "--test-freq=16", "--test-mini-batch-size=48"],
    "B": COMMON + ["--learning-rate=0.05", "--optimizer=rwsadagrad", "--data-randomize=day", "--max-ind-range=40",
                   "--mini-batch-size=64", "--nepochs=1", "--print-freq=4", "--test-freq=10"],
    "C": COMMON + ["--learning-rate=0.1", "--data-randomize=none", "--mini-batch-size=32", "--nepochs=1",
                   "--print-freq=10", "--test-freq=19", "--test-mini-batch-size=64", "--mlperf-logging"],
}
KEEP = re.compile(r"Sparse fea|Randomized|Defined|Split data|Finished training|Testing at|accuracy|^recall ")


def write_train_txt(path):
    rng = np.random.RandomState(1234)
    with open(path, "w") as f:
        for _ in range(N_LINES):
            ints = rng.geometric(0.05, 13) - 1
            ints[rng.rand(13) < 0.1] -= rng.randint(1, 4)            # negative counts: clipped to 0 by preprocessing
            z = (ints[0] > 20) * 1.5 + (ints[1] % 3 == 0) * 0.5 - 1.0
            fields = [str(int(rng.rand() < 1 / (1 + np.exp(-z))))]
            fields += ["" if rng.rand() < 0.15 else str(v) for v in ints]           # empty fields read as 0
            for c in CARD:
                v = min(int(rng.zipf(1.3)) - 1, c - 1)                 # skewed: most lines hit a few values
                fields.append("" if rng.rand() < 0.05 else "%08x" % ((v * 2654435761 + c) & 0x7FFFFFFF))
            f.write("\t".join(fields) + "\n")


def data_flags(d, processed):
    return ["--raw-data-file=" + os.path.join(d, "kaggle.txt"), "--processed-data-file=" + os.path.join(d, processed)]


def reference_cli(flags, cwd):
    r = subprocess.run([sys.executable, os.path.join(HERE, "ref_bin_driver.py")] + flags, cwd=cwd,
                       capture_output=True, text=True, env=dict(os.environ, DLRM_REFERENCE=REF))
    if r.returncode != 0:
        raise SystemExit("reference CLI failed:\n" + r.stdout[-2000:] + r.stderr[-2000:])
    return r.stdout


def dump_orders_and_batches(d, out):
    """The reference CriteoDataset on a copy of the processed file whose X_int[:, 0] is the row number: each split's
    rows then name their positions.  Batches come from the unmodified file."""
    sys.path[:0] = [REF]
    import dlrm_data_pytorch as dp

    with np.load(os.path.join(d, "kaggle_processed.npz")) as z:
        arrays = {k: z[k] for k in z.files}
    tag_dir = os.path.join(d, "tagged")
    os.makedirs(tag_dir)
    shutil.copy(os.path.join(d, "kaggle_day_count.npz"), tag_dir)
    tagged = dict(arrays, X_int=arrays["X_int"].copy())
    tagged["X_int"][:, 0] = np.arange(len(tagged["y"]))
    np.savez(os.path.join(tag_dir, "p.npz"), **tagged)

    def make(path, mode, split, mir=-1):
        with contextlib.redirect_stdout(io.StringIO()):
            return dp.CriteoDataset("kaggle", mir, 0.0, mode, split, os.path.join(path, "kaggle.txt"),
                                    os.path.join(path, "p.npz" if path == tag_dir else "kaggle_processed.npz"))

    rows = {}
    for mode in ("none", "day", "total"):
        np.random.seed(727)
        for split in ("train", "test"):
            rows["%s_%s" % (mode, split)] = np.array([r[0] for r in make(tag_dir, mode, split).X_int], np.int64)
        st = np.random.get_state()
        rows["rng_%s_keys" % mode], rows["rng_%s_pos" % mode] = st[1].copy(), np.int64(st[2])
        rows["%s_val" % mode] = np.array([r[0] for r in make(tag_dir, mode, "val").X_int], np.int64)
    # split "none" permutes local copies of the arrays and keeps none of them (:215-223): only its draw is recorded
    np.random.seed(5)
    make(tag_dir, "total", "none")
    st = np.random.get_state()
    rows["rng_split_none_keys"], rows["rng_split_none_pos"] = st[1].copy(), np.int64(st[2])
    np.savez_compressed(os.path.join(out, "kaggle_orders.npz"), **rows)

    batches = {}
    for name, mode, split, mir, bs in (("train", "total", "train", 40, 32), ("test", "none", "test", -1, 48)):
        np.random.seed(727)
        ds = make(d, mode, split, mir)
        for j, lo in enumerate(range(0, len(ds), bs)):
            X, lS_o, lS_i, T = dp.collate_wrapper_criteo_offset([ds[i] for i in range(lo, min(lo + bs, len(ds)))])
            batches["%s_%d_X" % (name, j)] = X.numpy()
            batches["%s_%d_lS_o" % (name, j)] = lS_o.numpy().astype(np.int32)
            batches["%s_%d_lS_i" % (name, j)] = lS_i.numpy().astype(np.int32)
            batches["%s_%d_T" % (name, j)] = T.numpy()
    np.savez_compressed(os.path.join(out, "kaggle_batches.npz"), **batches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden"))
    args = ap.parse_args()
    out = os.path.abspath(args.out)
    with tempfile.TemporaryDirectory() as tmp:             # the reference writes its TensorBoard run into the cwd
        write_train_txt(os.path.join(tmp, "kaggle.txt"))
        reference_cli(RUNS["A"] + data_flags(tmp, "kaggleAdDisplayChallenge_processed.npz"), tmp)   # preprocess
        for src, dst in (("kaggleAdDisplayChallenge_processed.npz", "kaggle_processed.npz"),
                         ("kaggle_day_count.npz", "kaggle_day_count.npz"),
                         ("kaggle_fea_count.npz", "kaggle_fea_count.npz")):
            shutil.copy(os.path.join(tmp, src), os.path.join(out, dst))
        data = tempfile.mkdtemp(dir=tmp)
        for f in ("kaggle_processed.npz", "kaggle_day_count.npz"):
            shutil.copy(os.path.join(out, f), data)
        for tag, flags in RUNS.items():
            with open(os.path.join(out, "cli_kaggle_%s.flags" % tag), "w") as fh:
                fh.write(" ".join(flags) + "\n")
            stdout = reference_cli(flags + data_flags(data, "kaggle_processed.npz"), tmp)
            lines = [ln for ln in stdout.splitlines() if KEEP.search(ln)]
            with open(os.path.join(out, "cli_kaggle_%s.txt" % tag), "w") as fh:
                fh.write("\n".join(lines) + "\n")
            print("tag %s: %d lines" % (tag, len(lines)))
        dump_orders_and_batches(data, out)


if __name__ == "__main__":
    main()
