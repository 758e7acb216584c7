"""Regenerate the per-day Criteo fixtures (`--memory-map`) and the reference's recorded runs on them
(tests/test_criteo_days_host.py, tests/test_gpu_criteo_days.py):

    python oracle/make_day_goldens.py [--out DIR]        # default: tests/golden

1. Writes a synthetic raw Kaggle train.txt (make_kaggle_goldens.write_train_txt: 7 days of 200 lines) and 24
   synthetic Terabyte `day_{d}` files cut from the same generator, of the unequal sizes TB_DAYS: day 5 (7 lines) is
   shorter than both recorded batch sizes (16 and 24), day 11 (48) is a multiple of both, and batches span three days.
   The sizes are chosen so that the reference's data_loader_terabyte._batch_generator never carries more than a
   batch across a short day (it raises "should not happen" when it does).
2. Runs the UNMODIFIED reference CLI once per dataset with --memory-map to preprocess them, then records runs K, T1,
   T2, T3 with the reordered days in place: cli_days_<tag>.flags / cli_days_<tag>.txt (kept stdout lines) and T1's
   saved checkpoint, cli_days_T1_ref.pt, which T3 evaluates.
3. Packs the reordered days (exact integers, stored here as int32; the reference writes float64) into
   days_kaggle.npz / days_terabyte.npz: `X_int_<d>`, `X_cat_<d>`, `y_<d>`, `total_per_file`, `counts`.
4. Dumps both reference loaders' batches (days_batches.npz): CriteoDataset(memory_map=True) under a torch DataLoader
   ("ds") and, for Terabyte, data_loader_terabyte.DataLoader ("tb"), for train and test at every recorded batch size.
   `<ds>_<loader>_<split>_<B>_ids` are the samples of each batch in order, read from days whose X_cat[:, 0] was
   replaced by the sample's global position (its day's offset plus its row), and `..._sizes` the batch sizes; the
   full collated batches (X, lS_i, T) of the unmodified days are kept for one batch size per dataset and split.
   numpy's global RNG state after both memory-map datasets are built is `<ds>_rng_keys` / `<ds>_rng_pos` (seed 727).

Test infrastructure: needs the reference checkout (DLRM_REFERENCE)."""
import argparse
import contextlib
import io
import os
import re
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import make_kaggle_goldens as MK  # noqa: E402

REF = MK.REF
TB_DAYS = [29, 50, 28, 44, 48, 7, 39, 48, 33, 50, 51, 48, 29, 32, 25, 36, 31, 44, 30, 49, 25, 59, 34, 61]
MODEL = ["--arch-sparse-feature-size=16", "--arch-mlp-bot=13-64-16", "--arch-mlp-top=64-1", "--data-generation=dataset",
         "--loss-function=bce", "--round-targets=True", "--numpy-rand-seed=727", "--memory-map"]
RUNS = {
    "K": MODEL + ["--data-set=kaggle", "--learning-rate=0.1", "--optimizer=sgd", "--mini-batch-size=32", "--nepochs=2",
                  "--print-freq=8", "--test-freq=16", "--test-mini-batch-size=48"],
    "T1": MODEL + ["--data-set=terabyte", "--learning-rate=0.05", "--optimizer=rwsadagrad", "--max-ind-range=40",
                   "--mini-batch-size=24", "--nepochs=1", "--print-freq=4", "--test-freq=10",
                   "--test-mini-batch-size=12"],
    "T2": MODEL + ["--data-set=terabyte", "--learning-rate=0.1", "--optimizer=sgd", "--mini-batch-size=16",
                   "--nepochs=2", "--print-freq=9", "--test-freq=20", "--test-mini-batch-size=16",
                   "--mlperf-logging"],
}
RUNS["T3"] = [f for f in RUNS["T1"] if not f.startswith("--test-freq")] + ["--inference-only"]
KEEP = re.compile(r"Sparse features|Finished training|Testing at|accuracy|^recall |Saved at|Training state|"
                  r"Testing state|Testing for inference")
# (dataset, batch sizes of train, batch sizes of test); the first of each is also kept as full batches
BATCHES = {"kaggle": ((32,), (48,)), "terabyte": ((24, 16), (12, 16))}


def data_flags(d, dataset):
    raw = os.path.join(d, "kaggle.txt" if dataset == "kaggle" else "day")
    return ["--raw-data-file=" + raw, "--processed-data-file=" + os.path.join(d, dataset + "_processed.npz")]


def day_file(d, dataset, day):
    return os.path.join(d, ("kaggle_day_%d" if dataset == "kaggle" else "day_%d") + "_reordered.npz") % day


def stem(d, dataset):
    return os.path.join(d, "kaggle" if dataset == "kaggle" else "day")


def pack(d, dataset, out):
    days = 7 if dataset == "kaggle" else 24
    arrays = {}
    with np.load(stem(d, dataset) + "_day_count.npz") as z:
        arrays["total_per_file"] = z["total_per_file"]
    with np.load(stem(d, dataset) + "_fea_count.npz") as z:
        arrays["counts"] = z["counts"]
    for day in range(days):
        with np.load(day_file(d, dataset, day)) as z:
            for k in ("X_int", "X_cat", "y"):
                a = z[k]
                if a.dtype != np.float64:
                    raise SystemExit("%s %s is %s, not float64" % (day_file(d, dataset, day), k, a.dtype))
                b = a.astype(np.int32)
                if not np.array_equal(b, a):
                    raise SystemExit("%s %s holds values that are not int32 integers" % (day_file(d, dataset, day), k))
                arrays["%s_%d" % (k, day)] = b
    np.savez_compressed(os.path.join(out, "days_%s.npz" % dataset), **arrays)
    return arrays


def dump_batches(d, dataset, arrays, rec):
    """Both reference loaders' batches on the days in `d` (see the module docstring)."""
    sys.path[:0] = [REF, os.path.join(HERE, "mlperf_stub")]
    import torch
    import data_loader_terabyte as dlt
    import dlrm_data_pytorch as dp

    days = len(arrays["total_per_file"])
    raw = data_flags(d, dataset)[0].split("=", 1)[1]
    tag = tempfile.mkdtemp(dir=d)
    off = np.concatenate([[0], np.cumsum(arrays["total_per_file"])])
    for f in ("_day_count.npz", "_fea_count.npz"):
        shutil.copy(stem(d, dataset) + f, stem(tag, dataset) + f)
    for day in range(days):
        x_cat = arrays["X_cat_%d" % day].astype(np.float64)
        x_cat[:, 0] = off[day] + np.arange(len(x_cat))
        np.savez_compressed(day_file(tag, dataset, day), X_int=arrays["X_int_%d" % day].astype(np.float64),
                            X_cat=x_cat, y=arrays["y_%d" % day].astype(np.float64))
    tag_raw = os.path.join(tag, os.path.basename(raw))

    def ds_loader(path, split, bs):
        with contextlib.redirect_stdout(io.StringIO()):
            ds = dp.CriteoDataset(dataset, -1, 0.0, "total", split, path, "", True)
        return torch.utils.data.DataLoader(ds, batch_size=bs, shuffle=False, num_workers=0,
                                           collate_fn=dp.collate_wrapper_criteo_offset, drop_last=False)

    def tb_loader(path, split, bs):
        return dlt.DataLoader(data_directory=os.path.dirname(path), data_filename=os.path.basename(path),
                              days=list(range(days - 1)) if split == "train" else [days - 1], batch_size=bs,
                              split=split)

    loaders = {"ds": ds_loader} if dataset == "kaggle" else {"ds": ds_loader, "tb": tb_loader}
    for split, sizes in zip(("train", "test"), BATCHES[dataset]):
        for bs in sizes:
            for name, make in loaders.items():
                ids, lens = [], []
                for X, lS_o, lS_i, T in make(tag_raw, split, bs):
                    ids.append(lS_i[0].numpy().astype(np.int32))
                    lens.append(len(T))
                key = "%s_%s_%s_%d" % (dataset, name, split, bs)
                rec[key + "_ids"], rec[key + "_sizes"] = np.concatenate(ids), np.asarray(lens, np.int32)
            if bs == sizes[0]:
                for j, (X, lS_o, lS_i, T) in enumerate(ds_loader(raw, split, bs)):
                    assert np.array_equal(lS_o.numpy(), np.tile(np.arange(len(T)), (26, 1)))
                    key = "%s_%s_%d" % (dataset, split, j)
                    rec[key + "_X"], rec[key + "_lS_i"] = X.numpy(), lS_i.numpy().astype(np.int32)
                    rec[key + "_T"] = T.numpy()
    np.random.seed(727)
    with contextlib.redirect_stdout(io.StringIO()):
        dp.CriteoDataset(dataset, -1, 0.0, "total", "train", raw, "", True)
        dp.CriteoDataset(dataset, -1, 0.0, "total", "test", raw, "", True)
    st = np.random.get_state()
    rec[dataset + "_rng_keys"], rec[dataset + "_rng_pos"] = st[1].copy(), np.int64(st[2])


def write_days(tmp):
    """Kaggle train.txt and the 24 Terabyte day files, cut from the same synthetic lines."""
    MK.write_train_txt(os.path.join(tmp, "kaggle.txt"))
    lines = open(os.path.join(tmp, "kaggle.txt")).read().splitlines(True)
    assert sum(TB_DAYS) <= len(lines)
    pos = 0
    for day, n in enumerate(TB_DAYS):
        with open(os.path.join(tmp, "day_%d" % day), "w") as f:
            f.writelines(lines[pos:pos + n])
        pos += n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden"))
    args = ap.parse_args()
    out = os.path.abspath(args.out)
    rec = {}
    with tempfile.TemporaryDirectory() as tmp:             # the reference writes its TensorBoard run into the cwd
        write_days(tmp)
        packs = {}
        for dataset, tag in (("kaggle", "K"), ("terabyte", "T2")):
            MK.reference_cli(RUNS[tag] + data_flags(tmp, dataset), tmp)        # preprocess (--memory-map)
            packs[dataset] = pack(tmp, dataset, out)
        data = tempfile.mkdtemp(dir=tmp)                   # the reordered days alone: no raw text, no intermediates
        for dataset, days in (("kaggle", 7), ("terabyte", 24)):
            for f in ("_day_count.npz", "_fea_count.npz"):
                shutil.copy(stem(tmp, dataset) + f, stem(data, dataset) + f)
            for day in range(days):
                shutil.copy(day_file(tmp, dataset, day), day_file(data, dataset, day))
        ckpt = os.path.join(tmp, "t1.pt")
        # the reference's torch.load takes torch's default weights_only=True, which refuses the numpy scalars its own
        # checkpoints hold; this checkpoint is the one T1 just wrote
        os.environ["TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD"] = "1"
        for tag in ("K", "T1", "T2", "T3"):
            flags = RUNS[tag]
            with open(os.path.join(out, "cli_days_%s.flags" % tag), "w") as fh:
                fh.write(" ".join(flags) + "\n")
            extra = (["--save-model=" + ckpt] if tag == "T1" else ["--load-model=" + ckpt] if tag == "T3" else [])
            dataset = "kaggle" if tag == "K" else "terabyte"
            stdout = MK.reference_cli(flags + data_flags(data, dataset) + extra, tmp)
            lines = [ln for ln in stdout.splitlines() if KEEP.search(ln)]
            with open(os.path.join(out, "cli_days_%s.txt" % tag), "w") as fh:
                fh.write("\n".join(lines) + "\n")
            print("tag %s: %d lines" % (tag, len(lines)))
            if tag == "T1":
                shutil.copy(ckpt, os.path.join(out, "cli_days_T1_ref.pt"))
        for dataset in ("kaggle", "terabyte"):
            dump_batches(data, dataset, packs[dataset], rec)
    np.savez_compressed(os.path.join(out, "days_batches.npz"), **rec)


if __name__ == "__main__":
    main()
