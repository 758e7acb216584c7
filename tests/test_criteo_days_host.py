"""Per-day Criteo files (dlrm_b200/criteo_days.py, the reference's --memory-map path) on the CPU: the member reader
against np.load, the batch plan against both reference loaders' recorded batches, the worker thread's stream and
seeking, the refusals, and the CLI's per-day path with a stand-in model and the device stream replaced by the host
oracle.  Fixtures: tests/golden/days_* and cli_days_* (oracle/make_day_goldens.py); the days are written back as
float64 savez_compressed files, as the reference stores them."""
import os
import zipfile

import numpy as np
import pytest
import torch

from dlrm_b200 import criteo, criteo_days as CD
from test_criteo_dataset_host import cli_on_cpu  # noqa: F401  (the CLI with a stand-in model, on the CPU)

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PACK = {ds: dict(np.load(os.path.join(GOLD, "days_%s.npz" % ds))) for ds in ("kaggle", "terabyte")}
REC = np.load(os.path.join(GOLD, "days_batches.npz"))


def write_days(tmp_path, dataset, dtype=np.float64, compress=True):
    """The packed fixture as the reference's per-day files under tmp_path; returns the --raw-data-file."""
    z = PACK[dataset]
    raw = str(tmp_path / ("kaggle.txt" if dataset == "kaggle" else "day"))
    files, count_file, fea_file = CD.day_files(dataset, raw)
    np.savez(count_file, total_per_file=z["total_per_file"])
    np.savez(fea_file, counts=z["counts"])
    save = np.savez_compressed if compress else np.savez
    for d, f in enumerate(files):
        save(f, X_cat=z["X_cat_%d" % d].astype(dtype), X_int=z["X_int_%d" % d].astype(dtype),
             y=z["y_%d" % d].astype(dtype))
    return raw


def host_batch(dataset, segments, mir=-1):
    """The reference's collate of the samples a plan names (the host oracle)."""
    z = PACK[dataset]
    items = []
    for d, lo, hi in segments:
        x_cat = z["X_cat_%d" % d][lo:hi]
        for i in range(hi - lo):
            items.append((z["X_int_%d" % d][lo + i], x_cat[i] % mir if mir > 0 else x_cat[i], z["y_%d" % d][lo + i]))
    return criteo.CriteoDataset.collate(items)


def plan_ids(dataset, plan):
    off = np.concatenate([[0], np.cumsum(PACK[dataset]["total_per_file"])])
    return [np.concatenate([off[d] + np.arange(lo, hi) for d, lo, hi in b]) for b in plan]


def recorded(dataset, split):
    """(loader, batch size) of every recorded batch list of `dataset` / `split` (keys <ds>_<loader>_<split>_<B>_ids)."""
    keys = [k.split("_") for k in REC.files]
    return sorted((k[1], int(k[3])) for k in keys if len(k) == 5 and k[0] == dataset and k[2] == split
                  and k[4] == "ids")


@pytest.mark.parametrize("compress", [True, False])
@pytest.mark.parametrize("dtype", [np.float64, np.int64, np.int32])
def test_member_reader_returns_what_np_load_returns(tmp_path, compress, dtype):
    raw = write_days(tmp_path, "terabyte", dtype, compress)
    files, _, _ = CD.day_files("terabyte", raw)
    for d in (0, 5, 23):
        with np.load(files[d]) as z:
            want = {k: z[k] for k in z.files}
        for name, cols in CD.MEMBERS:
            r = CD.MemberReader(files[d], name, cols)
            assert r.rows == len(want[name]) and r.dtype == np.dtype(dtype)
            got, row = np.empty_like(want[name]), 0
            while row < r.rows:                           # 7 rows at a time: 7 divides no day here
                k = min(7, r.rows - row)
                r.readinto(got[row:row + k], k)
                row += k
            r.close()
            assert np.array_equal(got, want[name]) and got.dtype == want[name].dtype
            r = CD.MemberReader(files[d], name, cols)
            r.skip(3)
            rest = np.empty_like(want[name][3:])
            r.readinto(rest, len(rest))
            r.close()
            assert np.array_equal(rest, want[name][3:])


def test_member_reader_reads_zip64_members(tmp_path):
    a = PACK["terabyte"]["X_cat_1"].astype(np.float64)
    p = tmp_path / "z.npz"
    with zipfile.ZipFile(p, "w", compression=zipfile.ZIP_DEFLATED) as zf, \
            zf.open("X_cat.npy", "w", force_zip64=True) as f:
        np.lib.format.write_array(f, a)
    r = CD.MemberReader(str(p), "X_cat", 26)
    got = np.empty_like(a)
    r.readinto(got, len(a))
    r.close()
    assert np.array_equal(got, a)


@pytest.mark.parametrize("dataset", ["kaggle", "terabyte"])
@pytest.mark.parametrize("split", ["train", "test"])
def test_batch_plan_equals_both_reference_loaders(dataset, split):
    got = recorded(dataset, split)
    sizes = {"kaggle": {"train": {32}, "test": {48}}, "terabyte": {"train": {24, 16}, "test": {12, 16}}}
    assert {b for _, b in got} == sizes[dataset][split]
    loaders = {name for name, _ in got}
    assert loaders == ({"ds"} if dataset == "kaggle" else {"ds", "tb"})
    for name, bs in got:
        key = "%s_%s_%s_%d" % (dataset, name, split, bs)
        p = CD.plan(PACK[dataset]["total_per_file"], split, bs)
        assert [sum(hi - lo for _, lo, hi in b) for b in p] == list(REC[key + "_sizes"])
        assert np.array_equal(np.concatenate(plan_ids(dataset, p)), REC[key + "_ids"]), key


def test_recorded_batches_cover_the_day_boundary_cases():
    """The Terabyte fixture has a day shorter than a batch, a day that is a multiple of it, and batches that span
    three days, at both recorded training batch sizes."""
    n = PACK["terabyte"]["total_per_file"]
    for bs in (24, 16):
        p = CD.plan(n, "train", bs)
        assert any(v < bs for v in n[:-1]) and any(v % bs == 0 for v in n[:-1])
        assert any(len(b) == 3 for b in p)
        assert sum(hi - lo for _, lo, hi in p[-1]) < bs       # a tail batch


@pytest.mark.parametrize("dataset,split,bs", [("kaggle", "train", 32), ("kaggle", "test", 48),
                                              ("terabyte", "train", 24), ("terabyte", "test", 12)])
def test_host_oracle_equals_the_recorded_batches(dataset, split, bs):
    p = CD.plan(PACK[dataset]["total_per_file"], split, bs)
    for j, segs in enumerate(p):
        X, lS_o, lS_i, T = host_batch(dataset, segs)
        key = "%s_%s_%d" % (dataset, split, j)
        assert torch.equal(X, torch.from_numpy(REC[key + "_X"]))
        assert torch.equal(lS_i, torch.from_numpy(REC[key + "_lS_i"]).long())
        assert torch.equal(T, torch.from_numpy(REC[key + "_T"]))
    assert "%s_%s_%d_X" % (dataset, split, len(p)) not in REC.files


def test_a_plan_off_by_one_at_a_day_boundary_fails_the_comparison():
    """Negative control: the batch that crosses the first day boundary takes one sample less from day 0."""
    n = PACK["terabyte"]["total_per_file"]
    p = CD.plan(n, "train", 24)
    j = next(i for i, b in enumerate(p) if len(b) > 1)
    (d0, lo0, hi0), (d1, lo1, hi1) = p[j][:2]
    bad = [list(b) for b in p]
    bad[j][0], bad[j][1] = (d0, lo0, hi0 - 1), (d1, lo1, hi1 + 1)
    assert [sum(hi - lo for _, lo, hi in b) for b in bad] == list(REC["terabyte_ds_train_24_sizes"])
    assert not np.array_equal(np.concatenate(plan_ids("terabyte", bad)), REC["terabyte_ds_train_24_ids"])
    X, _, _, _ = host_batch("terabyte", bad[j])
    assert not torch.equal(X, torch.from_numpy(REC["terabyte_train_%d_X" % j]))


def _stream(files, counts, segments, start, chunk_rows):
    """Every chunk the worker thread produces from `start`, as (position, rows of the three members)."""
    bufs = [np.zeros(CD.slot_bytes(chunk_rows), np.uint8) for _ in range(CD.SLOTS)]
    pr = CD._Producer(files, counts, segments, start, chunk_rows, bufs)
    out = []
    try:
        while True:
            c = pr.ready.get(timeout=60)
            if c is None or isinstance(c, BaseException):
                if c is not None:
                    raise c
                break
            members = []
            for m, (name, cols) in enumerate(CD.MEMBERS):
                dt = {0: np.float64, 1: np.int64, 2: np.int32}[c.codes[m]]
                a = bufs[c.slot][c.offsets[m]:c.offsets[m] + c.n * cols * np.dtype(dt).itemsize].view(dt)
                members.append(a.reshape(c.n, cols) if cols > 1 else a.copy())
            out.append((c.pos, [m.copy() for m in members]))
            pr.free.put(c.slot)
    finally:
        pr.close()
    return out


@pytest.mark.parametrize("split", ["train", "test"])
def test_stream_and_seek_give_the_samples_in_order(tmp_path, split):
    raw = write_days(tmp_path, "terabyte")
    files, _, _ = CD.day_files("terabyte", raw)
    z = PACK["terabyte"]
    n = z["total_per_file"]
    segs = CD.split_segments(n, split)
    full = [np.concatenate([z["%s_%d" % (k, d)][lo:hi] for d, lo, hi in segs]) for k in ("X_int", "X_cat", "y")]
    total = sum(hi - lo for _, lo, hi in segs)
    for start in [s for s in (0, 1, 29, 30, 100, 216) if s < total] + [total - 1]:
        chunks = _stream(files, n, segs, start, 11)
        assert chunks[0][0] == start
        pos = start
        for p, members in chunks:
            assert p == pos and len(members[2]) <= 11
            for m in range(3):
                assert np.array_equal(members[m], full[m][pos:pos + len(members[2])])
            pos += len(members[2])
        assert pos == len(full[2])


def test_a_resumed_stream_gives_the_batches_of_a_full_read():
    n = PACK["terabyte"]["total_per_file"]
    p = CD.plan(n, "train", 24)
    for j in (1, 7, len(p) - 1):
        assert CD.plan(n, "train", 24)[j:] == p[j:]
        assert sum(hi - lo for b in p[:j] for _, lo, hi in b) == 24 * j


def _bad_day(tmp_path, **members):
    z = PACK["terabyte"]
    d = dict(X_int=z["X_int_0"].astype(np.float64), X_cat=z["X_cat_0"].astype(np.float64),
             y=z["y_0"].astype(np.float64))
    d.update(members)
    p = str(tmp_path / "bad.npz")
    np.savez_compressed(p, **d)
    return p


def test_refusals_name_the_file_and_member(tmp_path):
    z = PACK["terabyte"]
    n = int(z["total_per_file"][0])
    x_int = z["X_int_0"].astype(np.float64)
    cases = [
        (dict(X_int=np.asfortranarray(x_int)), "member X_int is stored in Fortran order"),
        (dict(X_cat=z["X_cat_0"].astype(np.float32)), "member X_cat has dtype <f4"),
        (dict(y=z["y_0"].astype(">f8")), "member y has dtype >f8"),
        (dict(y=z["y_0"][:-1].astype(np.float64)), "members X_int, X_cat, y hold %d, %d, %d samples"
         % (n, n, n - 1)),
        (dict(X_int=x_int[:, :12]), "member X_int has shape (%d, 12), expected [n, 13]" % n),
    ]
    for kw, msg in cases:
        p = _bad_day(tmp_path, **kw)
        with pytest.raises(ValueError) as e:
            CD.open_day(p, n)
        assert str(e.value).startswith(p + ": ") and msg in str(e.value), str(e.value)
    p = _bad_day(tmp_path)
    with pytest.raises(ValueError, match="member X_int holds %d samples, the day count says %d" % (n, n + 1)):
        CD.open_day(p, n + 1)
    with zipfile.ZipFile(p, "a") as zf:
        zf.writestr("unrelated.txt", "x")
    CD.open_day(p, n)
    q = str(tmp_path / "no_y.npz")
    np.savez(q, X_int=x_int, X_cat=z["X_cat_0"].astype(np.float64))
    with pytest.raises(ValueError, match="member y.npy is missing"):
        CD.open_day(q, n)
    open(tmp_path / "text.npz", "w").write("not a zip")
    with pytest.raises(ValueError, match="text.npz: File is not a zip file"):
        CD.open_day(str(tmp_path / "text.npz"), n)


def test_stream_refuses_a_day_count_that_disagrees(tmp_path):
    raw = write_days(tmp_path, "terabyte")
    files, count_file, _ = CD.day_files("terabyte", raw)
    n = PACK["terabyte"]["total_per_file"].copy()
    n[3] += 1
    np.savez(count_file, total_per_file=n)
    with pytest.raises(ValueError, match=r"day_3_reordered.npz: member X_int holds 44 samples, the day count says 45"):
        CD.DayBatches("terabyte", raw, "train", 24, -1, "cpu")
    np.savez(count_file, total_per_file=n[:7])
    with pytest.raises(ValueError, match="7 days, terabyte has 24"):
        CD.DayBatches("terabyte", raw, "train", 24, -1, "cpu")
    os.remove(files[9])
    with pytest.raises(FileNotFoundError, match="day_9_reordered.npz"):
        CD.DayBatches("terabyte", raw, "train", 24, -1, "cpu")
    with pytest.raises(ValueError, match="val"):
        CD.split_segments(n, "val")


class HostDays:
    """The device stream, replaced by its host oracle: the plan over the packed fixture."""
    seen = []

    def __init__(self, dataset, raw_path, split, batch_size, max_ind_range, device):
        files, count_file, _ = CD.day_files(dataset, raw_path)
        assert all(os.path.exists(f) for f in files)
        self.dataset, self.mir = dataset, max_ind_range
        self.plan = CD.plan(np.load(count_file)["total_per_file"], split, batch_size)
        self.num_samples = sum(hi - lo for b in self.plan for _, lo, hi in b)
        HostDays.seen.append((split, batch_size))

    def __len__(self):
        return len(self.plan)

    def __getitem__(self, j):
        return host_batch(self.dataset, self.plan[j], self.mir)

    def close(self):
        pass


def _flags(tag):
    return open(os.path.join(GOLD, "cli_days_%s.flags" % tag)).read().split()


@pytest.mark.parametrize("tag,dataset,ntrain,ntest", [
    ("K", "kaggle", [32] * 37 + [16], [48, 48, 4]),
    ("T1", "terabyte", [24] * 36 + [5], [12, 12, 7]),
    ("T2", "terabyte", [16] * 54 + [5], [16, 15]),
])
def test_cli_tables_lines_and_batches(cli_on_cpu, capsys, monkeypatch, tmp_path, tag, dataset, ntrain, ntest):  # noqa: F811
    cli, rec = cli_on_cpu
    monkeypatch.setattr(CD, "DayBatches", HostDays)
    raw = write_days(tmp_path, dataset)
    flags = _flags(tag)
    cli.run(flags + ["--raw-data-file=" + raw, "--processed-data-file=" + str(tmp_path / "p.npz"), "--use-gpu"])
    out = capsys.readouterr().out.splitlines()
    mir = int(dict(f.split("=", 1) for f in flags if "=" in f).get("--max-ind-range", -1))
    counts = PACK[dataset]["counts"]
    assert rec["ln_emb"] == list(counts if mir <= 0 else np.minimum(counts, mir)) and rec["ln_bot"][0] == 13
    # no draw from numpy's global RNG before the model is built, as in the reference
    st = rec["rng_at_init"]
    assert np.array_equal(st[1], REC[dataset + "_rng_keys"]) and st[2] == int(REC[dataset + "_rng_pos"])
    gold = open(os.path.join(GOLD, "cli_days_%s.txt" % tag)).read().splitlines()
    head = gold[:gold.index("time/loss/accuracy (if enabled):")]
    assert [ln for ln in out if ln.startswith("Sparse features")] == head
    assert out.count("Reading pre-processed data=" + str(tmp_path / "p.npz")) == 2
    assert [ln for ln in out if ln.startswith("Testing at")] == [ln for ln in gold if ln.startswith("Testing at")]
    nep = int(dict(f.split("=", 1) for f in flags if "=" in f)["--nepochs"])
    passes = len([ln for ln in gold if ln.startswith("Testing at")])
    assert sorted(b for b, _ in rec["seen"]) == sorted(ntrain * nep + ntest * passes)
    assert len(ntrain) == len(CD.plan(PACK[dataset]["total_per_file"], "train", ntrain[0]))
    if mir > 0:
        assert max(m for _, m in rec["seen"]) < mir


def test_cli_test_batch_default_and_num_batches(cli_on_cpu, monkeypatch, tmp_path):  # noqa: F811
    cli, rec = cli_on_cpu
    monkeypatch.setattr(CD, "DayBatches", HostDays)
    HostDays.seen = []
    raw = write_days(tmp_path, "terabyte")
    flags = [f for f in _flags("T1") if not f.startswith(("--test-mini-batch-size", "--nepochs"))]
    cli.run(flags + ["--raw-data-file=" + raw, "--use-gpu", "--num-batches=5", "--test-freq=5", "--nepochs=2"])
    assert HostDays.seen == [("train", 24), ("test", 24)]
    # each epoch restarts at day 0 (the reference reads the next epoch at negative positions of its loaded day)
    assert [b for b, _ in rec["seen"]] == ([24] * 5 + [24, 7]) * 2


def test_cli_refuses_missing_days_naming_the_first(cli_on_cpu, tmp_path):  # noqa: F811
    cli, _ = cli_on_cpu
    raw = write_days(tmp_path, "kaggle")
    files, _, _ = CD.day_files("kaggle", raw)
    os.remove(files[4])
    os.remove(files[6])
    with pytest.raises(SystemExit) as e:
        cli.run(_flags("K") + ["--raw-data-file=" + raw, "--use-gpu"])
    msg = str(e.value)
    assert files[4] + " does not exist" in msg and files[6] not in msg
    assert "--data-generation=dataset is not supported" in msg and "per-day _reordered.npz files are not read" in msg
