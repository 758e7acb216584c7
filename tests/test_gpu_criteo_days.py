"""Per-day Criteo files streamed through device memory (dlrm_b200/criteo_days.py): the ingest kernel
(dlrm_b200_ingest_records) against a numpy conversion, every batch of every split through rings that wrap many
times against the host oracle and against criteo.DeviceBatches over the same samples held resident, the stream's
memory bound, bad data and access order, and the CLI's --memory-map path against the reference's recorded runs
K, T1, T2, T3 (tests/golden/cli_days_*, oracle/make_day_goldens.py)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from dlrm_b200 import _lib, criteo
from dlrm_b200 import criteo_days as CD
from test_criteo_days_host import PACK, host_batch, write_days

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
DEV = "cuda:0"
SENT = -123456789


def _ingest(x_int, x_cat, y, ring, dst):
    """One chunk (host numpy arrays in any accepted dtype) into `ring` (three int32 device tensors) at row dst;
    returns the error word."""
    C = ring[2].shape[0]
    srcs = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (x_int, x_cat, y)]
    bad = torch.full((1,), -1, dtype=torch.int64, device=DEV)
    _lib.check(_lib.lib().dlrm_b200_ingest_records(
        srcs[0].data_ptr(), CD.DTYPE_CODES[x_int.dtype], srcs[1].data_ptr(), CD.DTYPE_CODES[x_cat.dtype],
        srcs[2].data_ptr(), CD.DTYPE_CODES[y.dtype], len(y), 13, 26, ring[0].data_ptr(), ring[1].data_ptr(),
        ring[2].data_ptr(), C, dst, bad.data_ptr(), None), "ingest_records")
    torch.cuda.synchronize()
    return int(bad.item())


def _ring(C):
    return tuple(torch.full(s, SENT, dtype=torch.int32, device=DEV) for s in ((C, 13), (C, 26), (C,)))


def _chunk(rng, n):
    x_int = rng.randint(-5, 1 << 30, (n, 13))
    x_int[:, 0] = np.iinfo(np.int32).max
    x_int[:, 1] = np.iinfo(np.int32).min
    x_cat = rng.randint(0, (1 << 31) - 1, (n, 26))
    return x_int, x_cat, rng.randint(0, 2, n)


@pytest.mark.parametrize("dtypes", [("<f8",) * 3, ("<i8",) * 3, ("<i4",) * 3, ("<f8", "<i8", "<i4"),
                                    ("<i4", "<f8", "<i8")])
def test_ingest_equals_numpy_across_the_ring_wrap(dtypes):
    rng = np.random.RandomState(1)
    n, C, dst = 100, 150, 120                      # rows 120..149 then 0..69
    x_int, x_cat, y = _chunk(rng, n)
    ring = _ring(C)
    assert _ingest(x_int.astype(dtypes[0]), x_cat.astype(dtypes[1]), y.astype(dtypes[2]), ring, dst) == -1
    rows = (dst + np.arange(n)) % C
    want = [np.full(tuple(t.shape), SENT, np.int32) for t in ring]
    for w, a in zip(want, (x_int, x_cat, y)):
        w[rows] = a.astype(np.int32)
    for t, w in zip(ring, want):
        assert np.array_equal(t.cpu().numpy(), w)            # the target rows exactly, nothing else written


@pytest.mark.parametrize("member,value,dtype", [
    (0, 1.5, "<f8"), (0, float("nan"), "<f8"), (0, 2.0 ** 31, "<f8"), (0, -2.0 ** 31 - 1, "<f8"),
    (0, 1 << 31, "<i8"), (1, -1, "<i4"), (1, -1.0, "<f8"), (1, 0.25, "<f8"), (1, -(1 << 40), "<i8"),
    (2, 2, "<i4"), (2, -1, "<i8"), (2, 0.5, "<f8"), (2, float("inf"), "<f8")])
def test_ingest_reports_the_first_bad_row(member, value, dtype):
    rng = np.random.RandomState(2)
    n, C, dst = 90, 128, 70
    arrays = [a.astype(dtype) for a in _chunk(rng, n)]
    a = arrays[member]
    for r in (61, 37, 80):                           # the first bad row is 37, whatever the order it is met in
        if a.ndim == 2:
            a[r, 5 if member == 0 else 11] = value
        else:
            a[r] = value
    ring = _ring(C)
    assert _ingest(*arrays, ring, dst) == 37 * 4 + member
    # the bad value is not written; the good values of the bad rows are
    got = ring[member].cpu().numpy()
    rows = (dst + np.arange(n)) % C
    col = 5 if member == 0 else 11
    bad_vals = got[rows[37], col] if a.ndim == 2 else got[rows[37]]
    assert bad_vals == SENT
    outside = np.setdiff1d(np.arange(C), rows)
    for t in ring:
        assert (t.cpu().numpy()[outside] == SENT).all()


def test_ingest_rejects_bad_arguments():
    lib = _lib.lib()
    buf = torch.zeros(1 << 12, dtype=torch.int64, device=DEV)
    p = buf.data_ptr()
    for args, msg in [((0, 13, 26, 8, 0), b"n=0"), ((9, 13, 26, 8, 0), b"n=9 rows for a ring of 8"),
                      ((4, 13, 26, 8, 8), b"dst=8"), ((4, 0, 26, 8, 0), b"num_dense=0")]:
        n, nd, ns, C, dst = args
        assert lib.dlrm_b200_ingest_records(p, 0, p, 0, p, 0, n, nd, ns, p, p, p, C, dst, p, None) != 0
        assert msg in lib.dlrm_b200_last_error()
    assert lib.dlrm_b200_ingest_records(p, 3, p, 0, p, 0, 4, 13, 26, p, p, p, 8, 0, p, None) != 0
    assert b"dtype code 3" in lib.dlrm_b200_last_error()
    assert lib.dlrm_b200_ingest_records(p, 0, p, 0, p, 0, 4, 13, 26, p, p, p, 8, 0, None, None) != 0
    assert b"NULL" in lib.dlrm_b200_last_error()


def _resident(tmp_path, dataset, split, mir):
    """criteo.CriteoDataset over the same samples, resident: the days concatenated into one processed file,
    read in file order (the last day's array_split gives the test split its first ceil(n/2) samples)."""
    z = PACK[dataset]
    D = len(z["total_per_file"])
    d = tmp_path / "resident"
    d.mkdir(exist_ok=True)
    cat = {k: np.concatenate([z["%s_%d" % (k, i)] for i in range(D)]) for k in ("X_int", "X_cat", "y")}
    np.savez(d / "p.npz", counts=z["counts"], **cat)
    np.savez(d / ("kaggle_day_count.npz" if dataset == "kaggle" else "day_day_count.npz"),
             total_per_file=z["total_per_file"])
    raw = str(d / ("kaggle.txt" if dataset == "kaggle" else "day"))
    return criteo.CriteoDataset(dataset, mir, 0.0, "none", split, raw, str(d / "p.npz"))


@pytest.mark.parametrize("dataset,split,B,chunk,ring,mir", [
    ("terabyte", "train", 24, 7, 31, -1), ("terabyte", "train", 16, 5, 40, 40), ("terabyte", "test", 12, 4, 16, -1),
    ("terabyte", "train", 24, 64, 200, 7), ("kaggle", "train", 32, 9, 41, 40), ("kaggle", "test", 48, 13, 70, -1),
    ("terabyte", "train", 24, None, None, -1)])
def test_every_batch_matches_the_oracle_and_the_resident_assembly(tmp_path, dataset, split, B, chunk, ring, mir):
    raw = write_days(tmp_path, dataset)
    stream = CD.DayBatches(dataset, raw, split, B, mir, DEV, chunk_rows=chunk, ring_rows=ring)
    res = criteo.DeviceBatches(_resident(tmp_path, dataset, split, mir), B, DEV)
    p = CD.plan(PACK[dataset]["total_per_file"], split, B)
    assert len(stream) == len(res) == len(p)
    for epoch in range(2):                           # the second epoch restarts the stream at day 0
        for j in range(len(p)):
            X, lS_o, lS_i, T = (t.clone() for t in stream[j])
            n = X.shape[0]
            db = stream.batches[n][0]
            Xh, lS_oh, lS_ih, Th = host_batch(dataset, p[j], mir)
            assert torch.equal(lS_i.cpu(), lS_ih) and torch.equal(lS_o.cpu(), lS_oh) and torch.equal(T.cpu(), Th)
            assert torch.equal(db.offsets.reshape(-1)[:26 * (n + 1)].cpu(),
                               (torch.arange(26)[:, None] * n + torch.arange(n + 1)[None]).view(-1))
            Xr, _, lS_ir, Tr = res[j]
            assert torch.equal(X.view(torch.int32), Xr.view(torch.int32)) and torch.equal(lS_i, lS_ir)
    if ring is not None:
        assert stream.num_samples > 4 * ring or split == "test"     # the ring wrapped many times


def test_device_memory_does_not_depend_on_day_size(tmp_path):
    z = PACK["terabyte"]
    big = tmp_path / "big"
    big.mkdir()
    raw_small = write_days(tmp_path, "terabyte")
    raw_big = str(big / "day")
    files, count_file, fea_file = CD.day_files("terabyte", raw_big)
    np.savez(count_file, total_per_file=4 * z["total_per_file"])
    np.savez(fea_file, counts=z["counts"])
    for d, f in enumerate(files):
        np.savez_compressed(f, **{k: np.concatenate([z["%s_%d" % (k, d)]] * 4).astype(np.float64)
                                  for k in ("X_int", "X_cat", "y")})
    used = []
    for raw in (raw_small, raw_big):
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated(DEV)
        s = CD.DayBatches("terabyte", raw, "train", 24, -1, DEV, chunk_rows=64, ring_rows=24 + 4 * 64)
        for j in range(len(s) - 1):                  # full batches: the tail's DeviceBatch differs in size
            s[j]
        torch.cuda.synchronize()
        used.append((torch.cuda.memory_allocated(DEV) - before, s.device_bytes(), len(s)))
        s.close()
        del s
    assert used[0][:2] == used[1][:2] and used[1][2] > 3 * used[0][2]


def test_bad_data_stops_the_run_naming_the_file_and_row(tmp_path):
    raw = write_days(tmp_path, "terabyte")
    files, _, _ = CD.day_files("terabyte", raw)
    z = PACK["terabyte"]
    y = z["y_2"].astype(np.float64)
    y[9] = 3.0
    np.savez_compressed(files[2], X_int=z["X_int_2"].astype(np.float64), X_cat=z["X_cat_2"].astype(np.float64), y=y)
    s = CD.DayBatches("terabyte", raw, "train", 24, -1, DEV, chunk_rows=8, ring_rows=64)
    bad_pos = int(z["total_per_file"][:2].sum()) + 9          # sample 88: batch 3
    with pytest.raises(ValueError) as e:
        for j in range(len(s)):
            s[j]
    assert j <= bad_pos // 24 + 1
    assert str(e.value) == "%s: row 9: y holds a value that is not an integer in int32 range or a label outside " \
                           "{0, 1}" % files[2]


def test_access_is_sequential_with_skips_and_restarts(tmp_path):
    raw = write_days(tmp_path, "terabyte")
    s = CD.DayBatches("terabyte", raw, "train", 16, -1, DEV, chunk_rows=6, ring_rows=30)
    full = [tuple(t.clone() for t in s[j]) for j in range(len(s))]
    s2 = CD.DayBatches("terabyte", raw, "train", 16, -1, DEV, chunk_rows=6, ring_rows=30)
    for j in (0, 1, 7, 8, 30, 31, 0, 1, len(s) - 1):
        got = s2[j]
        assert all(torch.equal(a, b) for a, b in zip(got, full[j])), j
    with pytest.raises(IndexError, match="moves forward or restarts at 0"):
        s2[5]
    with pytest.raises(IndexError):
        s2[len(s)]
    s2[0]
    s2[1]
    with pytest.raises(IndexError, match="batch 1 requested after batch 1"):
        s2[1]


def _cli(tag, raw, extra=()):
    flags = open(os.path.join(GOLD, "cli_days_%s.flags" % tag)).read().split()
    cmd = [sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py")] + flags + ["--raw-data-file=" + raw, "--use-gpu"] \
        + list(extra)
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


@pytest.mark.parametrize("tag", ["K", "T1", "T2", "T3"])
def test_cli_matches_the_reference_run(tmp_path, tag):
    """fp32 CUDA-core GEMMs: every loss within 1e-5 of the reference's CPU run, the other kept lines identical.
    T3 evaluates the checkpoint the reference saved in T1."""
    raw = write_days(tmp_path, "kaggle" if tag == "K" else "terabyte")
    extra = ["--gemm=simt"] + (["--load-model=" + os.path.join(GOLD, "cli_days_T1_ref.pt")] if tag == "T3" else [])
    want = open(os.path.join(GOLD, "cli_days_%s.txt" % tag)).read().splitlines()
    got = _cli(tag, raw, extra).splitlines()
    loss = re.compile(r"Finished training it .* loss ([0-9.]+)")
    want_loss = [float(loss.match(ln).group(1)) for ln in want if loss.match(ln)]
    got_loss = [float(loss.match(ln).group(1)) for ln in got if loss.match(ln)]
    assert len(got_loss) == len(want_loss)
    np.testing.assert_allclose(got_loss, want_loss, rtol=0, atol=1e-5)
    other = re.compile(r"Sparse features|Testing at|accuracy|^recall |Saved at|Training state|Testing state|"
                       r"Testing for inference")
    assert [ln for ln in got if other.search(ln)] == [ln for ln in want if other.search(ln)]
