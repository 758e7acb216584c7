"""Preprocessed Criteo splits resident on the GPU: the batch assembly kernel (dlrm_b200_gather_records) against its
host oracle (CriteoDataset.__getitem__ + collate) and against the record decode (dlrm_b200_decode_records) of the same
samples, on every batch of every split; and the CLI's dataset path against the reference's recorded runs A-C
(tests/golden/cli_kaggle_*, oracle/make_kaggle_goldens.py)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from dlrm_b200 import _lib
from dlrm_b200 import binrecords as BR
from dlrm_b200 import criteo
from dlrm_b200.data import DeviceBatch, PackedLayout

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
RAW = os.path.join(GOLD, "kaggle.txt")
PRO = os.path.join(GOLD, "kaggle_processed.npz")
DEV = "cuda:0"


def _wide_fixture(tmp_path):
    """The golden fixture with values the Kaggle preprocessing never writes: dense counts above 2^24 (the int -> fp32
    conversion rounds) and negative or huge ids (the floor modulo folds them)."""
    rng = np.random.RandomState(0)
    with np.load(PRO) as z:
        d = {k: z[k] for k in z.files}
    n = len(d["y"])
    x_int = d["X_int"].copy()
    big = rng.rand(n, 13) < 0.1
    x_int[big] = rng.randint(1 << 24, (1 << 31) - 1, int(big.sum()))
    x_cat = d["X_cat"].astype(np.int32)
    x_cat[:, 20:] = rng.randint(-(1 << 31), (1 << 31) - 1, (n, 6))
    np.savez(tmp_path / "p.npz", X_int=x_int, X_cat=x_cat, y=d["y"], counts=d["counts"])
    np.savez(tmp_path / "kaggle_day_count.npz", total_per_file=np.full(7, n // 7))
    return str(tmp_path / "kaggle.txt"), str(tmp_path / "p.npz")


def _ulps(a, b):
    return (a.view(torch.int32).long() - b.view(torch.int32).long()).abs()


@pytest.mark.parametrize("wide", [False, True])
@pytest.mark.parametrize("max_ind_range", [-1, 0, 40])
def test_assembly_matches_the_host_oracle_on_every_batch(tmp_path, wide, max_ind_range):
    raw, pro = _wide_fixture(tmp_path) if wide else (RAW, PRO)
    np.random.seed(3)
    train = criteo.CriteoDataset("kaggle", max_ind_range, 0.0, "total", "train", raw, pro)
    splits = [train] + [criteo.CriteoDataset("kaggle", max_ind_range, 0.0, "total", s, raw, pro, data=train)
                        for s in ("test", "val")]
    log_ulps = checked = 0
    for ds, B in zip(splits, (37, 48, 64)):                          # every split ends in a short batch
        batches = criteo.DeviceBatches(ds, B, DEV)
        assert len(batches) == -(-len(ds) // B) and len(ds) % B
        for j in range(len(batches)):
            lo, hi = j * B, min((j + 1) * B, len(ds))
            X, lS_o, lS_i, T = (t.cpu() for t in batches[j])
            Xh, lS_oh, lS_ih, Th = criteo.CriteoDataset.collate(ds[lo:hi])
            assert torch.equal(lS_i, lS_ih) and torch.equal(lS_o, lS_oh) and torch.equal(T, Th)
            # the record decode of the same samples: bit for bit, including the fp32 log
            rows = ds.order[lo:hi]
            rec = np.concatenate([ds.y[rows, None], ds.X_int[rows], ds.X_cat[rows]], 1).astype(np.int32)
            db = DeviceBatch(PackedLayout(hi - lo, 26, 13, (hi - lo) * 26), DEV)
            BR.decode_records(torch.from_numpy(rec).to(DEV), max_ind_range, db)
            nb = batches.batches[hi - lo][0]
            for a, b in ((nb.X, db.X), (nb.target, db.target), (nb.offsets, db.offsets), (nb.indices, db.indices)):
                assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                   b.view(torch.int32) if b.dtype == torch.float32 else b)
            # torch.log on the CPU and logf on the GPU may round differently: at most 1 ulp apart
            u = _ulps(X, Xh)
            assert int(u.max()) <= 1
            log_ulps += int((u != 0).sum())
            checked += X.numel()
            if max_ind_range > 0:
                assert 0 <= int(lS_i.min()) and int(lS_i.max()) < max_ind_range
    print("gather: %d of %d log values differ from torch.log on the CPU by 1 ulp" % (log_ulps, checked))


def test_outputs_are_written_in_full_and_nothing_past_them():
    np.random.seed(3)
    ds = criteo.CriteoDataset("kaggle", 40, 0.0, "day", "train", RAW, PRO).to_device(DEV)
    n, G = 77, 64                                        # 77 = one full tile and a partial one
    X = torch.full((n * 13 + G,), float("nan"), device=DEV)
    T = torch.full((n + G,), float("nan"), device=DEV)
    off = torch.full((26 * (n + 1) + G,), -7, dtype=torch.int64, device=DEV)
    ind = torch.full((26 * n + G,), -7, dtype=torch.int64, device=DEV)
    ids = ds.dev[3][100:100 + n]
    X_int, X_cat, y = ds.dev[:3]
    _lib.check(_lib.lib().dlrm_b200_gather_records(X_int.data_ptr(), X_cat.data_ptr(), y.data_ptr(), ids.data_ptr(), n,
                                                   13, 26, 40, X.data_ptr(), T.data_ptr(), off.data_ptr(),
                                                   ind.data_ptr(), None))
    torch.cuda.synchronize()
    assert not X[:n * 13].isnan().any() and not T[:n].isnan().any()
    assert X[n * 13:].isnan().all() and T[n:].isnan().all()
    assert (off[:26 * (n + 1)] >= 0).all() and (off[26 * (n + 1):] == -7).all()
    assert (ind[:26 * n] >= 0).all() and (ind[26 * n:] == -7).all()
    Xh, _, lS_ih, Th = criteo.CriteoDataset.collate(ds[100:100 + n])
    assert torch.equal(ind[:26 * n].cpu().view(26, n), lS_ih) and torch.equal(T[:n].cpu().view(-1, 1), Th)
    assert torch.equal(off[:26 * (n + 1)].cpu(), (torch.arange(26)[:, None] * n + torch.arange(n + 1)[None]).view(-1))


def test_assembly_rejects_bad_arguments():
    lib = _lib.lib()
    buf = torch.zeros(1 << 16, dtype=torch.int64, device=DEV)
    p = buf.data_ptr()
    for n, nd, ns, msg in [(0, 13, 26, b"n=0"), (4, 0, 26, b"num_dense=0"), (4, 13, -1, b"num_sparse=-1"),
                           (4, 13, 200, b"num_sparse=200")]:
        assert lib.dlrm_b200_gather_records(p, p, p, p, n, nd, ns, -1, p, p, p, p, None) != 0
        assert msg in lib.dlrm_b200_last_error()
    assert lib.dlrm_b200_gather_records(p, p, p, None, 4, 13, 26, -1, p, p, p, p, None) != 0
    assert b"NULL" in lib.dlrm_b200_last_error()
    torch.cuda.synchronize()


def _cli(tag, extra=()):
    flags = open(os.path.join(GOLD, "cli_kaggle_%s.flags" % tag)).read().split()
    cmd = [sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py")] + flags + [
        "--raw-data-file=" + RAW, "--processed-data-file=" + PRO, "--use-gpu"] + list(extra)
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


@pytest.mark.parametrize("tag", ["A", "B", "C"])
def test_cli_matches_the_reference_run(tag):
    """fp32 CUDA-core GEMMs (--gemm=simt; these small MLPs take that path anyway): every loss within 1e-5 of the
    reference's CPU run, the dataset, test, accuracy and metric lines identical."""
    want = open(os.path.join(GOLD, "cli_kaggle_%s.txt" % tag)).read().splitlines()
    got = _cli(tag, ["--gemm=simt"]).splitlines()
    loss = re.compile(r"Finished training it .* loss ([0-9.]+)")
    want_loss = [float(loss.match(ln).group(1)) for ln in want if loss.match(ln)]
    got_loss = [float(loss.match(ln).group(1)) for ln in got if loss.match(ln)]
    assert len(got_loss) == len(want_loss) > 0
    np.testing.assert_allclose(got_loss, want_loss, rtol=0, atol=1e-5)
    other = re.compile(r"Sparse fea|Randomized|Defined|Split data|Testing at|accuracy|^recall ")
    assert [ln for ln in got if other.search(ln)] == [ln for ln in want if other.search(ln)]
