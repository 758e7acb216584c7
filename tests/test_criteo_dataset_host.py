"""Preprocessed Criteo dataset (dlrm_b200/criteo.py) on the CPU: split, sample order and numpy RNG consumption against
the reference CriteoDataset's recorded dump, items and collate against its recorded batches, and the CLI's dataset
path (table sizes, printed lines, batch counts, refusals) with a stand-in model and the device assembly replaced by
the host oracle.  Fixture: tests/golden/kaggle_* (oracle/make_kaggle_goldens.py)."""
import os
import re

import numpy as np
import pytest
import torch

from dlrm_b200 import criteo

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RAW = os.path.join(GOLD, "kaggle.txt")                     # never read: it names the day-count file
PRO = os.path.join(GOLD, "kaggle_processed.npz")
DATA = ["--raw-data-file=" + RAW, "--processed-data-file=" + PRO]
ORD = np.load(os.path.join(GOLD, "kaggle_orders.npz"))
COUNTS = np.load(PRO)["counts"]


def _flags(tag):
    return open(os.path.join(GOLD, "cli_kaggle_%s.flags" % tag)).read().split()


def _make(mode, split, data=None, mir=-1):
    return criteo.CriteoDataset("kaggle", mir, 0.0, mode, split, RAW, PRO, data=data)


def _state(key):
    st = np.random.get_state()
    return np.array_equal(st[1], ORD["rng_%s_keys" % key]) and st[2] == int(ORD["rng_%s_pos" % key])


@pytest.mark.parametrize("mode", ["none", "day", "total"])
def test_split_order_and_rng_state_match_the_reference(mode):
    np.random.seed(727)
    train = _make(mode, "train")
    test = _make(mode, "test", data=train)
    assert _state(mode)                      # the draws of both constructors, exactly: the model init comes next
    val = _make(mode, "val", data=train)
    for ds, split in ((train, "train"), (test, "test"), (val, "val")):
        assert np.array_equal(ds.order, ORD["%s_%s" % (mode, split)]), split
    assert (len(train), len(test), len(val)) == (1200, 100, 100)


def test_whole_set_split_draws_one_permutation():
    np.random.seed(5)
    ds = _make("total", "none")
    assert _state("split_none") and len(ds) == 1400
    np.random.seed(5)
    perm = np.random.permutation(1400)
    # the reference's X[perm] = X: position perm[i] holds row i
    assert np.array_equal(ds.order[perm], np.arange(1400))


def test_one_permutation_too_few_is_rejected():
    """Negative control for the comparison above: per-day shuffling that skips the last training day."""
    np.random.seed(727)
    days = np.array_split(np.arange(1400), np.cumsum([200] * 6))
    for i in range(5):
        days[i] = np.random.permutation(days[i])
    short = np.concatenate(days[:-1])
    assert not np.array_equal(short, ORD["day_train"])
    assert not _state("day")


@pytest.mark.parametrize("name,mode,split,mir,bs", [("train", "total", "train", 40, 32), ("test", "none", "test", -1, 48)])
def test_items_and_collate_match_the_recorded_batches(name, mode, split, mir, bs):
    np.random.seed(727)
    ds = _make(mode, split, mir=mir)
    rec = np.load(os.path.join(GOLD, "kaggle_batches.npz"))
    nb = 0
    for j, lo in enumerate(range(0, len(ds), bs)):
        X, lS_o, lS_i, T = criteo.CriteoDataset.collate([ds[i] for i in range(lo, min(lo + bs, len(ds)))])
        assert X.dtype == torch.float32 and lS_o.dtype == lS_i.dtype == torch.int64 and T.dtype == torch.float32
        assert torch.equal(X, torch.from_numpy(rec["%s_%d_X" % (name, j)]))
        assert torch.equal(lS_o, torch.from_numpy(rec["%s_%d_lS_o" % (name, j)]).long())
        assert torch.equal(lS_i, torch.from_numpy(rec["%s_%d_lS_i" % (name, j)]).long())
        assert torch.equal(T, torch.from_numpy(rec["%s_%d_T" % (name, j)]))
        nb += 1
    assert nb == len([k for k in rec.files if k.startswith(name + "_") and k.endswith("_X")])
    x_int, x_cat, y = ds[3]
    assert x_int.dtype == x_cat.dtype == np.int32 and (mir <= 0 or x_cat.max() < mir)


def test_dataset_refusals(tmp_path):
    with pytest.raises(FileNotFoundError, match="getCriteoAdData"):
        criteo.CriteoDataset("kaggle", -1, 0.0, "total", "train", RAW, str(tmp_path / "p.npz"))
    with pytest.raises(FileNotFoundError, match=re.escape(str(tmp_path / "kaggle_day_count.npz"))):
        criteo.CriteoDataset("kaggle", -1, 0.0, "total", "train", str(tmp_path / "kaggle.txt"), PRO)
    with pytest.raises(ValueError, match="_reordered.npz"):
        criteo.CriteoDataset("kaggle", -1, 0.0, "total", "train", RAW, PRO, memory_map=True)
    with pytest.raises(ValueError, match="not supported"):
        criteo.CriteoDataset("avazu", -1, 0.0, "total", "train", RAW, PRO)
    # the Terabyte set has 24 days: this 7-day fixture does not pass for it
    np.savez(tmp_path / "kaggle.txt_day_count.npz", total_per_file=np.full(7, 200))
    with pytest.raises(ValueError, match="7 days, terabyte has 24"):
        criteo.CriteoDataset("terabyte", -1, 0.0, "total", "train", str(tmp_path / "kaggle.txt"), PRO)


@pytest.fixture
def cli_on_cpu(monkeypatch):
    import dlrm_b200.cli as cli
    import dlrm_b200.dlrm_net as dn
    import dlrm_b200.metrics as mt
    import dlrm_b200.optim as fo

    rec = {"seen": [], "ln_emb": None, "ln_bot": None, "rng_at_init": None}

    class StandIn(torch.nn.Module):
        def __init__(self, m_spa, ln_emb, ln_bot, ln_top, **kw):
            super().__init__()
            rec["ln_emb"], rec["ln_bot"] = list(ln_emb), list(ln_bot)
            rec["rng_at_init"] = np.random.get_state()
            self.lin = torch.nn.Linear(int(ln_bot[0]), 1)
            self.loss_fn = torch.nn.BCELoss()
            self.n_tables = len(ln_emb)

        def forward(self, X, lS_o, lS_i):
            assert lS_o.shape == (self.n_tables, X.shape[0]) and lS_i.shape == (self.n_tables, X.shape[0])
            rec["seen"].append((X.shape[0], int(lS_i.max())))
            return torch.sigmoid(self.lin(X))

    class HostBatches:                       # the device assembly, replaced by its host oracle
        def __init__(self, ds, batch_size, device):
            self.ds, self.bs = ds, batch_size

        def __len__(self):
            return -(-len(self.ds) // self.bs)

        def __getitem__(self, j):
            return criteo.CriteoDataset.collate(self.ds[j * self.bs:min((j + 1) * self.bs, len(self.ds))])

    orig_to, orig_keys = torch.Tensor.to, mt.ScoreKeys
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: orig_to(self, *[x for x in a if isinstance(x, torch.dtype)]))
    monkeypatch.setattr(dn, "DLRM_Net", StandIn)
    monkeypatch.setattr(fo, "SGD", torch.optim.SGD)
    monkeypatch.setattr(fo, "RWSAdagrad", torch.optim.SGD)
    monkeypatch.setattr(criteo, "DeviceBatches", HostBatches)
    monkeypatch.setattr(mt, "ScoreKeys", lambda cap, device: orig_keys(cap, "cpu"))
    return cli, rec


@pytest.mark.parametrize("tag,mode,ntrain,ntest", [("A", "total", [32] * 37 + [16], [48, 48, 4]),
                                                   ("B", "day", [64] * 18 + [48], [64, 36]),
                                                   ("C", "none", [32] * 37 + [16], [64, 36])])
def test_cli_tables_lines_and_batches(cli_on_cpu, capsys, tag, mode, ntrain, ntest):
    cli, rec = cli_on_cpu
    flags = _flags(tag)
    cli.run(flags + DATA + ["--use-gpu"])
    out = capsys.readouterr().out.splitlines()
    mir = int(dict(f.split("=", 1) for f in flags if "=" in f).get("--max-ind-range", -1))
    want = COUNTS if mir <= 0 else np.minimum(COUNTS, mir)
    assert rec["ln_emb"] == list(want) and rec["ln_bot"][0] == 13
    # the model is built after both constructors drew from numpy's global RNG, as in the reference
    st = rec["rng_at_init"]
    assert np.array_equal(st[1], ORD["rng_%s_keys" % mode]) and st[2] == int(ORD["rng_%s_pos" % mode])
    gold = open(os.path.join(GOLD, "cli_kaggle_%s.txt" % tag)).read().splitlines()
    head = gold[:gold.index("time/loss/accuracy (if enabled):")]
    assert [ln for ln in out if ln in head or ln.startswith(("Sparse fea", "Defined", "Randomized", "Split data"))] == head
    assert "Reading pre-processed data=" + PRO in out
    assert [ln for ln in out if ln.startswith("Testing at")] == [ln for ln in gold if ln.startswith("Testing at")]
    nep = 2 if tag == "A" else 1
    passes = len([ln for ln in gold if ln.startswith("Testing at")])
    sizes = [b for b, _ in rec["seen"]]
    assert sorted(sizes) == sorted(ntrain * nep + ntest * passes)
    if mir > 0:
        assert max(m for _, m in rec["seen"]) < mir


def test_cli_num_batches_and_test_batch_default(cli_on_cpu):
    cli, rec = cli_on_cpu
    flags = [f for f in _flags("A") if not f.startswith(("--test-mini-batch-size", "--nepochs"))]
    cli.run(flags + DATA + ["--use-gpu", "--num-batches=5", "--test-freq=5"])
    # 5 training batches, then a test pass at the training batch size that also stops at 5 batches (as the reference)
    assert [b for b, _ in rec["seen"]] == [32] * 5 + [32, 32, 32, 4]


@pytest.mark.parametrize("extra,msg", [
    (["--memory-map"], "per-day _reordered.npz files are not read"),
    (["--data-set=avazu"], "--data-set=avazu is not supported"),
    (["--processed-data-file=/nonexistent/p.npz"], "/nonexistent/p.npz does not exist"),
    (["--raw-data-file=/nonexistent/kaggle.txt"], "/nonexistent/kaggle_day_count.npz does not exist"),
])
def test_cli_refusals(cli_on_cpu, extra, msg):
    cli, _ = cli_on_cpu
    with pytest.raises(SystemExit) as e:
        cli.run(_flags("A") + DATA + ["--use-gpu"] + extra)
    assert msg in str(e.value)
    if not msg.startswith("--data-set"):
        assert "--data-generation=dataset is not supported" in str(e.value)
    if "does not exist" in msg:
        assert "data_utils.getCriteoAdData" in str(e.value)


def test_cli_refuses_a_sharded_dataset_run(cli_on_cpu, monkeypatch):
    cli, _ = cli_on_cpu
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit) as e:
        cli.run(_flags("A") + DATA + ["--use-gpu"])
    assert "runs on one GPU" in str(e.value)


def test_preprocessing_flags_are_accepted_and_ignored(cli_on_cpu, capsys):
    cli, rec = cli_on_cpu
    cli.run(_flags("A") + DATA + ["--use-gpu", "--nepochs=1", "--data-sub-sample-rate=0.5", "--dataset-multiprocessing"])
    assert len([b for b, _ in rec["seen"] if b != 48 and b != 4]) == 38


def test_cli_mlperf_metric_line(cli_on_cpu, capsys):
    cli, _ = cli_on_cpu
    cli.run(_flags("C") + DATA + ["--use-gpu"])
    out = capsys.readouterr().out
    assert len(re.findall(r"^recall .* best accuracy 0\.000 %$", out, re.M)) == 2
