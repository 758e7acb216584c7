"""Host-side control flow of the CLI's MLPerf binary-loader path (--data-generation=dataset --mlperf-bin-loader) and of
--mlperf-logging, on CPU: a stand-in model, the device decode replaced by CriteoBinDataset.__getitem__ (its host
oracle) and the metric keys kept on the CPU.  Runs on the fixture of tests/golden/bin_* (oracle/make_bin_goldens.py)."""
import os
import re

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FLAGS = open(os.path.join(GOLD, "cli_bin_A.flags")).read().split()
DATA = ["--raw-data-file=" + os.path.join(GOLD, "bin_day"),
        "--processed-data-file=" + os.path.join(GOLD, "bin_processed.npz")]
METRIC = re.compile(r"recall \d\.\d{4}, precision \d\.\d{4}, f1 \d\.\d{4}, ap \d\.\d{4}, auc \d\.\d{4}, "
                    r"best auc \d\.\d{4}, accuracy \d+\.\d{3} %, best accuracy \d+\.\d{3} %")


@pytest.fixture
def cli_on_cpu(monkeypatch):
    import dlrm_b200.binrecords as br
    import dlrm_b200.cli as cli
    import dlrm_b200.dlrm_net as dn
    import dlrm_b200.metrics as mt
    import dlrm_b200.optim as fo

    rec = {"seen": [], "ln_emb": None, "items": []}

    class StandIn(torch.nn.Module):
        def __init__(self, m_spa, ln_emb, ln_bot, ln_top, **kw):
            super().__init__()
            rec["ln_emb"] = list(ln_emb)
            self.lin = torch.nn.Linear(int(ln_bot[0]), 1)
            self.loss_fn = torch.nn.BCELoss()
            self.n_tables = len(ln_emb)

        def forward(self, X, lS_o, lS_i):
            assert lS_o.shape == (self.n_tables, X.shape[0]) and len(lS_i) == self.n_tables
            rec["seen"].append((X.shape[0], max(int(i.max()) for i in lS_i)))
            return torch.sigmoid(self.lin(X))

    class HostBatches:                       # the device decode, replaced by its host oracle
        def __init__(self, ds, device):
            self.ds = ds

        def __len__(self):
            return len(self.ds)

        def __getitem__(self, j):
            rec["items"].append((self.ds.batch_size, j))
            return self.ds[j]

    orig_to, orig_keys = torch.Tensor.to, mt.ScoreKeys
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    # device moves are no-ops here; dtype conversions still happen
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: orig_to(self, *[x for x in a if isinstance(x, torch.dtype)]))
    monkeypatch.setattr(dn, "DLRM_Net", StandIn)
    monkeypatch.setattr(fo, "SGD", torch.optim.SGD)
    monkeypatch.setattr(br, "DeviceBatches", HostBatches)
    monkeypatch.setattr(mt, "ScoreKeys", lambda cap, device: orig_keys(cap, "cpu"))
    return cli, rec


def test_files_tables_batches_and_lines(cli_on_cpu, capsys):
    cli, rec = cli_on_cpu
    cli.run(FLAGS + DATA + ["--use-gpu"])
    out = capsys.readouterr().out.splitlines()
    assert rec["ln_emb"] == [1000, 7, 300, 20, 1000] + [11] * 21           # counts capped at --max-ind-range
    train = [b for b, _ in rec["seen"] if b != 256 and b != 232]
    assert len(train) == 2 * 32 and train[31] == 16 and set(train[:31]) == {64}   # 2000 = 31 x 64 + 16
    test = [b for b, _ in rec["seen"] if b in (256, 232)]
    assert test == [256, 256, 256, 232] * 8                                # 1000 = 3 x 256 + 232, 8 passes
    assert max(m for _, m in rec["seen"]) < 1000                           # ids folded by --max-ind-range
    body = [ln for ln in out if re.match(r"Finished|Testing at|recall", ln)]
    assert [ln.split()[0] for ln in body] == ["Finished", "Testing", "recall"] * 8
    assert body[1] == "Testing at - 8/32 of epoch 0," and body[-2] == "Testing at - 32/32 of epoch 1,"
    assert all(METRIC.fullmatch(ln) for ln in body[2::3])
    assert all(ln.endswith("best accuracy 0.000 %") for ln in body[2::3])  # the reference never updates it
    for ln in body[2::3]:                                                  # best auc = this pass's auc
        auc, best = re.search(r"auc (\S+), best auc (\S+),", ln).groups()
        assert auc == best


@pytest.mark.parametrize("flag,text", [("--mlperf-auc-threshold=1e-9", "MLPerf testing auc threshold 1e-09 reached"),
                                       ("--mlperf-acc-threshold=1e-9", "MLPerf testing accuracy threshold 1e-09 reached")])
def test_threshold_stops_both_loops(cli_on_cpu, capsys, flag, text):
    cli, rec = cli_on_cpu
    cli.run(FLAGS + DATA + ["--use-gpu", flag])
    out = capsys.readouterr().out
    assert text + ", stop training" in out
    assert out.count("Finished training") == 1 and out.count("recall ") == 1 and len(rec["seen"]) == 8 + 4


def test_checkpoint_holds_test_auc(cli_on_cpu, capsys, tmp_path):
    cli, _ = cli_on_cpu
    ck = str(tmp_path / "m.pt")
    cli.run(FLAGS + DATA + ["--use-gpu", "--nepochs=1", "--num-batches=8", "--save-model=" + ck])
    out = capsys.readouterr().out
    assert out.count("Saving model to " + ck) == 1
    sd = torch.load(ck, weights_only=False)
    auc = float(re.search(r" auc (\S+),", out).group(1))
    assert "test_auc" in sd and abs(sd["test_auc"] - auc) <= 5e-5 and sd["nbatches"] == 8 and sd["nbatches_test"] == 4


def _train_order(cli, rec, seed):
    del rec["items"][:]
    cli.run(FLAGS + DATA + ["--use-gpu", "--test-freq=-1", "--mlperf-bin-shuffle", "--numpy-rand-seed=%d" % seed])
    order = [j for b, j in rec["items"] if b == 64]
    return order[:32], order[32:]


def test_bin_shuffle_is_a_new_permutation_every_epoch_and_follows_the_seed(cli_on_cpu):
    cli, rec = cli_on_cpu
    e0, e1 = _train_order(cli, rec, 5)
    assert sorted(e0) == sorted(e1) == list(range(32)) and e0 != e1 and e0 != list(range(32))
    assert _train_order(cli, rec, 5) == (e0, e1)
    assert _train_order(cli, rec, 6)[0] != e0


def test_mlperf_logging_on_random_data(cli_on_cpu, capsys):
    cli, _ = cli_on_cpu
    base = ["--arch-sparse-feature-size=16", "--arch-embedding-size=64-16", "--arch-mlp-bot=5-16", "--arch-mlp-top=8-1",
            "--mini-batch-size=8", "--use-gpu", "--num-batches=4", "--test-freq=2", "--mlperf-logging",
            "--loss-function=bce"]
    cli.run(base + ["--round-targets=True"])
    out = capsys.readouterr().out
    assert len([ln for ln in out.splitlines() if METRIC.fullmatch(ln)]) == 2
    with pytest.raises(SystemExit) as e:
        cli.run(base)
    assert "--round-targets=True" in str(e.value)


@pytest.mark.parametrize("drop", ["--mlperf-bin-loader", "--memory-map", "--mlperf-logging", "--data-set=terabyte"])
def test_other_dataset_combinations_keep_the_refusal(cli_on_cpu, drop):
    cli, _ = cli_on_cpu
    with pytest.raises(SystemExit) as e:
        cli.run([f for f in FLAGS if f != drop] + DATA + ["--use-gpu"])
    assert "--data-generation=dataset is not supported" in str(e.value)


def test_missing_file_and_sharded_run_are_refused(cli_on_cpu, monkeypatch, tmp_path):
    cli, _ = cli_on_cpu
    with pytest.raises(SystemExit) as e:
        cli.run(FLAGS + ["--raw-data-file=" + str(tmp_path / "day"), DATA[1], "--use-gpu"])
    assert str(tmp_path / "day") + "_fea_count.npz does not exist" in str(e.value)
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit) as e:
        cli.run(FLAGS + DATA + ["--use-gpu"])
    assert "runs on one GPU" in str(e.value)


def test_mlperf_logging_refuses_a_sharded_random_run(cli_on_cpu, monkeypatch):
    cli, _ = cli_on_cpu
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit) as e:
        cli.run(["--arch-sparse-feature-size=16", "--arch-embedding-size=64-16", "--arch-mlp-bot=5-16",
                 "--arch-mlp-top=8-1", "--mini-batch-size=8", "--use-gpu", "--num-batches=4", "--test-freq=2",
                 "--mlperf-logging", "--round-targets=True", "--loss-function=bce"])
    assert "--mlperf-logging runs on one GPU" in str(e.value)


def test_final_save_reloads_under_mlperf_logging(cli_on_cpu, capsys, tmp_path, monkeypatch):
    """A run without test passes saves its final state; --mlperf-logging --load-model reads `test_auc` from it."""
    cli, _ = cli_on_cpu
    orig_load = torch.load
    monkeypatch.setattr(torch, "load", lambda f, map_location=None, **k: orig_load(f, map_location="cpu", **k))
    ck = str(tmp_path / "m.pt")
    cli.run(FLAGS + DATA + ["--use-gpu", "--nepochs=1", "--num-batches=4", "--test-freq=-1", "--save-model=" + ck])
    assert torch.load(ck, weights_only=False)["test_auc"] == 0.0
    capsys.readouterr()
    cli.run(FLAGS + DATA + ["--use-gpu", "--load-model=" + ck, "--inference-only"])
    out = capsys.readouterr().out
    assert "Testing state: accuracy = 0.000 %, auc = 0.000" in out and len(METRIC.findall(out)) == 1


def test_a_file_of_partial_records_is_refused_when_opened(tmp_path):
    from dlrm_b200.binrecords import CriteoBinDataset

    p = tmp_path / "bad.bin"
    p.write_bytes(b"\0" * (160 * 3 + 4))
    with pytest.raises(ValueError, match="not a whole number of 160-byte records"):
        CriteoBinDataset(str(p), None, batch_size=2)
