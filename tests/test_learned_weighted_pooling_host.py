"""Learned weighted pooling (--weighted-pooling=learned) without a GPU: the float64 restatement of the fused step
(oracle/learned_f64.py) against the live reference's recorded training (tests/golden/cfg0_learned.npz), the flag's way
from the command line to the model, and the refusals that stay (host tables, sharded runs)."""
import numpy as np
import pytest
import torch

from golden_util import Golden
from oracle import dlrm_numpy as O
from oracle.learned_f64 import OPT_ADAGRAD, learned_step_f64
from oracle.sparse_f64 import OPT_RWSADAGRAD, OPT_SGD

_OPT = {"sgd": OPT_SGD, "rwsadagrad": OPT_RWSADAGRAD, "adagrad": OPT_ADAGRAD}


@pytest.mark.parametrize("optname", ["sgd", "rwsadagrad", "adagrad"])
def test_float64_step_reproduces_the_reference_first_step(optname):
    """dY of every table from the float64 forward/backward of the initial model, then learned_step_f64: tables, v_W_l
    and every accumulator equal the reference's state after its first optimizer step."""
    g = Golden("cfg0_learned")
    p = g.params()
    X, off, idx, T = g.batch(0)
    p64 = dict(emb=[w.astype(np.float64) for w in p["emb"]], v_W_l=[v.astype(np.float64) for v in p["v_W_l"]],
               bot=[(W.astype(np.float64), b.astype(np.float64)) for W, b in p["bot"]],
               top=[(W.astype(np.float64), b.astype(np.float64)) for W, b in p["top"]])
    r = O.dlrm_backward(p64, X.astype(np.float64), off, idx, T.astype(np.float64), loss="bce", dtype=np.float64)
    assert abs(float(r["loss"]) - float(g[f"{optname}_losses"][0])) < 1e-6
    lr, opt = float(g[f"{optname}_lr"]), _OPT[optname]
    for k, n in enumerate(g.ln_emb):
        acc = {"sgd": None, "rwsadagrad": np.zeros(n, np.float32), "adagrad": np.zeros((n, g.m_spa), np.float32)}[optname]
        vsum = None if optname == "sgd" else np.zeros(n, np.float32)
        W2, acc2, v2, vs2, rows = learned_step_f64(p["emb"][k], acc, p["v_W_l"][k], vsum, idx[k], off[k], idx[k].size,
                                                   r["d_ly"][k], opt, lr, 1e-10)
        assert rows.size > 0
        np.testing.assert_allclose(W2, g[f"{optname}0_emb{k}"], rtol=2e-5, atol=1e-6)
        np.testing.assert_allclose(v2, g[f"{optname}0_v{k}"], rtol=2e-5, atol=1e-6)
        if optname == "rwsadagrad":
            np.testing.assert_allclose(acc2, g[f"{optname}0_mom{k}"], rtol=1e-4, atol=1e-12)
        if optname == "adagrad":
            np.testing.assert_allclose(acc2, g[f"{optname}0_acc{k}"], rtol=1e-4, atol=1e-12)
        if optname != "sgd":
            np.testing.assert_allclose(vs2, g[f"{optname}0_vsum{k}"], rtol=1e-4, atol=1e-12)
        untouched = np.setdiff1d(np.arange(n), rows)
        assert np.array_equal(v2[untouched], p["v_W_l"][k][untouched])      # a zero gradient: v stays as it was
        assert np.array_equal(g[f"{optname}0_v{k}"][untouched], p["v_W_l"][k][untouched])


def test_cli_flag_reaches_the_model(monkeypatch):
    """--weighted-pooling=learned goes to DLRM_Net as weighted_pooling="learned" with each optimizer."""
    import dlrm_b200.cli as cli
    import dlrm_b200.dlrm_net as dn
    import dlrm_b200.optim as fo

    got = []

    class StandIn(torch.nn.Module):
        def __init__(self, m_spa, ln_emb, ln_bot, ln_top, **kw):
            super().__init__()
            got.append(kw.get("weighted_pooling"))
            self.lin = torch.nn.Linear(int(ln_bot[0]), 1)
            self.loss_fn = torch.nn.MSELoss()

        def forward(self, X, lS_o, lS_i):
            return torch.sigmoid(self.lin(X))

    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)
    monkeypatch.setattr(dn, "DLRM_Net", StandIn)
    for name in ("SGD", "RWSAdagrad", "Adagrad"):
        monkeypatch.setattr(fo, name, torch.optim.SGD)
    base = ["--arch-sparse-feature-size=16", "--arch-embedding-size=64-16", "--arch-mlp-bot=5-16",
            "--arch-mlp-top=8-1", "--mini-batch-size=8", "--num-batches=1", "--use-gpu", "--weighted-pooling=learned"]
    for opt in ("sgd", "rwsadagrad", "adagrad"):
        cli.run(base + ["--optimizer=" + opt])
    assert got == ["learned"] * 3


def test_host_tables_refuse_weighted_pooling(monkeypatch):
    import dlrm_b200.cli as cli

    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    with pytest.raises(SystemExit) as e:
        cli.run(["--arch-sparse-feature-size=16", "--arch-embedding-size=64-16", "--arch-mlp-bot=5-16",
                 "--arch-mlp-top=8-1", "--mini-batch-size=8", "--num-batches=1", "--use-gpu",
                 "--weighted-pooling=learned", "--emb-host-tables=0"])
    assert "does not support weighted pooling" in str(e.value)


def test_model_refuses_learned_weights_on_host_tables_and_sharded_runs(monkeypatch):
    """The refusals name their reason before any device memory is touched (DLRM_Net checks host tables first; the
    engine refuses sharded placements)."""
    import dlrm_b200.dlrm_net as dn
    import dlrm_b200.engine as E

    with pytest.raises(SystemExit) as e:
        dn.DLRM_Net(16, [64, 16], [5, 16], [8, 1], arch_interaction_op="dot", weighted_pooling="learned",
                    emb_host_tables=[0])
    assert "host embedding tables do not support weighted pooling" in str(e.value)

    class Probe(E.Engine):                       # just the placement check of the constructor
        def __init__(self, shards, host=()):
            self.shards, self.host, self.total_rows = shards, list(host), 80
            self.learned_row_weights = True
            E.Engine._check_learned_placement(self)

    with pytest.raises(ValueError, match="not supported on sharded runs"):
        Probe([dict(table=0, rows=128, row_lo=0, row_n=64, part=0, nparts=2)])
    with pytest.raises(ValueError, match="host tables do not support weighted pooling"):
        Probe([dict(table=0, rows=64, row_lo=0, row_n=64, part=0, nparts=1)], host=[0])
    Probe([dict(table=0, rows=64, row_lo=0, row_n=64, part=0, nparts=1)])
