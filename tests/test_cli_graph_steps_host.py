"""Host side of --cuda-graph-steps: the flag, its refusals, and the static stage a batch is copied into (on the CPU:
the stage is plain tensors, the copies are the same ops on either device)."""
import pytest
import torch


def test_flag_parses_and_is_off_by_default():
    from dlrm_b200.cli import build_parser

    assert build_parser().parse_args([]).cuda_graph_steps is False
    assert build_parser().parse_args(["--cuda-graph-steps"]).cuda_graph_steps is True


@pytest.mark.parametrize("extra,env,msg", [
    (["--emb-dtype=fp16", "--data-generation=random"], "1", "needs --emb-dtype=fp32"),
    (["--data-generation=random"], "2", "runs on one GPU"),
    (["--data-generation=random"], "1", "needs --data-generation=dataset"),
    (["--data-generation=synthetic"], "1", "needs --data-generation=dataset"),
])
def test_refusals(monkeypatch, extra, env, msg):
    from dlrm_b200 import cli

    monkeypatch.setenv("WORLD_SIZE", env)
    with pytest.raises(SystemExit) as ei:
        cli.run(["--cuda-graph-steps"] + extra)
    assert str(ei.value).startswith("ERROR: --cuda-graph-steps") and msg in str(ei.value)


def test_stage_takes_full_batches_in_packed_layout():
    from dlrm_b200.graph_steps import _Stage

    B, T, m = 5, 3, 4
    st = _Stage(B, T, m, "cpu")
    X = torch.rand(B, m)
    lS_o = torch.arange(B).expand(T, B)
    lS_i = torch.randint(0, 100, (T, B))
    tgt = torch.rand(B, 1)
    assert st.fits(X, lS_o, lS_i)
    assert not st.fits(X[:4], lS_o[:, :4], lS_i[:, :4])
    assert not st.fits(X, lS_o, [lS_i[k] for k in range(T)])
    st.load_from(X, lS_o, lS_i, tgt)
    assert torch.equal(st.X, X) and torch.equal(st.target, tgt)
    assert torch.equal(st.indices.view(T, B), lS_i)
    want = torch.arange(T)[:, None] * B + torch.arange(B + 1)[None, :]
    assert torch.equal(st.offsets, want)
    assert st.sparse.include_last and st.sparse.batch == B and st.sparse.nnz_total == B * T
