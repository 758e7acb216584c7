"""Element-wise Adagrad (`--optimizer=adagrad`) on the host: the float64 / fp32 restatements of oracle/adagrad_f64.py
against torch.optim.Adagrad on CPU sparse and dense gradients, the fp32 kernel order within its bound, negative
controls that the GPU tests' checks must reject, the CLI accepting the flag, and the optimizer's state_dict layout
against torch's."""
import re

import numpy as np
import pytest
import torch

from oracle import adagrad_f64 as A
from oracle import sparse_f64 as S


def _wide(rng, shape, lo=-8, hi=2):
    return (rng.choice([-1.0, 1.0], shape) * np.exp2(rng.uniform(lo, hi, shape))).astype(np.float32)


@pytest.mark.parametrize("D", [1, 3, 16, 128])
def test_sparse_restatement_matches_torch_adagrad(D):
    """torch.optim.Adagrad on one embedding table, stepped three times with lr_decay on an uncoalesced sparse gradient
    with duplicates.  After every step, from torch's previous state: the touched rows' accumulators equal the fp32
    kernel order bit for bit (RN(g*g) then the add), weights and accumulators are within the bound of the float64
    step, and rows not in the batch keep weight AND accumulator."""
    rng = np.random.default_rng(D)
    R, lr, lr_decay, eps = 50, 0.05, 0.1, 1e-10
    W0 = _wide(rng, (R, D), -4, 0)
    idx = rng.integers(0, R // 2, 60)                      # duplicates; rows >= R // 2 never occur
    G = _wide(rng, (idx.size, D))
    gc = A.dense_rows_sparse_grad(R, D, idx, G).coalesce()
    rows, g = gc.indices()[0].numpy(), gc.values().numpy()
    np.testing.assert_array_equal(rows, S.coalesce(idx)[0])
    p = torch.nn.Parameter(torch.from_numpy(W0.copy()))
    opt = torch.optim.Adagrad([p], lr=lr, lr_decay=lr_decay, eps=eps)
    w, s = W0.copy(), np.zeros((R, D), np.float32)
    for step in (1, 2, 3):
        p.grad = A.dense_rows_sparse_grad(R, D, idx, G)
        opt.step()
        got_w, got_s = p.detach().numpy().copy(), opt.state[p]["sum"].numpy().copy()
        c = A.clr(lr, step, lr_decay)
        w32, s32 = A.step_f32(w[rows], s[rows], g, c, eps)
        w64, s64 = A.step_f64(w[rows], s[rows], g, c, eps)
        bw, bs = A.step_bound(w64, s64, g, c, eps)
        np.testing.assert_array_equal(got_s[rows], s32)
        S.check_within(got_w[rows], w64, bw, f"step {step}: torch weights vs float64")
        S.check_within(w32, w64, bw, f"step {step}: fp32 kernel order vs float64")
        S.check_within(got_s[rows], s64, bs, f"step {step}: torch accumulators vs float64")
        rest = np.setdiff1d(np.arange(R), rows)
        np.testing.assert_array_equal(got_w[rest], W0[rest])
        assert np.all(got_s[rest] == 0)
        w, s = got_w, got_s


def test_dense_parameters_take_the_rwsadagrad_dense_step():
    """torch.optim.Adagrad on a dense gradient is the dense branch the engine runs for RWSAdagrad
    (oracle/dense_f64.dense_step, OPT_RWSADAGRAD): sum += g*g; p -= clr g / (sqrt(sum) + eps)."""
    from oracle import dense_f64 as O

    rng = np.random.default_rng(0)
    p0, g = _wide(rng, (7, 9), -4, 0), _wide(rng, (7, 9))
    p = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = torch.optim.Adagrad([p], lr=0.05, eps=1e-10)
    p.grad = torch.from_numpy(g.copy())
    opt.step()
    want_p, want_s = O.dense_step(p0, g, np.zeros_like(p0), O.OPT_RWSADAGRAD, 0.05, 1e-10)
    bw, bs = A.step_bound(want_p, want_s, g, 0.05, 1e-10)
    S.check_within(p.detach().numpy(), want_p, bw, "dense weights")
    S.check_within(opt.state[p]["sum"].numpy(), want_s, bs, "dense sum")


@pytest.mark.parametrize("D", [1, 3, 16, 64, 128, 132, 256, 1000])
def test_fp32_kernel_order_is_within_the_bound(D):
    rng = np.random.default_rng(D + 1)
    n = 400
    w, g = _wide(rng, (n, D), -4, 2), _wide(rng, (n, D), -30, 4)
    s = np.where(rng.random((n, D)) < 0.3, 0, np.abs(_wide(rng, (n, D), -20, 4))).astype(np.float32)
    for lr, eps in ((0.05, 1e-10), (1.0, 1e-4), (3e-3, 0.0)):
        w32, s32 = A.step_f32(w, s, g, lr, eps)
        w64, s64 = A.step_f64(w, s, g, lr, eps)
        bw, bs = A.step_bound(w64, s64, g, lr, eps)
        assert S.check_within(w32, w64, bw, "weights") <= 1
        assert S.check_within(s32, s64, bs, "accumulators") <= 1


def test_negative_controls_are_rejected():
    """What the GPU tests compare must catch each of these wrong steps."""
    rng = np.random.default_rng(5)
    n, D, lr, eps = 2000, 16, 0.05, 1e-10
    w, g = _wide(rng, (n, D), -4, 0), _wide(rng, (n, D), -6, 2)
    s = _wide(rng, (n, D), -6, 2) ** 2
    w32, s32 = A.step_f32(w, s, g, lr, eps)
    w64, s64 = A.step_f64(w, s, g, lr, eps)
    bw, bs = A.step_bound(w64, s64, g, lr, eps)
    # FMA-contracted accumulator: the accumulators (compared bit for bit) differ
    _, sf = A.step_f32(w, s, g, lr, eps, fma_accumulator=True)
    assert not np.array_equal(sf, s32)
    # eps inside the square root: far outside the weight bound at small accumulators
    s_small = np.zeros_like(s)
    we, _ = A.step_f32(w, s_small, g * 1e-6, lr, 1e-4, eps_in_sqrt=True)
    w64e, s64e = A.step_f64(w, s_small, g * 1e-6, lr, 1e-4)
    bwe, _ = A.step_bound(w64e, s64e, g * 1e-6, lr, 1e-4)
    assert S.worst_ratio(we, w64e, bwe)[0] > 1
    # RWSAdagrad's row-wise mean instead of one accumulator per element
    wm, sm = A.step_f32(w, s, g, lr, eps, row_mean=True)
    assert S.worst_ratio(wm, w64, bw)[0] > 1 and S.worst_ratio(sm, s64, bs)[0] > 1
    # lr_decay ignored at step 3 (clr = lr instead of lr / (1 + 2 lr_decay))
    c = A.clr(lr, 3, 0.5)
    wd, _ = A.step_f32(w, s, g, lr, eps)
    w64d, s64d = A.step_f64(w, s, g, c, eps)
    bwd, _ = A.step_bound(w64d, s64d, g, c, eps)
    assert S.worst_ratio(wd, w64d, bwd)[0] > 1
    # stepping a row that is not in the batch (here with another row's gradient): its weight and accumulator move,
    # which the bitwise comparison of untouched rows catches
    wu, su = A.step_f32(w[:1], s[:1], g[1:2], lr, eps)
    assert not np.array_equal(wu, w[:1]) and not np.array_equal(su, s[:1])


# ---------------------------------------------------------------------------------------------- CLI + state_dict
@pytest.fixture
def cli_on_cpu(monkeypatch):
    import dlrm_b200.cli as cli
    import dlrm_b200.dlrm_net as dn
    import dlrm_b200.optim as fo

    class StandIn(torch.nn.Module):
        def __init__(self, m_spa, ln_emb, ln_bot, ln_top, **kw):
            super().__init__()
            self.lin = torch.nn.Linear(int(ln_bot[0]), 1)
            self.loss_fn = torch.nn.MSELoss()

        def forward(self, X, lS_o, lS_i):
            return torch.sigmoid(self.lin(X))

    made = []

    def adagrad(params, **kw):
        made.append(kw)
        return torch.optim.Adagrad(params, **kw)

    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)
    monkeypatch.setattr(dn, "DLRM_Net", StandIn)
    monkeypatch.setattr(fo, "Adagrad", adagrad)
    return cli, made


def test_cli_accepts_optimizer_adagrad_and_checkpoints_its_state(cli_on_cpu, capsys, tmp_path):
    cli, made = cli_on_cpu
    ck = str(tmp_path / "m.pt")
    cli.run(["--arch-sparse-feature-size=16", "--arch-embedding-size=64-16", "--arch-mlp-bot=5-16",
             "--arch-mlp-top=8-1", "--mini-batch-size=8", "--print-freq=1", "--use-gpu", "--num-batches=3",
             "--optimizer=adagrad", "--learning-rate=0.01", "--test-freq=3", "--save-model=" + ck])
    out = capsys.readouterr().out
    assert made == [dict(lr=0.01)]                         # opts[args.optimizer](parameters, lr=...)
    assert len(re.findall(r"Finished training it \d/3", out)) == 3
    sd = torch.load(ck, weights_only=False)["opt_state_dict"]
    assert set(sd["state"][0]) == {"step", "sum"} and float(sd["state"][0]["step"]) == 3.0


class _FakeEngine:
    """The memory layout dlrm_b200.optim reads: a dense arena holding the MLP parameters, a table arena and the
    element-wise accumulator arena (CPU tensors stand in for the device ones)."""

    def __init__(self, rows, D, dense_shapes):
        self.D, self.row_base = D, np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
        self.tables = torch.zeros((int(self.row_base[-1]), D))
        n = sum(int(np.prod(s)) for s in dense_shapes)
        self.dense, self.dense_state, self.acc_ew = torch.zeros(n), None, None
        self.opt_step, self.ensured = 0, []
        self.dense_params, o = [], 0
        for s in dense_shapes:
            self.dense_params.append(self.dense[o:o + int(np.prod(s))].view(s))
            o += int(np.prod(s))

    def ensure_optimizer_state(self, name):
        self.ensured.append(name)
        self.dense_state = torch.zeros_like(self.dense)
        self.acc_ew = torch.zeros_like(self.tables)

    def table(self, k):
        return self.tables[int(self.row_base[k]):int(self.row_base[k + 1])]

    def accumulator_ew(self, k):
        return self.acc_ew[int(self.row_base[k]):int(self.row_base[k + 1])]


def _fake_net(rows=(10, 4), D=3, dense_shapes=((5, 3), (5,))):
    import weakref

    class Net:
        pass

    net = Net()
    net._engine = _FakeEngine(list(rows), D, list(dense_shapes))
    params = []
    for t in [net._engine.table(k) for k in range(len(rows))] + net._engine.dense_params:
        p = torch.nn.Parameter(t, requires_grad=True)
        assert p.data_ptr() == t.data_ptr()
        p._dlrm_net = weakref.ref(net)
        params.append(p)
    return net, params


def test_state_dict_has_torch_adagrad_layout():
    from dlrm_b200.optim import Adagrad

    net, params = _fake_net()
    opt = Adagrad(params, lr=0.1, lr_decay=0.01)
    assert net._engine.ensured == ["adagrad"]
    eng = net._engine
    eng.opt_step = 4
    eng.acc_ew.uniform_()
    eng.dense_state.uniform_()
    sd = opt.state_dict()
    ref = torch.optim.Adagrad([torch.nn.Parameter(p.detach().clone()) for p in params], lr=0.1, lr_decay=0.01)
    for p in ref.param_groups[0]["params"]:
        p.grad = torch.ones_like(p)
    ref.step()
    rsd = ref.state_dict()
    assert set(sd["param_groups"][0]) == set(rsd["param_groups"][0])
    assert {k: v for k, v in sd["param_groups"][0].items() if k != "params"} == \
        {k: v for k, v in rsd["param_groups"][0].items() if k != "params"}
    assert sorted(sd["state"]) == sorted(rsd["state"])
    for i, st in sd["state"].items():
        assert set(st) == set(rsd["state"][i]) == {"step", "sum"}
        assert st["sum"].shape == rsd["state"][i]["sum"].shape == params[i].shape
        assert torch.is_tensor(st["step"]) and st["step"].dtype == rsd["state"][i]["step"].dtype and float(st["step"]) == 4
    assert torch.equal(sd["state"][0]["sum"], eng.accumulator_ew(0))
    # a torch.optim.Adagrad checkpoint (the reference CLI's opt_state_dict) loads back: sums and step
    rsd["state"][1]["sum"].fill_(0.25)
    rsd["state"][2]["sum"].fill_(0.5)
    opt.load_state_dict(rsd)
    assert eng.opt_step == 1
    assert torch.all(eng.accumulator_ew(1) == 0.25) and torch.all(eng.dense_state[:15] == 0.5)
    # and the layout written here loads into torch.optim.Adagrad
    ref2 = torch.optim.Adagrad([torch.nn.Parameter(p.detach().clone()) for p in params], lr=0.1)
    ref2.load_state_dict(opt.state_dict())
    assert torch.equal(ref2.state[ref2.param_groups[0]["params"][1]]["sum"], eng.accumulator_ew(1))


@pytest.mark.parametrize("kw,err", [(dict(maximize=True), ValueError), (dict(weight_decay=0.1), RuntimeError),
                                    (dict(initial_accumulator_value=0.1), ValueError)])
def test_adagrad_refuses_options_it_does_not_run(kw, err):
    from dlrm_b200.optim import Adagrad

    _, params = _fake_net()
    with pytest.raises(err):
        Adagrad(params, lr=0.1, **kw)
