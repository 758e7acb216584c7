"""The reference-facing surface on the GPU: `dlrm_b200.DLRM_Net` (module surface of
dlrm_s_pytorch.py:207-730) and the `dlrm_s_pytorch.py` command line, against the live-reference goldens."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from golden_util import Golden

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


def _net(g, gemm="tc", **kw):
    from dlrm_b200.dlrm_net import DLRM_Net

    np.random.seed(1)
    net = DLRM_Net(g.m_spa, np.array(g.ln_emb), np.array(g.ln_bot), np.array(g.ln_top),
                   arch_interaction_op=g.op, arch_interaction_itself=g.itself, sigmoid_bot=-1,
                   sigmoid_top=len(g.ln_top) - 2, loss_threshold=g.thr, loss_function=g.loss, device=DEV, gemm=gemm,
                   max_batch=g.B, **kw)
    p = g.params()
    sd = {}
    for k, W in enumerate(p["emb"]):
        sd[f"emb_l.{k}.weight"] = torch.from_numpy(W)
    for nm in ("bot", "top"):
        for i, (W, b) in enumerate(p[nm]):
            sd[f"{nm}_l.{2 * i}.weight"] = torch.from_numpy(W)
            sd[f"{nm}_l.{2 * i}.bias"] = torch.from_numpy(b)
    net.load_state_dict(sd)  # reference checkpoints use exactly these keys
    return net


def _batch(g, s):
    X, off, idx, T = g.batch(s)
    return (torch.from_numpy(X), torch.from_numpy(np.stack(off)), [torch.from_numpy(i) for i in idx],
            torch.from_numpy(T))


def test_state_dict_keys_and_parameter_order():
    g = Golden("cfg0")
    net = _net(g)
    keys = list(net.state_dict().keys())
    want = [f"emb_l.{k}.weight" for k in range(g.T)]
    for nm, ln in (("bot_l", g.ln_bot), ("top_l", g.ln_top)):
        for i in range(len(ln) - 1):
            want += [f"{nm}.{2 * i}.weight", f"{nm}.{2 * i}.bias"]
    assert keys == want
    shapes = [tuple(p.shape) for p in net.parameters()]
    assert shapes[:g.T] == [(n, g.m_spa) for n in g.ln_emb]
    assert len(net.bot_l) == 2 * (len(g.ln_bot) - 1) and len(net.top_l) == 2 * (len(g.ln_top) - 1)


@pytest.mark.parametrize("name,gemm", [("cfg0", "tc"), ("cfg0", "simt"), ("tiny_default", "tc"), ("cfg0_cat", "tc"),
                                       ("cfg0_itself_thr", "tc"), ("mini_cfg1", "tc")])
def test_module_forward_and_stages(name, gemm):
    g = Golden(name)
    net = _net(g, gemm)
    X, lS_o, lS_i, T = _batch(g, 0)
    with torch.no_grad():
        out = net(X, lS_o, lS_i)
    np.testing.assert_allclose(out.cpu().numpy(), g["f_out"], rtol=0, atol=1e-5)
    # the individual methods of the reference surface
    ly = net.apply_emb(lS_o, lS_i, net.emb_l, net.v_W_l)
    for k in range(g.T):
        if g.has(f"f_ly{k}"):
            assert np.array_equal(ly[k].cpu().numpy(), g[f"f_ly{k}"])
    x = net.apply_mlp(X, net.bot_l)
    np.testing.assert_allclose(x.cpu().numpy(), g["f_x"], rtol=2e-5, atol=2e-6)
    R = net.interact_features(x, ly)
    np.testing.assert_allclose(R.cpu().numpy(), g["f_R"], rtol=2e-5, atol=5e-6)
    p = net.apply_mlp(R, net.top_l)
    np.testing.assert_allclose(p.cpu().numpy(), g["f_p"], rtol=0, atol=1e-5)


@pytest.mark.parametrize("gemm", ["tc", "simt"])
def test_autograd_with_unmodified_torch_sgd(gemm):
    """Compatibility mode: E.backward() materialises the reference's sparse COO embedding grads,
    torch.optim.SGD steps them."""
    g = Golden("cfg0")
    net = _net(g, gemm)
    opt = torch.optim.SGD(net.parameters(), lr=float(g["sgd_lr"]))
    losses = []
    for s in range(g.nsteps):
        X, lS_o, lS_i, T = _batch(g, s)
        E = net.loss_fn(net(X, lS_o, lS_i), T.to(DEV))
        losses.append(float(E.item()))
        opt.zero_grad()
        E.backward()
        if s == 0:
            gr = net.emb_l[0].weight.grad
            assert gr.is_sparse and not gr.is_coalesced()
            gc = gr.coalesce()
            assert np.array_equal(gc._indices()[0].cpu().numpy(), g["g_emb0_rows"])
            np.testing.assert_allclose(gc._values().cpu().numpy(), g["g_emb0_vals"], rtol=1e-3, atol=1e-6)
        opt.step()
    np.testing.assert_allclose(losses, g["sgd_losses"], rtol=0, atol=2e-5)


@pytest.mark.parametrize("optname", ["sgd", "rwsadagrad"])
def test_fused_optimizers_match_reference_losses(optname):
    from dlrm_b200 import optim as fused

    g = Golden("cfg0")
    net = _net(g, "tc")
    cls = fused.SGD if optname == "sgd" else fused.RWSAdagrad
    opt = cls(net.parameters(), lr=float(g[f"{optname}_lr"]))
    losses = []
    for s in range(g.nsteps):
        X, lS_o, lS_i, T = _batch(g, s)
        E = net.loss_fn(net(X, lS_o, lS_i), T.to(DEV))
        losses.append(float(E.item()))
        opt.zero_grad()
        E.backward()
        opt.step()
    np.testing.assert_allclose(losses, g[f"{optname}_losses"], rtol=0, atol=2e-5 if optname == "sgd" else 3e-4)
    X, lS_o, lS_i, T = _batch(g, g.nsteps)
    with torch.no_grad():
        pa = net(X, lS_o, lS_i).cpu().numpy()
    err = np.abs(pa - g[f"{optname}_p_after"])
    assert np.median(err) < (3e-5 if optname == "sgd" else 5e-4)


@pytest.mark.parametrize("tag", ["A", "B"])
@pytest.mark.parametrize("gemm", ["tc", "simt"])
def test_cli_loss_curve_matches_reference_cli(tag, gemm):
    """Same flags, same numpy seed -> same inputs and initial weights as the reference CLI; the printed
    loss curve (6 SGD iterations, recorded from /root/reference in the build container) must match."""
    flags = open(os.path.join(ROOT, "tests", "golden", f"cli_cfg0_{tag}.flags")).read().split()
    want = [float(m.group(1)) for m in re.finditer(r"loss ([0-9.]+)",
                                                   open(os.path.join(ROOT, "tests", "golden", f"cli_cfg0_{tag}.txt")).read())]
    cmd = [sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py"), "--arch-sparse-feature-size=16",
           "--arch-embedding-size=1000-1000-1000", "--arch-mlp-bot=13-512-256-64-16", "--arch-mlp-top=512-256-1",
           "--mini-batch-size=128", "--data-generation=random", "--num-batches=6", "--print-freq=1",
           "--learning-rate=0.1", "--numpy-rand-seed=727", "--use-gpu", "--gemm", gemm] + flags
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    got = [float(m.group(1)) for m in re.finditer(r"Finished training it \d+/6 of epoch 0, .* loss ([0-9.]+)", r.stdout)]
    assert len(got) == 6, r.stdout
    np.testing.assert_allclose(got, want, rtol=0, atol=2e-5)


def test_eval_forward_with_grad_enabled_between_training_steps():
    """The reference's inference() loop runs the model WITHOUT no_grad (dlrm_s_pytorch.py:759-899).  A
    grad-enabled forward on another batch that is never followed by step() must not disturb the next
    training step (round-1 advisor finding: stale per-row list heads)."""
    from dlrm_b200 import optim as fused

    g = Golden("cfg0")
    net = _net(g, "tc")
    opt = fused.RWSAdagrad(net.parameters(), lr=float(g["rwsadagrad_lr"]))
    losses = []
    for s in range(g.nsteps):
        Xe, oe, ie, Te = _batch(g, g.nsteps)            # "evaluation" batch, grad enabled, no step
        _ = net(Xe, oe, ie)
        _ = net(Xe, oe, ie)
        X, lS_o, lS_i, T = _batch(g, s)
        E = net.loss_fn(net(X, lS_o, lS_i), T.to(DEV))
        losses.append(float(E.item()))
        opt.zero_grad()
        E.backward()
        opt.step()
    np.testing.assert_allclose(losses, g["rwsadagrad_losses"], rtol=0, atol=3e-4)
    assert int(net._engine.head.abs().sum().item()) == 0     # list heads are clean between steps
    for k in range(g.T):
        np.testing.assert_allclose(net._engine.momentum[int(net._engine.row_base[k]):int(net._engine.row_base[k + 1])]
                                   .cpu().numpy(), g[f"rwsadagrad_mom{k}"], rtol=2e-3, atol=1e-7)


def test_gradient_accumulation_fails_loudly():
    from dlrm_b200 import optim as fused

    g = Golden("cfg0")
    net = _net(g, "tc")
    opt = fused.SGD(net.parameters(), lr=0.1)
    X, lS_o, lS_i, T = _batch(g, 0)
    opt.zero_grad()
    net.loss_fn(net(X, lS_o, lS_i), T.to(DEV)).backward()
    with pytest.raises(RuntimeError, match="accumulation"):
        net.loss_fn(net(X, lS_o, lS_i), T.to(DEV)).backward()


_CLI_BASE = ["--arch-sparse-feature-size=16", "--arch-embedding-size=1000-1000-1000", "--arch-mlp-bot=13-512-256-64-16",
             "--arch-mlp-top=512-256-1", "--mini-batch-size=128", "--data-generation=random", "--num-batches=6",
             "--print-freq=1", "--learning-rate=0.1", "--numpy-rand-seed=727", "--use-gpu"]


def test_cli_test_pass_and_checkpoint_follow_the_reference(tmp_path):
    """--test-freq / --save-model: the printed lines (loss curve, 'Testing at', accuracy, 'Saving model') equal the
    reference CLI's run recorded in tests/golden/cli_cfg0_C.txt (the test set re-seeds numpy, so the training batches
    after a test pass differ from a run without one -- the same happens here), and the checkpoint carries the
    reference's key set (dlrm_s_pytorch.py:860-866, :1703-1715) with the reference's state_dict keys."""
    flags = open(os.path.join(ROOT, "tests", "golden", "cli_cfg0_C.flags")).read().split()
    want = [ln for ln in open(os.path.join(ROOT, "tests", "golden", "cli_cfg0_C.txt")).read().splitlines()
            if not ln.startswith("time/loss")]
    ck = str(tmp_path / "ours.pt")
    cmd = [sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py")] + _CLI_BASE + flags + ["--save-model=" + ck]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    got = [ln for ln in r.stdout.splitlines() if re.match(r"Finished| accuracy|Testing at|Saving model", ln)]
    assert len(got) == len(want), r.stdout
    for a, b in zip(got, want):
        if a.startswith("Finished"):
            la, lb = float(a.rsplit(" ", 1)[1]), float(b.rsplit(" ", 1)[1])
            assert a.rsplit(" ", 1)[0] == b.rsplit(" ", 1)[0] and abs(la - lb) < 2e-5, (a, b)
        elif a.startswith("Saving model"):
            assert b.startswith("Saving model")
        else:
            assert a == b
    ref = torch.load(os.path.join(ROOT, "tests", "golden", "cli_cfg0_C_ref.pt"), map_location="cpu", weights_only=False)
    ours = torch.load(ck, map_location="cpu", weights_only=False)
    assert set(ours.keys()) == set(ref.keys())
    assert list(ours["state_dict"].keys()) == list(ref["state_dict"].keys())
    for k in ("epoch", "iter", "nepochs", "nbatches", "nbatches_test"):
        assert ours[k] == ref[k], k
    assert abs(float(ours["test_acc"]) - float(ref["test_acc"])) < 1e-9
    assert abs(float(ours["train_loss"]) - float(ref["train_loss"])) < 2e-5
    for k, v in ref["state_dict"].items():          # same weights after the same 6 SGD steps
        np.testing.assert_allclose(ours["state_dict"][k].numpy(), v.numpy(), rtol=0, atol=1e-4)   # lr = 0.1


def test_cli_loads_a_reference_checkpoint_for_inference():
    """A checkpoint WRITTEN BY THE REFERENCE (tests/golden/cli_cfg0_C_ref.pt) loads through --load-model
    --inference-only; the test pass gives the accuracy the reference recorded in it."""
    flags = [f for f in open(os.path.join(ROOT, "tests", "golden", "cli_cfg0_C.flags")).read().split()
             if not f.startswith("--test-freq")]       # the checkpoint's architecture, no test pass while training
    ck = os.path.join(ROOT, "tests", "golden", "cli_cfg0_C_ref.pt")
    cmd = [sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py")] + _CLI_BASE + flags + \
        ["--load-model=" + ck, "--inference-only"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "Saved at: epoch = 0/1, batch = 6/6, ntbatch = 6" in r.stdout
    assert "Testing for inference only" in r.stdout
    assert " accuracy 51.693 %, best 51.693 %" in r.stdout


def test_checkpoint_resume_restores_optimizer_state(tmp_path):
    """--optimizer=rwsadagrad: opt_state_dict round-trips the row-wise accumulators ('momentum'), the dense
    accumulators ('sum') and the step count, with the reference optimizer's per-parameter keys
    (optim/rwsadagrad.py:86-100); resuming skips the batches already trained (:1430-1436)."""
    from dlrm_b200 import cli

    ck = str(tmp_path / "ada.pt")
    args = [a for a in _CLI_BASE if not a.startswith("--num-batches")] + \
        ["--round-targets=True", "--loss-function=bce", "--optimizer=rwsadagrad"]
    net = cli.run(args + ["--num-batches=4", "--test-freq=4", "--save-model=" + ck])
    sd = torch.load(ck, map_location="cpu", weights_only=False)
    assert sd["iter"] == 4 and sd["epoch"] == 0
    st = sd["opt_state_dict"]["state"]
    assert len(st) == 3 + 2 * 4 + 2 * 3
    assert all(set(st[i]) == {"step", "momentum"} and st[i]["momentum"].shape == (1000,) for i in range(3))
    assert all(set(st[i]) == {"step", "sum"} for i in range(3, len(st)))
    assert all(st[i]["step"] == 4 for i in st)
    assert float(st[0]["momentum"].abs().sum()) > 0 and float(st[3]["sum"].abs().sum()) > 0
    mom = net._engine.momentum.detach().cpu().clone()
    dsum = net._engine.dense_state.detach().cpu().clone()
    del net
    net2 = cli.run(args + ["--num-batches=4", "--load-model=" + ck])        # every batch skipped: state == checkpoint
    assert net2._engine.opt_step == 4
    np.testing.assert_array_equal(net2._engine.momentum.cpu().numpy(), mom.numpy())
    np.testing.assert_array_equal(net2._engine.dense_state.cpu().numpy(), dsum.numpy())
    for k, v in sd["state_dict"].items():
        np.testing.assert_array_equal(net2.state_dict()[k].cpu().numpy(), v.numpy())
