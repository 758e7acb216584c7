#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the LIVE reference (imported in place
from /root/reference; nothing is copied) on seeded inputs.  TEST INFRASTRUCTURE.

Run in the build container only (the reference does not exist on the GPU box):

    python oracle/make_goldens.py            # writes tests/golden/*.npz

Each fixture holds: the model weights (or the seed they are regenerated from by
oracle.dlrm_numpy.random_params -- weights are always COPIED INTO the reference
module, never obtained through seed equality, SURVEY.md §3.1), the inputs
produced by the reference generator dlrm_data_pytorch.generate_dist_input_batch
(:899-960) under np.random.seed(s), and the reference's outputs: every forward
stage, loss, dense grads, and parameters / RWSAdagrad momentum after N optimizer
steps (torch.optim.SGD and optim/rwsadagrad.py).
"""
import os
import sys

import numpy as np
import torch

REF = os.environ.get("DLRM_REFERENCE", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
# the repo root holds its own dlrm_s_pytorch.py (the drop-in CLI shim): the REFERENCE must come first
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)
for _m in ("dlrm_s_pytorch", "dlrm_data_pytorch"):
    sys.modules.pop(_m, None)          # never reuse an already-imported shim
_print = print  # extend_distributed overrides builtins.print on import

import dlrm_data_pytorch as dp  # noqa: E402
import dlrm_s_pytorch as R  # noqa: E402

assert os.path.realpath(os.path.dirname(R.__file__)) == os.path.realpath(REF), \
    "dlrm_s_pytorch resolved to %s, not to the reference" % R.__file__
assert hasattr(R, "DLRM_Net")

from oracle import dlrm_numpy as O  # noqa: E402
from oracle.golden_format import shrink  # noqa: E402

OUT = os.environ.get("DLRM_GOLDEN_OUT", os.path.join(ROOT, "tests", "golden"))


def build_ref(m_spa, ln_emb, ln_bot, ln_top, params, loss, itself=False, thr=0.0, op="dot",
              weighted=None):
    ref = R.DLRM_Net(m_spa, np.asarray(ln_emb), np.asarray(ln_bot), np.asarray(ln_top),
                     arch_interaction_op=op, arch_interaction_itself=itself, sigmoid_bot=-1,
                     sigmoid_top=len(ln_top) - 2, ndevices=-1, loss_threshold=thr,
                     loss_function=loss, weighted_pooling=weighted)
    with torch.no_grad():
        for k, W in enumerate(params["emb"]):
            ref.emb_l[k].weight.copy_(torch.from_numpy(W))
        for name, seq in (("bot", ref.bot_l), ("top", ref.top_l)):
            for i, (W, b) in enumerate(params[name]):
                seq[2 * i].weight.copy_(torch.from_numpy(W))
                seq[2 * i].bias.copy_(torch.from_numpy(b))
        if weighted is not None:  # "fixed": plain tensors (dlrm_s_pytorch.py:289-292,375)
            for k, w in enumerate(params["v_W_l"]):
                ref.v_W_l[k] = torch.from_numpy(w.copy())
    return ref


def ref_inputs(seed, m_den, ln_emb, B, lmax, fixed=False, round_targets=True):
    np.random.seed(seed)
    X, lS_o, lS_i = dp.generate_dist_input_batch(m_den, np.asarray(ln_emb), B, lmax, fixed,
                                                 "uniform", 0, 1, -1, 1)
    T = dp.generate_random_output_batch(B, 1, round_targets)
    return X, torch.stack(lS_o), lS_i, T


def pack_inputs(d, tag, X, lS_o, lS_i, T):
    d[f"{tag}X"] = X.numpy()
    d[f"{tag}off"] = lS_o.numpy()
    d[f"{tag}T"] = T.numpy()
    for k, i in enumerate(lS_i):
        d[f"{tag}idx{k}"] = i.numpy()


def stages(ref, X, lS_o, lS_i):
    x = ref.apply_mlp(X, ref.bot_l)
    ly = ref.apply_emb(lS_o, lS_i, ref.emb_l, ref.v_W_l)
    z = ref.interact_features(x, ly)
    p = ref.apply_mlp(z, ref.top_l)
    return x, ly, z, p


def case(name, m_spa, ln_emb, ln_bot, top_tail, B, lmax, loss, seed, nsteps=2, lr=0.1,
         store_params=True, itself=False, thr=0.0, op="dot", weighted=None, fixed=False,
         store_tables=None, shrunk=False):
    ln_emb = list(ln_emb)
    nf = len(ln_emb) + 1
    if op == "dot":
        num_int = (nf * (nf + 1)) // 2 + ln_bot[-1] if itself else (nf * (nf - 1)) // 2 + ln_bot[-1]
    else:
        num_int = nf * ln_bot[-1]
    ln_top = [num_int] + list(top_tail)
    rng = np.random.default_rng(seed)
    params = O.random_params(rng, m_spa, ln_emb, ln_bot, ln_top)
    if weighted is not None:
        params["v_W_l"] = [rng.uniform(0.5, 1.5, size=int(n)).astype(np.float32) for n in ln_emb]
    d = dict(m_spa=m_spa, ln_emb=np.array(ln_emb), ln_bot=np.array(ln_bot), ln_top=np.array(ln_top),
             B=B, lmax=lmax, loss=loss, seed=seed, lr=lr, nsteps=nsteps, itself=int(itself), thr=thr,
             op=op, weighted="" if weighted is None else weighted, store_params=int(store_params))
    if store_params:
        for k, W in enumerate(params["emb"]):
            d[f"emb{k}"] = W
        for nm in ("bot", "top"):
            for i, (W, b) in enumerate(params[nm]):
                d[f"{nm}W{i}"], d[f"{nm}b{i}"] = W, b
    if weighted is not None:
        for k, w in enumerate(params["v_W_l"]):
            d[f"vW{k}"] = w
    batches = [ref_inputs(seed + 1000 + s, ln_bot[0], ln_emb, B, lmax, fixed) for s in range(nsteps + 1)]
    for s, b in enumerate(batches):
        pack_inputs(d, f"b{s}_", *b)

    # ---- forward stages on batch 0 (fresh weights)
    ref = build_ref(m_spa, ln_emb, ln_bot, ln_top, params, loss, itself, thr, op, weighted)
    X, lS_o, lS_i, T = batches[0]
    x, ly, z, p = stages(ref, X, lS_o, lS_i)
    d["f_x"], d["f_R"], d["f_p"] = x.detach().numpy(), z.detach().numpy(), p.detach().numpy()
    for k in range(len(ly)):
        if store_tables is None or k in store_tables:
            d[f"f_ly{k}"] = ly[k].detach().numpy()
    out = ref(X, lS_o, lS_i)
    d["f_out"] = out.detach().numpy()
    if loss == "wbce":
        raise NotImplementedError
    E = ref.loss_fn(out, T)
    d["f_loss"] = np.float32(E.item())
    ref.zero_grad()
    E.backward()
    for nm, seq in (("bot", ref.bot_l), ("top", ref.top_l)):
        for i in range(len(seq) // 2):
            d[f"g_{nm}W{i}"] = seq[2 * i].weight.grad.numpy().copy()
            d[f"g_{nm}b{i}"] = seq[2 * i].bias.grad.numpy().copy()
    for k in range(len(ln_emb)):
        g = ref.emb_l[k].weight.grad
        assert g.is_sparse and not g.is_coalesced()
        assert torch.equal(g._indices()[0], lS_i[k])  # uncoalesced, input order (SURVEY §8 a9)
        gc = g.coalesce()
        if store_tables is None or k in store_tables:
            d[f"g_emb{k}_rows"] = gc._indices()[0].numpy().copy()
            d[f"g_emb{k}_vals"] = gc._values().numpy().copy()

    # ---- N optimizer steps, then forward on batch N: SGD and RWSAdagrad.
    # Parameters are recorded after step 1 (a pure function of the batch-0 grads
    # stored above -> tight optimizer check) and after step N (end-to-end check;
    # Adagrad's first steps divide by |g|, so entries with |g|~0 are ill-conditioned
    # and the tests compare those with robust statistics).
    def snapshot(tag, ref, opt, upto):
        for k in range(len(ln_emb)):
            W = ref.emb_l[k].weight.detach().numpy()
            touched = np.unique(np.concatenate([batches[s][2][k].numpy() for s in range(upto)]))
            if store_tables is None or k in store_tables:
                d[f"{tag}_emb{k}_rows"] = touched
                d[f"{tag}_emb{k}_vals"] = W[touched].copy()
            # untouched rows must be unchanged: checksum of the whole table
            d[f"{tag}_emb{k}_sum"] = np.float64(W.astype(np.float64).sum())
            if "rwsadagrad" in tag:
                d[f"{tag}_mom{k}"] = opt.state[ref.emb_l[k].weight]["momentum"].numpy().copy()
        for nm, seq in (("bot", ref.bot_l), ("top", ref.top_l)):
            for i in range(len(seq) // 2):
                Wt = seq[2 * i].weight.detach().numpy()
                if Wt.size <= 20000 or i == len(seq) // 2 - 1:
                    d[f"{tag}_{nm}W{i}"] = Wt.copy()
                d[f"{tag}_{nm}b{i}"] = seq[2 * i].bias.detach().numpy().copy()

    for optname in ("sgd", "rwsadagrad"):
        ref = build_ref(m_spa, ln_emb, ln_bot, ln_top, params, loss, itself, thr, op, weighted)
        olr = lr if optname == "sgd" else lr * 0.1
        d[f"{optname}_lr"] = olr
        if optname == "sgd":
            opt = torch.optim.SGD(ref.parameters(), lr=olr)
        else:
            opt = R.RowWiseSparseAdagrad.RWSAdagrad(ref.parameters(), lr=olr)
        losses = []
        for s in range(nsteps):
            X, lS_o, lS_i, T = batches[s]
            E = ref.loss_fn(ref(X, lS_o, lS_i), T)
            losses.append(E.item())
            opt.zero_grad()
            E.backward()
            opt.step()
            if s == 0:
                snapshot(optname + "1", ref, opt, 1)
        d[f"{optname}_losses"] = np.array(losses, dtype=np.float32)
        X, lS_o, lS_i, T = batches[nsteps]
        with torch.no_grad():
            d[f"{optname}_p_after"] = ref(X, lS_o, lS_i).numpy().copy()
        snapshot(optname, ref, opt, nsteps)
    for suffix, arrays in (shrink(d) if shrunk else {"": d}).items():
        path = os.path.join(OUT, name + suffix + ".npz")
        np.savez_compressed(path, **arrays)
        _print(f"wrote {path}  ({os.path.getsize(path) / 1e6:.2f} MB)  loss0={d['f_loss']:.6f}")


def embbag_order_check():
    """Re-verify SURVEY §8 a4: the reference CPU EmbeddingBag(sum) equals a
    sequential fp32 accumulation in index order, bit for bit."""
    rng = np.random.default_rng(7)
    for D in (2, 16, 64, 128):
        W = rng.standard_normal((5000, D)).astype(np.float32)
        X, off, idx = O.random_batch(rng, [5000], 257, lmax=40)
        E = torch.nn.EmbeddingBag(5000, D, mode="sum", sparse=True)
        E.weight.data = torch.from_numpy(W.copy())
        ref = E(torch.from_numpy(idx[0]), torch.from_numpy(off[0])).detach().numpy()
        mine = O.emb_bag_sum(W, idx[0], off[0])
        assert np.array_equal(ref, mine), f"EmbeddingBag order differs at D={D}"
    _print("EmbeddingBag(sum) == sequential fp32 order: bit-exact (D=2,16,64,128)")


def main(only=None):
    """only: iterable of fixture names to (re)generate (default: all)."""
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    embbag_order_check()
    global case
    _case = case

    def case(name, *a, **kw):  # noqa: F811
        if only is None or name in only:
            _case(name, *a, **kw)
    try:
        _main_cases(case)
    finally:
        case = _case


def _main_cases(case):
    # reference's own test arch (dlrm_s_pytorch.py:908-914 defaults; test/dlrm_s_test.sh)
    case("tiny_default", 2, [4, 3, 2], [4, 3, 2], [4, 2, 1], B=5, lmax=3, loss="mse", seed=11)
    # CFG0 (BASELINE.json configs[0])
    case("cfg0", 16, [1000, 1000, 1000], [13, 512, 256, 64, 16], [512, 256, 1], B=128, lmax=10,
         loss="bce", seed=22, shrunk=True)
    # CFG0 variants: diagonal-inclusive interaction + loss threshold; cat op; weighted pooling
    case("cfg0_itself_thr", 16, [1000, 800, 600], [13, 64, 16], [64, 1], B=64, lmax=10, loss="bce",
         seed=33, itself=True, thr=0.45)
    case("cfg0_cat", 16, [300, 200], [13, 32, 16], [32, 1], B=32, lmax=4, loss="mse", seed=44, op="cat")
    case("cfg0_weighted", 16, [300, 200, 100], [13, 32, 16], [32, 1], B=32, lmax=6, loss="bce",
         seed=55, weighted="fixed")
    # CFG1/2 shapes (D=128, T=26, same MLPs) with shrunk row counts and batch
    case("mini_cfg1", 128, [2000] * 25 + [40], [13, 512, 256, 128], [1024, 512, 256, 1], B=96,
         lmax=10, loss="bce", seed=66, store_params=False, store_tables=(0, 13, 25), shrunk=True)


if __name__ == "__main__":
    main(only=set(sys.argv[1:]) or None)
