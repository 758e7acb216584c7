#!/usr/bin/env python
"""Generate tests/golden/cfg0_learned.npz by training the LIVE reference model (imported in place from
/root/reference, as oracle/make_goldens.py does) with --weighted-pooling=learned on seeded inputs.  TEST
INFRASTRUCTURE; runs in the build container only (the reference does not exist on the GPU box):

    python oracle/make_learned_goldens.py

The fixture holds the initial model (tables, MLPs and v_W_l drawn from a seed, copied INTO the reference module), the
batches of oracle.make_goldens.ref_inputs, and for each optimizer (torch.optim.SGD, optim/rwsadagrad.py,
torch.optim.Adagrad): the loss of every step and, after the first and the last step, every table, v_W_l, the tables' accumulators (RWSAdagrad 'momentum'
[rows], Adagrad 'sum' [rows, D]) and v_W_l's 'sum'.  The loader is tests/golden_util.Golden.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import make_goldens as MG  # noqa: E402  (imports the live reference)
from oracle import dlrm_numpy as O  # noqa: E402

R = MG.R
NAME = "cfg0_learned"
# two list-path tables and one tiny table (<= 256 rows: the two-pass update)
M_SPA, LN_EMB, LN_BOT, TOP_TAIL = 16, [500, 300, 100], [13, 32, 16], [32, 1]
B, LMAX, SEED, NSTEPS = 64, 8, 77, 3
LRS = {"sgd": 0.1, "rwsadagrad": 0.02, "adagrad": 0.02}


def main():
    torch.manual_seed(0)
    nf = len(LN_EMB) + 1
    ln_top = [(nf * (nf - 1)) // 2 + LN_BOT[-1]] + TOP_TAIL
    rng = np.random.default_rng(SEED)
    params = O.random_params(rng, M_SPA, LN_EMB, LN_BOT, ln_top)
    params["v_W_l"] = [rng.uniform(0.5, 1.5, size=n).astype(np.float32) for n in LN_EMB]
    d = dict(m_spa=M_SPA, ln_emb=np.array(LN_EMB), ln_bot=np.array(LN_BOT), ln_top=np.array(ln_top), B=B, lmax=LMAX,
             loss="bce", seed=SEED, lr=LRS["sgd"], nsteps=NSTEPS, itself=0, thr=0.0, op="dot", weighted="learned",
             store_params=1)
    for k, W in enumerate(params["emb"]):
        d[f"emb{k}"] = W
        d[f"vW{k}"] = params["v_W_l"][k]
    for nm in ("bot", "top"):
        for i, (W, b) in enumerate(params[nm]):
            d[f"{nm}W{i}"], d[f"{nm}b{i}"] = W, b
    batches = [MG.ref_inputs(SEED + 1000 + s, LN_BOT[0], LN_EMB, B, LMAX) for s in range(NSTEPS)]
    for s, b in enumerate(batches):
        MG.pack_inputs(d, f"b{s}_", *b)
    opts = {"sgd": torch.optim.SGD, "rwsadagrad": R.RowWiseSparseAdagrad.RWSAdagrad, "adagrad": torch.optim.Adagrad}
    for name, cls in opts.items():
        ref = R.DLRM_Net(M_SPA, np.asarray(LN_EMB), np.asarray(LN_BOT), np.asarray(ln_top), arch_interaction_op="dot",
                         sigmoid_bot=-1, sigmoid_top=len(ln_top) - 2, ndevices=-1, loss_function="bce",
                         weighted_pooling="learned")
        with torch.no_grad():
            for k, W in enumerate(params["emb"]):
                ref.emb_l[k].weight.copy_(torch.from_numpy(W))
                ref.v_W_l[k].copy_(torch.from_numpy(params["v_W_l"][k]))
            for nm, seq in (("bot", ref.bot_l), ("top", ref.top_l)):
                for i, (W, b) in enumerate(params[nm]):
                    seq[2 * i].weight.copy_(torch.from_numpy(W))
                    seq[2 * i].bias.copy_(torch.from_numpy(b))
        assert [n for n, _ in ref.named_parameters()][3:6] == ["v_W_l.0", "v_W_l.1", "v_W_l.2"]
        opt = cls(ref.parameters(), lr=LRS[name])
        d[f"{name}_lr"] = LRS[name]
        losses = []
        for s in range(NSTEPS):
            X, lS_o, lS_i, T = batches[s]
            E = ref.loss_fn(ref(X, lS_o, lS_i), T)
            losses.append(E.item())
            opt.zero_grad()
            E.backward()
            opt.step()
            for k in range(len(LN_EMB) if s in (0, NSTEPS - 1) else 0):    # the state after the first and last step
                W, v = ref.emb_l[k].weight, ref.v_W_l[k]
                d[f"{name}{s}_emb{k}"] = W.detach().numpy().copy()
                d[f"{name}{s}_v{k}"] = v.detach().numpy().copy()
                if name == "rwsadagrad":
                    d[f"{name}{s}_mom{k}"] = opt.state[W]["momentum"].numpy().copy()
                if name == "adagrad":
                    d[f"{name}{s}_acc{k}"] = opt.state[W]["sum"].numpy().copy()
                if name != "sgd":
                    d[f"{name}{s}_vsum{k}"] = opt.state[v]["sum"].numpy().copy()
        d[f"{name}_losses"] = np.array(losses, dtype=np.float32)
    path = os.path.join(MG.OUT, NAME + ".npz")
    np.savez_compressed(path, **d)
    MG._print(f"wrote {path}  ({os.path.getsize(path) / 1e6:.2f} MB)  losses sgd={d['sgd_losses']}")


if __name__ == "__main__":
    main()
