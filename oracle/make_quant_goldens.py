#!/usr/bin/env python
"""Generate tests/golden/cfg0_quant.npz from the LIVE reference model (imported in place from /root/reference, as
oracle/make_goldens.py does): a seeded model copied INTO the reference's DLRM_Net, then quantize_embedding(8) and
quantize_embedding(4) (dlrm_s_pytorch.py:465-481) and its quantized forward (:430-450) on CPU.  TEST INFRASTRUCTURE;
runs in the build container only (the reference does not exist on the GPU box):

    python oracle/make_quant_goldens.py

The fixture holds the initial model (two list-size tables and one tiny table), per-row weights for the weighted case,
the batches of oracle.make_goldens.ref_inputs, and for bits in (8, 4): the packed tables emb_l_q[k] (q{bits}_emb{k},
uint8) and the reference's outputs on every batch, unweighted (q{bits}_p{s}) and with the fixed weights as v_W_l
(q{bits}_w_p{s}).
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
NAME = "cfg0_quant"
M_SPA, LN_EMB, LN_BOT, TOP_TAIL = 16, [500, 300, 100], [13, 32, 16], [32, 1]
B, LMAX, SEED, NBATCH = 64, 8, 91, 2


def _reference(params, ln_top, weights):
    ref = R.DLRM_Net(M_SPA, np.asarray(LN_EMB), np.asarray(LN_BOT), np.asarray(ln_top), arch_interaction_op="dot",
                     sigmoid_bot=-1, sigmoid_top=len(ln_top) - 2, ndevices=-1, loss_function="bce",
                     weighted_pooling=None if weights is None else "fixed")
    with torch.no_grad():
        for k, W in enumerate(params["emb"]):
            ref.emb_l[k].weight.copy_(torch.from_numpy(W))
        for nm, seq in (("bot", ref.bot_l), ("top", ref.top_l)):
            for i, (W, b) in enumerate(params[nm]):
                seq[2 * i].weight.copy_(torch.from_numpy(W))
                seq[2 * i].bias.copy_(torch.from_numpy(b))
    if weights is not None:
        ref.v_W_l = [torch.from_numpy(w) for w in weights]
    return ref


def main():
    torch.manual_seed(0)
    nf = len(LN_EMB) + 1
    ln_top = [(nf * (nf - 1)) // 2 + LN_BOT[-1]] + TOP_TAIL
    rng = np.random.default_rng(SEED)
    params = O.random_params(rng, M_SPA, LN_EMB, LN_BOT, ln_top)
    weights = [rng.uniform(0.5, 1.5, size=n).astype(np.float32) for n in LN_EMB]
    d = dict(m_spa=M_SPA, ln_emb=np.array(LN_EMB), ln_bot=np.array(LN_BOT), ln_top=np.array(ln_top), B=B, lmax=LMAX,
             seed=SEED, nbatch=NBATCH)
    for k, W in enumerate(params["emb"]):
        d[f"emb{k}"] = W
        d[f"vW{k}"] = weights[k]
    for nm in ("bot", "top"):
        for i, (W, b) in enumerate(params[nm]):
            d[f"{nm}W{i}"], d[f"{nm}b{i}"] = W, b
    batches = [MG.ref_inputs(SEED + 1000 + s, LN_BOT[0], LN_EMB, B, LMAX) for s in range(NBATCH)]
    for s, b in enumerate(batches):
        MG.pack_inputs(d, f"b{s}_", *b)
    for bits in (8, 4):
        for tag, w in (("", None), ("w_", weights)):
            ref = _reference(params, ln_top, w)
            ref.quantize_embedding(bits)
            assert ref.quantize_emb and ref.quantize_bits == bits
            if w is None:
                for k in range(len(LN_EMB)):
                    d[f"q{bits}_emb{k}"] = ref.emb_l_q[k].numpy().copy()
            with torch.no_grad():
                for s, (X, lS_o, lS_i, _) in enumerate(batches):
                    d[f"q{bits}_{tag}p{s}"] = ref(X, lS_o, lS_i).numpy().copy()
    path = os.path.join(MG.OUT, NAME + ".npz")
    np.savez_compressed(path, **d)
    MG._print(f"wrote {path}  ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
