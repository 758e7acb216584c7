"""Persistent tile-dataflow MLP chains (csrc/gemm_chain.cu) == one wgmma launch per layer, bit for bit:
same CTA program per tile, so every activation, gradient operand and weight-gradient slab must be identical.
(Parity of the per-layer path with the reference is tests/test_gpu_engine_tc.py / test_gpu_gemm_tc.py.)"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _run(use_chain, D, ln_emb, ln_bot, ln_top, B, tile_n=None, steps=2, seed=0):
    from oracle import dlrm_numpy as O
    from dlrm_b200.engine import Engine, sparse_from_reference

    rng = np.random.default_rng(seed)
    params = O.random_params(rng, D, ln_emb, ln_bot, ln_top)
    X, off, idx = O.random_batch(rng, ln_emb, B, ln_bot[0], 6)
    tgt = np.round(rng.random((B, 1))).astype(np.float32)
    old = os.environ.get("DLRM_CHAIN_TILE_N")
    if tile_n:
        os.environ["DLRM_CHAIN_TILE_N"] = str(tile_n)
    try:
        e = Engine(D, ln_emb, ln_bot, ln_top, loss="bce", sigmoid_top=len(ln_top) - 2, device=DEV, max_batch=B,
                   gemm="tc")
        e.use_chain = use_chain
        e.load_params(params)
        sp = sparse_from_reference([torch.from_numpy(o) for o in off], [torch.from_numpy(i) for i in idx], DEV)
        Xd, Td = torch.from_numpy(X).to(DEV), torch.from_numpy(tgt).to(DEV)
        losses = []
        for _ in range(steps):
            losses.append(float(e.train_step(Xd, sp, Td, 0.05, "rwsadagrad").item()))
        p = e.forward(Xd, sp).clone()
        torch.cuda.synchronize()
    finally:
        if tile_n:
            if old is None:
                os.environ.pop("DLRM_CHAIN_TILE_N", None)
            else:
                os.environ["DLRM_CHAIN_TILE_N"] = old
    out = dict(p=p.cpu(), dense=e.dense.clone().cpu(), grad=e.dense_grad.clone().cpu(), tables=e.tables.clone().cpu(),
               mom=e.momentum.clone().cpu(), dT=e.dT.clone().cpu(), dR=e.dR.clone().cpu(), T=e.Tbuf.clone().cpu())
    for which in ("bot", "top"):
        for i, (h, l, _) in enumerate(e.tc_in[which]):
            out["in_%s%d" % (which, i)] = torch.stack([h.float().cpu(), l.float().cpu()])
        for i, (h, l, _) in enumerate(e.tc_gz[which]):
            out["gz_%s%d" % (which, i)] = torch.stack([h.float().cpu(), l.float().cpu()])
    return losses, out, e


CASES = [
    # D, ln_emb, ln_bot, ln_top tail, B
    (128, [1000] * 4, [13, 512, 256, 128], [1024, 512, 256, 1], 2048),
    (128, [900, 700, 500], [13, 64, 128], [96, 64, 1], 300),      # ragged last m tile, narrow layers
    (16, [1000, 1000, 1000], [13, 512, 256, 64, 16], [512, 256, 1], 128),   # CFG0 shapes
]


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("order", [0, 2])
@pytest.mark.parametrize("tile_n", [None, 64])
def test_chain_is_bitwise_the_per_layer_path(case, tile_n, order):
    D, ln_emb, ln_bot, tail, B = CASES[case]
    F = len(ln_emb) + 1
    ln_top = [D + F * (F - 1) // 2] + tail
    from dlrm_b200 import _lib

    l0, a, e0 = _run(False, D, ln_emb, ln_bot, ln_top, B, tile_n)
    _lib.set_tunable("chain_order", order)     # 2 = m-tile-major task order
    try:
        l1, b, e1 = _run(True, D, ln_emb, ln_bot, ln_top, B, tile_n)
    finally:
        _lib.set_tunable("chain_order", 0)
    assert e1.tc_chains and all(c.info()["tasks"] > 0 for c in e1.tc_chains.values())
    bad = ["%s: max|diff|=%.3e of scale %.3e, %d elements" % (k, float((a[k] - b[k]).abs().max()), float(a[k].abs().max()),
                                                              int((a[k] != b[k]).sum()))
           for k in a if not torch.equal(a[k], b[k])]
    assert l0 == l1 and not bad, "chain differs from per-layer launches: losses %s vs %s\n%s" % (l0, l1, "\n".join(bad))
    # the kernel leaves its queue / completion counters zeroed (graph replays need no memset)
    for ctr in e1._chain_ctr.values():
        assert int(ctr.abs().sum().item()) == 0


def test_chain_graph_replay_and_launch_count():
    """Captured into a CUDA graph, replayed: same losses as eager; 4 GEMM launches per step instead of 17."""
    from dlrm_b200.engine import GraphedTrainStep
    import types

    D, ln_emb, ln_bot, tail, B = CASES[0]
    F = len(ln_emb) + 1
    ln_top = [D + F * (F - 1) // 2] + tail
    l_ref, _, _ = _run(True, D, ln_emb, ln_bot, ln_top, B, steps=5)
    from oracle import dlrm_numpy as O
    from dlrm_b200.engine import Engine, sparse_from_reference

    rng = np.random.default_rng(0)
    params = O.random_params(rng, D, ln_emb, ln_bot, ln_top)
    X, off, idx = O.random_batch(rng, ln_emb, B, ln_bot[0], 6)
    tgt = np.round(rng.random((B, 1))).astype(np.float32)
    e = Engine(D, ln_emb, ln_bot, ln_top, loss="bce", sigmoid_top=len(ln_top) - 2, device=DEV, max_batch=B, gemm="tc")
    e.use_chain = True
    e.load_params(params)
    sp = sparse_from_reference([torch.from_numpy(o) for o in off], [torch.from_numpy(i) for i in idx], DEV)
    st = types.SimpleNamespace(X=torch.from_numpy(X).to(DEV), target=torch.from_numpy(tgt).to(DEV), sparse=sp)
    g = GraphedTrainStep(e, st, 0.05, "rwsadagrad", warmup=0)     # capture = step 1
    got = []   # warmup=0: nothing ran before the capture, and the capture itself does not execute
    for _ in range(5):
        got.append(float(g.replay().item()))
    torch.cuda.synchronize()
    np.testing.assert_allclose(got, l_ref, rtol=0, atol=0)
    assert g.kernels_per_replay <= 14, g.kernels_per_replay
