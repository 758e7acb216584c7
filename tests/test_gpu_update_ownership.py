"""Row ownership in the embedding update: the training gather marks every occurrence that a later occurrence of the
same row superseded, and the update lets the one unmarked (last) occurrence of a row own it without reading the
row's list head.  Driven through the training gather (emb_forward(..., link=True)) on a mix of tables whose lists
have 1, 2-32 and more than 32 members, fixed-length bags with duplicates inside a bag, 32-position windows that
straddle table boundaries and a row-split shard; D = 128 runs the lean update kernel, D = 256 the general one.
Rows and accumulators against the numpy oracle, list heads and marks all zero afterwards, and two runs from the same
state bit-identical."""
import numpy as np
import pytest
import torch

from oracle import dlrm_numpy as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# rows and (fixed) bag length per table: lists of > 32 members (table 0), 2-32 (tables 1, 3), mostly 1 (table 2)
ROWS = [5, 300, 200003, 37, 2500]
HOT = [20, 8, 3, 1, 6]
B = 251            # odd: no table's positions start or end on a 32-position window boundary


def _batch(rng):
    off, idx = [], []
    for R, L in zip(ROWS, HOT):
        i = rng.integers(0, R, size=B * L).astype(np.int64)
        if L > 1:
            i[1] = i[0]                       # a duplicate inside one bag
        off.append((np.arange(B) * L).astype(np.int64))
        idx.append(i)
    return off, idx


def _run(split, D, opt, interleave):
    from dlrm_b200 import placement as P, sharding as S
    from dlrm_b200.engine import Engine, sparse_from_reference

    rng = np.random.default_rng(11 + D)
    off, idx = _batch(rng)
    F = len(ROWS) + 1
    kw = dict(device=DEV, max_batch=B, small_rows_max=0, interleave_momentum=interleave)
    if split:      # table 1 stored as two row-range shards (each scans every occurrence of the table)
        pl = P.plan(ROWS, [float(h) for h in HOT], 1, force_split=[1])
        ek = S.engine_kwargs(pl, 0, len(ROWS))
        shards = [(s.table, s.row_lo, s.row_hi) for s in pl.of_rank(0)]
        assert sum(1 for t, _, _ in shards if t == 1) == 2
        e = Engine(D, ek["ln_emb"], [4, D], [D + F * (F - 1) // 2, 1], shards=ek["shards"],
                   split_slots=ek["split_slots"], n_features=ek["n_features"], **kw)
    else:
        shards = [(t, 0, R) for t, R in enumerate(ROWS)]
        e = Engine(D, ROWS, [4, D], [D + F * (F - 1) // 2, 1], **kw)
    assert e.interleave == interleave
    W = [rng.standard_normal((R, D)).astype(np.float32) for R in ROWS]
    mom = [rng.uniform(0, 1, R).astype(np.float32) for R in ROWS]
    dY = rng.standard_normal((B, len(ROWS), D)).astype(np.float32)
    e.ensure_optimizer_state(opt)
    for j, (t, lo, hi) in enumerate(shards):
        e.table(j).copy_(torch.from_numpy(W[t][lo:hi]))
        if opt == "rwsadagrad":
            e.momentum[int(e.row_base[j]):int(e.row_base[j + 1])].copy_(torch.from_numpy(mom[t][lo:hi]))
    # index stream and gradient rows per local shard: every shard of a table gets the table's
    sp = sparse_from_reference([torch.from_numpy(off[t]) for t, _, _ in shards],
                               [torch.from_numpy(idx[t]) for t, _, _ in shards], DEV)
    dYs = torch.from_numpy(np.ascontiguousarray(dY[:, [t for t, _, _ in shards], :])).to(DEV)
    ns = len(shards)
    tables0 = e.tables.clone()
    mom0 = e.momentum.clone() if opt == "rwsadagrad" else None
    runs = []
    for _ in range(2):
        e.tables.copy_(tables0)
        if mom0 is not None:
            e.momentum.copy_(mom0)
        e.emb_forward(sp, link=True)
        e.emb_update(sp, dYs, ns * D, D, opt, 0.05)
        torch.cuda.synchronize()
        assert int(e.head.abs().sum().item()) == 0, "list heads not reset"
        assert int(e.mark.sum().item()) == 0, "superseded marks not cleared"
        runs.append((e.tables.clone(), e.momentum.clone() if mom0 is not None else None))
    assert torch.equal(runs[0][0], runs[1][0])
    if mom0 is not None:
        assert torch.equal(runs[0][1], runs[1][1])
    assert e.lib.dlrm_b200_check_device_errors(None) == 0
    for t in range(len(ROWS)):
        ind, val = O.sparse_grad(idx[t], off[t], dY[:, t, :])
        Wt, mt = W[t].copy(), mom[t].copy()
        if opt == "sgd":
            O.sgd_sparse(Wt, ind, val, 0.05)
        else:
            O.rwsadagrad_sparse(Wt, mt, ind, val, 0.05)
        for j, (tj, lo, hi) in enumerate(shards):
            if tj != t:
                continue
            np.testing.assert_allclose(e.table(j).cpu().numpy(), Wt[lo:hi], rtol=2e-5, atol=2e-5)
            if opt == "rwsadagrad":
                got_m = e.momentum[int(e.row_base[j]):int(e.row_base[j + 1])].cpu().numpy()
                np.testing.assert_allclose(got_m, mt[lo:hi], rtol=2e-5, atol=1e-7)


@pytest.mark.parametrize("opt", ["rwsadagrad", "sgd"])
@pytest.mark.parametrize("D", [128, 256])
@pytest.mark.parametrize("split", [False, True])
def test_update_ownership_through_the_training_gather(split, D, opt):
    _run(split, D, opt, interleave=True)


@pytest.mark.parametrize("opt", ["rwsadagrad", "sgd"])
def test_update_ownership_with_separate_accumulator_and_head_arrays(opt):
    """interleave=False: accumulator and list head in arrays of their own, reached through their strides."""
    _run(False, 128, opt, interleave=False)
