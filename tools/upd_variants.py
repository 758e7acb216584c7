"""Time the embedding update (and the training gather) of one workload for several kernel variants in ONE process:
   python tools/upd_variants.py [cfg3|cfg2] 0,2        (0 = the lean kernel, 2 = the general one)
prints one line per TUNE_UPD_LEAN value (median microseconds of the update launch group between CUDA events)."""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from dlrm_b200 import _lib, dist as ddist, placement as P  # noqa: E402
from dlrm_b200.data import DeviceBatch  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "cfg3"
variants = [int(v) for v in (sys.argv[2] if len(sys.argv) > 2 else "0,2").split(",")]
os.environ.update(RANK="0", WORLD_SIZE="1", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(bench._free_port()))
ddist.init_distributed("nccl")
dev = "cuda:0"
W = bench.workload(name, 1)
D, rows, ln_bot, ln_top = bench.model_dims(W)
cost = bench.lookups_per_sample(W)
pl = P.plan(rows, cost, 1)
de = ddist.DistEngine(D, rows, ln_bot, ln_top, local_batch=W["B"], device=dev, gemm="tc", exchange="p2p", placement=pl)
de.eng.init_params(100)
de.eng.ensure_optimizer_state("rwsadagrad")
eng = de.eng
ring = 6
if W["hot"] is not None:
    mh = ddist.MultiHotExchange(de, W["hot"], 13, 1)
    devr = [mh.fill_host(mh.host_buffer(), 1234, i, rows).to(dev) for i in range(ring)]
    sp = mh.sparse[0]

    def prep(i):
        mh.stage[0].copy_(devr[i % ring], non_blocking=True)
        mh.exchange(0)
else:
    hostb = [ddist.make_sharded_batch(1000 + i, rows, 0, 1, W["B"], 13, W["lmax"], placement=pl) for i in range(ring)]
    devb = []
    for hb, X, Tt in hostb:
        db = DeviceBatch(hb.layout, dev)
        db.load(hb, non_blocking=False)
        devb.append(db)
    st = DeviceBatch(hostb[0][0].layout, dev)
    st.load(hostb[0][0], non_blocking=False)
    sp = st.sparse

    def prep(i):
        db = devb[i % ring]
        n = db.layout.used(db.nnz)
        st.buf[:n].copy_(db.buf[:n], non_blocking=True)
eng.prepare(sp, train=True, batch=de.B)
eng.dT.normal_()
eng.head.zero_()
torch.cuda.synchronize()
for v in variants:
    _lib.set_tunable("upd_lean", v)
    evs = []
    for i in range(14):
        prep(i)
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        eng.emb_forward(sp, link=True)
        eng.reduce_partials(de.B)
        e1.record()
        eng.emb_update(sp, optimizer="rwsadagrad", lr=1e-6)
        e2.record()
        if i >= 4:
            evs.append((e0, e1, e2))
    torch.cuda.synchronize()
    assert int(eng.head.abs().sum().item()) == 0
    tg = float(np.median([a.elapsed_time(b) for a, b, _ in evs])) * 1e3
    tu = float(np.median([b.elapsed_time(c) for _, b, c in evs])) * 1e3
    print("%s upd_lean=%d  gather+link %.1f us  update %.1f us" % (name, v, tg, tu), flush=True)
