"""One-process-per-GPU DLRM: sharded embeddings (table-wise + row-split) + data-parallel MLPs.

Replaces `DLRM_Net.distributed_forward` (dlrm_s_pytorch.py:528-585) and `extend_distributed.py`
(`get_my_slice` :47-51, `get_split_lengths` :54-62, `alltoall` :541-576 and its autograd pair
`All2All_Req/Wait` :389-486, DDP of the MLPs :1329-1336):

  * where a table lives is decided by `placement.plan` (cost-balanced; hot / huge tables are ROW-SPLIT over
    all ranks) -- `placement.contiguous` reproduces the reference's `get_my_slice` slices;
  * every rank pools ITS shards for the GLOBAL batch, the pooled vectors (partial sums for a row-split
    table, added on arrival) are exchanged so that every rank ends up with ALL tables for ITS batch slice,
    inside the interaction operand T (forward), and the per-bag gradients travel the opposite way
    (backward) into the fused coalesce + row-wise-Adagrad update of every rank storing rows of the table;
  * the MLPs are replicated; their gradients are averaged with one NCCL all-reduce (DDP semantics:
    mean over ranks of the local-mean-loss gradients; embedding gradients are NOT averaged -- the
    reference's all-to-all backward simply routes them, `extend_distributed.py:467-486`).

Exchange back ends
  "nccl" : `all_to_all_single` on packed send/recv buffers (the reference's collective).
  "p2p"  : the gather kernel stores each pooled row directly into the owner rank's T buffer
           through peer-mapped memory (NVLink stores) and the update kernel reads the dY rows
           from the peers' dT buffers -- no staging buffers, no separate collective.

Launch: `torchrun --nproc-per-node N ...` (env RANK/LOCAL_RANK/WORLD_SIZE/MASTER_*).
"""
from __future__ import annotations

import os
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist


# ---------------------------------------------------------------------------- host-side layout logic
def table_slices(n_tables: int, world: int) -> List[Tuple[int, int]]:
    """Contiguous [start, end) table slice of every rank (extend_distributed.get_my_slice)."""
    k, m = divmod(n_tables, world)
    return [(r * k + min(r, m), (r + 1) * k + min(r + 1, m)) for r in range(world)]


def a2a_splits(n_tables: int, world: int, rank: int, local_batch: int, dim: int):
    """(send_splits, recv_splits) in ELEMENTS for the forward exchange of pooled vectors.

    send buffer of rank r : [world][local_batch][T_r][dim]   (sample-major: block d goes to rank d)
    recv buffer of rank r : [world][local_batch][T_s][dim]   (block s came from rank s)
    The backward exchange uses the same numbers with the roles swapped."""
    sl = table_slices(n_tables, world)
    t_mine = sl[rank][1] - sl[rank][0]
    send = [local_batch * t_mine * dim] * world
    recv = [local_batch * (e - s) * dim for s, e in sl]
    return send, recv


def scatter_recv_into_T(recv: torch.Tensor, Tbuf: torch.Tensor, n_tables: int, world: int,
                        local_batch: int, dim: int):
    """recv [sum_s B*T_s*D] -> Tbuf[:B, 1 + start_s : 1 + end_s, :] for every source rank s."""
    o = 0
    for s, e in table_slices(n_tables, world):
        n = local_batch * (e - s) * dim
        if e > s:
            Tbuf[:local_batch, 1 + s:1 + e, :].copy_(recv[o:o + n].view(local_batch, e - s, dim))
        o += n


def pack_dT_into_send(dT: torch.Tensor, gsend: torch.Tensor, n_tables: int, world: int,
                      local_batch: int, dim: int):
    """dT[:B, 1 + start_d : 1 + end_d, :] -> gsend block d (gradients of rank d's tables)."""
    o = 0
    for s, e in table_slices(n_tables, world):
        n = local_batch * (e - s) * dim
        if e > s:
            gsend[o:o + n].view(local_batch, e - s, dim).copy_(dT[:local_batch, 1 + s:1 + e, :])
        o += n


def push_route(n_tables: int, world: int, rank: int, local_batch: int, dim: int):
    """Where rank `rank`'s interact_bwd stores the gradient rows of every table (peer-memory exchange).

    Returns one (owner, offset, ld) per table t, in ELEMENTS: the row of local sample b goes to
    `recv_of(owner)[offset + b * ld : ... + dim]`.  The receive buffer of a rank with T_r tables is
    [world][local_batch][T_r][dim]; slab `rank` holds what this rank sends, so the owner's update kernel
    sees the same [global batch][T_r][dim] view the all-to-all path assembles (a2a_splits)."""
    out = []
    for r, (s, e) in enumerate(table_slices(n_tables, world)):
        for t in range(s, e):
            out.append((r, (rank * local_batch * (e - s) + (t - s)) * dim, (e - s) * dim))
    return out


def gather_route(n_tables: int, world: int, rank: int, dim: int):
    """Forward twin of push_route: byte-free description of where the gather of rank `rank` stores the
    pooled row of (global sample g, local table k): T_of(g // local_batch)[(g % local_batch), 1 + s + k, :]
    -> returns the element offset of feature (1 + s) inside one sample of T ([F, dim] per sample)."""
    s, _ = table_slices(n_tables, world)[rank]
    return (1 + s) * dim


def init_distributed(backend: Optional[str] = None):
    """Process-group bring-up from the torchrun environment (extend_distributed.init_distributed)."""
    if dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29500")
    if backend is None:
        backend = "nccl" if torch.cuda.is_available() else "gloo"
    import datetime

    # NCCL only brings the job up here (IPC handles, scalars, host-side barriers); the data path is our own kernels over
    # peer-mapped memory.  No NVLS / multicast resources are needed for that, and their setup is the slowest part of
    # creating a communicator on an NVSwitch box.
    os.environ.setdefault("NCCL_NVLS_ENABLE", "0")
    # generous: on a cold 8-GPU box the ranks finish importing / creating contexts minutes apart
    tmo = datetime.timedelta(seconds=float(os.environ.get("DLRM_PG_TIMEOUT_S", "1200")))
    if backend == "nccl":
        torch.cuda.set_device(local)
        dist.init_process_group(backend, rank=rank, world_size=world, device_id=torch.device("cuda", local), timeout=tmo)
    else:
        dist.init_process_group(backend, rank=rank, world_size=world, timeout=tmo)
    return rank, world


# one cudaIpcOpenMemHandle per exported allocation and PROCESS (a second open of the same handle fails)
_IPC_BASES = {}
_KEEP_ALIVE = []     # exported buffers must outlive their importers' mappings: engines are never freed


# ---------------------------------------------------------------------------- the sharded engine
class DistEngine:
    """exchange="p2p" (default on an NVSwitch box): both exchanges ride on our kernels' stores through
    peer-mapped memory, any placement.  exchange="nccl": `all_to_all_single` (the reference's collective),
    contiguous whole-table placement only."""

    def __init__(self, m_spa: int, ln_emb: Sequence[int], ln_bot: Sequence[int], ln_top: Sequence[int], *,
                 local_batch: int, device=None, gemm: str = "tc", loss: str = "bce", exchange: str = "nccl",
                 placement=None, cost: Optional[Sequence[float]] = None, split_forward: str = "partial",
                 semantics: str = "reference", **kw):
        from . import placement as P, sharding as S
        from .engine import Engine

        if gemm == "simt":
            raise SystemExit("ERROR: dlrm_b200.dist runs on the tensor-core path (gemm='tc' or 'tc_bf16')")
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.Tg = len(ln_emb)
        self.D = int(m_spa)
        self.B = int(local_batch)
        self.Bg = self.B * self.world
        self.exchange = exchange
        if exchange not in ("nccl", "p2p"):
            raise SystemExit("ERROR: exchange must be nccl or p2p")
        if placement is None:
            if exchange == "nccl":
                if self.Tg < self.world:
                    raise SystemExit("ERROR: only (%d) sparse features for (%d) devices, table partitions will fail"
                                     % (self.Tg, self.world))
                placement = P.contiguous(ln_emb, self.world)
            else:
                # fp16 tables: the plan's memory budget counts their real row size (fp32 keeps the plan's default)
                pkw = {"bytes_per_row": P.row_bytes(m_spa, "fp16")} if kw.get("emb_dtype") == "fp16" else {}
                placement = P.plan(ln_emb, cost if cost is not None else [1.0] * self.Tg, self.world, **pkw)
        self.pl = placement
        if exchange == "nccl" and (self.pl.split_tables() or
                                   [(s.table, s.rank) for s in sorted(self.pl.shards, key=lambda s: s.table)] !=
                                   [(s.table, s.rank) for s in sorted(P.contiguous(ln_emb, self.world).shards,
                                                                      key=lambda s: s.table)]):
            raise SystemExit("ERROR: exchange=nccl supports the reference's contiguous table slices only")
        self.mine = self.pl.of_rank(self.rank)
        self.Tl = len(self.mine)
        self.slices = table_slices(self.Tg, self.world)
        self.t0, self.t1 = self.slices[self.rank]
        if device is None:
            device = "cuda:%d" % torch.cuda.current_device()
        self.device = torch.device(device)
        ek = S.engine_kwargs(self.pl, self.rank, self.Tg)
        self.eng = Engine(m_spa, ek["ln_emb"], ln_bot, ln_top, n_features=ek["n_features"], shards=ek["shards"],
                          split_slots=ek["split_slots"], loss=loss, device=device, max_batch=self.B, gemm=gemm,
                          sigmoid_top=len(ln_top) - 2, **kw)
        e = self.eng
        f32 = torch.float32
        # "reference": every rank's loss is the mean over ITS batch slice, dense gradients are averaged (DDP) and
        # embedding gradients SUMMED over the ranks (the all-to-all backward just routes them,
        # extend_distributed.py:467-486) -- i.e. world x the single-process embedding gradient, exactly what
        # `torchrun dlrm_s_pytorch.py` computes.  "single_process": embedding gradients scaled by 1/world = the
        # gradient of the GLOBAL mean loss, so the run reproduces a single-process run of the whole batch (what
        # the live-reference goldens record).  The two differ by one scalar inside the interaction backward.
        if semantics not in ("reference", "single_process"):
            raise SystemExit("ERROR: semantics must be reference or single_process")
        self.semantics = semantics
        if semantics == "single_process":
            if exchange != "p2p":
                raise SystemExit("ERROR: semantics=single_process needs exchange=p2p")
            e.emb_grad_scale = 1.0 / self.world
        e.dense_sync_fn = self._dense_sync
        self._flag = torch.zeros(1, dtype=f32, device=self.device)
        if exchange == "p2p":
            self._setup_p2p()
            e.gather_fn, e.update_fn = self._gather_p2p, self._update_p2p
            if split_forward == "remote" and self.pl.split_tables():
                self._setup_remote_reads()
            elif split_forward not in ("partial", "remote"):
                raise SystemExit("ERROR: split_forward must be partial or remote")
        else:
            self.send_splits, self.recv_splits = a2a_splits(self.Tg, self.world, self.rank, self.B, self.D)
            self.send = torch.zeros(self.Bg * self.Tl * self.D, dtype=f32, device=self.device)
            self.recv = torch.zeros(sum(self.recv_splits), dtype=f32, device=self.device)
            self.gsend = torch.zeros(sum(self.recv_splits), dtype=f32, device=self.device)
            self.grecv = torch.zeros(self.Bg * self.Tl * self.D, dtype=f32, device=self.device)
            e.gather_fn, e.update_fn = self._gather, self._update

    # ------------------------------------------------------------------ peer-mapped exchange
    def _export(self, t):
        """handle of the cudaMalloc block holding t + t's byte offset inside it"""
        import ctypes as C
        from . import _lib as _l

        h = C.create_string_buffer(64)
        off = C.c_int64()
        _l.check(self.eng.lib.dlrm_b200_ipc_export(t.data_ptr(), h, C.byref(off)), "ipc_export")
        return h.raw, int(off.value)

    def _import(self, handle, offset):
        import ctypes as C
        from . import _lib as _l

        key = (self.device.index, handle)
        if key not in _IPC_BASES:
            base = C.c_void_p()
            _l.check(self.eng.lib.dlrm_b200_ipc_open(handle, self.device.index, C.byref(base)), "ipc_open")
            _IPC_BASES[key] = base.value
        return _IPC_BASES[key] + offset

    def share(self, tensors):
        """All-gather the IPC handles of `tensors` (same list on every rank); returns ptrs[rank][i] usable by
        kernels of THIS device (own tensors: their plain pointers)."""
        torch.cuda.synchronize()
        _KEEP_ALIVE.append(list(tensors))
        if self.world == 1:
            return [[t.data_ptr() for t in tensors]]
        mine = tuple(self._export(t) for t in tensors)
        allh = [None] * self.world
        dist.all_gather_object(allh, mine)
        out = []
        for r in range(self.world):
            if r == self.rank:
                out.append([t.data_ptr() for t in tensors])
            else:
                out.append([self._import(hd, off) for hd, off in allh[r]])
        return out

    def _setup_p2p(self):
        """Map every rank's interaction operand (+ partial-sum area) and gradient receive buffer into this process
        (CUDA IPC over NVLink).  Both directions PUSH: the gather stores pooled rows into the buffer of the rank
        that owns the sample, interact_bwd stores per-table gradient rows into the receive buffer of every rank
        storing rows of the table; every load on the data path stays local (L2-cacheable)."""
        import ctypes as C

        e = self.eng
        e._tc_prepare(self.B)    # final allocation of the dense-gradient arena (split-K slabs)
        # two barrier channels (slots + epoch each): 0 = embedding stream (gather / update), 1 = main
        # stream (dense-gradient sync).  Barriers of one channel are ordered by their stream on every
        # rank; the two streams may interleave differently across ranks, so they must not share slots.
        self._sig = torch.zeros(32, dtype=torch.int32, device=self.device)
        self._epoch = torch.zeros(2, dtype=torch.int32, device=self.device)
        W, B, D = self.world, self.B, self.D
        # gradient receive buffer: slab s = [B, Tl, D] written by rank s's interact_bwd (push over NVLink)
        self._grecv_p2p = torch.zeros(W * B * max(self.Tl, 1) * D, dtype=torch.float32, device=self.device)
        ptrs = self.share([e.TP, self._grecv_p2p, self._sig, e.dense_grad])
        pTP = [p[0] for p in ptrs]
        pdT = [p[1] for p in ptrs]
        psig = [p[2] for p in ptrs]
        pgrad = [p[3] for p in ptrs]
        # gather: pooled rows -> TP of the sample's owner at the engine's (globally consistent) route offsets
        self._peer_TP = (C.c_void_p * W)(*pTP)
        e.peer = (self._peer_TP, W, B)
        # update: slab s of MY receive buffer holds the gradient rows of rank s's samples, [B][Tl][D]
        slab = B * self.Tl * D * 4
        self._peer_dT = (C.c_void_p * W)(*[self._grecv_p2p.data_ptr() + s_ * slab for s_ in range(W)])
        e.peer_dY = (self._peer_dT, W, B)
        e.route_dy = [j * D for j in range(self.Tl)]
        e.dy_stride = self.Tl * D
        # interact_bwd: feature 0 stays local; feature 1 + t goes to slab `rank` of every rank storing rows of t
        from .sharding import grad_routes

        routes, first = grad_routes(self.pl, self.rank, B, D, e.F)
        dst = [e.dT.data_ptr() if r < 0 else pdT[r] + off * 4 for r, off, _ in routes]
        ld = [stride for _, _, stride in routes]
        n = len(dst)
        e.dT_route = ((C.c_void_p * n)(*dst), (C.c_int64 * n)(*ld), (C.c_int * (e.F + 1))(*first))
        self._peer_sig = [(C.c_void_p * W)(*[p + 64 * ch for p in psig]) for ch in range(2)]
        self._peer_grad = (C.c_void_p * W)(*pgrad)
        self.own_sync = os.environ.get("DLRM_P2P_NCCL_SYNC") != "1"   # our kernels instead of NCCL all_reduce
        if self.world == 1:
            e.dense_sync_fn = None            # nothing to average
        elif self.own_sync:
            e.dense_sync_fn = self._dense_sync_p2p
        _KEEP_ALIVE.append(self)
        if self.world > 1:
            dist.barrier()

    def _setup_remote_reads(self):
        """Map every rank's table arena: the forward of a row-split table then reads remote rows directly."""
        e = self.eng
        ptrs = self.share([e.tables])
        tabs = {}
        for t in self.pl.split_tables():
            sh = self.pl.of_table(t)
            bases = []
            for s in sh:
                own = self.pl.of_rank(s.rank)
                row0 = sum(o.local_rows for o in own[:own.index(s)])       # rows before shard s in the owner's arena
                bases.append(ptrs[s.rank][0] + row0 * e.ldw * e.esize)
            tabs[t] = (bases, sh[0].local_rows)
        e.use_remote_reads(tabs)
        e.remote_sample0 = self.rank * self.B

    def _barrier(self, channel: int = 0):
        """Device-side ordering across ranks on the current stream (no host sync)."""
        if self.world == 1:
            return
        if getattr(self, "own_sync", False):
            from . import _lib
            from .engine import _stream

            _lib.check(self.eng.lib.dlrm_b200_p2p_barrier(self._peer_sig[channel], self.rank, self.world,
                                                          self._epoch.data_ptr() + 4 * channel, _stream()),
                       "p2p_barrier")
            self.eng.n_launch += 1
        else:
            dist.all_reduce(self._flag)

    def _dense_sync_p2p(self):
        """Mean of the dense gradients over the ranks with our own two-shot all-reduce over NVLink."""
        from . import _lib
        from .engine import _stream

        self._barrier(1)      # every rank's gradient arena is complete
        _lib.check(self.eng.lib.dlrm_b200_p2p_allreduce_mean(self._peer_grad, self.rank, self.world,
                                                             self.eng.dense_numel, _stream()), "p2p_allreduce_mean")
        self.eng.n_launch += 1
        self._barrier(1)      # every slice has been written back everywhere

    def _gather_p2p(self, sp, link):
        e = self.eng
        # Peers must be done reading my T / partial area (interaction of the previous batch) before anybody's
        # pooled rows of this batch land in it.  Issued ALWAYS (training too): an evaluation forward between
        # two training steps must not race with a faster rank's next gather (round-1 advisor finding).
        self._barrier()
        e._mark("emb:barrier_pre_gather")
        e.emb_forward(sp, link=link)          # routed: stores go to the owners' buffers over NVLink
        e._mark("emb:gather")
        self._barrier()                       # every rank's pooled rows / partial sums have landed everywhere
        e._mark("emb:barrier_post_gather")
        e.reduce_partials(self.B)
        e._mark("emb:reduce_partials")

    def _update_p2p(self, sp, optimizer, clr):
        self._barrier()       # every rank's interact_bwd stores have landed in my receive buffer
        self.eng._mark("emb:barrier_pre_update")
        self.eng.emb_update(sp, optimizer=optimizer, lr=clr)

    # -- forward: pool local tables for the global batch, exchange, land in T
    def _gather(self, sp, link):
        e = self.eng
        e.emb_forward(sp, self.send, self.Tl * self.D, self.D, link)
        dist.all_to_all_single(self.recv, self.send, self.recv_splits, self.send_splits)
        scatter_recv_into_T(self.recv, e.Tbuf, self.Tg, self.world, self.B, self.D)

    # -- backward: route per-bag gradients to the table owners, fused coalesce + optimizer there
    def _update(self, sp, optimizer, clr):
        e = self.eng
        pack_dT_into_send(e.dT, self.gsend, self.Tg, self.world, self.B, self.D)
        dist.all_to_all_single(self.grecv, self.gsend, self.send_splits, self.recv_splits)
        e.emb_update(sp, self.grecv, self.Tl * self.D, self.D, optimizer, clr)

    def _dense_sync(self):
        dist.all_reduce(self.eng.dense_grad[:self.eng.dense_numel], op=dist.ReduceOp.AVG)

    def sync_dense_params_from_rank0(self):
        """DDP broadcasts rank 0's MLP weights at wrap time (SURVEY A: reference quirk)."""
        dist.broadcast(self.eng.dense, src=0)
        self.eng.mark_params_changed()

    def forward(self, X_local, sp_local_shards):
        return self.eng.forward(X_local, sp_local_shards)

    def train_step(self, X_local, sp_local_shards, target_local, lr, optimizer="rwsadagrad"):
        return self.eng.train_step(X_local, sp_local_shards, target_local, lr, optimizer)

    def nvlink_bytes_per_step(self, step_seconds: float, staged_index_bytes: int = 0, lookups=None) -> dict:
        """Bytes THIS rank pushes to its peers per training step (peer stores over NVLink) and what that is per
        second of step time (a lower bound of the link rate: the pushes happen inside three kernels, not all step)."""
        W, B, D = self.world, self.B, self.D
        remote = (W - 1) / W if W > 1 else 0.0
        fwd = len(self.mine) * self.Bg * D * 4 * remote                    # pooled rows / partial sums of all samples
        rd = 0.0
        if self.eng.remote_tables is not None:                              # remote-read forward of the split tables:
            nsplit = sum(1 for s in self.mine if not s.whole)               # no partial sums pushed, rows PULLED instead
            fwd -= nsplit * self.Bg * D * 4 * remote
            if lookups is not None:
                rd = sum(float(lookups[t]) for t in self.pl.split_tables()) * B * D * self.eng.esize * remote
        bwd = sum(sum(1 for s in self.pl.of_table(t) if s.rank != self.rank) for t in range(self.Tg)) * B * D * 4
        idx = staged_index_bytes * remote                                    # upper bound: split tables go to every rank
        tot = fwd + bwd + idx + rd
        return {"pooled_rows_fwd": fwd, "remote_rows_read_fwd": rd, "gradient_rows_bwd": bwd, "indices": idx,
                "total_bytes_per_rank_per_step": tot,
                "gb_per_s_over_step": tot / max(step_seconds, 1e-12) / 1e9, "measured_link_peak_gb_s": 770.0}

    def gather_bytes_per_step(self, lookups_per_sample: Sequence[float]) -> float:
        """Expected embedding-row bytes this rank reads per step (its share of every table's lookups)."""
        ld = 0.0
        for s in self.mine:
            ld += float(lookups_per_sample[s.table]) * (s.local_rows / max(s.rows, 1))
        return ld * self.Bg * self.D * self.eng.esize


# ---------------------------------------------------------------------------- fixed-length (multi-hot) inputs
class MultiHotExchange:
    """Index side of a sharded step for fixed-length bags (the MLPerf multi-hot workload).

    The reference hands every rank the whole global batch (dlrm_s_pytorch.py:528-544).  Here a rank receives
    only ITS samples -- one packed pinned host buffer [X | target | table 0 [B, L_0] | table 1 ...], int32
    indices, ONE H2D copy -- and `exchange()` pushes every table's block into the index buffer of the rank(s)
    storing rows of that table (peer stores over NVLink, one launch), at slot `rank` of the [world, B, L_t]
    global index array the gather / update kernels read.  Offsets are implicit (bag b = [b*L, (b+1)*L))."""

    def __init__(self, de: DistEngine, hot: Sequence[int], m_den: int = 13, nsets: int = 2):
        import ctypes as C

        self.de, self.hot, self.m_den, self.nsets = de, [int(h) for h in hot], m_den, nsets
        B, W, dev = de.B, de.world, de.device
        i32 = torch.int32
        # host / staging layout (bytes)
        self.off_x = 0
        self.off_t = B * m_den * 4
        o = self.off_t + B * 4
        o = (o + 15) // 16 * 16
        self.off_idx = []
        for L in self.hot:
            self.off_idx.append(o)
            o += (B * L * 4 + 15) // 16 * 16
        self.nbytes = o
        self.stage = [torch.zeros(self.nbytes, dtype=torch.uint8, device=dev) for _ in range(nsets)]
        # global index arrays of my shards, per set
        self.idxg = [[torch.zeros(W * B * self.hot[s.table], dtype=i32, device=dev) for s in de.mine]
                     for _ in range(nsets)]
        self.offs = {}
        for L in sorted(set(self.hot)):
            self.offs[L] = (torch.arange(W * B, dtype=torch.int64, device=dev) * L).to(i32)
        self.X = [st[self.off_x:self.off_x + B * m_den * 4].view(torch.float32).view(B, m_den) for st in self.stage]
        self.target = [st[self.off_t:self.off_t + B * 4].view(torch.float32).view(B, 1) for st in self.stage]
        from .engine import SparseInput

        self.sparse = [SparseInput(list(self.idxg[k]), [self.offs[self.hot[s.table]] for s in de.mine], W * B, False)
                       for k in range(nsets)]
        # copy lists: block of table t -> slot `rank` of idxg[j] on every rank storing rows of t
        self._copies = []
        if W > 1:
            ptrs = de.share([t for k in range(nsets) for t in self.idxg[k]])
        from .sharding import index_copies

        for k in range(nsets):
            src, dst, nb = [], [], []
            for t, r, j, off, n in index_copies(de.pl, de.rank, self.hot, B):
                nloc = len(de.pl.of_rank(r))
                if W > 1:
                    base = ptrs[r][k * nloc + j] if r != de.rank else self.idxg[k][j].data_ptr()
                else:
                    base = self.idxg[k][j].data_ptr()
                src.append(self.stage[k].data_ptr() + self.off_idx[t])
                dst.append(base + off * 4)
                nb.append(n * 4)
            self._copies.append((src, dst, nb))
        self._C = C

    def host_buffer(self, pin=True):
        buf = torch.zeros(self.nbytes, dtype=torch.uint8)
        return buf.pin_memory() if pin and torch.cuda.is_available() else buf

    def fill_host(self, buf, seed: int, step: int, rows: Sequence[int]):
        """This rank's samples of global step `step` (dlrm_b200/mlperf.py generator) into a host buffer."""
        from . import mlperf as M

        de, B = self.de, self.de.B
        X, T = M.dense_and_targets(seed, step, de.rank * B, B, self.m_den)
        buf[self.off_x:self.off_x + B * self.m_den * 4].view(torch.float32).view(B, self.m_den).copy_(torch.from_numpy(X))
        buf[self.off_t:self.off_t + B * 4].view(torch.float32).view(B, 1).copy_(torch.from_numpy(T))
        idx = M.multi_hot_batch(seed, step, rows, self.hot, de.rank * B, B, dtype=np.int32)
        for t, a in enumerate(idx):
            buf[self.off_idx[t]:self.off_idx[t] + a.size * 4].view(torch.int32).copy_(torch.from_numpy(a.reshape(-1)))
        return buf

    def upload(self, k: int, buf, non_blocking=True):
        self.stage[k].copy_(buf, non_blocking=non_blocking)
        return self.nbytes

    def exchange(self, k: int):
        """Push the staged index blocks of set k to their owners (current stream).  The consumers' gather is
        ordered behind it by the pre-gather barrier of DistEngine._gather_p2p."""
        from . import _lib
        from .engine import _stream

        C = self._C
        src, dst, nb = self._copies[k]
        for c0 in range(0, len(src), 64):
            n = len(src[c0:c0 + 64])
            _lib.check(self.de.eng.lib.dlrm_b200_block_copy((C.c_void_p * n)(*src[c0:c0 + 64]),
                                                            (C.c_void_p * n)(*dst[c0:c0 + 64]),
                                                            (C.c_int64 * n)(*nb[c0:c0 + 64]), n, _stream()),
                       "block_copy")
            self.de.eng.n_launch += 1


# ---------------------------------------------------------------------------- synthetic sharded batches
def make_sharded_batch(step_seed: int, ln_emb: Sequence[int], rank: int, world: int, local_batch: int,
                       m_den: int = 13, lmax: int = 10, pin: bool = True, placement=None):
    """Rank-local view of one GLOBAL synthetic batch of the `--data-generation=random` distribution (variable
    bag lengths): indices of the tables the rank stores rows of, for all world*local_batch samples (packed
    format, one entry per local shard) + the rank's slice of dense features and targets.  Every table has its
    own seed, so all ranks agree on the global batch."""
    from .data import HostBatch, PackedLayout, fill_batch
    from . import placement as P

    pl = placement if placement is not None else P.contiguous(ln_emb, world)
    tabs = [s.table for s in pl.of_rank(rank)]
    rows = [int(ln_emb[t]) for t in tabs]
    Bg = local_batch * world
    cap = int(Bg * sum(min(int(r), lmax) for r in rows))
    hb = HostBatch(PackedLayout(Bg, len(rows), m_den, max(cap, 1)), pin)
    fill_batch(hb, None, rows, lmax, table_seeds=[(step_seed, 7, t) for t in tabs])
    rng = np.random.default_rng([step_seed, 11])
    Xg = rng.random((Bg, m_den), dtype=np.float32)
    Tg = np.round(rng.random((Bg, 1), dtype=np.float32))
    sl = slice(rank * local_batch, (rank + 1) * local_batch)
    X = torch.from_numpy(Xg[sl].copy())
    T = torch.from_numpy(Tg[sl].copy())
    if pin and torch.cuda.is_available():
        X, T = X.pin_memory(), T.pin_memory()
    return hb, X, T
