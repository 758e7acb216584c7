"""Device-side engine of the DLRM hot path on one H100.

Owns the HBM layout (one table arena, one dense-parameter arena, activation/gradient buffers
written in place by the producing kernels) and sequences the C-ABI kernels of
``include/dlrm_b200.h`` for

    forward            == DLRM_Net.sequential_forward          (dlrm_s_pytorch.py:587-612)
    train_step         == forward + loss_fn_wrap + backward + optimizer.step()  (:1575-1621)

PyTorch is used for device memory and streams only; every FLOP/byte of the path runs in
libdlrm_b200.so.  No CPU fallback exists: a missing library or device raises.

HBM layout (fp32 unless noted)
  tables   [sum_k rows_k, D]   one allocation; table k = rows [row_base_k, row_base_k + rows_k)
                               (emb_dtype="fp16": fp16 rows [D halves | fp32 accumulator | int32 head | pad])
  momentum [sum_k rows_k]      RWSAdagrad row-wise accumulator (optim/rwsadagrad.py:91-95)
  acc_ew   [sum_k rows_k, D]   element-wise Adagrad accumulator (torch.optim.Adagrad 'sum'), a separate arena
                               allocated by the first Adagrad step; same row_base as the tables
  head     [sum_k rows_k] i32  per-row list heads for the sort-free coalesce (zero between steps)
  mark     [nnz] u8            per-occurrence superseded marks beside link[] (zero between steps)
  dense    [P]                 bot W0,b0,W1,b1,... top W0,b0,...  (+ grad arena, + Adagrad sums)
  T        [B, F, D]           interaction operand: feature 0 <- last bottom-MLP epilogue,
                               feature 1+k <- gather of table k (torch.cat K3 eliminated)
  R        [B, ldr]            [x | tril(T T^T)]  (ldr = num_int rounded up to a multiple of 4)
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os
import warnings
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import (ACT_NONE, ACT_RELU, ACT_SIGMOID, DTYPE_F16, DTYPE_F32, DTYPE_Q4, DTYPE_Q8, GEMM_SIMT_FP32,
                   LOSS_BCE, LOSS_MSE, LOSS_WBCE, OPT_ADAGRAD, OPT_RWSADAGRAD, OPT_SGD, EmbBwdTable, EmbFwdTable)

_LOSS = {"mse": LOSS_MSE, "bce": LOSS_BCE, "wbce": LOSS_WBCE}
_OPT = {"sgd": OPT_SGD, "rwsadagrad": OPT_RWSADAGRAD, "adagrad": OPT_ADAGRAD}
_LR_DECAY = ("rwsadagrad", "adagrad")     # optimizers whose step applies lr_decay: clr = lr / (1 + (step - 1) lr_decay)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


_M64 = (1 << 64) - 1


def _splitmix64(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def round_key(seed: int, step: int, table: int) -> int:
    """Stochastic-rounding key of a global table at optimizer step `step` (dlrm_emb_bwd_table_t.round_key): the hash
    prefix of (seed, step, table), keyed like the synthetic batches of mlperf.py."""
    base = ((seed * 0xD6E8FEB86659FD93) ^ ((step + 1) * 0x9E3779B97F4A7C15) ^ ((table + 1) * 0x165667B19E3779F9)) & _M64
    return _splitmix64(base)


def quant_row_bytes(dim: int, bits: int) -> int:
    """Bytes of one packed row-wise quantized row (fbgemm's layout): [dim uint8 | fp32 scale | fp32 bias] for 8 bits,
    [dim/2 bytes | fp16 scale | fp16 bias] for 4 bits."""
    return dim + 8 if bits == 8 else dim // 2 + 4


# Rows quantized per launch when a table is quantized from a float source: a host source (a checkpoint) crosses to the
# device one chunk at a time, so a load needs one chunk of device memory beyond the packed arena.
QUANT_CHUNK_ROWS = 1 << 20


def fp16_row_stride(dim: int) -> int:
    """Row stride (halves) of an fp16 table row [dim halves | fp32 accumulator | int32 head | pad], 16-byte aligned."""
    return (2 * dim + 8 + 15) // 16 * 16 // 2


@dataclass
class SparseInput:
    """Sparse side of one batch, on the device.

    reference format : ``indices[k]`` 1-D per table, ``offsets[k]`` [B] (lS_i / lS_o of
                       dlrm_s_pytorch.py:517); include_last = False.
    packed format    : all tables share one ``indices`` array, ``offsets[k]`` holds B+1 GLOBAL
                       positions into it; include_last = True (CUDA-graph friendly: sizes live on
                       the device, pointers never change).
    """
    indices: List[torch.Tensor]
    offsets: List[torch.Tensor]
    batch: int
    include_last: bool = False
    nnz_total: int = -1

    @property
    def idx_bytes(self) -> int:
        return self.indices[0].element_size()


class Engine:
    def __init__(self, m_spa: int, ln_emb: Sequence[int], ln_bot: Sequence[int], ln_top: Sequence[int],
                 *, op: str = "dot", itself: bool = False, sigmoid_bot: int = -1, sigmoid_top: int = -1,
                 loss: str = "bce", loss_threshold: float = 0.0, loss_ws=None, device="cuda:0",
                 max_batch: int = 2048, gemm: str = "simt", n_features: Optional[int] = None,
                 interleave_momentum: Optional[bool] = None, shards=None, split_slots=None, small_rows_max: int = 256,
                 emb_dtype: str = "fp32", round_seed: int = 0, host_tables: Sequence[int] = (),
                 host_cache_rows=0, host_cache_reserve: int = 1 << 31, learned_row_weights: bool = False):
        if not torch.cuda.is_available():
            raise RuntimeError("dlrm_b200.Engine needs a CUDA device (H100, sm_90a); there is no CPU path")
        self.device = torch.device(device)
        self.lib = _lib.lib()
        sm, major, minor = _lib.device_info(self.device.index or 0)
        self.sm_count = sm
        self.D = int(m_spa)
        self.ln_emb = [int(v) for v in ln_emb]
        self.ln_bot = [int(v) for v in ln_bot]
        self.ln_top = [int(v) for v in ln_top]
        self.T = len(self.ln_emb)                       # table shards stored on THIS device
        # What the local "tables" are (dlrm_b200/placement.py): shard j = rows [row_lo, row_lo + row_n) of global
        # table `table` (part `part` of `nparts`; nparts == 1: the whole table).  Default: every table whole.
        if shards is None:
            shards = [dict(table=k, rows=n, row_lo=0, row_n=n, part=0, nparts=1) for k, n in enumerate(self.ln_emb)]
        self.shards = [dict(s) for s in shards]
        if [int(s["row_n"]) for s in self.shards] != self.ln_emb:
            raise ValueError("ln_emb must list the LOCAL row count of every shard")
        if any(n <= 0 for n in self.ln_emb):       # (row_n == 0 means "the whole table" to the kernels)
            raise ValueError("every table / shard needs at least one row")
        n_glob = max([int(s["table"]) for s in self.shards], default=-1) + 1
        self.F = int(n_features) if n_features else n_glob + 1   # interaction features (global)
        # row-split tables of the GLOBAL placement, (table, nparts) each: the rank that owns a sample adds the
        # nparts partial sums of its bags (one slab of the partial area per part)
        if split_slots is None:
            seen = {}
            for sh in self.shards:
                if int(sh["nparts"]) > 1:
                    seen[int(sh["table"])] = int(sh["nparts"])
            split_slots = sorted(seen.items())
        self.split_slots = [(int(t), int(n)) for t, n in split_slots]
        self.slab_first = np.concatenate([[0], np.cumsum([n for _, n in self.split_slots])]).astype(np.int64)
        self.slot_of = {t: i for i, (t, _) in enumerate(self.split_slots)}
        self.small_rows_max = int(small_rows_max)
        self.op, self.itself = op, bool(itself)
        if op not in ("dot", "cat"):
            raise ValueError("arch_interaction_op=%s is not supported" % op)
        self.sigmoid_bot, self.sigmoid_top = int(sigmoid_bot), int(sigmoid_top)
        self.loss_kind = _LOSS[loss]
        self.loss_threshold = float(loss_threshold)
        if gemm not in ("simt", "tc", "tc_bf16"):
            raise ValueError("gemm must be simt | tc (bf16x3 split, fp32-grade) | tc_bf16")
        self.gemm_mode = gemm
        self.gemm = GEMM_SIMT_FP32          # back end of the fp32-pointer entry points
        self.tc = gemm != "simt"
        self.tc_x3 = 1 if gemm == "tc" else 0
        self.tc_B = -1                       # batch size the wgmma plans were built for
        self._pack_dirty = True
        self._tc_kept = {}                   # B -> wgmma state a captured CUDA graph runs on (kept, see _tc_keep)
        if self.ln_bot[-1] != self.D:
            raise ValueError("bottom MLP output %d != sparse feature size %d" % (self.ln_bot[-1], self.D))
        if op == "dot":
            self.num_int = self.D + (self.F * (self.F + 1) // 2 if itself else self.F * (self.F - 1) // 2)
        else:
            self.num_int = self.F * self.D
        if self.ln_top[0] != self.num_int:
            raise ValueError("# of feature interactions %d does not match first dimension of top mlp %d"
                             % (self.num_int, self.ln_top[0]))
        dev = self.device
        # ---- table row type.  fp16: rows are stored as IEEE halves, widened to fp32 by the gather and the update, and
        # written back with stochastic rounding keyed by (round_seed, opt_step, global table, global row, column).
        if emb_dtype not in ("fp32", "fp16", "int8", "int4"):
            raise ValueError("emb_dtype must be fp32, fp16, int8 or int4")
        self.emb_dtype = emb_dtype
        self.f16 = emb_dtype == "fp16"
        # Row-wise quantized tables (emb_dtype="int8" / "int4", or quantize_tables() on a float engine): the forward
        # gathers packed rows from `qtables`; nothing trains them.  quant_only: the float arena was never allocated.
        self.quant_bits = {"int8": 8, "int4": 4}.get(emb_dtype, 0)
        self.quant_only = self.quant_bits > 0
        self.qtables: Optional[torch.Tensor] = None
        if self.quant_only:
            self._check_quant_placement(self.quant_bits, host_tables, shards)
        self.round_seed = int(round_seed)
        self.wdtype = torch.float16 if self.f16 else torch.float32
        self.esize = 2 if self.f16 else 4          # bytes per stored table element
        if self.f16 and self.D % 8:
            raise ValueError("fp16 embedding tables need a dimension divisible by 8 (got %d)" % self.D)
        if self.f16 and interleave_momentum is False:
            raise ValueError("fp16 embedding tables always keep the accumulator and list head inside the row")
        # ---- tables
        rows = np.asarray(self.ln_emb, dtype=np.int64)
        self.row_base = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
        self.total_rows = int(self.row_base[-1])
        # Host tables (dlrm_b200/host_tables.py): their rows live in pinned host memory and the rows of each batch are
        # staged through HBM.  Every table keeps its rows in ONE arena, device or host; _abase[k] is its first row
        # there (== row_base[k] when no table is on the host).
        self.host = sorted(set(int(k) for k in host_tables))
        self.is_host = [k in self.host for k in range(self.T)]
        self._check_host_tables(interleave_momentum)
        self._check_host_cache(host_cache_rows, host_cache_reserve)
        self._abase, nb = [], [0, 0]
        for k, n in enumerate(self.ln_emb):
            self._abase.append(nb[self.is_host[k]])
            nb[self.is_host[k]] += n
        self.dev_rows, self.host_rows = nb
        # Row layout.  interleave (default when D % 4 == 0): [D weights | Adagrad accumulator | list head (int32) |
        # 2 pad], row stride D + 4 floats -- the two per-row words of the backward live in the row's own DRAM page.
        # The update kernel is bound by the RATE of random DRAM accesses, not by bytes: a 4-byte head[] read costs
        # about what a 512-byte row costs, so separate head / accumulator arrays would add two random accesses per
        # row.  The gather pays a little bandwidth for rows that are no longer 512-byte aligned (528-byte stride).
        # interleave=False: dense [rows, D] tables + separate accumulator / head arrays (round 1's layout).
        if interleave_momentum is None:
            interleave_momentum = self.f16 or ((self.D % 4 == 0) and os.environ.get("DLRM_ROW_META", "1") != "0")
        self.interleave = bool(interleave_momentum)
        # DLRM_ROW_PAD: floats appended to a row (>= 2: accumulator + list head).  4 keeps rows 16-B aligned (+3 % memory);
        # 16 keeps 512-B rows 64-B aligned (every row the same 8 DRAM atoms + 1 for the two words, +12.5 % memory).
        self.row_pad = max(4, (int(os.environ.get("DLRM_ROW_PAD", "4")) + 3) // 4 * 4)
        self.ldw = self.D + self.row_pad if self.interleave else self.D        # row stride in stored elements
        if self.f16:
            self.ldw = fp16_row_stride(self.D)      # D + 8 halves at D % 8 == 0: 272 bytes at D = 128
        if self.quant_only:
            self.interleave = False
            self.tables = self._head_sep = None
            self.qtables = torch.zeros((self.dev_rows, quant_row_bytes(self.D, self.quant_bits)), dtype=torch.uint8,
                                       device=dev)
        else:
            self.tables = torch.zeros((self.dev_rows, self.ldw), dtype=self.wdtype, device=dev)
            self._head_sep = None if self.interleave else torch.zeros(self.dev_rows, dtype=torch.int32, device=dev)
        self._host_init()
        self._momentum_sep: Optional[torch.Tensor] = None
        self.acc_ew: Optional[torch.Tensor] = None       # element-wise Adagrad accumulators [total_rows, D]
        self.row_weights: Optional[torch.Tensor] = None  # weighted pooling v_W_l, arena [total_rows]
        # Learned weighted pooling (--weighted-pooling=learned): v starts at one and the fused update steps it with its
        # rows (dv = <S, W_old>); RWSAdagrad / Adagrad keep its dense 'sum' in row_weight_sum [total_rows].
        self.learned_row_weights = bool(learned_row_weights)
        self.row_weight_sum: Optional[torch.Tensor] = None
        if self.learned_row_weights:
            self._check_learned_placement()
            self.row_weights = torch.ones(self.total_rows, dtype=torch.float32, device=dev)
        # ---- dense arena
        self.dense_slices = []  # (name, layer, kind, offset, shape)
        ofs = 0
        for name, ln in (("bot", self.ln_bot), ("top", self.ln_top)):
            for i in range(len(ln) - 1):
                n_in, n_out = ln[i], ln[i + 1]
                self.dense_slices.append((name, i, "W", ofs, (n_out, n_in)))
                ofs += n_out * n_in
                ofs = (ofs + 3) & ~3  # keep every tensor 16-byte aligned
                self.dense_slices.append((name, i, "b", ofs, (n_out,)))
                ofs += n_out
                ofs = (ofs + 3) & ~3
        self.dense_numel = ofs
        self.dense = torch.zeros(ofs, dtype=torch.float32, device=dev)
        self.dense_grad = torch.zeros(ofs, dtype=torch.float32, device=dev)
        self.dense_state: Optional[torch.Tensor] = None
        self.W = {"bot": [], "top": []}
        self.b = {"bot": [], "top": []}
        self.dW = {"bot": [], "top": []}
        self.db = {"bot": [], "top": []}
        for name, i, kind, o, shape in self.dense_slices:
            n = int(np.prod(shape))
            (self.W if kind == "W" else self.b)[name].append(self.dense[o:o + n].view(shape))
            (self.dW if kind == "W" else self.db)[name].append(self.dense_grad[o:o + n].view(shape))
        self.loss_ws = None
        if loss_ws is not None:
            self.loss_ws = torch.as_tensor(loss_ws, dtype=torch.float32, device=dev)
        self.opt_step = 0
        # While set (a CUDA graph being captured with GraphedTrainStep(device_lr=True)), the optimizer kernels read the
        # learning rate from this device float instead of taking it by value; `lr_scalar` is the engine's one.
        self.lr_dev: Optional[torch.Tensor] = None
        self.lr_scalar: Optional[torch.Tensor] = None
        self._marks = None      # phase timeline (bench.py --phases): list of (name, stream tag, CUDA event)
        # hooks replaced by dlrm_b200.dist for table-wise sharded runs
        self.gather_fn = None       # (sp, link) -> fills Tbuf[:, 1:, :] for the LOCAL batch
        self.update_fn = None       # (sp, optimizer, clr) -> embedding update from dT[:, 1:, :]
        self.dense_sync_fn = None   # () -> make dense_grad slab 0 the cross-rank mean gradient
        self.dT_route = None        # (void*[n], int64[n], int[F+1]): destinations of interact_bwd's rows per feature
        self.n_launch = 0            # kernels launched by this engine (bench: gpu_launches)
        self.peer = None             # sharded runs: (peer_out void*[world], world, local batch) for the gather
        self.peer_dY = None          #               (peer_dY void*[world], world, local batch) for the update
        # Row-split tables, forward variant "remote" (BASELINE north_star: P2P reads of remote rows): table ->
        # ([base pointer of every shard], rows per shard); the rank that owns a sample pools the whole bag itself,
        # reading each row from the rank that stores it, instead of every rank pooling a partial sum.
        self.emb_grad_scale = 1.0    # sharded runs: factor on the embedding gradient rows (DistEngine.semantics)
        self.remote_tables = None
        self.remote_sample0 = 0      # first global sample of THIS rank (its bags inside the global index streams)
        # side streams: the gather runs beside the bottom MLP, the weight-gradient GEMMs and the
        # embedding update beside the dgrad chain (independent work; parallel branches in the graph)
        self.s_emb = torch.cuda.Stream(device=self.device)
        self.s_wg = torch.cuda.Stream(device=self.device)
        self.s_small = torch.cuda.Stream(device=self.device)
        self._alloc_activations(int(max_batch))

    # ------------------------------------------------------------------ buffers
    def _alloc_activations(self, B: int):
        dev, f32 = self.device, torch.float32
        self.max_batch = B
        D, F = self.D, self.F
        # interaction operand T [B, F, D] followed by the partial-sum area of the row-split tables
        # [slab][B][D] (one slab per (split table, part)); ONE allocation, so that a peer needs one mapping
        n_slabs = int(self.slab_first[-1])
        self.TP = torch.zeros(B * F * D + n_slabs * B * D, dtype=f32, device=dev)
        self.Tbuf = self.TP[:B * F * D].view(B, F, D)
        self.part = self.TP[B * F * D:]
        self._set_default_routes()
        self.ldr = (self.num_int + 3) & ~3
        self.Rbuf = torch.zeros((B, self.ldr), dtype=f32, device=dev) if self.op == "dot" else None
        nb, nt = len(self.ln_bot) - 1, len(self.ln_top) - 1
        # post-activation outputs of every layer (last bottom layer lives in Tbuf[:, 0, :])
        self.bot_act = [torch.empty((B, self.ln_bot[i + 1]), dtype=f32, device=dev) for i in range(nb - 1)]
        self.top_act = [torch.empty((B, self.ln_top[i + 1]), dtype=f32, device=dev) for i in range(nt)]
        # gradients w.r.t. pre-activations
        self.bot_gz = [torch.empty((B, self.ln_bot[i + 1]), dtype=f32, device=dev) for i in range(nb - 1)]
        self.top_gz = [torch.empty((B, self.ln_top[i + 1]), dtype=f32, device=dev) for i in range(nt)]
        self.dT = torch.zeros((B, F, D), dtype=f32, device=dev)
        self.dR = torch.zeros((B, self.ldr), dtype=f32, device=dev) if self.op == "dot" else None
        self.loss_buf = torch.zeros(1, dtype=f32, device=dev)
        self.scratch = torch.zeros(1024, dtype=f32, device=dev)
        self.link = None  # int32 [2 * nnz capacity]
        self.mark = None  # uint8 [nnz capacity]: occurrence superseded by a later one of its row (zero between steps)
        self.dedup, self._filtered = None, False
        # Optional duplicate filter for the training gather / update (dlrm_emb_dedup_t).  It removes the gather's
        # list-head atomics but adds a memset + two small launches to the gather side and runs the general update
        # kernel instead of the lean one; OFF by default.
        self.use_filter = False

    def is_small(self, j: int) -> bool:
        """Tiny whole tables take the dense two-pass update (csrc/emb_small.cu) instead of the per-row lists."""
        sh = self.shards[j]
        return (int(sh["nparts"]) == 1 and self.ln_emb[j] <= self.small_rows_max and self.D % 4 == 0
                and self.D <= 512)

    def _set_default_routes(self):
        """Single-GPU routes.  out: (offset, sample stride) of shard j's pooled rows inside TP; dy: offset of
        shard j's gradient rows inside one sample of dT (sample stride F*D)."""
        from .sharding import out_routes

        B, F, D = self.max_batch, self.F, self.D
        self.route_out, self.route_dy = out_routes(self.shards, self.split_slots, B, F, D)
        self.dy_stride = F * D

    def _emb_forward_remote(self, sp: SparseInput, split, link: bool):
        """Row-split tables, remote-read variant: pool the bags of MY samples (rows fetched from the shards' owners
        through peer-mapped memory, summed in index order -> bit-identical to the reference), and -- training --
        thread the global occurrences that fall into my row ranges onto their lists (indices only)."""
        B = sp.batch if self.peer is None else self.peer[2]
        done = set()
        descs = []
        for k in split:
            t = int(self.shards[k]["table"])
            if t in done:
                continue
            done.add(t)
            ptrs, rps = self.remote_tables[t]
            d = _lib.EmbRemoteTable()
            for i, p_ in enumerate(ptrs):
                d.shard_weight[i] = p_
            d.num_shards, d.rows_per_shard, d.rows, d.ld = len(ptrs), int(rps), int(self.shards[k]["rows"]), self.ldw
            d.weight_dtype = DTYPE_F16 if self.f16 else DTYPE_F32
            es = sp.offsets[k].element_size()
            d.indices = sp.indices[k].data_ptr() if sp.indices[k].numel() else 0
            d.offsets = sp.offsets[k].data_ptr() + self.remote_sample0 * es     # my bags inside the global stream
            d.nnz = sp.indices[k].numel()
            d.out_off, d.out_stride = (1 + t) * self.D, self.F * self.D
            # offsets[b + 1] exists for my last bag unless it is the last bag of the global batch (reference format)
            last_global = self.remote_sample0 + B >= sp.batch
            descs.append((d, 1 if (sp.include_last or not last_global) else 0))
        for inc in (0, 1):
            group = [d for d, i in descs if i == inc]
            for c0 in range(0, len(group), 4):
                arr = (_lib.EmbRemoteTable * len(group[c0:c0 + 4]))(*group[c0:c0 + 4])
                _lib.check(self.lib.dlrm_b200_emb_bag_fwd_remote(arr, len(arr), self.D, B, sp.idx_bytes, inc,
                                                                 self.TP.data_ptr(), _stream()), "emb_bag_fwd_remote")
                self.n_launch += 1
        if link:
            for c0 in range(0, len(split), _lib.MAX_TABLES):
                ks = split[c0:c0 + _lib.MAX_TABLES]
                desc, _ = self._bwd_desc_chunk(sp, ks)
                _lib.check(self.lib.dlrm_b200_emb_bwd_link(desc, len(ks), sp.batch, sp.idx_bytes, int(sp.include_last),
                                                           self.link.data_ptr(), _stream()), "emb_bwd_link")
                self.n_launch += 1

    def use_remote_reads(self, tables=None):
        """Switch the row-split tables to the remote-read forward.  tables: {table: ([shard base pointers], rows per
        shard)}; None (single GPU): every shard is a local one."""
        if tables is None:
            tables = {}
            for t, n in self.split_slots:
                js = sorted((int(sh["part"]), j) for j, sh in enumerate(self.shards) if int(sh["table"]) == t)
                ptrs = [self.tables.data_ptr() + int(self.row_base[j]) * self.ldw * self.esize for _, j in js]
                rps = int(self.shards[js[0][1]]["row_n"])
                tables[t] = (ptrs, rps)
        self.remote_tables = tables

    def reduce_partials(self, B: int):
        """T[b, 1+t, :] = sum of the partial sums of every row-split table t (fixed part order)."""
        if not self.split_slots or self.remote_tables is not None:
            return
        n = len(self.split_slots)
        feat = (C.c_int * n)(*[1 + t for t, _ in self.split_slots])
        first = (C.c_int * (n + 1))(*[int(v) for v in self.slab_first])
        # slabs are laid out with the ALLOCATED batch as their stride: reduce over the full capacity rows
        _lib.check(self.lib.dlrm_b200_emb_reduce_partials(self.part.data_ptr(), self.Tbuf.data_ptr(), self.F * self.D,
                                                          self.max_batch, self.D, feat, first, n, _stream()),
                   "emb_reduce_partials")
        self.n_launch += 1

    def _ensure_link(self, nnz_total: int):
        if self.link is None or self.link.numel() < 2 * nnz_total:
            cap = max(2 * nnz_total, 1024)
            self.link = torch.empty(cap, dtype=torch.int32, device=self.device)
            self.mark = torch.zeros(cap // 2, dtype=torch.uint8, device=self.device)
            # duplicate filter (see include/dlrm_b200.h, dlrm_emb_dedup_t): ~8 hashed counters per occurrence
            n = max(nnz_total, 512)
            log2 = max(16, int(np.ceil(np.log2(8 * n))))
            self.filter = torch.zeros((1 << log2) + 4, dtype=torch.int32, device=self.device)
            self.flags = torch.zeros(n, dtype=torch.uint8, device=self.device)
            self.suspects = torch.zeros(n, dtype=torch.int32, device=self.device)
            d = _lib.EmbDedup()
            d.filter, d.log2_size = self.filter.data_ptr(), log2
            d.flags, d.suspects = self.flags.data_ptr(), self.suspects.data_ptr()
            self.dedup = d
        self._filtered = False

    # ------------------------------------------------------------------ host tables (csrc/host_tables.cu)
    def _check_host_tables(self, interleave_momentum):
        if not self.host:
            return
        bad = [k for k in self.host if not 0 <= k < self.T]
        if bad:
            raise ValueError("host_tables: table %d does not exist (%d tables)" % (bad[0], self.T))
        if self.f16:
            raise ValueError("host tables need fp32 rows: the stochastic rounding of fp16 tables is keyed by the row "
                             "index the update kernel sees, which is a staging slot for a host table")
        if any(int(s["nparts"]) != 1 or int(s["row_lo"]) != 0 or int(s["table"]) != k
               for k, s in enumerate(self.shards)):
            raise ValueError("host tables are not supported on sharded runs")
        tiny = [k for k in self.host if self.is_small(k)]
        if tiny:
            raise ValueError("host_tables: table %d has %d rows (<= small_rows_max=%d): tiny tables take the dense "
                             "two-pass update, which indexes the whole table on the device"
                             % (tiny[0], self.ln_emb[tiny[0]], self.small_rows_max))

    def _check_host_cache(self, rows, reserve):
        """Row cache of the host tables (host_cache_rows: 0 = none, "auto", or a row count rounded up to 32)."""
        from .host_tables import MAP_LIMIT

        self.cache_rows = 0
        self._cache_auto = rows == "auto"
        self._cache_reserve = int(reserve)
        if not self._cache_auto:
            rows = int(rows)
            if rows < 0:
                raise ValueError("host_cache_rows=%d: expected 0 (no cache), a row count or \"auto\"" % rows)
            self.cache_rows = (rows + 31) // 32 * 32
        if (self._cache_auto or self.cache_rows) and not self.host:
            raise ValueError("host_cache_rows: a host row cache needs host tables (host_tables=[...])")
        if self.cache_rows + 1 > MAP_LIMIT:
            raise ValueError("host_cache_rows=%d: cache rows + staging positions must fit the int32 slot map (<= %d)"
                             % (self.cache_rows, MAP_LIMIT))

    def _pinned_zeros(self, shape) -> torch.Tensor:
        """Zeros in page-locked host memory mapped at the same device address (cudaHostRegister on a plain CPU tensor:
        torch's pinned allocator would round every block up to a power of two)."""
        t = torch.zeros(shape, dtype=torch.float32)
        nbytes = t.numel() * 4
        if nbytes:
            _lib.check(self.lib.dlrm_b200_host_register(t.data_ptr(), nbytes), "host_register")
            self._pinned.append(t)
            self.pinned_bytes += nbytes
        return t

    def _host_init(self):
        self._pinned: List[torch.Tensor] = []
        self.pinned_bytes = 0
        self.tables_h = self._momentum_sep_h = self.acc_ew_h = None
        self._staged = None             # SparseInput whose host-table rows are in the staging arena
        self._staged_by_link = False
        self._staged_train = False
        self.stage_cap = 0
        self._arena_rows = 0            # cache rows + staging positions of the device arena
        self._cache_ready = False
        self._cache_dirty = False       # a training step may have left rows in the cache since the last flush
        self.cache_flushes = 0
        if not self.host:
            return
        import weakref

        self.tables_h = self._pinned_zeros((self.host_rows, self.ldw))
        self._map_base = {}
        n = 0
        for k in self.host:
            self._map_base[k] = n
            n += self.ln_emb[k]
        self.slot_map = torch.zeros(n, dtype=torch.int32, device=self.device)   # slot + 1 of a staged row, else 0
        self.stage_count = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._slot_idx = {}
        weakref.finalize(self, _unpin, self.lib, self._pinned)

    def _host_sync(self):
        """Host reads and writes of host rows wait for every staging copy the engine has enqueued.  With a row cache,
        every resident row is written back and the cache emptied first: the caller sees current rows, and whatever it
        writes through its view is what the next step stages.  The flush waits for every stream first (an insert may
        still run on the update's stream), and runs only if a training step ran since the last one."""
        torch.cuda.synchronize(self.device)
        if self._cache_dirty:
            self._flush_cache()
            torch.cuda.synchronize(self.device)

    def _flush_cache(self):
        """Every resident row back to host memory and the cache emptied (current stream; the caller has ordered it
        after the last insert)."""
        arr, st = self._host_desc(None)
        _lib.check(self.lib.dlrm_b200_host_cache_flush(arr, len(self.host), C.byref(st), self.D, _stream()),
                   "host_cache_flush")
        self.n_launch += 1
        self.cache_flushes += 1
        self._cache_dirty = False

    def _cache_row_bytes(self) -> int:
        """Device bytes of one cache row: its arena row and words, tag (8), last use (4), set lists (< 1)."""
        return (4 * self.ldw + (0 if self.interleave else 4) + (4 if self._momentum_sep_h is not None else 0)
                + (4 * self.D if self.acc_ew_h is not None else 0) + 13)

    def _init_cache(self, cap: int):
        """Size ("auto": from the free device memory when the first batch is staged, beside a staging arena of `cap`
        positions) and allocate the cache's metadata, once, before the first arena is laid out."""
        from .host_tables import auto_cache_rows

        dev = self.device
        if self._cache_auto:
            free, _ = torch.cuda.mem_get_info(dev)
            row = self._cache_row_bytes()
            stage = cap * (row - 13 + 4 + 8 + 8)        # arena rows, list, key, slot indices
            self.cache_rows = auto_cache_rows(free - stage, self._cache_reserve, row, self.host_rows)
            self._cache_auto = False
        N = self.cache_rows
        if N:
            self.cache_tag = torch.full((N,), -1, dtype=torch.int64, device=dev)
            self.cache_used = torch.zeros(N, dtype=torch.int32, device=dev)
            self.cache_step = torch.zeros(1, dtype=torch.int32, device=dev)
            self.cache_set_head = torch.zeros(N // 32, dtype=torch.int32, device=dev)
            self.cache_sets = torch.zeros(N // 32, dtype=torch.int32, device=dev)
            self.cache_nsets = torch.zeros(1, dtype=torch.int32, device=dev)
            self.cache_stats = torch.zeros(4, dtype=torch.int64, device=dev)
            self._cache_ready = True

    def _ensure_stage(self, cap: int, idx_bytes: int):
        """Device arena for the cache rows and `cap` staging positions (one slot per position of the batch).  When
        the staging grows, the cache is written back and emptied and the old arena released before the new one is
        allocated: there is never a second copy of the cache rows, so an "auto" cache sized at the first batch
        still fits when a later batch needs more staging."""
        from .host_tables import MAP_LIMIT

        dev = self.device
        if not self._cache_ready and (self._cache_auto or self.cache_rows):
            self._init_cache(cap)
        N = self.cache_rows
        if cap > self.stage_cap:
            if N + cap > MAP_LIMIT:
                raise ValueError("host tables: %d cache rows + %d staging positions do not fit the int32 slot map "
                                 "(<= %d)" % (N, cap, MAP_LIMIT))
            if N and self.stage_cap:
                if self._staged is not None:
                    self._stage_out(True)
                torch.cuda.synchronize(self.device)       # inserts on the update's stream have finished
                if self._cache_dirty:
                    self._flush_cache()
                self.stage_w = self.stage_head = self.stage_mom = self.stage_acc = None
            if N and cap > 256 * (N // 32):
                warnings.warn("host cache of %d rows: %d sets for up to %d misses per step; one warp walks each "
                              "set's misses, so a step can be slower than without the cache (use at least %d rows)"
                              % (N, N // 32, cap, (cap + 255) // 256 * 32), stacklevel=3)
            self.stage_cap = cap
            self._arena_rows = N + cap
            self.stage_w = torch.zeros((N + cap, self.ldw), dtype=torch.float32, device=dev)
            self.stage_head = None if self.interleave else torch.zeros(N + cap, dtype=torch.int32, device=dev)
            self.stage_list = torch.zeros(cap, dtype=torch.int32, device=dev)
            self.stage_key = torch.zeros(cap, dtype=torch.int64, device=dev)
            self.stage_mom = self.stage_acc = None
            self._slot_idx = {}
            if N:
                self.cache_set_next = torch.zeros(cap, dtype=torch.int32, device=dev)
        if self._momentum_sep_h is not None and self.stage_mom is None:
            self.stage_mom = torch.zeros(self._arena_rows, dtype=torch.float32, device=dev)
        if self.acc_ew_h is not None and self.stage_acc is None:
            self.stage_acc = torch.zeros((self._arena_rows, self.D), dtype=torch.float32, device=dev)
        if idx_bytes not in self._slot_idx:
            dt = torch.int64 if idx_bytes == 8 else torch.int32
            self._slot_idx[idx_bytes] = torch.zeros(self.stage_cap, dtype=dt, device=dev)

    def _pos_base(self, sp: SparseInput, k: int) -> int:
        """First global position of table k: packed batches' offsets are global already; reference-format tables
        are numbered back to back (the pair_base of the update)."""
        return 0 if sp.include_last else sum(int(sp.indices[j].numel()) for j in range(k))

    def _slot_ptr(self, sp: SparseInput, k: int) -> int:
        return self._slot_idx[sp.idx_bytes].data_ptr() + self._pos_base(sp, k) * sp.idx_bytes

    def _host_desc(self, sp: Optional[SparseInput], forward_only: bool = False):
        """Descriptors of the host tables and the arena for batch `sp` (None: no batch, for the cache flush)."""
        arr = (_lib.HostTable * len(self.host))()
        for n, k in enumerate(self.host):
            d = arr[n]
            d.weight = self.tables_h.data_ptr() + self._abase[k] * self.ldw * 4
            if self._momentum_sep_h is not None:
                d.momentum = self._momentum_sep_h.data_ptr() + self._abase[k] * 4
            if self.acc_ew_h is not None:
                d.acc_ew = self.acc_ew_h.data_ptr() + self._abase[k] * self.D * 4
            d.rows = self.ln_emb[k]
            d.map = self.slot_map.data_ptr() + self._map_base[k] * 4
            if sp is None:
                d.offsets = self.stage_count.data_ptr()        # never read
                continue
            d.indices = sp.indices[k].data_ptr() if sp.indices[k].numel() else 0
            d.offsets = sp.offsets[k].data_ptr()
            d.nnz = sp.indices[k].numel()
            d.pos_base = self._pos_base(sp, k)
        st = _lib.HostStage()
        st.weight, st.list, st.key = self.stage_w.data_ptr(), self.stage_list.data_ptr(), self.stage_key.data_ptr()
        st.momentum = _ptr(self.stage_mom) if self._momentum_sep_h is not None else None
        st.acc_ew = _ptr(self.stage_acc) if self.acc_ew_h is not None else None
        st.head = _ptr(self.stage_head)
        st.count, st.capacity, st.ld = self.stage_count.data_ptr(), self.stage_cap, self.ldw
        st.head_col = self._meta_col + 1 if self.interleave else -1
        st.slot_idx = next(iter(self._slot_idx.values())).data_ptr() if sp is None else \
            self._slot_idx[sp.idx_bytes].data_ptr()
        if self.cache_rows:
            st.cache_rows, st.cache_tag, st.cache_used = self.cache_rows, self.cache_tag.data_ptr(), \
                self.cache_used.data_ptr()
            st.step, st.set_head, st.set_next = self.cache_step.data_ptr(), self.cache_set_head.data_ptr(), \
                self.cache_set_next.data_ptr()
            st.sets, st.num_sets, st.stats = self.cache_sets.data_ptr(), self.cache_nsets.data_ptr(), \
                self.cache_stats.data_ptr()
            st.forward_only = int(forward_only)
        return arr, st

    def _stage_in(self, sp: SparseInput, by_link: bool = False, train: bool = True):
        """Stage the rows of this batch's host-table occurrences (current stream).  A staging left by a step that did
        not finish is written back first (its rows are unchanged or updated; either way they go home).  train=False:
        a pass without an update, which leaves the row cache as it is."""
        if self.use_filter:
            raise ValueError("host tables do not support the duplicate filter (use_filter)")
        if self.row_weights is not None:
            raise ValueError("host tables do not support weighted pooling: row_weights is indexed by the table row")
        if self._staged is not None:
            self._stage_out(True)
        if sp.include_last and len({sp.indices[k].data_ptr() for k in self.host}) > 1:
            raise ValueError("host tables: a packed batch must hold every table's indices in one array")
        cap = sp.nnz_total if sp.include_last else sum(int(i.numel()) for i in sp.indices)
        self._ensure_stage(max(int(cap), 1), sp.idx_bytes)
        arr, st = self._host_desc(sp, forward_only=not train)
        _lib.check(self.lib.dlrm_b200_host_stage_in(arr, len(self.host), C.byref(st), self.D, sp.batch, sp.idx_bytes,
                                                    int(sp.include_last), _stream()), "host_stage_in")
        self.n_launch += 2      # counter memset (with a cache, a training pass: begin kernel) + kernel
        if self.cache_rows and train:
            self._cache_dirty = True
        self._staged, self._staged_by_link, self._staged_train = sp, by_link, train

    def _stage_out(self, write: bool):
        """After the update: staged rows back to their host rows; forward only: release the slots."""
        if self._staged is None:
            return
        if self.cache_rows and not self._staged_train:
            write = False       # a pass without an update changed no row, and its misses are not cache candidates
        arr, st = self._host_desc(self._staged, forward_only=not self._staged_train)
        self._staged = None
        fn = self.lib.dlrm_b200_host_write_back if write else self.lib.dlrm_b200_host_release
        _lib.check(fn(arr, len(self.host), C.byref(st), self.D, _stream()), "host_write_back")
        self.n_launch += 2 if write and self.cache_rows else 1      # with a cache: insert kernel + write-back

    def _abandon_staging(self):
        """A step raised between stage-in and write-back: return the staged rows so that no slot stays claimed.  With
        a cache the misses are inserted as after an update (their rows are current either way), and the list heads of
        the cache slots are cleared, since a link may have set them for an update that never ran."""
        if self.host and self._staged is not None:
            with contextlib.suppress(Exception):
                self._stage_out(True)
                if self.cache_rows:
                    N = self.cache_rows
                    if self.interleave:
                        self.stage_w[:N, self._meta_col + 1].zero_()
                    else:
                        self.stage_head[:N].zero_()

    def host_cache_stats(self) -> dict:
        """Cumulative counters of the host row cache (synchronises): hits, inserts, evictions and staged (uncached)
        rows, each per distinct row of a training step; plus the cache size, the training steps seen and the flushes
        (a read of a host table's memory through table(k), momentum_of(k), accumulator_ew(k) or the module's
        state_dict / load_state_dict writes the cache back when a training step ran since the last flush; so does a
        growth of the staging arena).  All zero without a cache."""
        out = dict(hits=0, inserts=0, evictions=0, staged=0, rows=self.cache_rows, steps=0,
                   flushes=self.cache_flushes)
        if self._cache_ready:
            h, i, e, s = (int(v) for v in self.cache_stats.tolist())
            out.update(hits=h, inserts=i, evictions=e, staged=s, steps=int(self.cache_step.item()))
        return out

    def table(self, k: int) -> torch.Tensor:
        """[rows_k, D] view of table k (strided when the accumulator is interleaved; fp16 with emb_dtype="fp16").
        A host table's view is a CPU tensor of pinned memory, returned after the engine's work has completed."""
        if self.quant_only:
            raise RuntimeError("emb_dtype=%s: the engine stores only the packed rows of its tables (table_q(k)); their "
                               "float rows were never stored" % self.emb_dtype)
        if self.is_host[k]:
            self._host_sync()
            return self._rows_of(self.tables_h, k)[:, :self.D]
        return self._rows_of(self.tables, k)[:, :self.D]

    # ------------------------------------------------------------------ row-wise quantized tables (csrc/quant.cu)
    def _check_quant_placement(self, bits, host_tables, shards):
        if bits == 8 and self.D % 4 or bits == 4 and self.D % 8:
            raise ValueError("%d-bit quantized tables need an embedding dimension divisible by %d (got %d)"
                             % (bits, 4 if bits == 8 else 8, self.D))
        if host_tables:
            raise ValueError("quantized tables are device tables (host_tables is not supported)")
        if shards is not None and any(int(s["nparts"]) != 1 or int(s["table"]) != k for k, s in enumerate(shards)):
            raise ValueError("quantized tables are not supported on sharded runs")

    def _refuse_quantized(self, what: str):
        if self.quant_bits:
            raise RuntimeError("%s: the embedding tables are %d-bit row-wise quantized, which is inference-only "
                               "(forward and forward-only graphs)" % (what, self.quant_bits))

    def table_q(self, k: int) -> torch.Tensor:
        """[rows_k, quant_row_bytes] uint8 view of table k's packed rows: the bytes of
        torch.ops.quantized.embedding_bag_{byte,4bit}_prepack of its float rows."""
        if self.qtables is None:
            raise RuntimeError("the tables are not quantized (emb_dtype=\"int8\"/\"int4\" or quantize_tables())")
        return self._rows_of(self.qtables, k)

    def quantize_rows(self, k: int, src: torch.Tensor, r0: int = 0):
        """Quantize float rows src [n, D] (fp32 or fp16, device or host, e.g. an mmap-loaded checkpoint) into rows
        [r0, r0 + n) of table k's packed rows.  A host source crosses to the device QUANT_CHUNK_ROWS rows at a time;
        a device source is read in place at its row stride."""
        if self.qtables is None:
            raise RuntimeError("the tables are not quantized (emb_dtype=\"int8\"/\"int4\" or quantize_tables())")
        if src.dim() != 2 or src.shape[1] != self.D or src.dtype not in (torch.float32, torch.float16):
            raise ValueError("quantize_rows: expected fp32 / fp16 rows of shape [n, %d], got %s %s"
                             % (self.D, src.dtype, tuple(src.shape)))
        n = int(src.shape[0])
        if r0 < 0 or r0 + n > self.ln_emb[k]:
            raise ValueError("quantize_rows: rows [%d, %d) outside table %d (%d rows)" % (r0, r0 + n, k, self.ln_emb[k]))
        dst = self.table_q(k)
        qd = DTYPE_Q8 if self.quant_bits == 8 else DTYPE_Q4
        with torch.no_grad():
            for c0 in range(0, n, QUANT_CHUNK_ROWS):
                part = src[c0:c0 + QUANT_CHUNK_ROWS]
                if part.device != self.device or part.stride(1) != 1:
                    part = part.to(self.device).contiguous()
                _lib.check(self.lib.dlrm_b200_emb_quantize_rows(
                    part.data_ptr(), DTYPE_F16 if part.dtype == torch.float16 else DTYPE_F32, part.stride(0),
                    part.shape[0], self.D, dst[r0 + c0:].data_ptr(), qd, dst.stride(0), _stream()), "emb_quantize_rows")
                self.n_launch += 1
                del part

    def quantize_tables(self, bits: int):
        """DLRM_Net.quantize_embedding: pack every (device) float table into `bits`-bit rows; from then on the forward
        gathers the packed rows and the float tables stay as they are.  Training is refused afterwards."""
        if bits not in (4, 8):
            raise ValueError("only 4- and 8-bit row-wise quantization is supported (got %r)" % (bits,))
        if self.quant_only:
            raise RuntimeError("the tables are already %d-bit quantized (emb_dtype=%s)" % (self.quant_bits, self.emb_dtype))
        self._check_quant_placement(bits, self.host, self.shards)
        self.quant_bits = bits
        self.qtables = torch.zeros((self.dev_rows, quant_row_bytes(self.D, bits)), dtype=torch.uint8, device=self.device)
        for k in range(self.T):
            self.quantize_rows(k, self.table(k))

    def _rows_of(self, arena: torch.Tensor, k: int) -> torch.Tensor:
        """Rows of table k in `arena` (a device arena or its host twin; the table decides which)."""
        return arena[self._abase[k]:self._abase[k] + self.ln_emb[k]]

    def momentum_of(self, k: int) -> Optional[torch.Tensor]:
        """[rows_k] row-wise Adagrad accumulators of table k (a CPU view for a host table), or None."""
        if self.is_host[k]:
            self._host_sync()
            m = (self.tables_h.view(torch.float32)[:, self._meta_col] if self.interleave else self._momentum_sep_h)
        else:
            m = self.momentum
        return None if m is None else self._rows_of(m, k)

    @property
    def _meta_col(self) -> int:
        """Column of the accumulator in the 4-byte view of an interleaved row (the list head is the next one)."""
        return self.D * self.esize // 4

    @property
    def head(self) -> torch.Tensor:
        """Per-row list heads of the sort-free coalesce, [sum rows] int32 (a strided view when interleaved)."""
        return self.tables.view(torch.int32)[:, self._meta_col + 1] if self.interleave else self._head_sep

    @property
    def momentum(self) -> Optional[torch.Tensor]:
        """Row-wise Adagrad accumulator of every row, [sum rows] fp32 (a strided view when interleaved)."""
        return self.tables.view(torch.float32)[:, self._meta_col] if self.interleave else self._momentum_sep

    def _check_learned_placement(self):
        """Learned row weights are indexed by the table row: every table whole and in device memory."""
        if self.host:
            raise ValueError("host tables do not support weighted pooling: row_weights is indexed by the table row")
        if any(int(s["nparts"]) > 1 or int(s["table"]) != k for k, s in enumerate(self.shards)):
            raise ValueError("learned weighted pooling is not supported on sharded runs")

    def ensure_optimizer_state(self, optimizer: str):
        self._refuse_quantized("optimizer state")
        if optimizer == "rwsadagrad":
            if not self.interleave and self._momentum_sep is None:
                self._momentum_sep = torch.zeros(self.dev_rows, dtype=torch.float32, device=self.device)
                if self.host:
                    self._momentum_sep_h = self._pinned_zeros((self.host_rows,))
        if optimizer == "adagrad" and self.acc_ew is None:
            # One fp32 accumulator per table element (4 D bytes per row), in its own arena: the optimizer is created
            # after the tables are laid out (dlrm_s_pytorch.py builds DLRM_Net first), and moving the tables into an
            # interleaved [w | s] layout then would move every emb_l[k].weight.
            self.acc_ew = torch.zeros((self.dev_rows, self.D), dtype=torch.float32, device=self.device)
            if self.host:
                self.acc_ew_h = self._pinned_zeros((self.host_rows, self.D))
        if optimizer in _LR_DECAY and self.dense_state is None:
            self.dense_state = torch.zeros_like(self.dense)
        if optimizer in _LR_DECAY and self.learned_row_weights and self.row_weight_sum is None:
            self.row_weight_sum = torch.zeros(self.total_rows, dtype=torch.float32, device=self.device)

    def row_weight_sum_of(self, k: int) -> torch.Tensor:
        """[rows_k] Adagrad 'sum' of the learned row weights of table k (after ensure_optimizer_state)."""
        return self.row_weight_sum[int(self.row_base[k]):int(self.row_base[k + 1])]

    def accumulator_ew(self, k: int) -> torch.Tensor:
        """[rows_k, D] element-wise Adagrad accumulators of table k (after ensure_optimizer_state("adagrad"))."""
        if self.is_host[k]:
            self._host_sync()
            return self._rows_of(self.acc_ew_h, k)
        return self._rows_of(self.acc_ew, k)

    def _point_at_acc_ew(self, desc, ks):
        """Element-wise Adagrad: the descriptors of tables ks take the [rows, D] accumulator rows as `momentum`
        (a host table's: its staged rows)."""
        base = self.acc_ew.data_ptr()
        for n, k in enumerate(ks):
            desc[n].momentum = self.stage_acc.data_ptr() if self.is_host[k] else base + self._abase[k] * self.D * 4
            desc[n].mom_stride = self.D

    # ------------------------------------------------------------------ parameters
    def mark_params_changed(self):
        """Call after writing master weights from outside (the bf16 operand copies are stale)."""
        self._pack_dirty = True

    def load_params(self, params: dict):
        self._pack_dirty = True
        """params = dict(emb=[W_k], bot=[(W,b)...], top=[(W,b)...], v_W_l=None|[...]) of numpy /
        torch arrays (the layout of the oracle and of the reference's state_dict)."""
        if self.host and params.get("v_W_l") is not None:
            raise ValueError("host tables do not support weighted pooling: row_weights is indexed by the table row")
        with torch.no_grad():
            for k, Wk in enumerate(params["emb"]):     # fp16 tables: round to nearest
                self.table(k).copy_(torch.as_tensor(Wk, dtype=torch.float32))
            for name in ("bot", "top"):
                for i, (Wl, bl) in enumerate(params[name]):
                    self.W[name][i].copy_(torch.as_tensor(Wl, dtype=torch.float32))
                    self.b[name][i].copy_(torch.as_tensor(bl, dtype=torch.float32))
            if params.get("v_W_l") is not None:
                if self.row_weights is None:    # learned weights: written in place (parameters are views)
                    self.row_weights = torch.empty(self.total_rows, dtype=torch.float32, device=self.device)
                for k, w in enumerate(params["v_W_l"]):
                    self.row_weights[int(self.row_base[k]):int(self.row_base[k + 1])].copy_(
                        torch.as_tensor(w, dtype=torch.float32))

    def init_params(self, seed: int = 0):
        """Same distributions as create_emb / create_mlp (dlrm_s_pytorch.py:221-228, :280-284),
        drawn on the device (26 x 1e6 x 128 takes 150 s with the reference's numpy init)."""
        self._pack_dirty = True
        g = torch.Generator(device=self.device)
        g.manual_seed(seed)
        # row stride of an fp32 engine built with the same arguments (its default layout): fp16 tables draw like it
        ld32 = self.D + self.row_pad if (self.D % 4 == 0 and os.environ.get("DLRM_ROW_META", "1") != "0") else self.D
        with torch.no_grad():
            for k, n in enumerate(self.ln_emb):
                a = float(np.sqrt(1.0 / int(self.shards[k]["rows"])))      # the bound of the WHOLE table (:280-284)
                tk = self.table(k)
                for r0 in range(0, tk.shape[0], 1 << 24):                    # chunks: any temporary stays < 9 GB
                    if self.is_host[k]:
                        # the draw of a device engine: the same chunk of full rows (same sizes and row stride) on the
                        # device, its other words kept, then copied back out whole
                        hrows = self._rows_of(self.tables_h, k)[r0:r0 + (1 << 24)]
                        tmp = hrows.to(self.device)
                        tmp[:, :self.D].uniform_(-a, a, generator=g)
                        hrows.copy_(tmp)
                        del tmp
                    elif self.f16:
                        # the fp32 draw of an fp32 engine, rounded to nearest.  The draw goes into a view with the
                        # fp32 engine's sizes AND row stride: torch's generator maps values to elements through the
                        # iteration space of its output (split into 32-bit-indexable pieces by the byte span), so
                        # only an identical view draws identical values.
                        n = tk[r0:r0 + (1 << 24)].shape[0]
                        tmp = torch.empty((n, ld32), dtype=torch.float32, device=self.device)[:, :self.D]
                        tk[r0:r0 + (1 << 24)].copy_(tmp.uniform_(-a, a, generator=g))
                        del tmp
                    else:
                        tk[r0:r0 + (1 << 24)].uniform_(-a, a, generator=g)
            for name, ln in (("bot", self.ln_bot), ("top", self.ln_top)):
                for i in range(len(ln) - 1):
                    n, m = ln[i], ln[i + 1]
                    self.W[name][i].normal_(0.0, float(np.sqrt(2.0 / (m + n))), generator=g)
                    self.b[name][i].normal_(0.0, float(np.sqrt(1.0 / m)), generator=g)

    # ------------------------------------------------------------------ descriptors
    def _fwd_desc(self, sp: SparseInput, tables=None, route=None):
        """route: per-shard (offset, sample stride) of the pooled rows (None: the call-level [b, k, :] layout)."""
        ks = range(self.T) if tables is None else tables
        arr = (EmbFwdTable * len(ks))()
        for n, k in enumerate(ks):
            d = arr[n]
            sh = self.shards[k]
            if self.quant_bits:     # packed rows, ld in bytes
                d.ld = self.qtables.stride(0)
                d.weight = self.qtables.data_ptr() + self._abase[k] * d.ld
                d.weight_dtype = DTYPE_Q8 if self.quant_bits == 8 else DTYPE_Q4
            else:
                d.weight = self.tables.data_ptr() + self._abase[k] * self.ldw * self.esize
                d.ld = self.ldw
                d.weight_dtype = DTYPE_F16 if self.f16 else DTYPE_F32
            d.indices = sp.indices[k].data_ptr() if sp.indices[k].numel() else 0
            d.offsets = sp.offsets[k].data_ptr()
            d.row_weights = (self.row_weights.data_ptr() + int(self.row_base[k]) * 4
                             if self.row_weights is not None else None)
            d.nnz = sp.indices[k].numel()
            d.rows = int(sh["rows"])
            d.row_lo, d.row_n = int(sh["row_lo"]), int(sh["row_n"])
            if self.is_host[k]:      # the staged rows, read through the slot of every position
                d.weight, d.indices = self.stage_w.data_ptr(), self._slot_ptr(sp, k)
                d.rows, d.row_lo, d.row_n = self._arena_rows, 0, self._arena_rows
            if route is not None:
                d.out_off, d.out_stride = int(route[k][0]), int(route[k][1])
        return arr

    def _bwd_desc(self, sp: SparseInput, tables=None, dy_off=None):
        ks = range(self.T) if tables is None else tables
        arr = (EmbBwdTable * len(ks))()
        base = 0
        for n, k in enumerate(ks):
            d = arr[n]
            sh = self.shards[k]
            d.row_lo, d.row_n = int(sh["row_lo"]), int(sh["row_n"])
            if dy_off is not None:
                d.use_dy_off, d.dy_off = 1, int(dy_off[k])
            d.weight = self.tables.data_ptr() + self._abase[k] * self.ldw * self.esize
            if self.is_host[k]:
                d.weight, d.row_lo, d.row_n = self.stage_w.data_ptr(), 0, self._arena_rows
            d.ld = self.ldw
            if self.f16:
                d.weight_dtype = DTYPE_F16
                d.round_key = round_key(self.round_seed, self.opt_step, int(sh["table"]))
            if self.interleave:
                d.momentum = d.weight + self.D * self.esize
                d.mom_stride = self.ldw * self.esize // 4
            else:
                d.momentum = (self._momentum_sep.data_ptr() + self._abase[k] * 4
                              if self._momentum_sep is not None else None)
                if self.is_host[k]:
                    d.momentum = self.stage_mom.data_ptr() if self._momentum_sep is not None else None
                d.mom_stride = 1
            # tiny tables are neither linked nor list-updated (head NULL): emb_small_update handles them
            if self.is_small(k):
                d.head = None
            elif self.interleave:
                d.head, d.head_stride = d.weight + self.D * self.esize + 4, self.ldw * self.esize // 4
            elif self.is_host[k]:
                d.head, d.head_stride = self.stage_head.data_ptr(), 1
            else:
                d.head, d.head_stride = self._head_sep.data_ptr() + self._abase[k] * 4, 1
            d.mark = self.mark.data_ptr() if self.mark is not None else None
            d.indices = sp.indices[k].data_ptr() if sp.indices[k].numel() else 0
            d.offsets = sp.offsets[k].data_ptr()
            d.nnz = sp.indices[k].numel()
            d.rows = int(sh["rows"])
            if self.is_host[k]:
                d.indices, d.rows = self._slot_ptr(sp, k), self._arena_rows
            d.pair_base = 0 if sp.include_last else base
            base += sp.indices[k].numel()
            if self.learned_row_weights:
                d.row_weights = self.row_weights.data_ptr() + int(self.row_base[k]) * 4
                d.row_weight_sum = (self.row_weight_sum.data_ptr() + int(self.row_base[k]) * 4
                                    if self.row_weight_sum is not None else None)
        total = sp.nnz_total if sp.include_last else base
        return arr, total

    # ------------------------------------------------------------------ kernels
    def _act(self, which: str, i: int) -> int:
        sig = self.sigmoid_bot if which == "bot" else self.sigmoid_top
        return ACT_SIGMOID if i == sig else ACT_RELU

    def emb_forward(self, sp: SparseInput, out: Optional[torch.Tensor] = None, stride_sample: int = 0,
                    stride_table: int = 0, link: bool = False):
        """apply_emb for every local shard: one launch per <= 64 whole tables + one for the row-split shards.
        out is None (the engine's own forward): pooled rows go where `route_out` says -- feature slot 1+t of the
        interaction operand (of the rank that owns the sample, on a sharded run) for a whole table, the shard's
        slab of the partial-sum area for a row-split one.  Explicit `out`: out[b, k, :] with the given strides.
        link=True (training) also threads every index occurrence onto its per-row list (step 1 of the
        sort-free coalesce) inside the same kernel."""
        chk = _lib.check
        if link:
            self._refuse_quantized("training gather")
            total = sp.nnz_total if sp.include_last else sum(int(i.numel()) for i in sp.indices)
            self._ensure_link(total)
        # host tables: stage the rows first (unless emb_link already staged this batch for its update)
        stage = bool(self.host) and not (self._staged is sp and self._staged_by_link)
        if stage:
            self._stage_in(sp, train=link)
        routed = out is None
        route = self.route_out if routed else [(k * stride_table, stride_sample) for k in range(self.T)]
        whole = [k for k in range(self.T) if int(self.shards[k]["nparts"]) == 1]
        split = [k for k in range(self.T) if int(self.shards[k]["nparts"]) > 1]
        remote = routed and self.remote_tables is not None and bool(split)
        if remote:
            self._emb_forward_remote(sp, split, link)
            split = []
        use_filter = self.use_filter and not split and not any(self.is_small(k) for k in range(self.T))
        peer = self.peer if routed else None
        base = self.TP.data_ptr() if routed else out.data_ptr()
        first = True
        for group in (whole, split):
            for c0 in range(0, len(group), _lib.MAX_TABLES):
                ks = group[c0:c0 + _lib.MAX_TABLES]
                desc = self._fwd_desc(sp, ks, route)
                bdesc = self._bwd_desc_chunk(sp, ks)[0] if link else None
                dd = C.byref(self.dedup) if (link and use_filter) else None
                if link and use_filter and first:
                    self.filter.zero_()     # counters + suspect count
                first = False
                if peer is not None:
                    chk(self.lib.dlrm_b200_emb_bag_fwd_p2p(desc, bdesc, len(ks), self.D, sp.batch, sp.idx_bytes,
                                                           int(sp.include_last), self.link.data_ptr() if link else None,
                                                           peer[0], peer[1], peer[2], 0, 0, dd, _stream()),
                        "emb_bag_fwd_p2p")
                elif link:
                    chk(self.lib.dlrm_b200_emb_bag_fwd_train(desc, bdesc, len(ks), self.D, sp.batch, sp.idx_bytes,
                                                             int(sp.include_last), self.link.data_ptr(), base,
                                                             0, 0, dd, _stream()), "emb_bag_fwd_train")
                else:
                    chk(self.lib.dlrm_b200_emb_bag_fwd(desc, len(ks), self.D, sp.batch, sp.idx_bytes,
                                                       int(sp.include_last), base, 0, 0, _stream()), "emb_bag_fwd")
                self.n_launch += 1
        if link:
            self._filtered = use_filter
            if use_filter:
                self.emb_classify(sp)
        elif stage:
            self._stage_out(False)      # forward only: nothing will update the staged rows

    def mlp_forward(self, which: str, x: torch.Tensor, ldx: int, B: int, outs: List[torch.Tensor],
                    lds: List[int], upto: Optional[int] = None):
        ln = self.ln_bot if which == "bot" else self.ln_top
        for i in range(len(ln) - 1 if upto is None else upto):
            K, N = ln[i], ln[i + 1]
            _lib.check(self.lib.dlrm_b200_linear_fwd(x.data_ptr(), ldx, self.W[which][i].data_ptr(), K,
                                                     self.b[which][i].data_ptr(), outs[i].data_ptr(),
                                                     lds[i], B, N, K, self._act(which, i), self.gemm,
                                                     _stream()), "linear_fwd")
            self.n_launch += 1
            x, ldx = outs[i], lds[i]

    def _bot_outs(self, B):
        outs = list(self.bot_act) + [self.Tbuf]
        lds = [t.shape[1] for t in self.bot_act] + [self.F * self.D]
        return outs, lds

    def _top_in(self):
        if self.op == "dot":
            return self.Rbuf, self.ldr
        return self.Tbuf, self.F * self.D

    # ---- fused head (last top layer with a single output; csrc/head.cu)
    @property
    def has_head(self) -> bool:
        return self.ln_top[-1] == 1 and len(self.ln_top) >= 3

    def _head(self, B: int, target: Optional[torch.Tensor], train: bool):
        """p (+ loss, gz, dW/db of the last layer and the gradient w.r.t. its input)."""
        nt = len(self.ln_top) - 1
        K = self.ln_top[nt - 1]
        h = self.top_act[nt - 2]
        need = int(self.lib.dlrm_b200_head_scratch_bytes(B, K))
        if getattr(self, "head_scratch", None) is None or self.head_scratch.numel() < need:
            self.head_scratch = torch.zeros(need, dtype=torch.uint8, device=self.device)
        gprev = gh = gl = None
        ldg = ldb = 0
        if train:
            if self.tc and (nt - 2) < self.ntc["top"]:
                gh_t, gl_t, ldb = self.tc_gz["top"][nt - 2]
                gh, gl = gh_t.data_ptr(), gl_t.data_ptr()
            else:
                gprev, ldg = self.top_gz[nt - 2].data_ptr(), self.top_gz[nt - 2].shape[1]
        _lib.check(self.lib.dlrm_b200_head_fused(
            h.data_ptr(), h.shape[1], self.W["top"][nt - 1].data_ptr(), self.b["top"][nt - 1].data_ptr(),
            _ptr(target), _ptr(self.loss_ws), B, K, self._act("top", nt - 1), self._act("top", nt - 2),
            self.loss_kind, self.loss_threshold, self.top_act[nt - 1].data_ptr(),
            self.loss_buf.data_ptr() if target is not None else None,
            self.top_gz[nt - 1].data_ptr() if target is not None else None,
            self.dW["top"][nt - 1].data_ptr() if train else None,
            self.db["top"][nt - 1].data_ptr() if train else None,
            gprev, ldg, gh, gl, ldb, self.head_scratch.data_ptr(), _stream()), "head_fused")
        self.n_launch += 1

    def forward(self, X: torch.Tensor, sp: SparseInput, *, link: bool = False, skip_head: bool = False) -> torch.Tensor:
        """sequential_forward.  X [B, m_den] fp32 on the device.  Returns p [B, n_out] (a view of an
        engine buffer, valid until the next call); clamped iff 0 < loss_threshold < 1.
        link=True: training forward (gather also builds the per-row occurrence lists);
        skip_head=True: leave the final 1-output layer to the fused head in backward()."""
        B = X.shape[0]   # MLP / interaction batch (== sp.batch except under table-wise sharding)
        if B > self.max_batch:
            self._alloc_activations(B)
        if self.tc:
            return self._tc_forward(X, sp, link, skip_head)
        FD = self.F * self.D
        outs, lds = self._bot_outs(B)
        self.mlp_forward("bot", X, X.stride(0), B, outs, lds)
        if self.T:
            self.emb_forward(sp, link=link)
            self.reduce_partials(B)
        if self.op == "dot":
            _lib.check(self.lib.dlrm_b200_interact_fwd(self.Tbuf.data_ptr(), FD, self.Rbuf.data_ptr(),
                                                       self.ldr, B, self.F, self.D, int(self.itself),
                                                       _stream()), "interact_fwd")
            self.n_launch += 1
        xin, ldx = self._top_in()
        self.mlp_forward("top", xin, ldx, B, self.top_act, [t.shape[1] for t in self.top_act],
                         upto=(len(self.ln_top) - 2) if self.has_head else None)
        if self.has_head and not skip_head:
            self._head(B, None, False)
        p = self.top_act[-1][:B]
        if 0.0 < self.loss_threshold < 1.0:
            return torch.clamp(p, self.loss_threshold, 1.0 - self.loss_threshold)
        return p

    def prepare(self, sp: SparseInput, train: bool = True, batch: Optional[int] = None):
        """Allocate every lazily-created buffer / wgmma plan for this batch shape (no kernels that
        change parameters): required before CUDA-graph capture."""
        B = batch if batch is not None else sp.batch
        if B > self.max_batch:
            self._alloc_activations(B)
        if train and self.T:
            self._ensure_link(sp.nnz_total if sp.include_last else sum(int(i.numel()) for i in sp.indices))
        small = [k for k in range(self.T) if self.is_small(k)]
        if train and small:
            self._ensure_small_scratch(max(sum(self.ln_emb[k] for k in small[c0:c0 + 32])
                                           for c0 in range(0, len(small), 32)), B)
        if self.host:
            self._ensure_stage(max(int(sp.nnz_total if sp.include_last else sum(int(i.numel()) for i in sp.indices)),
                                   1), sp.idx_bytes)
        if self.has_head:
            nt = len(self.ln_top) - 1
            need = int(self.lib.dlrm_b200_head_scratch_bytes(B, self.ln_top[nt - 1]))
            if getattr(self, "head_scratch", None) is None or self.head_scratch.numel() < need:
                self.head_scratch = torch.zeros(need, dtype=torch.uint8, device=self.device)
        if self.tc:
            self._tc_prepare(B)
        torch.cuda.synchronize()

    def emb_classify(self, sp: SparseInput):
        """After a filtered training gather (counters still L2-hot): flag suspects, link only those."""
        for c0 in range(0, self.T, _lib.MAX_TABLES):
            ks = list(range(c0, min(self.T, c0 + _lib.MAX_TABLES)))
            desc, _ = self._bwd_desc_chunk(sp, ks)
            _lib.check(self.lib.dlrm_b200_emb_bwd_classify(desc, len(ks), sp.batch, sp.idx_bytes,
                                                           int(sp.include_last), self.link.data_ptr(),
                                                           C.byref(self.dedup), _stream()), "emb_bwd_classify")
            self.n_launch += 2

    def emb_link(self, sp: SparseInput):
        """Thread this batch's (table,row) occurrences onto per-row lists.  Indices only: may be
        issued on a side stream, concurrently with the forward pass."""
        self._refuse_quantized("emb_link")
        total = sp.nnz_total if sp.include_last else sum(int(i.numel()) for i in sp.indices)
        self._ensure_link(total)
        if self.host and self._staged is not sp:
            self._stage_in(sp, by_link=True)
        for c0 in range(0, self.T, _lib.MAX_TABLES):
            ks = list(range(c0, min(self.T, c0 + _lib.MAX_TABLES)))
            desc, _ = self._bwd_desc_chunk(sp, ks)
            _lib.check(self.lib.dlrm_b200_emb_bwd_link(desc, len(ks), sp.batch, sp.idx_bytes,
                                                       int(sp.include_last), self.link.data_ptr(),
                                                       _stream()), "emb_bwd_link")
            self.n_launch += 1
        self._filtered = False

    def _bwd_desc_chunk(self, sp, ks, dy_off=None):
        # pair_base must be global over ALL tables of the batch, not per chunk
        arr, total = self._bwd_desc(sp, range(self.T), dy_off)
        sub = (EmbBwdTable * len(ks))()
        for n, k in enumerate(ks):
            C.memmove(C.byref(sub[n]), C.byref(arr[k]), C.sizeof(EmbBwdTable))
        return sub, total

    def emb_update(self, sp: SparseInput, dY: Optional[torch.Tensor] = None, stride_sample: int = 0,
                   stride_table: int = 0, optimizer: str = "rwsadagrad", lr: float = 0.01, eps: float = 1e-10):
        """Fused embedding backward + sparse optimizer for every local shard (coalesce + row update in place).
        dY is None: the gradient rows are where `route_dy` says (dT, or the receive slabs of a sharded run);
        explicit dY: dY[b, k, :] with the given strides.  Tiny tables go through the dense two-pass kernels."""
        self._refuse_quantized("emb_update")
        routed = dY is None
        dy_off = self.route_dy if routed else [k * stride_table for k in range(self.T)]
        ss = self.dy_stride if routed else stride_sample
        peer = self.peer_dY if routed else None
        base = None if peer is not None else (self.dT.data_ptr() if routed else dY.data_ptr())
        big = [k for k in range(self.T) if not self.is_small(k)]
        small = [k for k in range(self.T) if self.is_small(k)]
        if self.host and self._staged is not sp:
            raise RuntimeError("host tables: emb_update needs this batch staged by forward(link=True) or emb_link()")
        # The tiny-table kernels (few, long-running CTAs) go FIRST, on their own stream: they take their SM slots and the
        # grid-stride list-path update fills the rest of the machine beside them (different tables, no ordering needed).
        side = bool(small) and bool(big) and os.environ.get("DLRM_SMALL_SIDE", "1") != "0"
        if side:
            self._fork(self.s_small)
        with (torch.cuda.stream(self.s_small) if side else contextlib.nullcontext()):
            for c0 in range(0, len(small), 32):
                ks = small[c0:c0 + 32]
                desc, _ = self._bwd_desc_chunk(sp, ks, dy_off)
                if optimizer == "adagrad":
                    self._point_at_acc_ew(desc, ks)
                rows = sum(self.ln_emb[k] for k in ks)
                self._ensure_small_scratch(rows, sp.batch)
                args = (desc, len(ks), self.D, sp.batch, sp.idx_bytes, int(sp.include_last), base,
                        peer[0] if peer is not None else None, peer[1] if peer is not None else 0,
                        peer[2] if peer is not None else 0, ss, _OPT[optimizer], lr)
                tail = (eps, self.small_scratch.data_ptr(), self.small_scratch.numel() * 4, _stream())
                if self.lr_dev is None:
                    _lib.check(self.lib.dlrm_b200_emb_bwd_small_update(*args, *tail), "emb_bwd_small_update")
                else:
                    _lib.check(self.lib.dlrm_b200_emb_bwd_small_update_lr_dev(*args, self.lr_dev.data_ptr(), *tail),
                               "emb_bwd_small_update_lr_dev")
                self.n_launch += 2
        for c0 in range(0, len(big), _lib.MAX_TABLES):
            ks = big[c0:c0 + _lib.MAX_TABLES]
            desc, _ = self._bwd_desc_chunk(sp, ks, dy_off)
            if optimizer == "adagrad":
                self._point_at_acc_ew(desc, ks)
            dd = C.byref(self.dedup) if self._filtered else None
            if peer is not None:
                if self.lr_dev is not None:
                    raise RuntimeError("a device learning rate is not supported on sharded runs")
                _lib.check(self.lib.dlrm_b200_emb_bwd_update_p2p(desc, len(ks), self.D, sp.batch, sp.idx_bytes,
                                                                 int(sp.include_last), self.link.data_ptr(), peer[0],
                                                                 peer[1], peer[2], ss, 0, _OPT[optimizer], lr, eps, dd,
                                                                 _stream()), "emb_bwd_update_p2p")
            elif self.lr_dev is None:
                _lib.check(self.lib.dlrm_b200_emb_bwd_update(desc, len(ks), self.D, sp.batch, sp.idx_bytes,
                                                             int(sp.include_last), self.link.data_ptr(), base, ss, 0,
                                                             _OPT[optimizer], lr, eps, dd, _stream()), "emb_bwd_update")
            else:
                _lib.check(self.lib.dlrm_b200_emb_bwd_update_lr_dev(desc, len(ks), self.D, sp.batch, sp.idx_bytes,
                                                                    int(sp.include_last), self.link.data_ptr(), base,
                                                                    ss, 0, _OPT[optimizer], lr,
                                                                    self.lr_dev.data_ptr(), eps, dd, _stream()),
                           "emb_bwd_update_lr_dev")
            self.n_launch += 1
        if self.host:
            self._stage_out(True)       # same stream as the update: the rows go home before anything reads them
        if side:
            self._join(self.s_small)

    def _ensure_small_scratch(self, rows: int, batch: int):
        need = int(self.lib.dlrm_b200_emb_bwd_small_scratch_bytes(rows, self.D, batch))
        if getattr(self, "small_scratch", None) is None or self.small_scratch.numel() * 4 < need:
            self.small_scratch = torch.zeros(max(need // 4, 1), dtype=torch.float32, device=self.device)

    def mlp_backward(self, which: str, x_in: torch.Tensor, ldx: int, in_act: int, B: int,
                     acts: List[torch.Tensor], act_ld: List[int], gz: List[torch.Tensor],
                     gz_ld: List[int], dx: Optional[torch.Tensor], lddx: int):
        """gz[-1] holds the gradient w.r.t. the last pre-activation.  Produces dW/db for every
        layer and (if dx is given) the gradient w.r.t. the stack input, times in_act'(x_in)."""
        ln = self.ln_bot if which == "bot" else self.ln_top
        s = _stream()
        nl = len(ln) - 1
        if which == "top" and self.has_head and not getattr(self, "_external_gz", False):
            nl -= 1  # the fused head already produced that layer's gradients
        for i in reversed(range(nl)):
            K, N = ln[i], ln[i + 1]
            xin, ldxi = (x_in, ldx) if i == 0 else (acts[i - 1], act_ld[i - 1])
            _lib.check(self.lib.dlrm_b200_linear_wgrad(gz[i].data_ptr(), gz_ld[i], xin.data_ptr(), ldxi,
                                                       self.dW[which][i].data_ptr(), K,
                                                       self.db[which][i].data_ptr(), B, N, K, self.gemm, s),
                       "linear_wgrad")
            self.n_launch += 2  # GEMM + column sum (bias grad)
            if i > 0:
                _lib.check(self.lib.dlrm_b200_linear_dgrad(gz[i].data_ptr(), gz_ld[i],
                                                           self.W[which][i].data_ptr(), K,
                                                           acts[i - 1].data_ptr(), act_ld[i - 1],
                                                           self._act(which, i - 1), gz[i - 1].data_ptr(),
                                                           gz_ld[i - 1], B, N, K, self.gemm, s),
                           "linear_dgrad")
                self.n_launch += 1
            elif dx is not None:
                _lib.check(self.lib.dlrm_b200_linear_dgrad(gz[0].data_ptr(), gz_ld[0],
                                                           self.W[which][0].data_ptr(), K,
                                                           _ptr(x_in) if in_act != ACT_NONE else None, ldx,
                                                           in_act, dx.data_ptr(), lddx, B, N, K, self.gemm, s),
                           "linear_dgrad")
                self.n_launch += 1

    def loss_and_grad(self, target: torch.Tensor, B: int, want_grad: bool = True):
        p = self.top_act[-1]
        n = B * p.shape[1]
        last = self._act("top", len(self.ln_top) - 2)
        _lib.check(self.lib.dlrm_b200_loss_fwd_bwd(p.data_ptr(), target.data_ptr(), _ptr(self.loss_ws), n,
                                                   self.loss_kind, self.loss_threshold, last,
                                                   self.loss_buf.data_ptr(),
                                                   self.top_gz[-1].data_ptr() if want_grad else None,
                                                   self.scratch.data_ptr(), _stream()), "loss_fwd_bwd")
        self.n_launch += 1
        return self.loss_buf

    def backward(self, X: torch.Tensor, sp: SparseInput, target: torch.Tensor, update=None):
        """Everything between the loss and the parameter gradients.  Leaves dense grads in
        dense_grad and the per-bag embedding grads in dT[:, 1:, :].  update=(optimizer, clr) also
        applies the fused embedding update (on a side stream on the tensor-core path)."""
        self._refuse_quantized("backward")
        B = X.shape[0]
        FD = self.F * self.D
        if self.tc:
            return self._tc_backward(X, sp, target, update)
        ext = getattr(self, "_external_gz", False)
        if ext:
            pass                          # top_gz[-1] was filled by backward_from_output_grad()
        elif self.has_head:
            self._head(B, target, True)   # p, loss, gz, dW/db of the last layer, gz of the layer below
        else:
            self.loss_and_grad(target, B)
        top_ld = [t.shape[1] for t in self.top_act]
        xin, ldx = self._top_in()
        bot_last_act = self._act("bot", len(self.ln_bot) - 2)
        if self.op == "dot":
            self.mlp_backward("top", xin, ldx, ACT_NONE, B, self.top_act, top_ld, self.top_gz, top_ld,
                              self.dR, self.ldr)
            if self.dT_route is not None:
                self._interact_bwd_routed(B, bot_last_act, None, None, 0, _stream())
            else:
                _lib.check(self.lib.dlrm_b200_interact_bwd(self.Tbuf.data_ptr(), FD, self.dR.data_ptr(), self.ldr,
                                                           self.dT.data_ptr(), FD, B, self.F, self.D,
                                                           int(self.itself), bot_last_act, _stream()),
                           "interact_bwd")
            self.n_launch += 1
        else:
            # cat: dR == dT; feature 0 additionally goes through the bottom MLP's last activation
            self.mlp_backward("top", xin, ldx, ACT_NONE, B, self.top_act, top_ld, self.top_gz, top_ld,
                              None, 0)
            K, N = self.ln_top[0], self.ln_top[1]
            s = _stream()
            Wp = self.W["top"][0].data_ptr()
            _lib.check(self.lib.dlrm_b200_linear_dgrad(self.top_gz[0].data_ptr(), top_ld[0], Wp, K,
                                                       self.Tbuf.data_ptr(), FD, bot_last_act,
                                                       self.dT.data_ptr(), FD, B, N, self.D, self.gemm, s),
                       "linear_dgrad")
            if self.T:
                _lib.check(self.lib.dlrm_b200_linear_dgrad(self.top_gz[0].data_ptr(), top_ld[0],
                                                           Wp + self.D * 4, K, None, 0, ACT_NONE,
                                                           self.dT.data_ptr() + self.D * 4, FD, B, N,
                                                           K - self.D, self.gemm, s), "linear_dgrad")
            self.n_launch += 2
        acts, lds = self._bot_outs(B)
        gz = list(self.bot_gz) + [self.dT]
        gz_ld = [t.shape[1] for t in self.bot_gz] + [FD]
        self.mlp_backward("bot", X, X.stride(0), ACT_NONE, B, acts, lds, gz, gz_ld, None, 0)

    def sync_update(self):
        """Make the current stream wait for an embedding update left running by
        train_step(join_update=False)."""
        self._join(self.s_emb)

    # ---- entry points used by the DLRM_Net facade (dlrm_b200/dlrm_net.py)
    def backward_from_output_grad(self, X: torch.Tensor, sp: SparseInput, gp: torch.Tensor):
        """Backward pass started from dE/dp computed OUTSIDE (autograd of the module's output).
        Leaves dense grads in dense_grad (slabs) and per-bag embedding grads in dT[:, 1:, :]."""
        self._refuse_quantized("backward")
        B = X.shape[0]
        nt = len(self.ln_top) - 1
        p = self.top_act[nt - 1]
        n = B * p.shape[1]
        _lib.check(self.lib.dlrm_b200_act_bwd(gp.data_ptr(), p.data_ptr(), self.top_gz[nt - 1].data_ptr(), n,
                                              self._act("top", nt - 1), self.loss_threshold, _stream()), "act_bwd")
        self.n_launch += 1
        self._external_gz = True
        try:
            self.backward(X, sp, None)
        finally:
            self._external_gz = False

    def reduced_dW(self, which: str, i: int) -> torch.Tensor:
        """Weight gradient of layer i with the split-K slabs folded (a new tensor)."""
        if not self.tc or i >= self.ntc[which]:
            return self.dW[which][i].clone()
        P, ns = self.dense_numel, self.tc_splits[(which, i)]
        o = self._dense_off[(which, i, "W")]
        n = self.dW[which][i].numel()
        return sum(self.dense_grad[s * P + o:s * P + o + n] for s in range(ns)).view_as(self.dW[which][i])

    def reduced_db(self, which: str, i: int) -> torch.Tensor:
        if not self.tc or i >= self.ntc[which]:
            return self.db[which][i].clone()
        P, ns = self.dense_numel, self.tc_splits[(which, i)]
        o = self._dense_off[(which, i, "b")]
        n = self.db[which][i].numel()
        return sum(self.dense_grad[s * P + o:s * P + o + n] for s in range(ns)).view_as(self.db[which][i])

    def mlp_only(self, which: str, x: torch.Tensor) -> torch.Tensor:
        """apply_mlp as a stand-alone call (fp32 CUDA-core kernels; no autograd)."""
        ln = self.ln_bot if which == "bot" else self.ln_top
        B = x.shape[0]
        outs = [torch.empty((B, ln[i + 1]), dtype=torch.float32, device=self.device) for i in range(len(ln) - 1)]
        self.mlp_forward(which, x, x.stride(0), B, outs, [o.shape[1] for o in outs])
        return outs[-1]

    def interact_only(self, B: int) -> torch.Tensor:
        """interact_features on the current contents of Tbuf[:B]; returns R [B, num_int]."""
        FD = self.F * self.D
        _lib.check(self.lib.dlrm_b200_interact_fwd(self.Tbuf.data_ptr(), FD, self.Rbuf.data_ptr(), self.ldr, B,
                                                   self.F, self.D, int(self.itself), _stream()), "interact_fwd")
        self.n_launch += 1
        return self.Rbuf[:B, :self.num_int]

    def dense_step(self, optimizer: str, lr: float, eps: float = 1e-10):
        if self.lr_dev is None:
            _lib.check(self.lib.dlrm_b200_dense_update(self.dense.data_ptr(), self.dense_grad.data_ptr(),
                                                       _ptr(self.dense_state), self.dense_numel, _OPT[optimizer],
                                                       lr, eps, _stream()), "dense_update")
        else:
            _lib.check(self.lib.dlrm_b200_dense_update_lr_dev(self.dense.data_ptr(), self.dense_grad.data_ptr(),
                                                              _ptr(self.dense_state), self.dense_numel,
                                                              _OPT[optimizer], lr, self.lr_dev.data_ptr(), eps,
                                                              _stream()), "dense_update_lr_dev")
        self.n_launch += 1

    def train_step(self, X: torch.Tensor, sp: SparseInput, target: torch.Tensor, lr: float,
                   optimizer: str = "rwsadagrad", lr_decay: float = 0.0, link_done: bool = False,
                   join_update: bool = True):
        """forward + loss + backward + optimizer.step().  Returns the loss (1-element device
        tensor, not synchronised).

        join_update=False (tensor-core path): the embedding update is left running on the embedding
        stream; the NEXT step's gather is ordered behind it on that stream, so the update of step i
        overlaps the bottom MLP of step i+1 (the dense optimizer does not depend on it).  The caller
        must then use a different batch buffer for the next step and call `sync_update()` before
        reading the tables from another stream."""
        self._refuse_quantized("train_step")
        self.ensure_optimizer_state(optimizer)
        self._join_update = bool(join_update) or not self.tc
        try:
            self.forward(X, sp, link=not link_done, skip_head=True)
            self.opt_step += 1
            clr = lr / (1.0 + (self.opt_step - 1.0) * lr_decay) if optimizer in _LR_DECAY else lr
            if self.tc:
                self.backward(X, sp, target, update=(optimizer, clr))
            else:
                self.backward(X, sp, target)
                if self.T:
                    self.emb_update(sp, optimizer=optimizer, lr=clr)
        except BaseException:
            self._abandon_staging()
            raise
        self.dense_apply(optimizer, clr)
        return self.loss_buf



    def dense_apply(self, optimizer: str, clr: float, eps: float = 1e-10):
        """Dense branch of optimizer.step() (+ the cross-rank mean of the gradients on a sharded run)."""
        if self.tc:
            if self.dense_sync_fn is not None:
                self._dense_update_pack(-2, 0.0)      # fold the split-K slabs into slab 0
                self._mark("dense_fold")
                self.dense_sync_fn()                  # cross-rank mean of the dense gradients
                self._mark("dense_allreduce")
                self._dense_update_pack(_OPT[optimizer], clr, eps, single_slab=True)
            else:
                self._dense_update_pack(_OPT[optimizer], clr, eps)
            self._mark("dense_update")
        else:
            if self.dense_sync_fn is not None:
                self.dense_sync_fn()
            self.dense_step(optimizer, clr, eps)

    def apply_optimizer(self, sp: SparseInput, optimizer: str, clr: float, eps: float = 1e-10, linked: bool = False):
        """optimizer.step() on the gradients the last backward() left in the engine's buffers: embedding rows
        (through the sharded exchange when there is one), then the dense parameters."""
        if self.T or self.update_fn is not None:
            try:
                if not linked and self.T:
                    self.emb_link(sp)
                if self.update_fn is not None:
                    self.update_fn(sp, optimizer, clr)
                else:
                    self.emb_update(sp, optimizer=optimizer, lr=clr, eps=eps)
            except BaseException:
                self._abandon_staging()
                raise
        self.dense_apply(optimizer, clr, eps)

    # ================================================================== wgmma path
    # Layers whose output width is >= 16 run on tensor cores (all bottom layers, the top layers
    # up to the final 256 -> 1 layer, which stays on the fp32 CUDA-core kernels).  Every fp32
    # activation / gradient / weight is kept as a (hi, lo) bf16 pair, activations carry a
    # constant-1 column and weights a bias column, so the bias add and the bias gradient come
    # out of the GEMMs themselves.
    def _interact_bwd_routed(self, B, bot_last_act, g0h, g0l, ldg0, stream):
        """interact_bwd whose per-feature gradient rows go straight to their (possibly remote) consumers."""
        dst, ld, first = self.dT_route
        _lib.check(self.lib.dlrm_b200_interact_bwd_p2p(self.Tbuf.data_ptr(), self.F * self.D, self.dR.data_ptr(),
                                                       self.ldr, dst, ld, first, float(self.emb_grad_scale), B, self.F,
                                                       self.D, int(self.itself),
                                                       bot_last_act, g0h, g0l, ldg0, stream),
                   "interact_bwd_p2p")

    def _mark(self, name: str):
        """Phase timeline: a timing event on the current stream (only while `_marks` is a list; never in a graph)."""
        if self._marks is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self._marks.append((name, ev))

    def _fork(self, side):
        """side stream starts after everything enqueued so far on the current stream."""
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        side.wait_event(ev)

    def _join(self, side):
        ev = torch.cuda.Event()
        ev.record(side)
        torch.cuda.current_stream().wait_event(ev)

    def _tc_n(self, which: str) -> int:
        ln = self.ln_bot if which == "bot" else self.ln_top
        n = 0
        for i in range(len(ln) - 1):
            if ln[i + 1] >= 16:
                n += 1
            else:
                break
        if which == "bot" and n != len(ln) - 1:
            return 0
        return n

    def _tc_keep(self):
        """Keep the current wgmma state (operand buffers, weight copies, plans) alive for its batch size: a captured
        CUDA graph runs on it, so a step at another batch size must not release it, and _tc_setup restores it when
        that batch size comes back."""
        self._tc_kept[self.tc_B] = (self.ntc, self.tc_in, self.tc_gz, self.tc_W, self.tc_plans, self.tc_splits,
                                    self._dense_off, self.dense_grad)

    def _tc_setup(self, B: int):
        kept = self._tc_kept.get(B)
        if kept is not None:
            if kept[7] is not self.dense_grad:
                raise RuntimeError("the weight-gradient arena was reallocated after a CUDA graph was captured at "
                                   "batch %d: prepare the largest batch before capturing" % B)
            (self.ntc, self.tc_in, self.tc_gz, self.tc_W, self.tc_plans, self.tc_splits,
             self._dense_off, _) = kept
            self.tc_B = B
            self._pack_dirty = True       # this state's weight copies missed the updates made at other batch sizes
            return
        dev, bf = self.device, torch.bfloat16
        # operand rows padded to 64 bf16 = 128 bytes: every row of a (hi, lo) operand then starts on a 128-byte line,
        # so a TMA box row (64 or 128 bytes) covers whole 32-byte sectors (an ld of 1032 put every other 64-byte row
        # across three sectors)
        r64 = lambda v: (v + 63) // 64 * 64
        self.tc_B = B
        self.ntc = {"bot": self._tc_n("bot"), "top": self._tc_n("top")}
        self.tc_in, self.tc_gz, self.tc_W = {}, {}, {}
        self.tc_plans = {"fwd": {}, "dgrad": {}, "wgrad": {}}
        x3 = self.tc_x3
        P = self.dense_numel
        # split-K factors asked of the weight-gradient plans (upper bounds: room for that many gradient slabs);
        # tc_splits, the slabs every reduction folds, is what each plan reports it writes
        want_splits, self.tc_splits = {}, {}
        smax = 1
        for which in ("bot", "top"):
            ln = self.ln_bot if which == "bot" else self.ln_top
            for i in range(self.ntc[which]):
                tiles = ((ln[i + 1] + 127) // 128) * ((ln[i] + 1 + 127) // 128)
                sk = max(1, min(8, (120 + tiles - 1) // tiles, (B + 63) // 64))
                want_splits[(which, i)] = sk
                smax = max(smax, sk)
        if self.dense_grad.numel() < smax * P:
            self.dense_grad = torch.zeros(smax * P, dtype=torch.float32, device=dev)
            self.dW, self.db = {"bot": [], "top": []}, {"bot": [], "top": []}
            for name, i, kind, o, shape in self.dense_slices:
                n = int(np.prod(shape))
                (self.dW if kind == "W" else self.db)[name].append(self.dense_grad[o:o + n].view(shape))
        self._dense_off = {}
        for name, i, kind, o, shape in self.dense_slices:
            self._dense_off[(name, i, kind)] = o
        for which in ("bot", "top"):
            ln = self.ln_bot if which == "bot" else self.ln_top
            ntc = self.ntc[which]
            ins, gzs, Ws = [], [], []
            for i in range(ntc):
                K, N = ln[i], ln[i + 1]
                Kp, Np = r64(K + 1), r64(N)
                h = torch.zeros((B, Kp), dtype=bf, device=dev)
                l = torch.zeros((B, Kp), dtype=bf, device=dev)
                h[:, K] = 1.0  # constant-1 column: bias folded into the GEMM
                ins.append((h, l, Kp))
                gzs.append((torch.zeros((B, Np), dtype=bf, device=dev), torch.zeros((B, Np), dtype=bf, device=dev), Np))
                Ws.append((torch.zeros((N, Kp), dtype=bf, device=dev), torch.zeros((N, Kp), dtype=bf, device=dev), Kp))
            self.tc_in[which], self.tc_gz[which], self.tc_W[which] = ins, gzs, Ws
        FD = self.F * self.D
        for which in ("bot", "top"):
            ln = self.ln_bot if which == "bot" else self.ln_top
            ntc = self.ntc[which]
            nl = len(ln) - 1
            for i in range(ntc):
                K, N = ln[i], ln[i + 1]
                ih, il, Kp = self.tc_in[which][i]
                wh, wl, _ = self.tc_W[which][i]
                gh, gl, Np = self.tc_gz[which][i]
                # ---- forward: Y = act(X W^T + b): bias added in fp32 in the epilogue (the constant-1 column of
                # the activations only serves the weight-gradient GEMM: a K of 512 stays 8 k-blocks, not 9)
                kw = dict(A_hi=ih.data_ptr(), A_lo=il.data_ptr(), lda=Kp, a_mn_major=0,
                          B_hi=wh.data_ptr(), B_lo=wl.data_ptr(), ldb=Kp, b_mn_major=0,
                          M=B, N=N, K=K, mode_x3=x3, split_k=1, act=self._act(which, i),
                          bias=self.b[which][i].data_ptr())
                if i + 1 < ntc:
                    oh, ol, Kp2 = self.tc_in[which][i + 1]
                    kw.update(out_hi=oh.data_ptr(), out_lo=ol.data_ptr(), ld_out=Kp2)
                if which == "bot" and i == nl - 1:
                    kw.update(out_f32=self.Tbuf.data_ptr(), ld_f32=FD)
                elif which == "top" and (i == ntc - 1):
                    kw.update(out_f32=self.top_act[i].data_ptr(), ld_f32=self.top_act[i].shape[1])
                self.tc_plans["fwd"][(which, i)] = _lib.GemmTcPlan(**kw)
                # ---- wgrad: [dW | db] = gz^T [X | 1]   (both operands read MN-major, split-K slabs)
                oW = self._dense_off[(which, i, "W")]
                ob = self._dense_off[(which, i, "b")]
                self.tc_plans["wgrad"][(which, i)] = _lib.GemmTcPlan(
                    A_hi=gh.data_ptr(), A_lo=gl.data_ptr(), lda=Np, a_mn_major=1,
                    B_hi=ih.data_ptr(), B_lo=il.data_ptr(), ldb=Kp, b_mn_major=1,
                    M=N, N=K + 1, K=B, mode_x3=x3, split_k=want_splits[(which, i)],
                    out_f32=self.dense_grad.data_ptr() + oW * 4, ld_f32=K, slab_stride=P,
                    out_col=self.dense_grad.data_ptr() + ob * 4, col_index=K, col_slab_stride=P)
                # a plan never launches an empty split: slabs past this count keep whatever an earlier step left
                self.tc_splits[(which, i)] = self.tc_plans["wgrad"][(which, i)].info()["splits"]
                # ---- dgrad: gz_prev = (gz W) * act'(input activation)
                if i > 0:
                    ph, pl, Np_prev = self.tc_gz[which][i - 1]
                    self.tc_plans["dgrad"][(which, i)] = _lib.GemmTcPlan(
                        A_hi=gh.data_ptr(), A_lo=gl.data_ptr(), lda=Np, a_mn_major=0,
                        B_hi=wh.data_ptr(), B_lo=wl.data_ptr(), ldb=Kp, b_mn_major=1,
                        M=B, N=K, K=N, mode_x3=x3, split_k=1,
                        mask_act=self._act(which, i - 1), mask_hi=ih.data_ptr(), mask_lo=il.data_ptr(), ldmask=Kp,
                        out_hi=ph.data_ptr(), out_lo=pl.data_ptr(), ld_out=Np_prev)
                elif which == "top" and self.op == "dot":
                    self.tc_plans["dgrad"][(which, 0)] = _lib.GemmTcPlan(
                        A_hi=gh.data_ptr(), A_lo=gl.data_ptr(), lda=Np, a_mn_major=0,
                        B_hi=wh.data_ptr(), B_lo=wl.data_ptr(), ldb=Kp, b_mn_major=1,
                        M=B, N=K, K=N, mode_x3=x3, split_k=1,
                        out_f32=self.dR.data_ptr(), ld_f32=self.ldr)
        self._pack_dirty = True

    def _split(self, x: torch.Tensor, ldx: int, M: int, N: int, hl):
        h, l, ld = hl
        _lib.check(self.lib.dlrm_b200_split_bf16(x.data_ptr(), ldx, M, N, h.data_ptr(), l.data_ptr(), ld,
                                                 _stream()), "split_bf16")
        self.n_launch += 1

    def _dense_update_pack(self, opt_code: int, lr: float, eps: float = 1e-10, single_slab: bool = False):
        """optimizer step on every dense layer + bf16 operand refresh; opt_code -1 = refresh only,
        -2 = only fold the split-K gradient slabs into slab 0."""
        layers = []
        P = self.dense_numel
        for which in ("bot", "top"):
            ln = self.ln_bot if which == "bot" else self.ln_top
            for i in range(len(ln) - 1):
                d = _lib.DenseLayer()
                oW, ob = self._dense_off[(which, i, "W")], self._dense_off[(which, i, "b")]
                d.W = self.dense.data_ptr() + oW * 4
                d.b = self.dense.data_ptr() + ob * 4
                if self.dense_state is not None:
                    d.sW = self.dense_state.data_ptr() + oW * 4
                    d.sb = self.dense_state.data_ptr() + ob * 4
                d.dW = self.dense_grad.data_ptr() + oW * 4
                d.db = self.dense_grad.data_ptr() + ob * 4
                d.slab_stride = P
                d.N, d.K = ln[i + 1], ln[i]
                if i < self.ntc[which]:
                    wh, wl, Kp = self.tc_W[which][i]
                    d.pack_hi, d.pack_lo, d.ld_pack = wh.data_ptr(), wl.data_ptr(), Kp
                    d.num_slabs = self.tc_splits[(which, i)] if (opt_code >= 0 or opt_code == -2) and not single_slab else 1
                else:
                    d.num_slabs = 1
                layers.append(d)
        for c0 in range(0, len(layers), 16):
            chunk = layers[c0:c0 + 16]
            arr = (_lib.DenseLayer * len(chunk))(*chunk)
            if self.lr_dev is None or opt_code < 0:
                _lib.check(self.lib.dlrm_b200_dense_update_pack(arr, len(chunk), opt_code, lr, eps, _stream()),
                           "dense_update_pack")
            else:
                _lib.check(self.lib.dlrm_b200_dense_update_pack_lr_dev(arr, len(chunk), opt_code, lr,
                                                                       self.lr_dev.data_ptr(), eps, _stream()),
                           "dense_update_pack_lr_dev")
            self.n_launch += 1

    def _tc_prepare(self, B: int):
        if self.tc_B != B:
            self._tc_setup(B)
        if self._pack_dirty:
            self._dense_update_pack(-1, 0.0)
            self._pack_dirty = False

    def _tc_mlp_forward(self, which: str, B: int, skip_head: bool = False):
        ln = self.ln_bot if which == "bot" else self.ln_top
        s = _stream()
        ntc = self.ntc[which]
        for i in range(ntc):
            self.tc_plans["fwd"][(which, i)].run(s)
            self.n_launch += 1
        nl = len(ln) - 1
        if which == "top" and self.has_head:
            nl -= 1
            if not skip_head:
                self._head(B, None, False)
        # fp32 CUDA-core suffix (layers narrower than 16 outputs)
        for i in range(ntc, nl):
            K, N = ln[i], ln[i + 1]
            x = self.top_act[i - 1]
            _lib.check(self.lib.dlrm_b200_linear_fwd(x.data_ptr(), x.shape[1], self.W[which][i].data_ptr(), K,
                                                     self.b[which][i].data_ptr(), self.top_act[i].data_ptr(),
                                                     self.top_act[i].shape[1], B, N, K, self._act(which, i),
                                                     GEMM_SIMT_FP32, s), "linear_fwd")
            self.n_launch += 1

    def _tc_forward(self, X: torch.Tensor, sp: SparseInput, link: bool = False, skip_head: bool = False) -> torch.Tensor:
        B = X.shape[0]
        self._tc_prepare(B)
        if self.ntc["bot"] == 0 or self.ntc["top"] == 0 or self.op != "dot":
            raise RuntimeError("gemm='tc' needs op='dot' and MLP layers of width >= 16; use gemm='simt'")
        FD = self.F * self.D
        gather = self.T > 0 or self.gather_fn is not None
        self._mark("begin")
        if gather:   # gather (+ link) beside the bottom MLP
            self._fork(self.s_emb)
            with torch.cuda.stream(self.s_emb):
                if self.gather_fn is not None:
                    self.gather_fn(sp, link)
                else:
                    self.emb_forward(sp, link=link)
                    self._mark("emb:gather")
                    self.reduce_partials(B)
                    self._mark("emb:reduce_partials")
        self._split(X, X.stride(0), B, self.ln_bot[0], self.tc_in["bot"][0])
        self._tc_mlp_forward("bot", B)
        self._mark("bot_fwd")
        if gather:
            self._join(self.s_emb)
            self._mark("join_gather")
        rh, rl, ldrb = self.tc_in["top"][0]
        if self.D % 4 == 0:
            # R goes straight to the (hi, lo) operand pair of the first top-MLP GEMM
            _lib.check(self.lib.dlrm_b200_interact_fwd_ex(self.Tbuf.data_ptr(), FD, None, self.ldr, rh.data_ptr(),
                                                          rl.data_ptr(), ldrb, B, self.F, self.D, int(self.itself),
                                                          _stream()), "interact_fwd_ex")
            self.n_launch += 1
        else:
            _lib.check(self.lib.dlrm_b200_interact_fwd(self.Tbuf.data_ptr(), FD, self.Rbuf.data_ptr(), self.ldr, B,
                                                       self.F, self.D, int(self.itself), _stream()), "interact_fwd")
            self.n_launch += 1
            self._split(self.Rbuf, self.ldr, B, self.num_int, self.tc_in["top"][0])
        self._mark("interact_fwd")
        self._tc_mlp_forward("top", B, skip_head)
        self._mark("top_fwd")
        p = self.top_act[-1][:B]
        if 0.0 < self.loss_threshold < 1.0:
            return torch.clamp(p, self.loss_threshold, 1.0 - self.loss_threshold)
        return p

    def _tc_mlp_backward(self, which: str, B: int):
        """gz of the last tensor-core layer is ready on the current stream.  The dgrads stay on this stream (the
        critical chain); every wgrad only feeds the final dense update and goes to the side stream."""
        for i in reversed(range(self.ntc[which])):
            self._fork(self.s_wg)   # gz_i was produced by the previous launch on this stream
            with torch.cuda.stream(self.s_wg):
                self.tc_plans["wgrad"][(which, i)].run(_stream())
            self.n_launch += 1
            pl = self.tc_plans["dgrad"].get((which, i))
            if pl is not None:
                pl.run(_stream())
                self.n_launch += 1

    def _tc_backward(self, X: torch.Tensor, sp: SparseInput, target: torch.Tensor, update=None):
        B = X.shape[0]
        FD = self.F * self.D
        s = _stream()
        nt, ntc = len(self.ln_top) - 1, self.ntc["top"]
        top_ld = [t.shape[1] for t in self.top_act]
        head_to_tc = False
        if getattr(self, "_external_gz", False):
            pass                          # top_gz[nt-1] given; the fp32 suffix below handles layer nt-1
        elif self.has_head:
            self._head(B, target, True)
            head_to_tc = (nt - 2) < ntc   # head wrote the bf16 gradient pair of layer nt-2 directly
            nt -= 1
        else:
            self.loss_and_grad(target, B)
        # fp32 suffix of the top MLP
        for i in reversed(range(ntc, nt)):
            K, N = self.ln_top[i], self.ln_top[i + 1]
            xin = self.top_act[i - 1]
            _lib.check(self.lib.dlrm_b200_linear_wgrad(self.top_gz[i].data_ptr(), top_ld[i], xin.data_ptr(),
                                                       xin.shape[1], self.dW["top"][i].data_ptr(), K,
                                                       self.db["top"][i].data_ptr(), B, N, K, GEMM_SIMT_FP32, s),
                       "linear_wgrad")
            _lib.check(self.lib.dlrm_b200_linear_dgrad(self.top_gz[i].data_ptr(), top_ld[i],
                                                       self.W["top"][i].data_ptr(), K, xin.data_ptr(),
                                                       xin.shape[1], self._act("top", i - 1),
                                                       self.top_gz[i - 1].data_ptr(), top_ld[i - 1], B, N, K,
                                                       GEMM_SIMT_FP32, s), "linear_dgrad")
            self.n_launch += 3
        if not head_to_tc:
            self._split(self.top_gz[ntc - 1], top_ld[ntc - 1], B, self.ln_top[ntc], self.tc_gz["top"][ntc - 1])
        self._mark("head+loss")
        self._tc_mlp_backward("top", B)
        self._mark("top_bwd_dgrad")
        bot_last_act = self._act("bot", len(self.ln_bot) - 2)
        g0h, g0l, ldg0 = self.tc_gz["bot"][-1]
        if self.dT_route is not None:
            self._interact_bwd_routed(B, bot_last_act, g0h.data_ptr(), g0l.data_ptr(), ldg0, s)
        else:
            _lib.check(self.lib.dlrm_b200_interact_bwd_ex(self.Tbuf.data_ptr(), FD, self.dR.data_ptr(), self.ldr,
                                                          self.dT.data_ptr(), FD, B, self.F, self.D,
                                                          int(self.itself), bot_last_act, g0h.data_ptr(),
                                                          g0l.data_ptr(), ldg0, s),
                       "interact_bwd_ex")
        self.n_launch += 1
        self._mark("interact_bwd")
        has_emb = self.T > 0 or self.update_fn is not None
        if update is not None and has_emb:
            # fused coalesce + sparse optimizer beside the bottom-MLP backward
            opt, clr = update
            upd = (lambda: self.update_fn(sp, opt, clr)) if self.update_fn is not None else \
                (lambda: self.emb_update(sp, optimizer=opt, lr=clr))
            self._fork(self.s_emb)
            with torch.cuda.stream(self.s_emb):
                upd()
                self._mark("emb:update")
        self._tc_mlp_backward("bot", B)
        self._mark("bot_bwd_dgrad")
        self._join(self.s_wg)
        self._mark("join_wgrads")
        if update is not None and has_emb and getattr(self, "_join_update", True):
            self._join(self.s_emb)
            self._mark("join_update")


def _unpin(lib, tensors):
    """Unregister the pinned host arenas of a collected engine (after its last staging copy)."""
    with contextlib.suppress(Exception):
        torch.cuda.synchronize()
    for t in tensors:
        with contextlib.suppress(Exception):
            lib.dlrm_b200_host_unregister(t.data_ptr())


def _refuse_graphed_f16(eng: "Engine"):
    # The stochastic-rounding key of an fp16 table depends on the optimizer step and travels in the update's launch
    # parameters: a replayed graph would round every step with the bits of the captured one.
    if eng.f16:
        raise RuntimeError("fp16 embedding tables train with eager steps: a captured training step would replay one "
                           "step's stochastic-rounding bits on every replay")


class GraphedTrainSteps:
    """K consecutive training steps over K static batch buffers in ONE CUDA graph.  Inside the graph
    the embedding update of step j overlaps the bottom MLP of step j+1 (train_step(join_update=False));
    only the last update is joined.  `losses[j]` holds the loss of step j after a replay."""

    def __init__(self, eng: "Engine", stages, lr: float, optimizer: str = "rwsadagrad", warmup: int = 2):
        _refuse_graphed_f16(eng)
        self.eng, self.stages, self.lr, self.optimizer = eng, list(stages), lr, optimizer
        self.K = len(self.stages)
        eng.ensure_optimizer_state(optimizer)
        self.losses = torch.zeros(self.K, dtype=torch.float32, device=eng.device)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(warmup, 1)):
                self._eager()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        n0 = eng.n_launch
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._eager()
        self.kernels_per_replay = eng.n_launch - n0

    def _eager(self):
        for j, st in enumerate(self.stages):
            loss = self.eng.train_step(st.X, st.sparse, st.target, self.lr, self.optimizer,
                                       join_update=(j == self.K - 1))
            self.losses[j:j + 1].copy_(loss)
        return self.losses

    def replay(self):
        self.graph.replay()
        self.eng.n_launch += self.kernels_per_replay
        self.eng.opt_step += self.K
        self.eng._cache_dirty = bool(self.eng.cache_rows)      # the steps may have inserted into the row cache
        return self.losses


class GraphedTrainStep:
    """One training step (forward, loss, backward, fused embedding + dense optimizer) captured
    into a CUDA graph over a static packed device batch: per step the host issues one H2D (or D2D)
    copy of the packed inputs and one graph launch instead of ~35 kernel launches.  By default the
    learning rate is baked into the graph (re-capture to change it).  device_lr=True: the optimizer
    kernels read it from the engine's device scalar `eng.lr_scalar`, which replay(lr, lr_decay) sets
    before every launch, so a schedule can change it from step to step.

    The engine may run eager steps at other batch sizes between replays: the wgmma state the graph
    runs on is kept (Engine._tc_keep) and restored before the next replay.  Buffers that only grow
    (activations, occurrence lists, staging arena, scratch) must already have their final size when
    the graph is captured: prepare the largest batch first."""

    def __init__(self, eng: "Engine", stage, lr: float, optimizer: str = "rwsadagrad", warmup: int = 3,
                 train: bool = True, X: Optional[torch.Tensor] = None, target: Optional[torch.Tensor] = None,
                 pre=None, device_lr: bool = False):
        """pre: optional callable run (and captured) before the step, e.g. the index exchange of a sharded run."""
        if train:
            _refuse_graphed_f16(eng)
        self.eng, self.stage, self.train, self.pre = eng, stage, train, pre
        # table-wise sharded runs: the dense slice / targets are separate static tensors
        self.X = X if X is not None else stage.X
        self.target = target if target is not None else stage.target
        self.B = self.X.shape[0]
        self.lr, self.optimizer, self.device_lr = lr, optimizer, bool(device_lr)
        if train or not eng.quant_bits:
            eng.ensure_optimizer_state(optimizer)
        if self.device_lr and eng.lr_scalar is None:
            eng.lr_scalar = torch.zeros(1, dtype=torch.float32, device=eng.device)
        if warmup > 0:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(warmup):   # allocates every lazily-created buffer / plan outside capture
                    self._eager()
            torch.cuda.current_stream().wait_stream(side)
        else:
            eng.prepare(stage.sparse, train, batch=self.X.shape[0])  # allocate lazily-created buffers
        torch.cuda.synchronize()
        n0, step0 = eng.n_launch, eng.opt_step
        self.graph = torch.cuda.CUDAGraph()
        if self.device_lr:
            eng.lr_dev = eng.lr_scalar
        try:
            with torch.cuda.graph(self.graph):
                self.out = self._eager()
        finally:
            eng.lr_dev = None
        if self.device_lr:
            eng.opt_step = step0        # the capture did not run a step: replay() counts them
        self.kernels_per_replay = eng.n_launch - n0
        if eng.tc:
            eng._tc_keep()

    def _eager(self):
        st = self.stage
        if self.pre is not None:
            self.pre()
        if self.train:
            return self.eng.train_step(self.X, st.sparse, self.target, self.lr, self.optimizer)
        return self.eng.forward(self.X, st.sparse)

    def replay(self, lr: Optional[float] = None, lr_decay: float = 0.0):
        """lr, lr_decay (device_lr graphs): the step's learning rate is computed as train_step computes it, at the
        step this replay runs (clr = lr / (1 + (step - 1) lr_decay) for rwsadagrad and adagrad, else lr); lr=None
        takes the lr given at capture."""
        eng = self.eng
        if eng.tc and eng.tc_B != self.B:
            eng._tc_prepare(self.B)      # an eager step at another batch size ran since the last replay
        if self.device_lr and self.train:
            lr = self.lr if lr is None else lr
            step = eng.opt_step + 1
            clr = lr / (1.0 + (step - 1.0) * lr_decay) if self.optimizer in _LR_DECAY else lr
            eng.lr_scalar.fill_(clr)
        elif lr is not None or lr_decay:
            raise ValueError("this graph's learning rate is baked in (capture with device_lr=True to set it per replay)")
        self.graph.replay()
        eng.n_launch += self.kernels_per_replay
        if self.train:
            eng.opt_step += 1
            eng._cache_dirty = bool(eng.cache_rows)
        return self.out


def sparse_from_reference(lS_o, lS_i, device) -> SparseInput:
    """lS_o: [T,B] tensor or list; lS_i: list of 1-D tensors or stacked 2-D tensor
    (dlrm_s_pytorch.py:129-145 conventions).  Moves to `device` if needed (no dtype change)."""
    if isinstance(lS_i, torch.Tensor):
        lS_i = [lS_i[k] for k in range(lS_i.shape[0])]
    if isinstance(lS_o, torch.Tensor):
        lS_o = [lS_o[k] for k in range(lS_o.shape[0])]
    idx = [t.to(device).contiguous() for t in lS_i]
    off = [t.to(device).contiguous() for t in lS_o]
    B = int(off[0].numel()) if off else 0
    if idx and off and idx[0].dtype != off[0].dtype:
        raise RuntimeError("indices and offsets must have the same dtype (int64 or int32)")
    return SparseInput(idx, off, B, False)
