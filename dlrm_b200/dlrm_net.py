"""`DLRM_Net` -- the reference's module surface (dlrm_s_pytorch.py:207-730) over the H100 engine.

Call-compatible with the reference for the hot path (SURVEY.md §8 b1):
  * constructor keyword signature of `dlrm_s_pytorch.py:296-317` (no-arg construction allowed);
  * methods `create_mlp`, `create_emb`, `apply_mlp`, `apply_emb`, `interact_features`, `forward`,
    `sequential_forward` with the reference's argument meaning;
  * attributes `emb_l`, `v_W_l`, `bot_l`, `top_l`, `ndevices`, `loss_fn`, `loss_threshold`, ...;
  * `parameters()` order (tables, bottom MLP, top MLP) and `state_dict()` keys
    `emb_l.{k}.weight`, `bot_l.{2i}.{weight,bias}`, `top_l.{2i}.{weight,bias}` -- reference
    checkpoints load with `load_state_dict`;
  * errors for unsupported options are `sys.exit("ERROR: ...")` strings, as in the reference.

Parameters are VIEWS into the engine's HBM arenas (one table arena, one dense arena), so the kernels,
`state_dict()` and any torch optimizer see the same memory.  `E.backward()` works: the whole forward is
one autograd node whose backward runs the engine's backward kernels.  Embedding gradients are either
  - handed to a fused optimizer of `dlrm_b200.optim` (no [nnz, D] gradient is ever materialised), or
  - materialised as the reference's uncoalesced sparse COO tensors (`emb_l[k].weight.grad`) so an
    unmodified `torch.optim.SGD` keeps working (compatibility mode, slower; fp32 tables only).
`emb_dtype=torch.float16` stores the tables as fp16 (`emb_l[k].weight` is an fp16 strided parameter): lookups widen
the rows to fp32, the fused optimizers update them in fp32 and store them with stochastic rounding.  `state_dict()`
then holds fp16 tables; an fp32 checkpoint loads with round-to-nearest, an fp16 one into an fp32 model exactly.
`emb_host_tables="auto" | [k, ...]` keeps those tables in pinned host memory (dlrm_b200/host_tables.py): their
`emb_l[k].weight` are CPU tensors, so `state_dict()` / `load_state_dict()` and checkpoints are unchanged, and every step
stages the rows the batch touches through HBM.  "auto" moves the largest tables until the rest fits in free device
memory.  `emb_host_cache=N | "auto"` also keeps up to N of their rows in HBM between steps (a 32-way set-associative
cache, least recently used way replaced; "auto": the device memory free at the first batch beyond `host_reserve`).
A cached row's host copy is then stale: `emb_l[k].weight` of a host table shows the current rows only after
`state_dict()`, `load_state_dict()`, `engine.table(k)` or the optimizer's `state_dict()`, which write the cache back
(and empty it).  A training loop that calls none of them never writes it back.  QR / mixed-dimension embeddings and `parallel_forward` are outside the path
(SURVEY §2) and exit with an error when requested.
Row-wise quantized tables (inference only): `quantize_embedding(bits)` packs the float tables into fbgemm's 8- or 4-bit
rows, `emb_l_q[k]`, and the forward pools those from then on (the float tables stay).  `emb_dtype="int8" | "int4"` builds
a model whose float tables are never allocated: the initial draw and `load_state_dict` quantize each table as it is
written, and `state_dict()` is refused.  Either way the pooled rows are bit-identical to the reference's CPU ops.
"""
from __future__ import annotations

import sys
from typing import List, Optional

import numpy as np
import torch
import torch.nn as nn

from .engine import Engine, SparseInput, sparse_from_reference

# Above this many table elements the reference's numpy initialisation (one np.random.uniform call per
# table, 150 s for 26 x 1e6 x 128) is replaced by the same distribution drawn on the device.
_NUMPY_INIT_MAX = 50_000_000


def _uniform_(tab: torch.Tensor, a: float, gen):
    """U(-a, a) drawn in fp32 on the device (fp16 tables: that draw rounded to nearest)."""
    if tab.dtype == torch.float32:
        tab.uniform_(-a, a, generator=gen)
    else:
        tab.copy_(torch.empty(tab.shape, dtype=torch.float32, device=tab.device).uniform_(-a, a, generator=gen))


class _TableView(nn.Module):
    """Stands in for nn.EmbeddingBag(n, m, mode="sum", sparse=True): holds `.weight`."""

    def __init__(self, weight: torch.Tensor):
        super().__init__()
        self.weight = nn.Parameter(weight, requires_grad=True)
        self.num_embeddings, self.embedding_dim = weight.shape
        self.mode, self.sparse = "sum", True

    def extra_repr(self):
        return "%d, %d, mode=sum (dlrm_b200 arena view)" % (self.num_embeddings, self.embedding_dim)


class _LinearView(nn.Module):
    """Stands in for nn.Linear: `.weight` [out, in] and `.bias` [out] are views of the dense arena."""

    def __init__(self, weight: torch.Tensor, bias: torch.Tensor):
        super().__init__()
        self.weight = nn.Parameter(weight, requires_grad=True)
        self.bias = nn.Parameter(bias, requires_grad=True)
        self.out_features, self.in_features = weight.shape

    def extra_repr(self):
        return "in_features=%d, out_features=%d (dlrm_b200 arena view)" % (self.in_features, self.out_features)


class _DLRMForward(torch.autograd.Function):
    """sequential_forward as one autograd node (inputs: dense_x and every parameter)."""

    @staticmethod
    def forward(ctx, net, sp, train, dense_x, *params):
        eng = net._engine
        # The per-row occurrence lists of the sort-free coalesce (head[] / link[]) are built by
        # optimizer.step() itself, never here: a grad-enabled forward that is NOT followed by a step (the
        # reference's inference() loop, a skipped step, two forwards before one backward) would otherwise
        # leave stale list heads behind for the next update to follow.
        linked = False
        p = eng.forward(dense_x, sp, link=linked)
        ctx.net, ctx.sp, ctx.x, ctx.nparams, ctx.linked = net, sp, dense_x, len(params), linked
        return p.clone()

    @staticmethod
    def backward(ctx, gp):
        net, eng = ctx.net, ctx.net._engine
        eng.backward_from_output_grad(ctx.x, ctx.sp, gp.contiguous())
        grads: List[Optional[torch.Tensor]] = []
        if net._fused_opt is None and eng.host:
            raise RuntimeError("dlrm_b200: host embedding tables are trained by the fused optimizers of "
                               "dlrm_b200.optim (SGD, RWSAdagrad, Adagrad); create one before calling backward()")
        if net._fused_opt is None and net.weighted_pooling == "learned":
            raise RuntimeError("dlrm_b200: learned weighted pooling (v_W_l) is trained by the fused optimizers of "
                               "dlrm_b200.optim (SGD, RWSAdagrad, Adagrad); create one before calling backward()")
        if net._fused_opt is None and eng.f16:
            raise RuntimeError("dlrm_b200: fp16 embedding tables are trained by the fused optimizers of "
                               "dlrm_b200.optim (SGD, RWSAdagrad); create one before calling backward()")
        if net._fused_opt is not None:
            if net._pending is not None:
                raise RuntimeError("dlrm_b200: backward() called twice before optimizer.step(): gradient "
                                   "accumulation is not supported by the fused optimizers (the second "
                                   "micro-batch would overwrite the first)")
            net._pending = (ctx.sp, ctx.linked)          # consumed by the fused optimizer's step()
            return (None, None, None, None) + (None,) * ctx.nparams
        grads += net._materialise_sparse_grads(ctx.sp)
        for name in ("bot", "top"):
            for i in range(len(eng.W[name])):
                grads.append(eng.reduced_dW(name, i))
                grads.append(eng.reduced_db(name, i))
        return (None, None, None, None) + tuple(grads)


class DLRM_Net(nn.Module):
    def __init__(self, m_spa=None, ln_emb=None, ln_bot=None, ln_top=None, arch_interaction_op=None,
                 arch_interaction_itself=False, sigmoid_bot=-1, sigmoid_top=-1, sync_dense_params=True,
                 loss_threshold=0.0, ndevices=-1, qr_flag=False, qr_operation="mult", qr_collisions=0,
                 qr_threshold=200, md_flag=False, md_threshold=200, weighted_pooling=None,
                 loss_function="bce", *, device=None, gemm="tc", max_batch=2048, loss_weights=None,
                 emb_dtype=torch.float32, round_seed=0, emb_host_tables=None, emb_host_cache=None):
        super().__init__()
        self._engine: Optional[Engine] = None
        self._fused_opt = None
        self._pending = None
        if (m_spa is None or ln_emb is None or ln_bot is None or ln_top is None
                or arch_interaction_op is None):
            return  # reference allows an empty shell (dlrm_s_pytorch.py:320-326)
        if emb_dtype in (torch.float16, "fp16", "float16"):
            emb_dtype = "fp16"
        elif emb_dtype in (torch.float32, "fp32", "float32"):
            emb_dtype = "fp32"
        elif emb_dtype not in ("int8", "int4"):
            sys.exit("ERROR: emb_dtype must be torch.float32, torch.float16, \"int8\" or \"int4\"")
        if emb_dtype == "fp16" and int(m_spa) % 8:
            sys.exit("ERROR: fp16 embedding tables need an embedding dimension divisible by 8")
        if emb_dtype in ("int8", "int4"):
            if int(m_spa) % (4 if emb_dtype == "int8" else 8):
                sys.exit("ERROR: %s row-wise quantized tables need an embedding dimension divisible by %d"
                         % (emb_dtype, 4 if emb_dtype == "int8" else 8))
            if emb_host_tables:
                sys.exit("ERROR: quantized embedding tables are kept in device memory (emb_host_tables is not supported)")
        if qr_flag or md_flag:
            sys.exit("ERROR: --qr-flag / --md-flag embeddings are outside the dlrm_b200 hot path")
        if arch_interaction_op not in ("dot", "cat"):
            sys.exit("ERROR: --arch-interaction-op=" + str(arch_interaction_op) + " is not supported")
        if loss_function not in ("mse", "bce", "wbce"):
            sys.exit("ERROR: --loss-function=" + loss_function + " is not supported")
        self.ndevices = ndevices
        self.output_d = 0
        self.arch_interaction_op = arch_interaction_op
        self.arch_interaction_itself = arch_interaction_itself
        self.sync_dense_params = sync_dense_params
        self.loss_threshold = loss_threshold
        self.loss_function = loss_function
        self.weighted_pooling = ("learned" if weighted_pooling is not None and weighted_pooling != "fixed"
                                 else weighted_pooling)
        self.qr_flag, self.md_flag = False, False
        self.quantize_emb, self.emb_l_q, self.quantize_bits = False, [], 32
        self._quant_only = emb_dtype in ("int8", "int4")
        ln_emb = np.asarray(ln_emb).astype(np.int64)
        ln_bot = np.asarray(ln_bot).astype(np.int64)
        ln_top = np.asarray(ln_top).astype(np.int64)
        if device is None:
            device = "cuda:%d" % torch.cuda.current_device() if torch.cuda.is_available() else "cuda:0"
        widths_ok = all(int(v) >= 16 for v in ln_bot[1:]) and int(ln_top[1]) >= 16 if len(ln_top) > 1 else False
        if gemm != "simt" and (arch_interaction_op != "dot" or not widths_ok):
            gemm = "simt"  # tiny / cat architectures: fp32 CUDA-core kernels (still device code)
        loss_ws = None
        if loss_function == "wbce":
            loss_ws = loss_weights if loss_weights is not None else [1.0, 1.0]
            self.loss_ws = torch.tensor(np.asarray(loss_ws, dtype=float))
        self._dist = None
        import torch.distributed as tdist

        host = []
        if emb_host_tables:
            if emb_dtype == "fp16":
                sys.exit("ERROR: host embedding tables need fp32 rows (the stochastic rounding of fp16 tables is keyed "
                         "by the row index the update kernel sees)")
            if weighted_pooling is not None:
                sys.exit("ERROR: host embedding tables do not support weighted pooling (row weights are indexed by "
                         "table row)")
            if tdist.is_available() and tdist.is_initialized() and tdist.get_world_size() > 1:
                sys.exit("ERROR: host embedding tables are not supported on sharded runs")
            if emb_host_tables == "auto":
                from .host_tables import auto_host_tables

                free, _ = torch.cuda.mem_get_info(torch.device(device) if device is not None else None)
                try:
                    host = auto_host_tables(ln_emb.tolist(), 4 * int(m_spa) + 8, free, self.host_reserve(m_spa, ln_emb))
                except ValueError as e:
                    sys.exit("ERROR: " + str(e))
            else:
                host = sorted(set(int(k) for k in emb_host_tables))
        if emb_host_cache and not host:
            sys.exit("ERROR: a host row cache (emb_host_cache) needs host embedding tables (emb_host_tables)")

        if self._quant_only and tdist.is_available() and tdist.is_initialized() and tdist.get_world_size() > 1:
            sys.exit("ERROR: quantized embedding tables are not supported on sharded runs")
        if tdist.is_available() and tdist.is_initialized() and tdist.get_world_size() > 1:
            # one process per GPU (the reference: ext_dist.my_size > 1, dlrm_s_pytorch.py:352-365): tables are
            # placed over the ranks (dlrm_b200/placement.py), the MLPs replicated; max_batch is the GLOBAL batch
            from .dist import DistEngine

            world = tdist.get_world_size()
            if gemm == "simt":
                sys.exit("ERROR: distributed runs use the tensor-core path (MLP widths >= 16, dot interaction)")
            if max_batch % world:
                sys.exit("ERROR: batch_size %d can not split across %d ranks evenly" % (max_batch, world))
            self._dist = DistEngine(int(m_spa), ln_emb.tolist(), ln_bot.tolist(), ln_top.tolist(),
                                    local_batch=max_batch // world, device=device, gemm=gemm, loss=loss_function,
                                    exchange="p2p", itself=arch_interaction_itself, sigmoid_bot=sigmoid_bot,
                                    loss_threshold=loss_threshold, loss_ws=loss_ws, emb_dtype=emb_dtype,
                                    round_seed=round_seed)
            self._engine = self._dist.eng
            self.local_shards = list(self._dist.mine)
        else:
            self._engine = Engine(int(m_spa), ln_emb.tolist(), ln_bot.tolist(), ln_top.tolist(),
                                  op=arch_interaction_op, itself=arch_interaction_itself,
                                  sigmoid_bot=sigmoid_bot, sigmoid_top=sigmoid_top, loss=loss_function,
                                  loss_threshold=loss_threshold, loss_ws=loss_ws, device=device,
                                  max_batch=max_batch, gemm=gemm, emb_dtype=emb_dtype, round_seed=round_seed,
                                  interleave_momentum=None if emb_dtype == "fp16" else False, host_tables=host,
                                  host_cache_rows=emb_host_cache or 0,
                                  host_cache_reserve=self.host_reserve(m_spa, ln_emb),
                                  learned_row_weights=self.weighted_pooling == "learned")
        self._m_spa, self._ln_emb = int(m_spa), ln_emb
        # same construction (and numpy RNG consumption) order as the reference: tables, bottom, top
        if ndevices <= 1:
            self.emb_l, w_list = self.create_emb(m_spa, ln_emb, weighted_pooling)
            self.v_W_l = w_list
        if self._quant_only:
            self.quantize_emb, self.quantize_bits = True, self._engine.quant_bits
            self.emb_l_q = [self._engine.table_q(k) for k in range(self._engine.T)]
        self.bot_l = self.create_mlp(ln_bot, sigmoid_bot)
        self.top_l = self.create_mlp(ln_top, sigmoid_top)
        if loss_function == "mse":
            self.loss_fn = torch.nn.MSELoss(reduction="mean")
        elif loss_function == "bce":
            self.loss_fn = torch.nn.BCELoss(reduction="mean")
        else:
            self.loss_fn = torch.nn.BCELoss(reduction="none")
        if self._dist is not None:
            self._dist.sync_dense_params_from_rank0()    # DDP broadcasts rank 0's MLPs at wrap time (:1329-1336)
        self.register_load_state_dict_post_hook(lambda m, k: m._engine.mark_params_changed())
        import weakref

        ref = weakref.ref(self)
        for p in self.parameters():
            p._dlrm_net = ref

    @staticmethod
    def host_reserve(m_spa, ln_emb) -> int:
        """Device bytes "auto" keeps free beside the tables: 2 GiB of activations and workspace, plus the largest table
        once, which a large table's initial draw uses on the device before it is copied to host memory."""
        big = int(np.sum(ln_emb)) * int(m_spa) > _NUMPY_INIT_MAX
        return (1 << 31) + (int(np.max(ln_emb)) * int(m_spa) * 4 if big else 0)

    def state_dict(self, *args, **kwargs):
        if self._engine is not None and self._engine.quant_only:
            raise RuntimeError("dlrm_b200: this model was built with emb_dtype=%r: its float embedding tables were never "
                               "stored, so there is no state_dict (emb_l_q[k] holds the packed rows)"
                               % self._engine.emb_dtype)
        if self._engine is not None and self._engine.host:
            self._engine._host_sync()       # host rows may still be on their way back from the last step
        return super().state_dict(*args, **kwargs)

    def load_state_dict(self, state_dict, *args, **kwargs):
        eng = self._engine
        if eng is not None and eng.quant_only:
            # the reference's emb_l.{k}.weight (fp32 or fp16, on any device, e.g. an mmap load) is quantized table by
            # table, QUANT_CHUNK_ROWS rows at a time; the rest loads as usual
            state_dict = dict(state_dict)
            for k in range(eng.T):
                w = state_dict.pop("emb_l.%d.weight" % k, None)
                if w is None:
                    if kwargs.get("strict", args[0] if args else True):
                        raise RuntimeError("dlrm_b200: load_state_dict: missing key emb_l.%d.weight" % k)
                    continue
                if tuple(w.shape) != (eng.ln_emb[k], eng.D):
                    raise RuntimeError("dlrm_b200: load_state_dict: emb_l.%d.weight has shape %s, the model's table is "
                                       "[%d, %d]" % (k, tuple(w.shape), eng.ln_emb[k], eng.D))
                eng.quantize_rows(k, w.detach())
        if eng is not None and eng.host:
            eng._host_sync()
        out = super().load_state_dict(state_dict, *args, **kwargs)
        if eng is not None and self.quantize_emb and not eng.quant_only:
            for k in range(eng.T):          # quantize_embedding() was called: the packed rows follow the new tables
                eng.quantize_rows(k, eng.table(k))
        return out

    # ------------------------------------------------------------------ construction
    def create_mlp(self, ln, sigmoid_layer):
        eng = self._engine
        ln = [int(v) for v in np.asarray(ln)]
        which = "bot" if ln == eng.ln_bot and not hasattr(self, "bot_l") else "top"
        if ln != (eng.ln_bot if which == "bot" else eng.ln_top):
            sys.exit("ERROR: create_mlp called with layer sizes that differ from the constructed model")
        layers = []
        for i in range(len(ln) - 1):
            n, m = ln[i], ln[i + 1]
            W = np.random.normal(0.0, np.sqrt(2 / (m + n)), size=(m, n)).astype(np.float32)
            bt = np.random.normal(0.0, np.sqrt(1 / m), size=m).astype(np.float32)
            with torch.no_grad():
                eng.W[which][i].copy_(torch.from_numpy(W))
                eng.b[which][i].copy_(torch.from_numpy(bt))
            layers.append(_LinearView(eng.W[which][i], eng.b[which][i]))
            layers.append(nn.Sigmoid() if i == sigmoid_layer else nn.ReLU())
        eng.mark_params_changed()
        return nn.Sequential(*layers)

    def create_emb(self, m, ln, weighted_pooling=None):
        eng = self._engine
        ln = np.asarray(ln)
        emb_l, v_W_l = nn.ModuleList(), []
        big = int(ln.sum()) * int(m) > _NUMPY_INIT_MAX
        gen = None
        if big:
            gen = torch.Generator(device=eng.device)
            gen.manual_seed(int(np.random.randint(0, 2 ** 31 - 1)))
        if self._dist is not None:
            # This rank keeps only the rows it stores (the reference skips non-local tables BEFORE drawing,
            # dlrm_s_pytorch.py:252-254, so its ranks' numpy streams diverge).  Here every rank draws every table in
            # order and keeps its slices: the initial model is the single-process model for the same seed.
            if weighted_pooling is not None:
                sys.exit("ERROR: weighted pooling is not supported on distributed runs")
            mine = {}
            for j, sh in enumerate(eng.shards):
                mine.setdefault(int(sh["table"]), []).append((j, int(sh["row_lo"]), int(sh["row_n"])))
            views = {}
            for k in range(ln.size):
                n = int(ln[k])
                a = float(np.sqrt(1 / n))
                W = None if big else np.random.uniform(low=-a, high=a, size=(n, int(m))).astype(np.float32)
                for j, lo, cnt in mine.get(k, []):
                    tab = eng.table(j)
                    with torch.no_grad():
                        if big:
                            _uniform_(tab, a, gen)
                        else:
                            tab.copy_(torch.from_numpy(W[lo:lo + cnt]))
                    views[j] = _TableView(tab)
            for j in range(len(eng.shards)):
                emb_l.append(views[j])
                v_W_l.append(None)
            return emb_l, v_W_l
        for k in range(ln.size):
            n = int(ln[k])
            a = float(np.sqrt(1 / n))
            if eng.quant_only:
                # the float model's draw for the same seed (same generator, same order), quantized as its
                # quantize_embedding() would quantize it.  A device draw maps values to elements through the sizes and
                # strides of its output, so it goes into a whole [n, m] table with the fp32 model's row stride (m: that
                # model's engine is built with interleave_momentum=False); drawing in chunks would draw other values.
                # The fp32 temporary is one table (20.5 GB for a 40 M-row MLPerf table), freed before the next.
                with torch.no_grad():
                    if big:
                        W = torch.empty((n, int(m)), dtype=torch.float32, device=eng.device)
                        assert W.stride() == (int(m), 1)
                        _uniform_(W, a, gen)
                    else:
                        W = torch.from_numpy(np.random.uniform(low=-a, high=a, size=(n, int(m))).astype(np.float32))
                    eng.quantize_rows(k, W)
                    del W
                if weighted_pooling is None:
                    v_W_l.append(None)
                elif not eng.learned_row_weights:
                    v_W_l.append(torch.ones(n, dtype=torch.float32, device=eng.device))
                continue
            tab = eng.table(k)
            with torch.no_grad():
                if big and eng.is_host[k]:
                    # the draw of a device table (same sizes and strides), then copied to host memory
                    tmp = torch.empty(tab.shape, dtype=torch.float32, device=eng.device)
                    _uniform_(tmp, a, gen)
                    tab.copy_(tmp)
                    del tmp
                elif big:
                    _uniform_(tab, a, gen)
                else:  # bit-identical to the reference for the same numpy seed (dlrm_s_pytorch.py:280-284)
                    W = np.random.uniform(low=-a, high=a, size=(n, int(m))).astype(np.float32)
                    tab.copy_(torch.from_numpy(W))
            emb_l.append(_TableView(tab))
            if weighted_pooling is None:
                v_W_l.append(None)
            elif not eng.learned_row_weights:
                v_W_l.append(torch.ones(n, dtype=torch.float32, device=eng.device))
        if weighted_pooling is not None and eng.learned_row_weights:
            # Parameters that share storage with the engine's arena (ones, as the reference's torch.ones(n)): the fused
            # update steps them, state_dict() reads and load_state_dict() writes the arena
            eng.row_weights.fill_(1.0)
            v_W_l = nn.ParameterList([nn.Parameter(eng.row_weights[int(eng.row_base[k]):int(eng.row_base[k + 1])])
                                      for k in range(ln.size)])
        elif weighted_pooling is not None:
            eng.row_weights = torch.cat(v_W_l)
            v_W_l = [eng.row_weights[int(eng.row_base[k]):int(eng.row_base[k + 1])] for k in range(ln.size)]
        return emb_l, v_W_l

    # ------------------------------------------------------------------ reference methods
    def _sparse(self, lS_o, lS_i) -> SparseInput:
        return sparse_from_reference(lS_o, lS_i, self._engine.device)

    def apply_mlp(self, x, layers):
        """Forward of one MLP stack (no autograd through this stand-alone entry point)."""
        eng = self._engine
        which = "bot" if layers is self.bot_l else "top"
        x = x.to(eng.device).contiguous()
        return eng.mlp_only(which, x).clone()

    def apply_emb(self, lS_o, lS_i, emb_l=None, v_W_l=None):
        """list of T pooled tensors [B, D] (views of the interaction operand, features 1..T)."""
        eng = self._engine
        sp = self._sparse(lS_o, lS_i)
        if sp.batch > eng.max_batch:
            eng._alloc_activations(sp.batch)
        eng.emb_forward(sp)
        eng.reduce_partials(sp.batch)
        return [eng.Tbuf[:sp.batch, 1 + k, :] for k in range(eng.T)]

    def interact_features(self, x, ly):
        eng = self._engine
        B = x.shape[0]
        Tb = eng.Tbuf[:B]
        if x.data_ptr() != Tb.data_ptr():
            Tb[:, 0, :].copy_(x)
        for k, y in enumerate(ly):
            if y.data_ptr() != Tb[:, 1 + k, :].data_ptr():
                Tb[:, 1 + k, :].copy_(y)
        if self.arch_interaction_op == "cat":
            return Tb.reshape(B, -1).clone()
        return eng.interact_only(B).clone()

    def forward(self, dense_x, lS_o, lS_i):
        if self._dist is not None:
            return self.distributed_forward(dense_x, lS_o, lS_i)
        if self.ndevices > 1:
            sys.exit("ERROR: single-process multi-GPU (parallel_forward) is replaced by one process per GPU: "
                     "launch the same command with torchrun --nproc-per-node N (distributed_forward)")
        return self.sequential_forward(dense_x, lS_o, lS_i)

    def sequential_forward(self, dense_x, lS_o, lS_i):
        eng = self._engine
        sp = self._sparse(lS_o, lS_i)
        x = dense_x.to(eng.device, dtype=torch.float32).contiguous()
        params = list(self.parameters())
        if self._fused_opt is None:
            eng.mark_params_changed()   # a torch optimizer may have written the master weights
        return _DLRMForward.apply(self, sp, torch.is_grad_enabled(), x, *params)

    def parallel_forward(self, dense_x, lS_o, lS_i):
        return self.forward(dense_x, lS_o, lS_i)

    def distributed_forward(self, dense_x, lS_o, lS_i):
        """dlrm_s_pytorch.py:528-585: every rank receives the whole batch, keeps the dense rows of ITS batch slice and
        the index streams of the tables IT stores rows of, and returns the logits of its slice.  The exchange of
        the pooled vectors (and of their gradients in backward) rides on the gather / interaction-backward kernels'
        peer stores instead of an all-to-all."""
        if self._dist is None:
            sys.exit("ERROR: distributed_forward needs torch.distributed initialised with more than one rank "
                     "(launch with torchrun)")
        de, eng = self._dist, self._engine
        batch_size = dense_x.size()[0]
        if batch_size < de.world:
            sys.exit("ERROR: batch_size (%d) must be larger than number of ranks (%d)" % (batch_size, de.world))
        if batch_size % de.world != 0:
            sys.exit("ERROR: batch_size %d can not split across %d ranks evenly" % (batch_size, de.world))
        if batch_size != de.Bg:
            sys.exit("ERROR: distributed_forward was built for a global batch of %d, got %d" % (de.Bg, batch_size))
        if isinstance(lS_i, torch.Tensor):
            lS_i = [lS_i[k] for k in range(lS_i.shape[0])]
        if isinstance(lS_o, torch.Tensor):
            lS_o = [lS_o[k] for k in range(lS_o.shape[0])]
        if len(lS_o) != de.Tg or len(lS_i) != de.Tg:
            sys.exit("ERROR: corrupted model input detected in distributed_forward call")
        sp = sparse_from_reference([lS_o[s.table] for s in de.mine], [lS_i[s.table] for s in de.mine], eng.device)
        x = dense_x[de.rank * de.B:(de.rank + 1) * de.B].to(eng.device, dtype=torch.float32).contiguous()
        params = list(self.parameters())
        return _DLRMForward.apply(self, sp, torch.is_grad_enabled(), x, *params)

    def quantize_embedding(self, bits):
        """dlrm_s_pytorch.py:465-481: pack every table into fbgemm's row-wise `bits`-bit rows (emb_l_q[k], the bytes of
        torch.ops.quantized.embedding_bag_{byte,4bit}_prepack) and pool from them from now on.  The float tables stay,
        so state_dict() is unchanged; training is refused afterwards (it would step the float tables while the forward
        serves the packed ones)."""
        if bits not in (4, 8):
            sys.exit("ERROR: quantize_embedding supports 4 and 8 bits (got %r)" % (bits,))
        if self._dist is not None:
            sys.exit("ERROR: quantized embedding tables are not supported on sharded runs")
        eng = self._engine
        if eng.quant_only:
            sys.exit("ERROR: the tables are already %d-bit quantized (emb_dtype=%s)" % (eng.quant_bits, eng.emb_dtype))
        try:
            eng.quantize_tables(int(bits))
        except ValueError as e:
            sys.exit("ERROR: " + str(e))
        self.emb_l_q = [eng.table_q(k) for k in range(eng.T)]
        self.quantize_emb, self.quantize_bits = True, int(bits)

    # ------------------------------------------------------------------ gradients for torch optimizers
    def _materialise_sparse_grads(self, sp: SparseInput):
        """The reference's uncoalesced sparse COO gradients (SURVEY §8 a9): indices = lS_i[k],
        values[j] = d_ly_k[bag of j].  Compatibility path for unmodified torch optimizers."""
        eng = self._engine
        B = sp.batch
        out = []
        for k in range(eng.T):
            idx = sp.indices[k]
            off = sp.offsets[k][:B]
            nnz = idx.numel() if not sp.include_last else int(sp.offsets[k][B].item() - sp.offsets[k][0].item())
            start = 0 if not sp.include_last else int(sp.offsets[k][0].item())
            ind = idx[start:start + nnz]
            bag = torch.searchsorted(off.contiguous(), torch.arange(start, start + nnz, device=idx.device),
                                     right=True) - 1
            vals = eng.dT[:B, 1 + k, :][bag]
            out.append(torch.sparse_coo_tensor(ind.view(1, -1).long(), vals, (eng.ln_emb[k], eng.D)))
        return out

    def to(self, *args, **kwargs):  # parameters already live in device arenas
        dev = args[0] if args else kwargs.get("device")
        if dev is not None and torch.device(dev).type == "cpu":
            sys.exit("ERROR: dlrm_b200.DLRM_Net has no CPU path")
        return self
