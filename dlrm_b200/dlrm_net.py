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
    unmodified `torch.optim.SGD` keeps working (compatibility mode, slower).
QR / mixed-dimension embeddings, quantised embeddings and `parallel_forward` are outside the path
(SURVEY §2) and exit with an error when requested.
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
                 loss_function="bce", *, device=None, gemm="tc", max_batch=2048, loss_weights=None):
        super().__init__()
        self._engine: Optional[Engine] = None
        self._fused_opt = None
        self._pending = None
        if (m_spa is None or ln_emb is None or ln_bot is None or ln_top is None
                or arch_interaction_op is None):
            return  # reference allows an empty shell (dlrm_s_pytorch.py:320-326)
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
        if self.weighted_pooling == "learned":
            sys.exit("ERROR: learned weighted pooling is not supported by dlrm_b200 (fixed only)")
        self.qr_flag, self.md_flag = False, False
        self.quantize_emb, self.emb_l_q, self.quantize_bits = False, [], 32
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
                                    loss_threshold=loss_threshold, loss_ws=loss_ws)
            self._engine = self._dist.eng
            self.local_shards = list(self._dist.mine)
        else:
            self._engine = Engine(int(m_spa), ln_emb.tolist(), ln_bot.tolist(), ln_top.tolist(),
                                  op=arch_interaction_op, itself=arch_interaction_itself,
                                  sigmoid_bot=sigmoid_bot, sigmoid_top=sigmoid_top, loss=loss_function,
                                  loss_threshold=loss_threshold, loss_ws=loss_ws, device=device,
                                  max_batch=max_batch, gemm=gemm, interleave_momentum=False)
        self._m_spa, self._ln_emb = int(m_spa), ln_emb
        # same construction (and numpy RNG consumption) order as the reference: tables, bottom, top
        if ndevices <= 1:
            self.emb_l, w_list = self.create_emb(m_spa, ln_emb, weighted_pooling)
            self.v_W_l = w_list
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
                            tab.uniform_(-a, a, generator=gen)
                        else:
                            tab.copy_(torch.from_numpy(W[lo:lo + cnt]))
                    views[j] = _TableView(tab)
            for j in range(len(eng.shards)):
                emb_l.append(views[j])
                v_W_l.append(None)
            return emb_l, v_W_l
        for k in range(ln.size):
            n = int(ln[k])
            tab = eng.table(k)
            a = float(np.sqrt(1 / n))
            with torch.no_grad():
                if big:
                    tab.uniform_(-a, a, generator=gen)
                else:  # bit-identical to the reference for the same numpy seed (dlrm_s_pytorch.py:280-284)
                    W = np.random.uniform(low=-a, high=a, size=(n, int(m))).astype(np.float32)
                    tab.copy_(torch.from_numpy(W))
            emb_l.append(_TableView(tab))
            if weighted_pooling is None:
                v_W_l.append(None)
            else:
                v_W_l.append(torch.ones(n, dtype=torch.float32, device=eng.device))
        if weighted_pooling is not None:
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
        sys.exit("ERROR: 4 and 8-bit quantization on GPU is not supported")

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
