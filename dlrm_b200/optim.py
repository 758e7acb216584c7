"""Fused optimizers for `dlrm_b200.DLRM_Net` with the constructor signatures the reference uses
(`opts[args.optimizer](parameters, lr=args.learning_rate)`, dlrm_s_pytorch.py:1342-1369):

    SGD(params, lr)          == torch.optim.SGD with sparse embedding gradients
    RWSAdagrad(params, lr)   == optim/rwsadagrad.py (row-wise sparse Adagrad; dense params: Adagrad)
    Adagrad(params, lr)      == torch.optim.Adagrad (element-wise; embedding tables take sparse gradients)

`step()` launches the fused kernels (coalesce + row update in place, dense update + operand
refresh) on the gradients the last `backward()` left in the engine's buffers: no [nnz, D] sparse
gradient tensor exists.  The reference refuses Adagrad/RWSAdagrad on GPU (:1339-1340); here they run
on the device.  `param_groups[0]["lr"]` is honoured every step, so `LRPolicyScheduler` works.
"""
from __future__ import annotations

import numpy as np
import torch



class NotEngineParameters(RuntimeError):
    """The parameters handed to a fused optimizer are not those of a dlrm_b200.DLRM_Net: its step runs on the engine's
    memory, so it cannot serve them."""


class _Fused(torch.optim.Optimizer):
    _name = "sgd"

    def __init__(self, params, lr=1e-2, lr_decay=0.0, weight_decay=0.0, initial_accumulator_value=0.0,
                 eps=1e-10):
        params = list(params)
        if weight_decay != 0.0:
            raise RuntimeError("weight_decay option is not compatible with sparse gradients")
        if initial_accumulator_value != 0.0:
            raise ValueError("initial_accumulator_value != 0 is not supported")
        super().__init__(params, dict(lr=lr, lr_decay=lr_decay, eps=eps))
        net = None
        for g in self.param_groups:
            for p in g["params"]:
                net = getattr(p, "_dlrm_net", None) or net
        if net is None:
            raise NotEngineParameters("dlrm_b200.optim optimizers take the parameters of a dlrm_b200.DLRM_Net")
        self.net = net() if callable(net) else net
        self.net._engine.ensure_optimizer_state(self._name)    # refuses quantized (inference-only) tables
        self.net._fused_opt = self

    def zero_grad(self, set_to_none: bool = True):
        self.net._pending = None      # discards a backward() whose step() was skipped
        for g in self.param_groups:
            for p in g["params"]:
                p.grad = None

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        net, eng = self.net, self.net._engine
        pend = net._pending
        if pend is None:
            return loss
        sp, linked = pend
        g = self.param_groups[0]
        eng.opt_step += 1
        clr = g["lr"] / (1.0 + (eng.opt_step - 1.0) * g["lr_decay"]) if self._name != "sgd" else g["lr"]
        eng.apply_optimizer(sp, self._name, clr, g["eps"], linked)
        net._pending = None
        return loss


    # ------------------------------------------------------------------ checkpoint (opt_state_dict)
    def _state_view(self, p):
        """('momentum', [rows] view) for an embedding table, ('sum', same-shape view) for an MLP parameter or a
        learned row-weight vector v_W_l[k]: the engine memory that holds the reference's per-parameter state
        (optim/rwsadagrad.py:86-100).  Adagrad: ('sum', [rows, D] view) for an embedding table too
        (torch.optim.Adagrad's state)."""
        eng = self.net._engine
        lo = eng.dense.data_ptr()
        if lo <= p.data_ptr() < lo + eng.dense.numel() * 4:
            off = (p.data_ptr() - lo) // 4
            return "sum", eng.dense_state[off:off + p.numel()].view(p.shape)
        if getattr(self.net, "weighted_pooling", None) == "learned":
            lo = eng.row_weights.data_ptr()
            if lo <= p.data_ptr() < lo + eng.row_weights.numel() * 4:
                k = int(np.searchsorted(eng.row_base, (p.data_ptr() - lo) // 4, side="right")) - 1
                return "sum", eng.row_weight_sum_of(k)
        for k in range(len(eng.row_base) - 1):
            if eng.table(k).data_ptr() == p.data_ptr():
                if self._name == "adagrad":
                    return "sum", eng.accumulator_ew(k)
                return "momentum", eng.momentum_of(k)
        raise RuntimeError("parameter is not backed by the engine's memory")

    def state_dict(self):
        """torch.optim's layout with the reference optimizer's keys: RWSAdagrad keeps 'step' and, per parameter,
        'momentum' ([rows], embedding tables) or 'sum' (dense parameters); Adagrad keeps torch.optim.Adagrad's
        {'step': tensor(float), 'sum': <the parameter's shape>} per parameter; SGD has no state."""
        eng = self.net._engine
        params = [p for g in self.param_groups for p in g["params"]]
        state = {}
        if self._name == "rwsadagrad":
            for i, p in enumerate(params):
                kind, view = self._state_view(p)
                state[i] = {"step": int(eng.opt_step), kind: view.detach().clone()}
        elif self._name == "adagrad":
            for i, p in enumerate(params):
                kind, view = self._state_view(p)
                state[i] = {"step": torch.tensor(float(eng.opt_step)), kind: view.detach().clone()}
        group = {k: v for k, v in self.param_groups[0].items() if k != "params"}
        group["params"] = list(range(len(params)))
        return {"state": state, "param_groups": [group], "opt_step": int(eng.opt_step)}

    @torch.no_grad()
    def load_state_dict(self, sd):
        eng = self.net._engine
        params = [p for g in self.param_groups for p in g["params"]]
        for k, v in sd["param_groups"][0].items():
            if k != "params":
                self.param_groups[0][k] = v
        step = int(sd.get("opt_step", 0))
        for i, st in sd.get("state", {}).items():
            kind, view = self._state_view(params[int(i)])
            if kind not in st:
                raise KeyError("optimizer state of parameter %d has no '%s'" % (int(i), kind))
            view.copy_(torch.as_tensor(st[kind]).to(view.device))
            step = max(step, int(st.get("step", 0)))
        eng.opt_step = step


class SGD(_Fused):
    _name = "sgd"


class RWSAdagrad(_Fused):
    _name = "rwsadagrad"


class Adagrad(_Fused):
    """torch.optim.Adagrad with the element-wise accumulator of every table row on the device: a step updates the
    rows of the batch (sum += g*g, w -= clr * g / (sqrt(sum) + eps) per element, clr = lr / (1 + (step - 1)
    lr_decay)) and leaves every other row and its accumulator alone; the MLP parameters take the same dense step.
    The accumulator arena adds 4 * D bytes per table row.  param_groups carry torch.optim.Adagrad's keys, so a
    checkpoint of the reference's `--optimizer=adagrad` loads here and one written here loads into
    torch.optim.Adagrad."""
    _name = "adagrad"

    def __init__(self, params, lr=1e-2, lr_decay=0.0, weight_decay=0.0, initial_accumulator_value=0.0, eps=1e-10,
                 foreach=None, *, maximize=False, differentiable=False, fused=None):
        if maximize:
            raise ValueError("maximize=True is not supported")
        if differentiable:
            raise ValueError("differentiable=True is not supported")
        super().__init__(params, lr=lr, lr_decay=lr_decay, weight_decay=weight_decay,
                         initial_accumulator_value=initial_accumulator_value, eps=eps)
        for g in self.param_groups:
            g.update(weight_decay=0, initial_accumulator_value=0, foreach=foreach, maximize=False,
                     differentiable=False, fused=fused)
