"""CPU restatement (numpy) of the DLRM_Net hot path -- TEST INFRASTRUCTURE ONLY.

This file is the *checker* for the CUDA path.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import it.  Nothing under ``dlrm_b200/`` does.

Parity pin: every function here is checked against the LIVE reference
(`/root/reference/dlrm_s_pytorch.py`, imported in place) by
``oracle/make_goldens.py`` and against the committed fixtures
``tests/golden/*.npz`` by ``tests/test_oracle_golden.py``.  The reference holds
no golden vectors of its own for this path (SURVEY.md §4/§8c), so the pin is
"outputs of the reference itself run in the build container", script committed.

The arithmetic of the reference lives in an un-vendored dependency: ``torch``
(ATen CPU kernels; ``requirements.txt:5`` unpinned, 2.11.0+cu128 installed).
The functions below restate the published algorithm of each ATen op at the
reference's call sites:

  emb_bag_sum      dlrm_s_pytorch.py:452-457  nn.EmbeddingBag(mode="sum")
  mlp_forward      dlrm_s_pytorch.py:208-246, 399-405  Linear + ReLU / Sigmoid
  interact_dot     dlrm_s_pytorch.py:483-504  cat -> bmm -> strict-lower-tri -> cat
  interact_cat     dlrm_s_pytorch.py:505-507
  loss_forward     dlrm_s_pytorch.py:148-156, 385-393  MSELoss / BCELoss(mean) / wbce
  dlrm_forward     dlrm_s_pytorch.py:587-612  sequential_forward
  dlrm_backward    autograd of the above (dlrm_s_pytorch.py:1613)
  rwsadagrad_*     optim/rwsadagrad.py:73-152
  sgd_*            torch.optim.SGD (dlrm_s_pytorch.py:1343), sparse add

All float math is float32 unless ``dtype=np.float64`` is requested (used as a
"ground truth" to bound rounding error of both the reference and the kernels).
"""

from __future__ import annotations

import numpy as np

# --------------------------------------------------------------------------
# embedding bag (sum pooling)            ref: dlrm_s_pytorch.py:407-462
# --------------------------------------------------------------------------


def bag_bounds(off, nnz):
    """[start, end) of every bag.  The last bag runs to ``nnz`` (EmbeddingBag
    without include_last_offset), ref dlrm_s_pytorch.py:453-457."""
    off = np.asarray(off, dtype=np.int64)
    end = np.empty_like(off)
    end[:-1] = off[1:]
    if off.size:
        end[-1] = nnz
    return off, end


def emb_bag_sum(W, idx, off, psw=None, dtype=np.float32):
    """out[b,:] = sum_{j in bag b} psw[j] * W[idx[j],:], accumulated
    SEQUENTIALLY in index order starting from 0 (one accumulator per output
    element).  The reference CPU kernel is bit-identical to this order
    (SURVEY.md §8 a4, re-verified by make_goldens.py).  Empty bag -> zeros."""
    W = np.asarray(W)
    idx = np.asarray(idx, dtype=np.int64)
    start, end = bag_bounds(off, idx.size)
    B = start.size
    out = np.zeros((B, W.shape[1]), dtype=dtype)
    if B == 0:
        return out
    length = end - start
    lmax = int(length.max()) if B else 0
    for j in range(lmax):  # position inside the bag: sequential dependence
        live = np.nonzero(length > j)[0]
        rows = W[idx[start[live] + j]].astype(dtype, copy=False)
        if psw is not None:
            w = np.asarray(psw, dtype=dtype)[start[live] + j][:, None]
            # ATen accumulates with a fused multiply-add; emulate the single
            # rounding in float64 when running in float32.
            if dtype == np.float32:
                acc = out[live].astype(np.float64) + w.astype(np.float64) * rows.astype(np.float64)
                out[live] = acc.astype(np.float32)
            else:
                out[live] = out[live] + w * rows
        else:
            out[live] = out[live] + rows
    return out


def apply_emb(tables, lS_o, lS_i, v_W_l=None, dtype=np.float32):
    """List over tables; ref dlrm_s_pytorch.py:407-462.  ``v_W_l[k]`` is the
    per-row weight vector gathered by the indices (`:425-428`)."""
    ly = []
    for k, W in enumerate(tables):
        idx = np.asarray(lS_i[k], dtype=np.int64)
        psw = None
        if v_W_l is not None and v_W_l[k] is not None:
            psw = np.asarray(v_W_l[k])[idx]
        ly.append(emb_bag_sum(W, idx, lS_o[k], psw, dtype))
    return ly


# --------------------------------------------------------------------------
# MLP                                     ref: dlrm_s_pytorch.py:208-246,399-405
# --------------------------------------------------------------------------


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def mlp_forward(x, layers, sigmoid_layer=-1, dtype=np.float32, keep=False):
    """layers = [(W[out,in], b[out]), ...]; activation i is Sigmoid iff
    i == sigmoid_layer else ReLU (`:237-241`).  Returns last activation, or the
    list of all layer outputs (post-activation) when keep=True."""
    acts = []
    h = np.asarray(x, dtype=dtype)
    for i, (W, b) in enumerate(layers):
        z = h @ np.asarray(W, dtype=dtype).T + np.asarray(b, dtype=dtype)
        h = sigmoid(z).astype(dtype) if i == sigmoid_layer else np.maximum(z, 0).astype(dtype)
        acts.append(h)
    return acts if keep else h


# --------------------------------------------------------------------------
# interaction                             ref: dlrm_s_pytorch.py:483-515
# --------------------------------------------------------------------------


def tril_indices(nf, itself=False):
    """Row-major strict (or diagonal-inclusive) lower triangle: (1,0),(2,0),(2,1)...
    ref `:499-501`."""
    offset = 1 if itself else 0
    li = np.array([i for i in range(nf) for j in range(i + offset)], dtype=np.int64)
    lj = np.array([j for i in range(nf) for j in range(i + offset)], dtype=np.int64)
    return li, lj


def interact_dot(x, ly, itself=False, dtype=np.float32):
    B, d = x.shape
    T = np.concatenate([x] + list(ly), axis=1).reshape(B, -1, d).astype(dtype, copy=False)
    Z = np.einsum("bik,bjk->bij", T, T).astype(dtype)  # bmm(T, T^T)
    li, lj = tril_indices(T.shape[1], itself)
    Zflat = Z[:, li, lj]
    return np.concatenate([x.astype(dtype, copy=False), Zflat], axis=1)


def interact_cat(x, ly):
    return np.concatenate([x] + list(ly), axis=1)


# --------------------------------------------------------------------------
# loss                                    ref: dlrm_s_pytorch.py:148-156,385-393
# --------------------------------------------------------------------------


def loss_forward(p, t, kind="bce", loss_ws=None):
    p = np.asarray(p)
    t = np.asarray(t, dtype=p.dtype)
    if kind == "mse":
        return np.mean((p - t) ** 2, dtype=p.dtype)
    # torch BCELoss clamps log() at -100
    with np.errstate(divide="ignore"):
        lp = np.maximum(np.log(p), -100.0)
        l1p = np.maximum(np.log1p(-p), -100.0)
    per = -(t * lp + (1.0 - t) * l1p)
    if kind == "bce":
        return np.mean(per, dtype=p.dtype)
    if kind == "wbce":
        w = np.asarray(loss_ws, dtype=p.dtype)[t.reshape(-1).astype(np.int64)].reshape(t.shape)
        return np.mean(w * per, dtype=p.dtype)
    raise ValueError(kind)


def loss_backward(p, t, kind="bce", loss_ws=None):
    """dL/dp for reduction=mean.  BCE backward follows ATen
    binary_cross_entropy_backward: (p - t) / max((1-p)*p, 1e-12)."""
    p = np.asarray(p)
    t = np.asarray(t, dtype=p.dtype)
    n = p.size
    if kind == "mse":
        return (2.0 * (p - t) / n).astype(p.dtype)
    g = (p - t) / np.maximum((1.0 - p) * p, 1e-12)
    if kind == "wbce":
        w = np.asarray(loss_ws, dtype=p.dtype)[t.reshape(-1).astype(np.int64)].reshape(t.shape)
        g = g * w
    return (g / n).astype(p.dtype)


# --------------------------------------------------------------------------
# full forward / backward                 ref: dlrm_s_pytorch.py:587-612, :1613
# --------------------------------------------------------------------------


def dlrm_forward(params, X, lS_o, lS_i, *, op="dot", itself=False, loss_threshold=0.0,
                 sigmoid_bot=-1, sigmoid_top=None, dtype=np.float32, keep=False):
    """params = dict(emb=[W_k], bot=[(W,b)...], top=[(W,b)...], v_W_l=None|[...]).
    Returns p [B,1] (or a dict of every stage when keep=True)."""
    if sigmoid_top is None:
        sigmoid_top = len(params["top"]) - 1
    bot_acts = mlp_forward(X, params["bot"], sigmoid_bot, dtype, keep=True)
    x = bot_acts[-1]
    ly = apply_emb(params["emb"], lS_o, lS_i, params.get("v_W_l"), dtype)
    R = interact_dot(x, ly, itself, dtype) if op == "dot" else interact_cat(x, ly)
    top_acts = mlp_forward(R, params["top"], sigmoid_top, dtype, keep=True)
    p = top_acts[-1]
    z = p
    if 0.0 < loss_threshold < 1.0:
        z = np.clip(p, loss_threshold, 1.0 - loss_threshold)
    if keep:
        return dict(x=x, ly=ly, R=R, p=p, z=z, bot_acts=bot_acts, top_acts=top_acts)
    return z


def _mlp_backward(x_in, acts, layers, sigmoid_layer, g_out, dtype):
    """Backprop through Linear+act stack.  Returns (dx_in, [(dW,db)...])."""
    grads = [None] * len(layers)
    g = g_out
    for i in reversed(range(len(layers))):
        W, _ = layers[i]
        y = acts[i]
        if i == sigmoid_layer:
            gz = g * (1.0 - y) * y  # sigmoid_backward: grad * (1 - y) * y
        else:
            gz = g * (y > 0)  # threshold_backward
        gz = gz.astype(dtype)
        h_in = x_in if i == 0 else acts[i - 1]
        dW = gz.T @ np.asarray(h_in, dtype=dtype)
        db = gz.sum(axis=0, dtype=dtype)
        grads[i] = (dW.astype(dtype), db.astype(dtype))
        g = gz @ np.asarray(W, dtype=dtype)
    return g.astype(dtype), grads


def dlrm_backward(params, X, lS_o, lS_i, target, *, loss="bce", loss_ws=None, op="dot",
                  itself=False, loss_threshold=0.0, sigmoid_bot=-1, sigmoid_top=None,
                  dtype=np.float32, relu_masks=None):
    """Manual backprop of loss(dlrm_forward(...)).  Returns dict with
    loss, p, bot/top grads [(dW,db)], and per-table dense-by-bag grads
    ``d_ly[k]`` [B,D] (the reference's sparse COO grad has values
    d_ly[k][bag_of(j)] at index lS_i[k][j], uncoalesced; SURVEY §8 a9).

    relu_masks = dict(bot=[y_0, ...], top=[y_0, ...]) (entries may be None): the
    backward of ReLU layer i passes the gradient where y_i > 0 instead of where
    this forward's own output is positive.  A checker that hands in the
    activations of the implementation under test gets the gradient of the same
    piecewise-linear branch, so a pre-activation within rounding of 0 is not a
    disagreement of a whole term.  Only the backward changes: p, z and the loss
    are this forward's own and are not recomputed, so the forward of the
    implementation is held by whatever the checker asserts about them."""
    if sigmoid_top is None:
        sigmoid_top = len(params["top"]) - 1
    f = dlrm_forward(params, X, lS_o, lS_i, op=op, itself=itself, loss_threshold=loss_threshold,
                     sigmoid_bot=sigmoid_bot, sigmoid_top=sigmoid_top, dtype=dtype, keep=True)
    if relu_masks is not None:
        for name, sig in (("bot", sigmoid_bot), ("top", sigmoid_top)):
            acts = f[name + "_acts"]
            for i, y in enumerate(relu_masks.get(name) or []):
                if y is not None and i != sig:
                    # values stay this forward's (the other branch's output stands in where it is 0)
                    acts[i] = np.where(np.asarray(y) > 0, np.where(acts[i] > 0, acts[i], y), 0).astype(dtype)
        f["x"] = f["bot_acts"][-1]
    p, z = f["p"], f["z"]
    L = loss_forward(z, target, loss, loss_ws)
    gz = loss_backward(z, np.asarray(target, dtype=dtype), loss, loss_ws)
    if 0.0 < loss_threshold < 1.0:  # clamp backward: pass where lo <= p <= hi
        gz = gz * ((p >= loss_threshold) & (p <= 1.0 - loss_threshold))
    dR, top_grads = _mlp_backward(f["R"], f["top_acts"], params["top"], sigmoid_top, gz, dtype)
    x, ly = f["x"], f["ly"]
    B, d = x.shape
    if op == "dot":
        T = np.concatenate([x] + list(ly), axis=1).reshape(B, -1, d).astype(dtype, copy=False)
        nf = T.shape[1]
        li, lj = tril_indices(nf, itself)
        dZ = np.zeros((B, nf, nf), dtype=dtype)
        dZ[:, li, lj] = dR[:, d:]
        dT = np.einsum("bij,bjk->bik", dZ + dZ.transpose(0, 2, 1), T).astype(dtype)
        dT[:, 0, :] += dR[:, :d]
    else:
        dT = dR.reshape(B, -1, d).copy()
    dx = dT[:, 0, :]
    d_ly = [np.ascontiguousarray(dT[:, 1 + k, :]) for k in range(len(ly))]
    _, bot_grads = _mlp_backward(np.asarray(X, dtype=dtype), f["bot_acts"], params["bot"],
                                 sigmoid_bot, dx, dtype)
    return dict(loss=L, p=p, z=z, top_grads=top_grads, bot_grads=bot_grads, d_ly=d_ly, fwd=f)


def bag_of_position(off, nnz):
    """offset2bag: for every index position j the bag it belongs to."""
    start, end = bag_bounds(off, nnz)
    out = np.zeros(nnz, dtype=np.int64)
    for b in range(start.size):
        out[start[b]:end[b]] = b
    return out


def sparse_grad(idx, off, d_ly_k):
    """(indices, values) of the reference's uncoalesced sparse COO gradient of
    one table (SURVEY §8 a9): values[j] = d_ly_k[bag_of(j)]."""
    idx = np.asarray(idx, dtype=np.int64)
    return idx, d_ly_k[bag_of_position(off, idx.size)]


# --------------------------------------------------------------------------
# optimizers                              ref: optim/rwsadagrad.py:73-152
# --------------------------------------------------------------------------


def coalesce(indices, values):
    """Sum duplicates; unique indices ascending (torch coalesce())."""
    uniq, inv = np.unique(indices, return_inverse=True)
    out = np.zeros((uniq.size, values.shape[1]), dtype=values.dtype)
    np.add.at(out, inv, values)  # sequential in original order
    return uniq, out


def rwsadagrad_sparse(W, momentum, indices, values, lr, eps=1e-10, step=1, lr_decay=0.0):
    """In-place row-wise sparse Adagrad on one table.  ref optim/rwsadagrad.py:115-143:
    g = coalesce(grad); momentum[rows] += mean_d(g^2); std = sqrt(momentum[rows]) + eps;
    W[rows] += -clr * g / std."""
    clr = lr / (1.0 + (step - 1.0) * lr_decay)
    rows, g = coalesce(np.asarray(indices, dtype=np.int64), values)
    if g.size == 0:
        return
    dt = W.dtype
    momentum[rows] += np.mean(g.astype(dt) ** 2, axis=1, dtype=dt)
    std = np.sqrt(momentum[rows]).astype(dt) + dt.type(eps)
    W[rows] += (dt.type(-clr) * (g / std[:, None])).astype(dt)


def adagrad_dense(p, state_sum, g, lr, eps=1e-10, step=1, lr_decay=0.0):
    """Dense branch of RWSAdagrad, ref optim/rwsadagrad.py:145-148."""
    clr = lr / (1.0 + (step - 1.0) * lr_decay)
    dt = p.dtype
    state_sum += g * g
    std = np.sqrt(state_sum).astype(dt) + dt.type(eps)
    p += (dt.type(-clr) * (g / std)).astype(dt)


def sgd_sparse(W, indices, values, lr):
    """torch.optim.SGD on a sparse grad: W.add_(g, alpha=-lr); duplicates add."""
    np.add.at(W, np.asarray(indices, dtype=np.int64), (-lr * values).astype(W.dtype))


def sgd_dense(p, g, lr):
    p += (-lr * g).astype(p.dtype)


def train_step(params, state, X, lS_o, lS_i, target, *, lr, optimizer="rwsadagrad",
               loss="bce", **kw):
    """One fwd+bwd+update, in place on params/state.  ref dlrm_s_pytorch.py:1575-1621.
    state = dict(step=int, mom=[...per table...], bot=[(sW,sb)...], top=[...])."""
    dtype = kw.get("dtype", np.float32)
    r = dlrm_backward(params, X, lS_o, lS_i, target, loss=loss, **kw)
    state["step"] = state.get("step", 0) + 1
    for k, W in enumerate(params["emb"]):
        ind, val = sparse_grad(lS_i[k], lS_o[k], r["d_ly"][k])
        if optimizer == "rwsadagrad":
            rwsadagrad_sparse(W, state["mom"][k], ind, val, lr, step=state["step"])
        else:
            sgd_sparse(W, ind, val, lr)
    for name in ("bot", "top"):
        for i, (W, b) in enumerate(params[name]):
            dW, db = r[name + "_grads"][i]
            if optimizer == "rwsadagrad":
                sW, sb = state[name][i]
                adagrad_dense(W, sW, dW, lr, step=state["step"])
                adagrad_dense(b, sb, db, lr, step=state["step"])
            else:
                sgd_dense(W, dW, lr)
                sgd_dense(b, db, lr)
    return r


def new_state(params):
    return dict(
        step=0,
        mom=[np.zeros(W.shape[0], dtype=np.float32) for W in params["emb"]],
        bot=[(np.zeros_like(W), np.zeros_like(b)) for W, b in params["bot"]],
        top=[(np.zeros_like(W), np.zeros_like(b)) for W, b in params["top"]],
    )


# --------------------------------------------------------------------------
# synthetic inputs, own generator (same distribution as
# dlrm_data_pytorch.py:899-960 / torchrec_dlrm/multi_hot.py:86-108; NOT the
# same RNG stream -- parity inputs come from the reference generator via goldens)
# --------------------------------------------------------------------------


def random_batch(rng, ln_emb, B, m_den=13, lmax=10, fixed=False, per_table_L=None, unique=True):
    X = rng.random((B, m_den), dtype=np.float32)
    lS_o, lS_i = [], []
    for k, R in enumerate(ln_emb):
        R = int(R)
        if per_table_L is not None:
            lens = np.full(B, int(per_table_L[k]), dtype=np.int64)
        elif fixed:
            lens = np.full(B, lmax, dtype=np.int64)
        else:
            lens = np.round(np.maximum(1.0, rng.random(B) * min(R, lmax))).astype(np.int64)
        tot = int(lens.sum())
        raw = np.round(rng.random(tot) * (R - 1)).astype(np.int64)
        bag = np.repeat(np.arange(B, dtype=np.int64), lens)
        if unique:  # per-bag sorted unique, like np.unique in the reference generator
            order = np.lexsort((raw, bag))
            raw, bag = raw[order], bag[order]
            keep = np.ones(tot, dtype=bool)
            keep[1:] = (raw[1:] != raw[:-1]) | (bag[1:] != bag[:-1])
            raw, bag = raw[keep], bag[keep]
        cnt = np.bincount(bag, minlength=B)
        off = np.zeros(B, dtype=np.int64)
        off[1:] = np.cumsum(cnt)[:-1]
        lS_o.append(off)
        lS_i.append(raw)
    return X, lS_o, lS_i


def random_params(rng, m_spa, ln_emb, ln_bot, ln_top):
    """Same distributions as create_emb/create_mlp (`:221-228`, `:280-284`)."""
    emb = [rng.uniform(-np.sqrt(1 / n), np.sqrt(1 / n), size=(int(n), m_spa)).astype(np.float32)
           for n in ln_emb]

    def mlp(ln):
        out = []
        for i in range(len(ln) - 1):
            n, m = int(ln[i]), int(ln[i + 1])
            W = rng.normal(0.0, np.sqrt(2 / (m + n)), size=(m, n)).astype(np.float32)
            b = rng.normal(0.0, np.sqrt(1 / m), size=m).astype(np.float32)
            out.append((W, b))
        return out

    return dict(emb=emb, bot=mlp(ln_bot), top=mlp(ln_top), v_W_l=None)
