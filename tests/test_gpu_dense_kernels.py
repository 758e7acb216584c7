"""The dense-path kernels called one by one through the C ABI and compared with the float64 restatements of
oracle/dense_f64.py: interaction forward / backward (bulk-copy and fallback forward, float2 and one-column backward,
MAXF 8 / 32 / 64), the fused head, the loss, act_bwd, the dense optimizer, dense_update_pack, split_bf16 and the fp32
SIMT linear layer.

Every output is prefilled with NaN, and the regions a kernel must not write (pad columns, the constant-1 column of the
bf16 operand, rows past the batch, outputs a mode does not produce, masters on a fold-only call) with a sentinel that
is compared bit for bit afterwards.  Bounds follow each kernel's order of operations (oracle/dense_f64.py states
them); results that the kernel computes with reproducible arithmetic are compared bit for bit: the bf16 splits against
torch's round-to-nearest-even, the slab fold, and repeated calls.  The worst err/bound ratio of every kernel family is
printed at the end of the module (`pytest -s`)."""
import json
import os

import numpy as np
import pytest
import torch

from dlrm_b200 import _lib
from oracle import dense_f64 as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = -7.75e33                 # fp32 sentinel of regions that must stay untouched
SENT16 = 0x7E5A                 # bf16 sentinel (a NaN payload no rounding produces)
NAN16 = 0x7FC1
WORST = {}


def _record(family, r):
    WORST[family] = max(WORST.get(family, 0.0), float(r))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst err/bound per kernel family: " + json.dumps({k: float("%.3g" % v) for k, v in sorted(WORST.items())}))


@pytest.fixture
def tunable():
    """Set process-wide kernel knobs for one test; the previous values (DLRM_TUNE or the default 0) come back after."""
    env = {k.strip(): int(v) for k, v in (kv.split("=") for kv in filter(None, os.environ.get("DLRM_TUNE", "").split(",")))}
    prev = {}

    def set_(name, value):
        prev.setdefault(name, env.get(name, 0))
        _lib.set_tunable(name, value)

    try:
        yield set_
    finally:
        for name, value in prev.items():
            _lib.set_tunable(name, value)


def L():
    return _lib.lib()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _ok(rc, what):
    _lib.check(rc, what)


def _error(rc):
    assert rc != 0
    return L().dlrm_b200_last_error().decode()


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _f32buf(rows, cols, inner=None):
    """[rows, cols] fp32 sentinel buffer with NaN in the [inner rows, inner cols] block the kernel must write."""
    t = torch.full((rows, cols), SENT, dtype=torch.float32, device=DEV)
    if inner is not None:
        t[:inner[0], :inner[1]] = float("nan")
    return t


def _bf16buf(rows, cols, inner=None):
    t = torch.full((rows, cols), SENT16, dtype=torch.int16, device=DEV)
    if inner is not None:
        t[:inner[0], :inner[1]] = NAN16
    return t


def _u16(t):
    return t.cpu().numpy().view(np.uint16)


def _outside_untouched(t, inner, what):
    """Everything of buffer t outside its [:inner[0], :inner[1]] block still holds the sentinel, bit for bit."""
    a = t.cpu().numpy()
    mask = np.ones(a.shape, bool)
    mask[:inner[0], :inner[1]] = False
    ref = np.full(a.shape, SENT16 if a.dtype == np.int16 else SENT, a.dtype)
    assert np.array_equal(a[mask].view(np.uint8), ref[mask].view(np.uint8)), what + ": wrote outside its output"


def _same_bits(a, b, what):
    a, b = a.cpu().numpy() if torch.is_tensor(a) else a, b.cpu().numpy() if torch.is_tensor(b) else b
    assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), what


def _mat(rng, rows, cols, ld, off=0, kind="normal", scale=1.0):
    """fp32 device matrix [rows, cols] with row stride ld, `off` floats past an aligned base; padding is random too
    (a kernel that reads it computes something else)."""
    n = max(rows * ld, 1) + off
    a = (rng.standard_normal(n) * scale).astype(np.float32)
    buf = _cuda(a)
    v = buf[off:off + rows * ld].view(rows, ld)
    if kind == "relu":
        v.clamp_(min=0.0)
    elif kind == "unit":
        v.copy_(_cuda(rng.uniform(0, 1, (rows, ld)).astype(np.float32)))
    return v, buf


def _ld(dim, aligned):
    """row stride larger than the minimum: a multiple of 4 (vector loads) or, misaligned, not a multiple of 4"""
    if aligned:
        return (dim + 3) // 4 * 4 + 4
    return dim + 1 if (dim + 1) % 4 else dim + 2


# ================================================================================================ interaction
def _npairs(F, itself):
    return F * (F + 1) // 2 if itself else F * (F - 1) // 2


def _fwd_spb(F, D, itself, bulk):
    """samples per CTA the forward launcher picks (interact.cu): bulk copy up to 100 KB, fallback up to 56 KB"""
    nb = (F + 2) // 3
    Fp, tps, npairs = 3 * nb, nb * (nb + 1) // 2, _npairs(F, itself)
    spb = max(1, 192 // tps)
    if bulk:
        per = (Fp * D + ((npairs + 3) & ~3)) * 4
        while spb > 1 and spb * per + 16 > 100 * 1024:
            spb -= 1
        if spb * per + 16 <= 200 * 1024:
            return spb
        spb = max(1, 192 // tps)
    per = (Fp * (D + 1) + npairs) * 4
    while spb > 1 and spb * per > 56 * 1024:
        spb -= 1
    return spb


def _bwd_spb(F, D, two):
    F4 = (F + 3) & ~3
    spb = max(1, 128 // (D // 2 if two else D))
    while spb > 1 and spb * F * F4 * 4 > 48 * 1024:
        spb -= 1
    return spb


def _pick_b(spb, sel):
    return [1, max(spb - 1, 1), spb + 1, 2049][sel]


def _x_values(rng, T3, mask0):
    """feature 0 = the bottom MLP's output: relu -> >= 0, sigmoid -> (0, 1); both with exact zeros"""
    x = T3[:, 0, :]
    if mask0 == O.ACT_RELU:
        x.clamp_(min=0.0)
    elif mask0 == O.ACT_SIGMOID:
        x.copy_(_cuda(rng.uniform(0, 1, tuple(x.shape)).astype(np.float32)))
    x[:, ::3] = 0.0


def _interact_fwd_call(T, ldt, B, F, D, itself, R=None, ldr=0, bf=None):
    Rh, Rl, ldrb = bf if bf is not None else (None, None, 0)
    return L().dlrm_b200_interact_fwd_ex(T.data_ptr(), ldt, R.data_ptr() if R is not None else None, ldr,
                                         Rh.data_ptr() if Rh is not None else None,
                                         Rl.data_ptr() if Rl is not None else None, ldrb, B, F, D, itself, _st())


def _run_interact_fwd(F, D, itself, B, off=0, seed=0, bf16=False, with_R=True):
    rng = np.random.default_rng(seed)
    ldt = F * D + 4
    T, _ = _mat(rng, B, ldt, ldt, off)
    T3 = T[:, :F * D].view(B, F, D)
    _x_values(rng, T3, O.ACT_RELU)
    ncols = D + _npairs(F, itself)
    ldr = ncols + 3
    R = _f32buf(B + 2, ldr, (B, ncols)) if with_R else None
    bf = None
    if bf16:
        ldrb = (ncols + 1 + 7) // 8 * 8
        Rh, Rl = _bf16buf(B + 1, ldrb, (B, ncols)), _bf16buf(B + 1, ldrb, (B, ncols))
        Rh[:, ncols], Rl[:, ncols] = 0x3F80, 0          # the constant-1 bias column next to R
        bf = (Rh, Rl, ldrb)
    _ok(_interact_fwd_call(T, ldt, B, F, D, itself, R, ldr, bf), "interact_fwd_ex")
    torch.cuda.synchronize()
    return T3, R, bf, ncols


def _check_interact_fwd(F, D, itself, B, off=0, seed=0, bf16=False):
    T3, R, bf, ncols = _run_interact_fwd(F, D, itself, B, off, seed, bf16)
    want, bound = O.interact_fwd(T3.cpu().numpy(), itself)
    Rk = R[:B, :ncols].cpu().numpy()
    _record("interact_fwd", O.check_within(Rk, want, bound, f"interact_fwd F={F} D={D} itself={itself} B={B}"))
    _outside_untouched(R, (B, ncols), "interact_fwd R")
    T3b, R2, bf2, _ = _run_interact_fwd(F, D, itself, B, off, seed, bf16)
    _same_bits(R, R2, "interact_fwd: repeated call differs")
    if bf16:
        Rh, Rl, ldrb = bf
        hi, lo = O.split_bf16(Rk)
        assert np.array_equal(_u16(Rh[:B, :ncols]), hi) and np.array_equal(_u16(Rl[:B, :ncols]), lo), \
            "bf16 pair is not the split of R"
        assert np.all(_u16(Rh[:, ncols]) == 0x3F80) and np.all(_u16(Rl[:, ncols]) == 0), "constant-1 column written"
        for t in (Rh, Rl):
            c = t.clone()
            c[:, ncols] = SENT16
            _outside_untouched(c, (B, ncols), "interact_fwd bf16 pair")
        _same_bits(Rh, bf2[0], "interact_fwd: repeated bf16 hi differs")
        # R = NULL (the engine's call): the same pair
        _, _, bf3, _ = _run_interact_fwd(F, D, itself, B, off, seed, True, with_R=False)
        _same_bits(Rh, bf3[0], "interact_fwd_ex without R: hi differs")
        _same_bits(Rl, bf3[1], "interact_fwd_ex without R: lo differs")


FS = [1, 2, 3, 4, 8, 9, 27, 32, 33, 40, 64]
DS = [1, 2, 3, 4, 16, 17, 100, 128, 256]
INTERACT = [(F, D, (i + j) % 2, (i + 2 * j) % 3) for i, F in enumerate(FS) for j, D in enumerate(DS)]


@pytest.mark.parametrize("F,D,itself,sel", INTERACT)
def test_interact_fwd(F, D, itself, sel):
    bulk = D % 4 == 0
    B = _pick_b(_fwd_spb(F, D, itself, bulk), sel)
    _check_interact_fwd(F, D, itself, B, seed=F * 1000 + D, bf16=bulk)


@pytest.mark.parametrize("F,D,itself,B,off", [
    (27, 128, 0, 2049, 0), (64, 16, 1, 2049, 0), (9, 17, 0, 2049, 0), (4, 2, 1, 2049, 0),
    (27, 128, 1, 37, 1), (8, 16, 0, 25, 1), (33, 4, 1, 9, 1),       # misaligned T: fallback kernel at D % 4 == 0
    (64, 400, 0, 3, 0),        # bulk copy, one sample of 114 KB per CTA
    (64, 201, 1, 3, 0),        # fallback with more than 48 KB of shared memory
])
def test_interact_fwd_edges(F, D, itself, B, off):
    _check_interact_fwd(F, D, itself, B, off=off, seed=B + D, bf16=(off == 0 and D % 4 == 0))


def test_interact_fwd_too_large_is_an_error_without_launch():
    rng = np.random.default_rng(1)
    F, D, B = 64, 770, 2
    T, _ = _mat(rng, B, F * D, F * D)
    ncols = D + _npairs(F, 0)
    R = _f32buf(B, ncols)
    msg = _error(_interact_fwd_call(T, F * D, B, F, D, 0, R, ncols))
    assert "200 KB" in msg and "D=770" in msg, msg
    torch.cuda.synchronize()
    _outside_untouched(R, (0, 0), "interact_fwd error path")
    Rh, Rl = _bf16buf(B, 16), _bf16buf(B, 16)
    msg = _error(_interact_fwd_call(T, 6, B, 2, 3, 0, None, 0, (Rh, Rl, 16)))
    assert "bf16" in msg, msg


def _run_interact_bwd(F, D, itself, B, mask0, off=0, seed=0):
    rng = np.random.default_rng(seed)
    ldt = F * D + 2
    T, _ = _mat(rng, B, ldt, ldt, off)
    T3 = T[:, :F * D].view(B, F, D)
    _x_values(rng, T3, mask0)
    ncols = D + _npairs(F, itself)
    lddr = ncols + 2 + ncols % 2                 # even: the float2 kernel needs 8-byte aligned dR rows
    dR, _ = _mat(rng, B, lddr, lddr)
    lddt, ldg = F * D + 2, D + 2
    dT = _f32buf(B + 1, lddt, (B, F * D))
    gh, gl = _bf16buf(B + 1, ldg, (B, D)), _bf16buf(B + 1, ldg, (B, D))
    _ok(L().dlrm_b200_interact_bwd_ex(T.data_ptr(), ldt, dR.data_ptr(), lddr, dT.data_ptr(), lddt, B, F, D, itself,
                                      mask0, gh.data_ptr(), gl.data_ptr(), ldg, _st()), "interact_bwd_ex")
    torch.cuda.synchronize()
    return T3, dR[:, :ncols], dT, gh, gl


def _check_interact_bwd(F, D, itself, B, mask0, off=0, seed=0):
    T3, dR, dT, gh, gl = _run_interact_bwd(F, D, itself, B, mask0, off, seed)
    want, bound = O.interact_bwd(T3.cpu().numpy(), dR.cpu().numpy(), itself, mask0)
    got = dT[:B, :F * D].cpu().numpy().reshape(B, F, D)
    _record("interact_bwd", O.check_within(got, want, bound, f"interact_bwd F={F} D={D} itself={itself} B={B} "
                                                             f"mask={mask0}"))
    _outside_untouched(dT, (B, F * D), "interact_bwd dT")
    hi, lo = O.split_bf16(got[:, 0, :])
    assert np.array_equal(_u16(gh[:B, :D]), hi) and np.array_equal(_u16(gl[:B, :D]), lo), "g0 pair is not dT[:, 0]"
    _outside_untouched(gh, (B, D), "interact_bwd g0 hi")
    _outside_untouched(gl, (B, D), "interact_bwd g0 lo")
    _, _, dT2, gh2, _ = _run_interact_bwd(F, D, itself, B, mask0, off, seed)
    _same_bits(dT, dT2, "interact_bwd: repeated call differs")
    _same_bits(gh, gh2, "interact_bwd: repeated g0 differs")


@pytest.mark.parametrize("F,D,itself,sel", INTERACT)
def test_interact_bwd(F, D, itself, sel):
    B = _pick_b(_bwd_spb(F, D, D % 2 == 0), sel)
    _check_interact_bwd(F, D, itself, B, mask0=(F + D) % 3, seed=F * 1000 + D + 7)


@pytest.mark.parametrize("F,D,itself,B,mask0,off", [
    (27, 128, 0, 2049, 1, 0), (64, 16, 1, 2049, 2, 0), (9, 17, 0, 2049, 1, 0),
    (40, 16, 1, 17, 2, 1), (8, 128, 0, 3, 1, 1), (64, 2, 1, 129, 1, 1),   # T one float off: one column per thread
    (64, 400, 0, 5, 2, 0),
])
def test_interact_bwd_edges(F, D, itself, B, mask0, off):
    _check_interact_bwd(F, D, itself, B, mask0, off=off, seed=B + D)


@pytest.mark.parametrize("F,D,itself,mask0", [(3, 4, 1, 1), (40, 100, 0, 2), (64, 16, 1, 1), (33, 128, 0, 0)])
def test_interact_bwd_one_column_per_thread(tunable, F, D, itself, mask0):
    tunable("interact_bwd_cols", 1)
    _check_interact_bwd(F, D, itself, _bwd_spb(F, D, False) + 1, mask0, seed=F + D)


def test_interact_bwd_more_than_64_features_is_an_error_without_launch():
    rng = np.random.default_rng(2)
    F, D, B = 65, 4, 3
    T, _ = _mat(rng, B, F * D, F * D)
    dR, _ = _mat(rng, B, D + _npairs(F, 0), D + _npairs(F, 0))
    dT = _f32buf(B, F * D)
    msg = _error(L().dlrm_b200_interact_bwd_ex(T.data_ptr(), F * D, dR.data_ptr(), dR.shape[1], dT.data_ptr(), F * D,
                                               B, F, D, 0, 0, None, None, 0, _st()))
    assert "num_features=65" in msg, msg
    torch.cuda.synchronize()
    _outside_untouched(dT, (0, 0), "interact_bwd error path")


# ================================================================================================ fused head
WS = np.array([0.3, 2.5], np.float32)


def _head_inputs(rng, B, K, act_prev, kind, specials=None):
    ldh = K + 3
    h, _ = _mat(rng, B, ldh, ldh, 0, {O.ACT_RELU: "relu", O.ACT_SIGMOID: "unit"}.get(act_prev, "normal"))
    if act_prev == O.ACT_RELU:
        h.view(-1)[::5] = 0.0
    w = (rng.standard_normal(K) / np.sqrt(K)).astype(np.float32)
    bias = np.array([0.1], np.float32)
    if kind == O.LOSS_MSE:
        t = rng.uniform(0, 1, B).astype(np.float32)
    else:
        t = rng.integers(0, 2, B).astype(np.float32)
        if kind == O.LOSS_BCE:
            t[::4] = rng.uniform(0, 1, len(t[::4]))
    if specials is not None:      # rows whose pre-activation is exactly v: h = [v, 0, ...], w[0] = 1, bias 0
        w[0], bias[0] = 1.0, 0.0
        for r, v in enumerate(specials[:B]):
            h[r].zero_()
            h[r, 0] = float(v)
    return h, _cuda(w), _cuda(bias), _cuda(t), ldh


def _head_call(h, ldh, w, bias, t, B, K, act_last, act_prev, kind, thr, out, scratch, mode):
    train, target = mode == "train", mode != "infer"
    f = lambda x: x.data_ptr() if x is not None else None  # noqa: E731
    return L().dlrm_b200_head_fused(
        h.data_ptr(), ldh, w.data_ptr(), bias.data_ptr(), f(t) if target else None, f(out["ws"]), B, K, act_last,
        act_prev, kind, thr, f(out["p"]), f(out["loss"]), f(out["gz"]), f(out["dW"]) if train else None,
        f(out["db"]) if train else None, f(out["gprev"]), out["gprev"].shape[1], f(out["gh"]), f(out["gl"]),
        out["gh"].shape[1], scratch.data_ptr(), _st())


def _head_outputs(B, K, mode):
    """NaN where the mode produces output, the sentinel everywhere else"""
    lo, tr = mode != "infer", mode == "train"
    return dict(ws=_cuda(WS), p=_f32buf(1, B + 1, (1, B)), loss=_f32buf(1, 2, (1, 1) if lo else None),
                gz=_f32buf(1, B + 1, (1, B) if lo else None), dW=_f32buf(1, K + 1, (1, K) if tr else None),
                db=_f32buf(1, 2, (1, 1) if tr else None), gprev=_f32buf(B + 1, K + 2, (B, K) if tr else None),
                gh=_bf16buf(B + 1, K + 4, (B, K) if tr else None), gl=_bf16buf(B + 1, K + 4, (B, K) if tr else None))


def _check_head(B, K, act_last, act_prev, kind, thr, rows, mode, out, h, w, bias, t):
    what = f"head B={B} K={K} act_last={act_last} act_prev={act_prev} loss={kind} thr={thr} rows={rows} {mode}"
    hn, wn, bn, tn = h[:, :K].cpu().numpy(), w.cpu().numpy(), bias.cpu().numpy(), t.cpu().numpy()
    p = out["p"][0, :B].cpu().numpy()
    want, bound = O.head_p(hn, wn, bn, act_last)
    _record("head_p", O.check_within(p, want, bound, what + " p"))
    _outside_untouched(out["p"], (1, B), what + " p")
    if mode == "infer":
        for k in ("loss", "gz", "dW", "db", "gprev", "gh", "gl"):
            _outside_untouched(out[k], (0, 0), what + " " + k)
        return
    per, g, per_b, g_b = O.loss_terms(p, tn, WS, kind, thr, act_last)
    gz = out["gz"][0, :B].cpu().numpy()
    _record("head_gz", O.check_within(gz, g, g_b, what + " gz"))
    _outside_untouched(out["gz"], (1, B), what + " gz")
    depth = O.head_depth(B, rows)
    loss, lb = O.loss_reduce_bound(per, per_b, depth, B)
    _record("head_loss", O.check_within(out["loss"][0, :1].cpu().numpy(), np.array([loss]), lb, what + " loss"))
    _outside_untouched(out["loss"], (1, 1), what + " loss")
    if mode == "loss":
        for k in ("dW", "db", "gprev", "gh", "gl"):
            _outside_untouched(out[k], (0, 0), what + " " + k)
        return
    bw = O.head_backward(hn, wn, gz, act_prev, depth)
    _record("head_dW", O.check_within(out["dW"][0, :K].cpu().numpy(), *bw["dW"], what=what + " dW"))
    _record("head_dW", O.check_within(out["db"][0, :1].cpu().numpy(), np.array([bw["db"][0]]), bw["db"][1],
                                      what + " db"))
    gp = out["gprev"][:B, :K].cpu().numpy()
    _record("head_gprev", O.check_within(gp, *bw["gprev"], what=what + " gprev"))
    hi, lo = O.split_bf16(gp)
    assert np.array_equal(_u16(out["gh"][:B, :K]), hi) and np.array_equal(_u16(out["gl"][:B, :K]), lo), \
        what + ": gprev pair is not the split of gprev"
    for k, inner in (("dW", (1, K)), ("db", (1, 1)), ("gprev", (B, K)), ("gh", (B, K)), ("gl", (B, K))):
        _outside_untouched(out[k], inner, what + " " + k)


def _head_case(B, K, act_last, act_prev, kind, thr, rows, mode, tunable, seed, specials=None):
    """Three calls on one scratch: inputs A, B, A.  Each is checked; the first and third must agree bit for bit (the
    grid-reduction counter is reset by every call, and the result is deterministic)."""
    tunable("head_rows", rows)
    scratch = torch.zeros(int(L().dlrm_b200_head_scratch_bytes(B, K)), dtype=torch.uint8, device=DEV)
    outs = []
    for call, s in enumerate((seed, seed + 1, seed)):
        rng = np.random.default_rng(s)
        h, w, bias, t, ldh = _head_inputs(rng, B, K, act_prev, kind, specials)
        out = _head_outputs(B, K, mode)
        _ok(_head_call(h, ldh, w, bias, t, B, K, act_last, act_prev, kind, thr, out, scratch, mode), "head_fused")
        torch.cuda.synchronize()
        _check_head(B, K, act_last, act_prev, kind, thr, rows, mode, out, h, w, bias, t)
        outs.append(out)
    for k in outs[0]:
        _same_bits(outs[0][k], outs[2][k], f"head: repeated call differs in {k}")


HEAD_BK = [(1, 1), (15, 31), (16, 33), (17, 256), (33, 1000), (2048, 256), (2049, 33), (16, 1), (33, 31),
           (2048, 1000), (1, 1000), (2049, 256), (15, 1), (17, 33)]
HEAD = [(al, ap, kind) for al in (0, 1, 2) for ap in (0, 1, 2) for kind in (0, 1, 2)]


@pytest.mark.parametrize("act_last,act_prev,kind", HEAD)
def test_head_training(tunable, act_last, act_prev, kind):
    i = HEAD.index((act_last, act_prev, kind))
    B, K = HEAD_BK[i % len(HEAD_BK)]
    thr = 0.0 if act_last == O.ACT_SIGMOID else 0.05 if kind != O.LOSS_MSE else 0.0   # BCE needs z in [0, 1]
    _head_case(B, K, act_last, act_prev, kind, thr, (16, 32)[i % 2], "train", tunable, seed=100 + i)


@pytest.mark.parametrize("mode", ["loss", "infer"])
@pytest.mark.parametrize("B,K,rows", [(1, 1, 16), (17, 33, 32), (2049, 256, 16), (2048, 1000, 32)])
def test_head_loss_only_and_inference(tunable, mode, B, K, rows):
    _head_case(B, K, O.ACT_SIGMOID, O.ACT_RELU, O.LOSS_BCE, 0.0, rows, mode, tunable, seed=B + K)


_, _LO, _HI = O.clamp_limits(0.45)
UNIT_SPECIALS = [_LO, _HI, 0.0, 1.0, 0.3, 0.5, 0.7, float(np.nextafter(np.float32(_LO), np.float32(0))),
                 float(np.nextafter(np.float32(_HI), np.float32(1))), 0.45, 0.55]


@pytest.mark.parametrize("act_last", [0, 1, 2])
@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("thr", [0.0, 0.45])
def test_head_saturation_and_clamp_boundary(tunable, act_last, kind, thr):
    """Pre-activations of exactly +-30 and +-100 (sigmoid gives p = 1, 1e-13, 1 and 0: the -100 log clamp and the
    1e-12 floor), and, for the identity and relu heads, p exactly at thr, 1 - thr and their neighbours."""
    if act_last == O.ACT_SIGMOID:
        specials = ([30.0, -30.0, 100.0, -100.0, 0.0] * 7)[:33]
    else:
        specials = (UNIT_SPECIALS * 3)[:33]
    _head_case(33, 31, act_last, O.ACT_SIGMOID, kind, thr, 16 + 16 * (kind % 2), "train", tunable,
               seed=7 + kind, specials=specials)


# ================================================================================================ loss, act_bwd
def _loss_p(rng, n, last_act):
    p = rng.uniform(0, 1, n).astype(np.float32)
    p[:6] = [_LO, _HI, 0.0, 1.0, 0.45, 0.55][:n] if n >= 6 else p[:6]
    if last_act == O.ACT_RELU:
        p[::7] = 0.0
    return p


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 5000])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_loss_fwd_bwd(n, kind):
    rng = np.random.default_rng(n + kind)
    last_act = (n + kind) % 3
    thr = 0.45 if n % 2 else 0.0
    p = _loss_p(rng, n, last_act)
    t = rng.integers(0, 2, n).astype(np.float32) if kind else rng.uniform(0, 1, n).astype(np.float32)
    pd, td, ws = _cuda(p), _cuda(t), _cuda(WS)
    scratch = torch.zeros(1024, dtype=torch.float32, device=DEV)
    per, g, per_b, g_b = O.loss_terms(p, t, WS, kind, thr, last_act)
    loss, lb = O.loss_reduce_bound(per, per_b, O.loss_depth(n), n)
    results = []
    for with_gz in (True, False, True):
        lo_ = _f32buf(1, 2, (1, 1))
        gz = _f32buf(1, n + 1, (1, n) if with_gz else None)
        _ok(L().dlrm_b200_loss_fwd_bwd(pd.data_ptr(), td.data_ptr(), ws.data_ptr(), n, kind, thr, last_act,
                                       lo_.data_ptr(), gz.data_ptr() if with_gz else None, scratch.data_ptr(), _st()),
            "loss_fwd_bwd")
        torch.cuda.synchronize()
        what = f"loss n={n} kind={kind} act={last_act} thr={thr}"
        _record("loss", O.check_within(lo_[0, :1].cpu().numpy(), np.array([loss]), lb, what))
        _outside_untouched(lo_, (1, 1), what + " loss")
        if with_gz:
            _record("loss_gz", O.check_within(gz[0, :n].cpu().numpy(), g, g_b, what + " gz"))
            _outside_untouched(gz, (1, n), what + " gz")
        else:
            _outside_untouched(gz, (0, 0), what + " gz (NULL)")
        results.append((lo_, gz))
    _same_bits(results[0][0], results[1][0], "loss differs with and without gz")
    _same_bits(results[0][1], results[2][1], "loss_fwd_bwd: repeated call differs")


@pytest.mark.parametrize("act_kind", [0, 1, 2])
@pytest.mark.parametrize("thr", [0.45, 0.0, 1.0, -0.5, 1.5])
def test_act_bwd(act_kind, thr):
    rng = np.random.default_rng(int(thr * 10) + 10 + act_kind)
    n = 1000
    y = _loss_p(rng, n, act_kind)
    gy = rng.standard_normal(n).astype(np.float32)
    gz = _f32buf(1, n + 1, (1, n))
    gyd, yd = _cuda(gy), _cuda(y)
    _ok(L().dlrm_b200_act_bwd(gyd.data_ptr(), yd.data_ptr(), gz.data_ptr(), n, act_kind, thr, _st()), "act_bwd")
    torch.cuda.synchronize()
    want, bound = O.act_bwd(gy, y, act_kind, thr)
    _record("act_bwd", O.check_within(gz[0, :n].cpu().numpy(), want, bound, f"act_bwd act={act_kind} thr={thr}"))
    _outside_untouched(gz, (1, n), "act_bwd")


# ================================================================================================ dense optimizer
@pytest.mark.parametrize("n", [1, 255, 257, 5000])
@pytest.mark.parametrize("opt", [0, 1])
def test_dense_update(n, opt):
    rng = np.random.default_rng(n + opt)
    p, g = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
    s = rng.uniform(0, 1, n).astype(np.float32)
    lr, eps = 0.01, 1e-8
    outs = []
    for _ in range(2):
        pd, sd, gd = _cuda(np.append(p, np.float32(SENT))), _cuda(np.append(s, np.float32(SENT))), _cuda(g)
        _ok(L().dlrm_b200_dense_update(pd.data_ptr(), gd.data_ptr(), sd.data_ptr() if opt else None, n, opt, lr, eps,
                                       _st()), "dense_update")
        torch.cuda.synchronize()
        outs.append((pd.cpu().numpy(), sd.cpu().numpy()))
    pw, sw = O.dense_step_f32(p, g, s, opt, lr, eps)
    pk, sk = outs[0]
    assert pk[n] == np.float32(SENT) and sk[n] == np.float32(SENT)
    d = int(O.ulp_diff(pk[:n], pw).max())
    _record("dense_update_ulp", d)
    assert d <= 1, d
    assert int(O.ulp_diff(sk[:n], sw).max()) <= 1
    _same_bits(outs[0][0], outs[1][0], "dense_update: repeated call differs")


LAYERS = [(7, 13), (33, 64), (1, 300), (5, 1)]      # N (K + 1) = 98, 2145, 301, 10: layers end inside a 256-block


def _pack_layers(rng, shapes, slabs, opt, null_grads=False):
    layers, keep = [], []
    for N, K in shapes:
        W, b = _cuda(rng.standard_normal((N, K)).astype(np.float32)), _cuda(rng.standard_normal(N).astype(np.float32))
        sW, sb = _cuda(rng.uniform(0, 1, (N, K)).astype(np.float32)), _cuda(rng.uniform(0, 1, N).astype(np.float32))
        stride = N * K + N + 3
        G = _cuda(rng.standard_normal((slabs, stride)).astype(np.float32))
        ldp = K + 1 + 3
        hi, lo = _bf16buf(N + 1, ldp), _bf16buf(N + 1, ldp)
        d = _lib.DenseLayer()
        d.W, d.b, d.sW, d.sb = W.data_ptr(), b.data_ptr(), sW.data_ptr(), sb.data_ptr()
        if not null_grads:
            d.dW, d.db = G.data_ptr(), G.data_ptr() + 4 * N * K
        d.pack_hi, d.pack_lo = hi.data_ptr(), lo.data_ptr()
        d.slab_stride, d.N, d.K, d.ld_pack, d.num_slabs = stride, N, K, ldp, slabs
        layers.append(d)
        keep.append(dict(W=W, b=b, sW=sW, sb=sb, G=G, hi=hi, lo=lo, N=N, K=K))
    return (_lib.DenseLayer * len(layers))(*layers), keep


def _snap(keep):
    return [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in lay.items()} for lay in keep]


def _run_pack(shapes, slabs, opt, seed, null_grads=False):
    rng = np.random.default_rng(seed)
    arr, keep = _pack_layers(rng, shapes, slabs, opt, null_grads)
    before = _snap(keep)
    _ok(L().dlrm_b200_dense_update_pack(arr, len(shapes), opt, 0.01, 1e-8, _st()), "dense_update_pack")
    torch.cuda.synchronize()
    return before, keep


def _check_pack(shapes, slabs, opt, seed, null_grads=False):
    before, keep = _run_pack(shapes, slabs, opt, seed, null_grads)
    for li, (b0, k) in enumerate(zip(before, keep)):
        N, K = k["N"], k["K"]
        what = f"dense_update_pack layer {li} N={N} K={K} slabs={slabs} opt={opt}"
        G0 = b0["G"].cpu().numpy()
        fold = O.fold_slabs_f32([G0[s, :N * K + N] for s in range(slabs)])
        if opt == -2:
            Gw = G0.copy()
            Gw[0, :N * K + N] = fold
            _same_bits(k["G"], Gw, what + ": fold")
        else:
            _same_bits(k["G"], b0["G"], what + ": gradients written")
        if opt in (-2, -1):
            for name in ("W", "b"):
                _same_bits(k[name], b0[name], what + ": master " + name + " changed")
        else:
            s0 = np.concatenate([b0["sW"].cpu().numpy().ravel(), b0["sb"].cpu().numpy()])
            p0 = np.concatenate([b0["W"].cpu().numpy().ravel(), b0["b"].cpu().numpy()])
            pw, sw = O.dense_step_f32(p0, fold, s0, opt, 0.01, 1e-8)
            pk = np.concatenate([k["W"].cpu().numpy().ravel(), k["b"].cpu().numpy()])
            d = int(O.ulp_diff(pk, pw).max())
            _record("dense_update_ulp", d)
            assert d <= 1, (what, d)
            if opt == O.OPT_RWSADAGRAD:
                sk = np.concatenate([k["sW"].cpu().numpy().ravel(), k["sb"].cpu().numpy()])
                assert int(O.ulp_diff(sk, sw).max()) <= 1, what
        if opt != O.OPT_RWSADAGRAD:
            for name in ("sW", "sb"):
                _same_bits(k[name], b0[name], what + ": Adagrad state changed")
        if opt == -2:
            _outside_untouched(k["hi"], (0, 0), what + ": pack written on fold")
            _outside_untouched(k["lo"], (0, 0), what + ": pack written on fold")
            continue
        hi, lo = O.split_bf16(O.pack_layer(k["W"].cpu().numpy(), k["b"].cpu().numpy()))
        assert np.array_equal(_u16(k["hi"][:N, :K + 1]), hi) and np.array_equal(_u16(k["lo"][:N, :K + 1]), lo), \
            what + ": pack is not the split of [W | b]"
        _outside_untouched(k["hi"], (N, K + 1), what + ": pack hi")
        _outside_untouched(k["lo"], (N, K + 1), what + ": pack lo")
    return keep


@pytest.mark.parametrize("opt", [-2, -1, 0, 1])
@pytest.mark.parametrize("slabs", [1, 2, 3, 4])
def test_dense_update_pack(opt, slabs):
    k1 = _check_pack(LAYERS, slabs, opt, seed=slabs)
    k2 = _check_pack(LAYERS, slabs, opt, seed=slabs)
    for a, b in zip(k1, k2):
        for name in ("W", "b", "sW", "sb", "G", "hi", "lo"):
            _same_bits(a[name], b[name], "dense_update_pack: repeated call differs in " + name)


def test_dense_update_pack_only_reads_no_gradient():
    """optimizer -1 with dW = db = NULL (allowed by the header): refreshes the pack, leaves the masters alone."""
    _check_pack(LAYERS, 2, -1, seed=11, null_grads=True)


def test_dense_update_pack_sixteen_layers():
    rng = np.random.default_rng(12)
    shapes = [(int(rng.integers(1, 40)), int(rng.integers(1, 70))) for _ in range(16)]
    _check_pack(shapes, 3, O.OPT_RWSADAGRAD, seed=13)


def test_dense_update_pack_rejects_before_launch():
    rng = np.random.default_rng(14)
    arr, keep = _pack_layers(rng, [(3, 4)] * 17, 1, 0)
    before = _snap(keep)
    assert "at most 16" in _error(L().dlrm_b200_dense_update_pack(arr, 17, 0, 0.01, 1e-8, _st()))
    assert "optimizer" in _error(L().dlrm_b200_dense_update_pack(arr, 1, -3, 0.01, 1e-8, _st()))
    arr[1].N, arr[1].K = 1 << 16, (1 << 15) - 1         # N (K + 1) = 2^31 parameters
    assert "parameters" in _error(L().dlrm_b200_dense_update_pack(arr, 2, 0, 0.01, 1e-8, _st()))
    torch.cuda.synchronize()
    for b0, k in zip(before, keep):
        for name in ("W", "b", "G", "hi"):
            _same_bits(k[name], b0[name], "rejected call wrote " + name)


# ================================================================================================ split_bf16
def _split_values(rng, n):
    u = [0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000, 0x4B7F8000, 0x00008000, 0x00018000, 0x80008000,
         0x00000001, 0x807FFFFF, 0x007FFFFF, 0x00800000, 0x00000000, 0x80000000, 0x7F7F7FFF, 0x7F7F8000,
         0x7F7FFFFF, 0xFF7F7FFF, 0xFF7F8000, 0x7F7EFFFF, 0x7F7F0000, 0x3F80FFFF, 0x3F807FFF]
    x = np.concatenate([np.array(u, np.uint32).view(np.float32),
                        (rng.standard_normal(n) * 10.0 ** rng.uniform(-30, 30, n)).astype(np.float32)])
    return x[:n]


@pytest.mark.parametrize("M,N,with_lo", [(37, 29, True), (37, 29, False), (300, 257, True), (1, 1, True)])
def test_split_bf16(M, N, with_lo):
    rng = np.random.default_rng(M + N)
    ldx, ldo = N + 4, N + 6
    X, _ = _mat(rng, M, ldx, ldx)
    X[:, :N] = _cuda(_split_values(rng, M * N).reshape(M, N))
    hi, lo = _bf16buf(M + 1, ldo, (M, N)), _bf16buf(M + 1, ldo, (M, N))
    _ok(L().dlrm_b200_split_bf16(X.data_ptr(), ldx, M, N, hi.data_ptr(), lo.data_ptr() if with_lo else None, ldo,
                                 _st()), "split_bf16")
    torch.cuda.synchronize()
    h, lw = O.split_bf16(X[:, :N].cpu().numpy())
    assert np.array_equal(_u16(hi[:M, :N]), h), "split_bf16 hi is not round-to-nearest-even"
    _outside_untouched(hi, (M, N), "split_bf16 hi")
    if with_lo:
        assert np.array_equal(_u16(lo[:M, :N]), lw), "split_bf16 lo"
        _outside_untouched(lo, (M, N), "split_bf16 lo")
    else:
        c = lo.clone()
        c[:M, :N] = SENT16
        assert torch.all(lo[:M, :N] == NAN16), "lo = NULL: lo written"
        _outside_untouched(c, (0, 0), "split_bf16 lo")


# ================================================================================================ SIMT linear
SIMT = [(1, 1, 1), (13, 13, 13), (63, 64, 65), (64, 65, 63), (65, 63, 64), (1024, 13, 64), (13, 1024, 1),
        (1, 65, 1024), (64, 1, 13), (65, 1024, 1024), (1024, 1024, 63), (65535, 13, 13), (65537, 1, 64),
        (13, 65537, 13), (13, 13, 65535), (1, 13, 65537)]


def _simt_operands(rng, shape, aligned, op, act_kind):
    M, N, K = shape
    off = 0 if aligned else 1
    if op == "fwd":
        X, _ = _mat(rng, M, _ld(K, aligned), _ld(K, aligned), off)
        W, _ = _mat(rng, N, _ld(K, aligned), _ld(K, aligned), off, scale=1 / np.sqrt(K))
        return X, W
    if op == "dgrad":
        dY, _ = _mat(rng, M, _ld(N, aligned), _ld(N, aligned), off)
        W, _ = _mat(rng, N, _ld(K, aligned), _ld(K, aligned), off, scale=1 / np.sqrt(N))
        Xa, _ = _mat(rng, M, _ld(K, aligned), _ld(K, aligned), off,
                     {O.ACT_RELU: "relu", O.ACT_SIGMOID: "unit"}.get(act_kind, "normal"))
        if act_kind == O.ACT_RELU:
            Xa.view(-1)[::5] = 0.0
        return dY, W, Xa
    dY, _ = _mat(rng, M, _ld(N, aligned), _ld(N, aligned), off)
    X, _ = _mat(rng, M, _ld(K, aligned), _ld(K, aligned), off)
    return dY, X


def _simt_run(shape, aligned, op, act_kind, seed):
    M, N, K = shape
    rng = np.random.default_rng(seed)
    ops = _simt_operands(rng, shape, aligned, op, act_kind)
    off = 0 if aligned else 1
    if op == "fwd":
        X, W = ops
        bias = _cuda(rng.standard_normal(N + off).astype(np.float32))[off:]
        ldy = _ld(N, aligned)
        Y = _f32buf(M + 1, ldy, (M, N))
        _ok(L().dlrm_b200_linear_fwd(X.data_ptr(), X.shape[1], W.data_ptr(), W.shape[1], bias.data_ptr(), Y.data_ptr(),
                                     ldy, M, N, K, act_kind, 0, _st()), "linear_fwd")
        torch.cuda.synchronize()
        want, bound = O.linear_fwd(X[:, :K].cpu().numpy(), W[:, :K].cpu().numpy(), bias.cpu().numpy(), act_kind)
        return [(Y, (M, N), want, bound, "simt_fwd")]
    if op == "dgrad":
        dY, W, Xa = ops
        lddx = _ld(K, aligned)
        dX = _f32buf(M + 1, lddx, (M, K))
        _ok(L().dlrm_b200_linear_dgrad(dY.data_ptr(), dY.shape[1], W.data_ptr(), W.shape[1], Xa.data_ptr(),
                                       Xa.shape[1], act_kind, dX.data_ptr(), lddx, M, N, K, 0, _st()), "linear_dgrad")
        torch.cuda.synchronize()
        want, bound = O.linear_dgrad(dY[:, :N].cpu().numpy(), W[:, :K].cpu().numpy(), Xa[:, :K].cpu().numpy(),
                                     act_kind)
        return [(dX, (M, K), want, bound, "simt_dgrad")]
    dY, X = ops
    lddw = _ld(K, aligned)
    dW = _f32buf(N + 1, lddw, (N, K))
    with_db = act_kind != O.ACT_NONE                      # wgrad has no activation: the knob selects dbias on / off
    db = _f32buf(1, N + 1, (1, N))
    _ok(L().dlrm_b200_linear_wgrad(dY.data_ptr(), dY.shape[1], X.data_ptr(), X.shape[1], dW.data_ptr(), lddw,
                                   db.data_ptr() if with_db else None, M, N, K, 0, _st()), "linear_wgrad")
    torch.cuda.synchronize()
    (w_, wb), (d_, dbb) = O.linear_wgrad(dY[:, :N].cpu().numpy(), X[:, :K].cpu().numpy())
    res = [(dW, (N, K), w_, wb, "simt_wgrad")]
    if with_db:
        res.append((db, (1, N), d_[None, :], dbb[None, :], "simt_dbias"))
    else:
        assert torch.isnan(db[0, :N]).all(), "dbias = NULL: dbias written"
    return res


@pytest.mark.parametrize("op", ["fwd", "dgrad", "wgrad"])
@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("shape", SIMT)
def test_simt_linear(shape, aligned, op):
    i = SIMT.index(shape)
    act_kind = (i + (op == "dgrad")) % 3
    seed = i * 10 + aligned
    res = _simt_run(shape, aligned, op, act_kind, seed)
    again = _simt_run(shape, aligned, op, act_kind, seed)
    for (buf, inner, want, bound, fam), (buf2, *_rest) in zip(res, again):
        got = buf[:inner[0], :inner[1]].cpu().numpy()
        _record(fam, O.check_within(got, want, bound, f"{fam} M,N,K={shape} aligned={aligned} act={act_kind}"))
        _outside_untouched(buf, inner, fam)
        _same_bits(buf, buf2, fam + ": repeated call differs")


def test_simt_wgrad_with_empty_batch_gives_exact_zeros():
    rng = np.random.default_rng(15)
    N, K = 65, 13
    dY, _ = _mat(rng, 1, N, N)
    X, _ = _mat(rng, 1, K, K)
    dW, db = _f32buf(N + 1, K + 3, (N, K)), _f32buf(1, N + 1, (1, N))
    _ok(L().dlrm_b200_linear_wgrad(dY.data_ptr(), N, X.data_ptr(), K, dW.data_ptr(), K + 3, db.data_ptr(), 0, N, K, 0,
                                   _st()), "linear_wgrad")
    torch.cuda.synchronize()
    assert torch.all(dW[:N, :K] == 0) and torch.all(db[0, :N] == 0)
    _outside_untouched(dW, (N, K), "wgrad M=0 dW")
    _outside_untouched(db, (1, N), "wgrad M=0 db")
