"""256-row wgmma GEMM tiles (tile_m = 256) against 128-row tiles: every output buffer bit for bit, pads and guard
rows included, at the cfg3 forward / dgrad shapes (batch 8192) and at the edges (ragged M and N, every epilogue
option, all four operand majornesses, bf16x3 and bf16); the same outputs against float64 references; which plans
the automatic choice makes 256 rows high; and the tile heights plan_create refuses."""
import pytest
import torch

from gemm_tc_check import ACC_MAX, DEV, SENTINEL_BF16, U, split

pytestmark = pytest.mark.gpu

B3 = 8192      # the cfg3 batch


def _cases():
    c = []
    # the cfg3 plans as the engine builds them: forward (K-major, bias + relu, (hi, lo) out; the last top layer fp32),
    # dgrad (B MN-major, relu-gradient mask, (hi, lo) out; top layer 0 fp32 into the interaction gradient)
    for x3 in (1, 0):
        c += [
            dict(name="top_fwd0", M=B3, N=1024, K=479, x3=x3, a_mn=0, b_mn=0, act=1, bias=1, outs="bf"),
            dict(name="top_fwd1", M=B3, N=1024, K=1024, x3=x3, a_mn=0, b_mn=0, act=1, bias=1, outs="bf"),
            dict(name="top_fwd2", M=B3, N=512, K=1024, x3=x3, a_mn=0, b_mn=0, act=1, bias=1, outs="bf"),
            dict(name="top_fwd3", M=B3, N=256, K=512, x3=x3, a_mn=0, b_mn=0, act=1, bias=1, outs="f32"),
            dict(name="top_dgrad0", M=B3, N=479, K=1024, x3=x3, a_mn=0, b_mn=1, outs="f32"),
            dict(name="top_dgrad1", M=B3, N=1024, K=1024, x3=x3, a_mn=0, b_mn=1, mask=1, outs="bf"),
            dict(name="top_dgrad2", M=B3, N=1024, K=512, x3=x3, a_mn=0, b_mn=1, mask=1, outs="bf"),
            dict(name="top_dgrad3", M=B3, N=512, K=256, x3=x3, a_mn=0, b_mn=1, mask=1, outs="bf"),
            dict(name="bot_fwd0", M=B3, N=512, K=13, x3=x3, a_mn=0, b_mn=0, act=1, bias=1, outs="bf"),
        ]
    # ragged M (not a multiple of 256, a tile that is half empty, fewer rows than one tile), N tails
    for M in (B3 - 64, 384, 200):
        c.append(dict(name="ragged_m", M=M, N=256, K=200, x3=1, a_mn=0, b_mn=0, act=1, bias=1, outs="f32 bf T"))
    for N in (479, 1025):
        c.append(dict(name="n_tail", M=1024, N=N, K=136, x3=1, a_mn=0, b_mn=1, mask=1, outs="f32 bf T"))
    # every epilogue option
    c += [
        dict(name="sigmoid", M=600, N=200, K=256, x3=1, a_mn=0, b_mn=0, act=2, bias=1, outs="f32 bf"),
        dict(name="mask_sigmoid", M=600, N=200, K=256, x3=1, a_mn=0, b_mn=1, mask=2, outs="f32 bf T"),
        dict(name="hi_only", M=600, N=200, K=256, x3=1, a_mn=0, b_mn=0, act=1, outs="bf T", no_lo=True),
        dict(name="f32_unaligned_rows", M=600, N=131, K=256, x3=1, a_mn=0, b_mn=0, outs="f32", ldf_exact=1),
    ]
    # all four majornesses, with a K tail inside a 32-wide and inside a 64-wide k block
    for a_mn in (0, 1):
        for b_mn in (0, 1):
            for K in (40, 328):
                for x3 in (1, 0):
                    c.append(dict(name="major", M=520, N=300, K=K, x3=x3, a_mn=a_mn, b_mn=b_mn, outs="f32 bf T"))
    return c


CASES = _cases()


def _id(c):
    return "-".join("%s%s" % (k, str(v).replace(" ", "+")) for k, v in c.items())


def _operands(case):
    M, N, K = case["M"], case["N"], case["K"]
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    A = torch.randn(M, K, generator=g)
    Bm = torch.randn(N, K, generator=g)
    if case.get("act") == 2:
        A = A * (2.0 / K ** 0.5)         # sigmoid out of saturation
    Ah, Al = split(A)
    Bh, Bl = split(Bm)
    bias = torch.randn(N, generator=g) if case.get("bias") else None
    ymask = None
    if case.get("mask"):
        ymask = torch.rand(M, N, generator=g) - (0.3 if case["mask"] == 1 else 0.0)
    return A, Bm, Ah, Al, Bh, Bl, bias, ymask


def _lay(t, mn):
    """bf16 [rows, K] -> device, K-major or MN-major ([K, rows]), leading dimension padded to 8 with NaN."""
    if mn:
        t = t.t().contiguous()
    r, cols = t.shape
    out = torch.full((r, (cols + 7) // 8 * 8 + 8), float("nan"), dtype=t.dtype)
    out[:, :cols] = t
    return out.to(DEV)


class _Inputs:
    def __init__(self, case):
        self.case = case
        A, Bm, Ah, Al, Bh, Bl, bias, ymask = _operands(case)
        self.host = (A, Bm, Ah, Al, Bh, Bl, bias, ymask)
        self.dAh, self.dAl = _lay(Ah, case["a_mn"]), _lay(Al, case["a_mn"])
        self.dBh, self.dBl = _lay(Bh, case["b_mn"]), _lay(Bl, case["b_mn"])
        self.dbias = bias.to(DEV) if bias is not None else None
        if ymask is not None:
            mh, ml = split(ymask)
            self.mh, self.ml = _lay(mh, 0), _lay(ml, 0)


def _run(inp, tile_m):
    """Runs the plan at this tile height on fresh sentinel-filled outputs; returns (outputs, info)."""
    from dlrm_b200 import _lib

    c = inp.case
    M, N, K = c["M"], c["N"], c["K"]
    kw = dict(A_hi=inp.dAh.data_ptr(), A_lo=inp.dAl.data_ptr(), lda=inp.dAh.stride(0), a_mn_major=c["a_mn"],
              B_hi=inp.dBh.data_ptr(), B_lo=inp.dBl.data_ptr(), ldb=inp.dBh.stride(0), b_mn_major=c["b_mn"],
              M=M, N=N, K=K, mode_x3=c["x3"], split_k=1, act=c.get("act", 0), tile_n=128, tile_m=tile_m)
    if c.get("mask"):
        kw.update(mask_act=c["mask"], mask_hi=inp.mh.data_ptr(), mask_lo=inp.ml.data_ptr(), ldmask=inp.mh.stride(0))
    if inp.dbias is not None:
        kw.update(bias=inp.dbias.data_ptr())
    outs = {}
    ldf = N if c.get("ldf_exact") else (N + 3) // 4 * 4 + 4
    if "f32" in c["outs"]:
        outs["f32"] = torch.full((M + 2, ldf), float("nan"), device=DEV)
        kw.update(out_f32=outs["f32"].data_ptr(), ld_f32=ldf, slab_stride=M * ldf)
    no_lo = c.get("no_lo", False)
    if "bf" in c["outs"]:
        ldo = (N + 7) // 8 * 8 + 8
        outs["hi"] = torch.full((M + 2, ldo), SENTINEL_BF16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
        outs["lo"] = torch.full_like(outs["hi"], 0).view(torch.int16).fill_(SENTINEL_BF16).view(torch.bfloat16)
        kw.update(out_hi=outs["hi"].data_ptr(), out_lo=None if no_lo else outs["lo"].data_ptr(), ld_out=ldo)
    if "T" in c["outs"]:
        ldt = (M + 7) // 8 * 8 + 8
        outs["Thi"] = torch.full((N + 2, ldt), SENTINEL_BF16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
        outs["Tlo"] = torch.full_like(outs["Thi"], 0).view(torch.int16).fill_(SENTINEL_BF16).view(torch.bfloat16)
        kw.update(outT_hi=outs["Thi"].data_ptr(), outT_lo=None if no_lo else outs["Tlo"].data_ptr(), ld_outT=ldt)
    plan = _lib.GemmTcPlan(**kw)
    info = plan.info()
    plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return outs, info


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _check_f64(inp, outs):
    """The outputs against float64: fp32 within the fp32-accumulation bound of the products the kernel forms (as
    gemm_tc_check), (hi + lo) within 3e-5 (x3) / 1e-5 (bf16) of sum |a||b| plus the split's own representation error."""
    c = inp.case
    M, N = c["M"], c["N"]
    A, Bm, Ah, Al, Bh, Bl, bias, ymask = (t.to(DEV).double() if t is not None else None for t in inp.host)
    if c["x3"]:
        ref, ref3 = A @ Bm.t(), Ah @ Bh.t() + Ah @ Bl.t() + Al @ Bh.t()
        scale3 = Ah.abs() @ Bh.abs().t() + Ah.abs() @ Bl.abs().t() + Al.abs() @ Bh.abs().t()
    else:
        ref = ref3 = Ah @ Bh.t()
        scale3 = Ah.abs() @ Bh.abs().t()
    scale = (A.abs() @ Bm.abs().t()).clamp_min(1e-30)
    if bias is not None:
        ref, ref3 = ref + bias[None, :], ref3 + bias[None, :]
        scale, scale3 = scale + bias.abs()[None, :], scale3 + bias.abs()[None, :]
    act, mask = c.get("act", 0), c.get("mask", 0)
    want = ref.clamp_min(0) if act == 1 else torch.sigmoid(ref) if act == 2 else ref
    if mask:
        mh, ml = split(ymask.float())
        y = mh.double() + ml.double()
        want = want * ((mh.double() > 0).double() if mask == 1 else (1 - y) * y)
    denom = scale if act != 2 else scale.clamp_min(1.0)
    tol = 3e-5 if c["x3"] else 1e-5
    if "f32" in outs:
        got = outs["f32"][:M, :N].double()
        assert ((got - want).abs() / denom).max().item() <= tol
        if act != 2 and mask != 2:
            n = (3 if c["x3"] else 1) * c["K"] + 1
            ref3a = ref3.clamp_min(0) if act == 1 else ref3
            if mask == 1:
                ref3a = ref3a * (split(ymask.float())[0].double() > 0).double()
            acc = ((got - ref3a).abs() / (n ** 0.5 * U * scale3).clamp_min(1e-300)).max().item()
            assert acc <= ACC_MAX, acc
    no_lo = c.get("no_lo", False)
    tol_bf = tol + (2.0 ** -8 if no_lo else 2e-5)
    if "hi" in outs:
        got = outs["hi"][:M, :N].double() + (0 if no_lo else outs["lo"][:M, :N].double())
        assert ((got - want).abs() / denom).max().item() <= tol_bf
    if "Thi" in outs:
        got = (outs["Thi"][:N, :M].double() + (0 if no_lo else outs["Tlo"][:N, :M].double())).t()
        assert ((got - want).abs() / denom).max().item() <= tol_bf


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_tall_tile_bit_identical(case):
    inp = _Inputs(case)
    tall, info_tall = _run(inp, 256)
    short, info_short = _run(inp, 128)
    assert info_tall["tile_m"] == 256 and info_short["tile_m"] == 128, (info_tall, info_short)
    assert info_tall["ctas"] == -(-case["N"] // 128) * -(-case["M"] // 256), info_tall
    for k in tall:
        assert torch.equal(_bits(tall[k]), _bits(short[k])), k
    _check_f64(inp, tall)


def test_cfg3_plan_heights():
    """A cfg3 engine at batch 8192: 256-row tiles for the forward and dgrad plans whose 256 x 128 grid keeps >= 120
    CTAs (the engine pads operand rows to 128 bytes); 128 rows for the rest (top forward 3 and the narrow bottom
    layers, whose grids would be 64 CTAs or fewer, and every split-K weight-gradient plan)."""
    from dlrm_b200 import mlperf as Mp
    from dlrm_b200.engine import Engine

    ln_top = Mp.ln_top()
    eng = Engine(Mp.DIM, [1000] * len(Mp.TABLE_ROWS), list(Mp.LN_BOT), ln_top, loss="bce",
                 sigmoid_top=len(ln_top) - 2, device=DEV, max_batch=B3, gemm="tc")
    eng._tc_setup(B3)
    got = {(kind, which, i): p.info()["tile_m"] for kind in ("fwd", "dgrad", "wgrad")
           for (which, i), p in eng.tc_plans[kind].items()}
    tall = {("fwd", "top", 0), ("fwd", "top", 1), ("fwd", "top", 2),
            ("dgrad", "top", 0), ("dgrad", "top", 1), ("dgrad", "top", 2), ("dgrad", "top", 3),
            # the bottom MLP's layers with 512 outputs: 128 CTAs at 256 rows
            ("fwd", "bot", 0), ("dgrad", "bot", 1)}
    want = {k: 256 if k in tall else 128 for k in got}
    assert got == want


def test_tile_m_refusals():
    from dlrm_b200 import _lib

    bf = torch.bfloat16
    a = torch.zeros((512, 256), dtype=bf, device=DEV)
    f = torch.zeros((8, 512, 512), device=DEV)
    base = dict(A_hi=a.data_ptr(), A_lo=a.data_ptr(), lda=256, a_mn_major=0, B_hi=a.data_ptr(), B_lo=a.data_ptr(),
                ldb=256, b_mn_major=0, M=512, N=512, K=256, mode_x3=1, split_k=1, out_f32=f.data_ptr(), ld_f32=512,
                slab_stride=512 * 512)
    for over, msg in ((dict(tile_m=64), "tile_m must be"), (dict(tile_m=256, split_k=4), "no split-K"),
                      (dict(tile_m=256, tile_n=64), "128-wide tile")):
        with pytest.raises(RuntimeError, match=msg):
            _lib.GemmTcPlan(**dict(base, **over))
    assert _lib.GemmTcPlan(**dict(base, tile_n=128, tile_m=256)).info()["tile_m"] == 256
    assert _lib.GemmTcPlan(**dict(base, tile_n=128)).info()["tile_m"] == 128   # 2 x 4 CTAs: too few for 256 rows
    big = torch.zeros((8192, 256), dtype=bf, device=DEV)
    fb = torch.zeros((8192, 1024), device=DEV)
    wide = dict(base, A_hi=big.data_ptr(), A_lo=big.data_ptr(), M=8192, N=1024, out_f32=fb.data_ptr(), ld_f32=1024,
                slab_stride=8192 * 1024)
    assert _lib.GemmTcPlan(**dict(wide, B_hi=fb.data_ptr(), B_lo=fb.data_ptr(), ldb=1024,
                                  b_mn_major=1)).info()["tile_m"] == 256
    assert _lib.GemmTcPlan(**dict(wide, B_hi=fb.data_ptr(), B_lo=fb.data_ptr(), ldb=256)).info()["tile_m"] == 256
    # a K-major operand whose rows are not 128-byte aligned keeps 128 rows
    assert _lib.GemmTcPlan(**dict(wide, B_hi=fb.data_ptr(), B_lo=fb.data_ptr(), ldb=264)).info()["tile_m"] == 128
    odd = torch.zeros((8192, 264), dtype=bf, device=DEV)
    assert _lib.GemmTcPlan(**dict(wide, A_hi=odd.data_ptr(), A_lo=odd.data_ptr(), lda=264, B_hi=fb.data_ptr(),
                                  B_lo=fb.data_ptr(), ldb=1024, b_mn_major=1)).info()["tile_m"] == 128
