"""wgmma GEMM plans at the shapes where a plan goes wrong: uneven split-K, K tails inside a split, rings deeper than
a split, ragged M / N, every tile width x majorness, poisoned operand pads -- one pytest id per case, all through
gemm_tc_check.run_case (float64 references, untouched-output sentinels, two bit-identical runs, the
fp32-accumulation bound) -- and the argument errors plan_create refuses."""
import pytest
import torch

from gemm_tc_check import DEV, run_case

pytestmark = pytest.mark.gpu
WG = dict(x3=1, a_mn=1, b_mn=1, outs="f32 col")     # the weight-gradient form: both operands MN-major, slabs + column


def _cases():
    c = []
    # uneven split-K: (k blocks, splits asked) -> last split shorter / fewer slabs than asked / ring deeper than a split
    for num_kb, sk in [(5, 2), (9, 8), (11, 8), (13, 4), (33, 8), (3, 8)]:
        c.append(dict(M=160, N=70, K=64 * num_kb, split_k=sk, **WG))
        c.append(dict(M=160, N=70, K=64 * num_kb, split_k=sk, x3=0, a_mn=0, b_mn=0, outs="f32"))
    for tail in (8, 56):                                 # the last split ends in a K tail
        c.append(dict(M=200, N=33, K=64 * 10 + tail, split_k=8, poison=True, **WG))
        c.append(dict(M=200, N=33, K=64 * 10 + tail, split_k=8, x3=1, a_mn=0, b_mn=1, outs="f32", poison=True))
    c.append(dict(M=130, N=40, K=40, split_k=4, poison=True, **WG))           # K < 64 with splits asked
    c.append(dict(M=130, N=40, K=8, x3=1, a_mn=0, b_mn=0, outs="f32 bf T", poison=True))
    c.append(dict(M=1024, N=14, K=700, split_k=8, poison=True, **WG))         # the engine's tail batch
    for M in (1, 63, 64, 65, 127, 129):
        c.append(dict(M=M, N=72, K=136, x3=1, a_mn=0, b_mn=0, act=1, outs="f32 bf T", bias=1, poison=True))
        c.append(dict(M=M, N=72, K=136, split_k=2, poison=True, **WG))
    for N in (1, 8, 31, 33, 65, 127, 129):
        c.append(dict(M=140, N=N, K=200, x3=1, a_mn=0, b_mn=1, mask=1, outs="f32 bf T", poison=True))
        c.append(dict(M=140, N=N, K=200, x3=0, a_mn=0, b_mn=0, outs="bf", poison=True))
    for tn in (32, 64, 128):
        for a_mn, b_mn in [(0, 0), (0, 1), (1, 0), (1, 1)]:
            c.append(dict(M=200, N=150, K=328, x3=1, a_mn=a_mn, b_mn=b_mn, tile_n=tn, outs="f32 bf", poison=True))
    c.append(dict(M=96, N=71, K=192, split_k=3, ldf_exact=1, poison=True, **WG))   # fp32 rows not 16-byte aligned
    c.append(dict(M=99, N=64, K=128, x3=1, a_mn=0, b_mn=1, mask=2, outs="bf T", poison=True))
    # K-major operands whose NaN pad starts inside a 16-byte segment (K % 8 != 0), one side and both
    for K in (13, 70, 134, 257):
        for a_mn, b_mn in [(0, 0), (0, 1), (1, 0)]:
            c.append(dict(M=150, N=90, K=K, x3=1, a_mn=a_mn, b_mn=b_mn, outs="f32 bf", poison=True))
        c.append(dict(M=150, N=90, K=K, x3=0, a_mn=0, b_mn=0, act=1, outs="f32", bias=1, poison=True))
    c.append(dict(M=150, N=90, K=64 * 9 + 13, x3=1, a_mn=0, b_mn=0, split_k=4, outs="f32", poison=True))  # tail in the last split
    c.append(dict(M=150, N=90, K=64 * 4 + 6, x3=0, a_mn=0, b_mn=0, split_k=8, outs="f32", poison=True))
    # values: every lo exactly 0; magnitudes 2^+-60 (the products stay O(1))
    for vals in ("bf16", "big"):
        c.append(dict(M=140, N=100, K=200, x3=1, a_mn=0, b_mn=0, act=1, outs="f32 bf T", vals=vals))
        c.append(dict(M=140, N=100, K=448, split_k=4, vals=vals, **WG))
    # masks: -0.0, +0.0, the smallest bf16 of either sign (relu); exactly 0 and 1 (sigmoid); in the 16-byte path, with a
    # leading dimension that is not a multiple of 8, and from a base that is only 2-byte aligned (element-wise path)
    for layout in (dict(), dict(mask_ld=3), dict(mask_off=1), dict(mask_ld=5, mask_off=1)):
        c.append(dict(M=140, N=96, K=128, x3=1, a_mn=0, b_mn=1, mask=1, outs="f32 bf", mask_edge=True, poison=True, **layout))
        c.append(dict(M=140, N=70, K=128, x3=1, a_mn=0, b_mn=1, mask=2, outs="f32 bf", mask_edge=True, poison=True, **layout))
    # hi outputs alone
    c.append(dict(M=140, N=96, K=128, x3=1, a_mn=0, b_mn=0, act=1, outs="bf T", no_lo=True))
    c.append(dict(M=77, N=70, K=136, x3=0, a_mn=0, b_mn=1, mask=1, outs="f32 bf T", no_lo=True, poison=True))
    return c


CASES = _cases()


def _id(c):
    return "-".join("%s%s" % (k, str(v).replace(" ", "+")) for k, v in c.items())


@pytest.fixture(scope="module")
def worst():
    """Worst err / tolerance and worst accumulation ratio per precision over the cases that ran, printed once."""
    w = {}
    yield w
    print("\nwgmma GEMM worst ratios:", {k: "%.3g" % v for k, v in sorted(w.items())})


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_plan(case, worst):
    r = run_case(**case)
    fam = "x3" if case["x3"] else "x1"
    worst[fam + " err/tol"] = max(worst.get(fam + " err/tol", 0.0), r.err / r.tol if r.tol else float("inf"))
    if r.acc is not None:
        worst[fam + " acc"] = max(worst.get(fam + " acc", 0.0), r.acc)
    print(r.name, "err/tol=%.3g" % (r.err / r.tol if r.tol else float("inf")), r.detail)
    assert r.ok, "%s: err=%.3e tol=%.1e %s" % (r.name, r.err, r.tol, r.detail)
    if case.get("tile_n") == 32 and case["b_mn"]:
        assert r.info["tile_n"] == 64, r.info          # MN-major boxes are 64 wide: the plan widens the tile


# ------------------------------------------------------------------------------------------ refusals
def _desc(**over):
    bf = torch.bfloat16
    M, N, K = 64, 40, 128
    t = dict(a=torch.zeros((M, K), dtype=bf, device=DEV), b=torch.zeros((N, K), dtype=bf, device=DEV),
             f=torch.zeros((8, M, N), device=DEV), o=torch.zeros((M, N), dtype=bf, device=DEV),
             c=torch.zeros((8, M), device=DEV))
    kw = dict(A_hi=t["a"].data_ptr(), A_lo=t["a"].data_ptr(), lda=K, a_mn_major=0, B_hi=t["b"].data_ptr(),
              B_lo=t["b"].data_ptr(), ldb=K, b_mn_major=0, M=M, N=N, K=K, mode_x3=1, split_k=1,
              out_f32=t["f"].data_ptr(), ld_f32=N, slab_stride=M * N)
    for k, v in over.items():
        kw[k] = v(t) if callable(v) else v
    return kw, t


REFUSALS = {
    "empty": (dict(M=0), "empty problem"),
    "null_lo_x3": (dict(A_lo=None), "NULL operand"),
    "misaligned_operand": (dict(A_hi=lambda t: t["a"].data_ptr() + 2), "16-byte"),
    "ld_not_multiple_of_8": (dict(lda=132), "16-byte"),
    "ld_out_not_multiple_of_8": (dict(out_hi=lambda t: t["o"].data_ptr(), ld_out=36), "ld_out"),
    "split_k_bf16_output": (dict(split_k=2, out_hi=lambda t: t["o"].data_ptr(), ld_out=40), "split-K"),
    "split_k_activation": (dict(split_k=2, act=1), "split-K"),
    "split_k_bias": (dict(split_k=2, bias=lambda t: t["c"].data_ptr()), "split-K"),
    "mask_without_pointer": (dict(mask_act=1), "mask_hi"),
    "out_col_without_out_f32": (dict(out_f32=None, out_col=lambda t: t["c"].data_ptr(), col_index=39, col_slab_stride=64),
                                "out_col needs out_f32"),
    "col_index_negative": (dict(out_col=lambda t: t["c"].data_ptr(), col_index=-1, col_slab_stride=64), "last column"),
    "col_index_past_n": (dict(out_col=lambda t: t["c"].data_ptr(), col_index=40, col_slab_stride=64), "last column"),
    "col_index_inside": (dict(out_col=lambda t: t["c"].data_ptr(), col_index=7, col_slab_stride=64), "last column"),
}


@pytest.mark.parametrize("what", sorted(REFUSALS))
def test_plan_create_refuses(what):
    from dlrm_b200 import _lib

    over, msg = REFUSALS[what]
    kw, keep = _desc(**over)
    with pytest.raises(RuntimeError, match=msg):
        _lib.GemmTcPlan(**kw)


def test_plan_create_accepts_the_unmodified_descriptor():
    from dlrm_b200 import _lib

    kw, keep = _desc()
    assert _lib.GemmTcPlan(**kw).info()["splits"] == 1
