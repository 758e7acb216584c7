"""Exhaustive check of the wgmma GEMM (dlrm_b200_gemm_tc_*) against float64 references.
Usable as a CLI (full table, never stops at the first failure -- one GPU call tells everything):

    python tests/gemm_tc_check.py [report.txt]

and from pytest (tests/test_gpu_gemm_tc.py).  Test infrastructure."""
import collections
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DEV = "cuda:0"


def split(x: torch.Tensor):
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


SENTINEL_BF16 = 0x7FC1          # a NaN no kernel produces: what an output element holds until it is written
U = 2.0 ** -24
# Largest accepted fp32-accumulation error in units of sqrt(n) 2^-24 sum|a||b| (n addends).  Empirical: the worst
# case of this file and of tests/test_gpu_gemm_tc_edges.py measures 0.59 on an H100 (K from 8 to 2112, both
# precisions, 1 to 8 splits); a k block dropped or read twice moves the sum by about sum|a||b| / num_kb, hundreds of
# times this at every K the suite runs.
ACC_MAX = 2.0


def sentinel(shape):
    return torch.full(shape, SENTINEL_BF16, dtype=torch.int16, device=DEV).view(torch.bfloat16)


def untouched(t):
    return bool((t.view(torch.int16) == SENTINEL_BF16).all())


Result = collections.namedtuple("Result", "name err tol ok detail info acc")


def pad_cols(t: torch.Tensor, mult=8, fill=0.0, extra=0):
    """[r, c] -> [r, ld] with ld = c rounded up to `mult`, plus `extra` columns, the pad holding `fill`."""
    r, c = t.shape
    cp = (c + mult - 1) // mult * mult + extra
    out = torch.full((r, cp), fill, dtype=t.dtype, device=t.device)
    out[:, :c] = t
    return out


def run_case(M, N, K, x3, a_mn, b_mn, tile_n=0, split_k=1, act=0, mask=0, outs="f32", seed=0, bias=0, ldf_exact=0,
             poison=False, vals="", mask_edge=False, mask_ld=0, mask_off=0, no_lo=False):
    """Returns Result(name, max_rel_err, tolerance, ok, detail, info, acc).  Every plan runs twice (bit-identical
    outputs) and must leave every output element outside [M, N] -- leading-dimension pads, guard rows, the diverted
    column, slabs the plan does not write -- as it found it.
      poison     the operands' and the mask's pads hold NaN, and every pad is at least 8 elements wide
      vals       "bf16": operands exactly representable in bf16 (every lo is 0);  "big": A scaled by 2^60, B by 2^-60
      mask_edge  the mask is made of the values where a mask test goes wrong: relu -0.0, +0.0, the smallest positive
                 and negative bf16, +-1; sigmoid exactly 0, exactly 1, 0.5 and random values
      mask_ld    extra mask columns (a leading dimension that is not a multiple of 8);  mask_off: mask base offset in
                 elements (1: 2-byte aligned only)
      no_lo      out_lo / outT_lo are NULL: the bf16 outputs are hi alone
    The fp32 output of a plan without sigmoid is also compared with the exact value of the products the kernel forms
    (ref3): acc = err / (sqrt(n) 2^-24 sum|a||b|), n the number of addends, must stay under ACC_MAX."""
    from dlrm_b200 import _lib

    name = (f"M{M} N{N} K{K} x3={x3} a_mn={a_mn} b_mn={b_mn} tn={tile_n} sk={split_k} act={act} mask={mask} {outs}"
            + (" bias" if bias else "") + (" ldf=N" if ldf_exact else "") + (" poison" if poison else "")
            + (" " + vals if vals else "") + (" mask_edge" if mask_edge else "")
            + (f" mask_ld+{mask_ld}" if mask_ld else "") + (f" mask_off={mask_off}" if mask_off else "")
            + (" no_lo" if no_lo else ""))
    fill, extra = (float("nan"), 8) if poison else (0.0, 0)
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(N, K, generator=g)
    # awkward magnitudes: exercise the lo terms
    A = A * (1 + 0.01 * torch.randn(M, K, generator=g))
    if act == 2:  # keep sigmoid out of saturation so its absolute error is meaningful
        A = A * (2.0 / K ** 0.5)
    if vals == "bf16":
        A, B = A.bfloat16().float(), B.bfloat16().float()
    elif vals == "big":
        A, B = A * 2.0 ** 60, B * 2.0 ** -60
    Ah, Al = split(A)
    Bh, Bl = split(B)
    # operands in the requested majorness
    def lay(h, l, mn):
        if mn:
            h, l = h.t().contiguous(), l.t().contiguous()
        return pad_cols(h, fill=fill, extra=extra).to(DEV), pad_cols(l, fill=fill, extra=extra).to(DEV)
    dAh, dAl = lay(Ah, Al, a_mn)
    dBh, dBl = lay(Bh, Bl, b_mn)
    if x3:
        ref = A.double() @ B.double().t()
        # what hi*hi + hi*lo + lo*hi computes exactly:
        ref3 = (Ah.double() @ Bh.double().t() + Ah.double() @ Bl.double().t() + Al.double() @ Bh.double().t())
    else:
        ref = Ah.double() @ Bh.double().t()
        ref3 = ref
    bvec = None
    if bias:
        bvec = torch.randn(N, generator=g)
        ref, ref3 = ref + bvec.double()[None, :], ref3 + bvec.double()[None, :]
        dbias = bvec.to(DEV)
    scale = (A.double().abs() @ B.double().abs().t()).clamp_min(1e-30)
    if bias:
        scale = scale + bvec.double().abs()[None, :]
    ymask = None
    if mask:
        ymask = torch.rand(M, N, generator=g) - 0.3 if mask == 1 else torch.rand(M, N, generator=g)
        if mask_edge:
            tiny = 2.0 ** -133                                  # the smallest positive bf16 (a subnormal)
            pick = torch.tensor([-0.0, 0.0, tiny, -tiny, 1.0, -1.0] if mask == 1 else [0.0, 1.0, 0.5, float("nan")])
            chosen = pick[torch.randint(0, pick.numel(), (M, N), generator=g)]
            ymask = torch.where(torch.isnan(chosen), ymask, chosen)
        mh, ml = split(ymask)

        def lay_mask(t):     # [M, ld] view that starts mask_off elements into its buffer; ld % 8 != 0 with mask_ld
            t = pad_cols(t, fill=fill, extra=extra)
            buf = torch.full((M * (t.shape[1] + mask_ld) + mask_off,), fill, dtype=t.dtype)
            v = buf[mask_off:].view(M, t.shape[1] + mask_ld)
            v[:, :N] = t[:, :N]
            return buf.to(DEV)[mask_off:].view(M, t.shape[1] + mask_ld)
        dmh, dml = lay_mask(mh), lay_mask(ml)
        y = mh.double() + ml.double()
        fac = (mh.double() > 0).double() if mask == 1 else (1 - y) * y
    kw = dict(A_hi=dAh.data_ptr(), A_lo=dAl.data_ptr(), lda=dAh.stride(0), a_mn_major=a_mn,
              B_hi=dBh.data_ptr(), B_lo=dBl.data_ptr(), ldb=dBh.stride(0), b_mn_major=b_mn,
              M=M, N=N, K=K, mode_x3=x3, split_k=split_k, tile_n=tile_n, act=act, mask_act=mask)
    if mask:
        kw.update(mask_hi=dmh.data_ptr(), mask_lo=dml.data_ptr(), ldmask=dmh.stride(0))
    if bias:
        kw.update(bias=dbias.data_ptr())
    nslab = max(split_k, 1)
    ldf = N if ldf_exact else (N + 3) // 4 * 4
    of32 = torch.full((nslab, M, ldf), float("nan"), device=DEV)
    ocol = torch.full((nslab, M), float("nan"), device=DEV)
    ldo = (N + 7) // 8 * 8
    ldt = (M + 7) // 8 * 8
    # two guard rows behind every bf16 output
    ohi, olo = sentinel((M + 2, ldo)), sentinel((M + 2, ldo))
    othi, otlo = sentinel((N + 2, ldt)), sentinel((N + 2, ldt))
    use_col = "col" in outs
    if "f32" in outs or use_col:
        kw.update(out_f32=of32.data_ptr(), ld_f32=ldf, slab_stride=M * ldf)
    if use_col:
        kw.update(out_col=ocol.data_ptr(), col_index=N - 1, col_slab_stride=M)
    if "bf" in outs:
        kw.update(out_hi=ohi.data_ptr(), out_lo=None if no_lo else olo.data_ptr(), ld_out=ldo)
    if "T" in outs:
        kw.update(outT_hi=othi.data_ptr(), outT_lo=None if no_lo else otlo.data_ptr(), ld_outT=ldt)
    try:
        plan = _lib.GemmTcPlan(**kw)
        info = plan.info()
        plan.run(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        first = [t.clone() for t in (of32, ocol, ohi, olo, othi, otlo)]
        plan.run(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
    except Exception as e:  # noqa: BLE001
        return Result(name, float("inf"), 0.0, False, "EXC " + str(e)[:200], None, None)
    structural = []
    if not all(torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                           b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32))
               for a, b in zip(first, (of32, ocol, ohi, olo, othi, otlo))):
        structural.append("second run differs")
    # the plan's geometry: no empty split, one CTA per (n tile, m tile, split)
    num_kb = (K + 63) // 64
    per = -(-num_kb // min(max(split_k, 1), num_kb))
    splits = -(-num_kb // per)
    if info["splits"] != splits or info["ctas"] != -(-N // info["tile_n"]) * -(-M // 128) * splits:
        structural.append("plan geometry: want %d splits" % splits)
    if not (torch.isnan(of32[splits:]).all() and torch.isnan(ocol[splits:]).all()):
        structural.append("a slab past the plan's splits was written")
    if not torch.isnan(of32[:, :, N:]).all():
        structural.append("fp32 pad columns written")
    if "f32" not in outs and "col" not in outs and not (torch.isnan(of32).all() and torch.isnan(ocol).all()):
        structural.append("fp32 output written without out_f32")
    for nm, t, rows, cols, used in (("out_hi", ohi, M, N, "bf" in outs), ("out_lo", olo, M, N, "bf" in outs and not no_lo),
                                    ("outT_hi", othi, N, M, "T" in outs), ("outT_lo", otlo, N, M, "T" in outs and not no_lo)):
        if not (untouched(t[rows:]) and untouched(t[:, cols:]) and (used or untouched(t))):
            structural.append(nm + " written outside [rows, cols]")
    want = ref.clone()
    want3 = ref3.clone()
    if act == 1:
        want, want3 = want.clamp_min(0), want3.clamp_min(0)
    elif act == 2:
        want, want3 = torch.sigmoid(want), torch.sigmoid(want3)
    if mask:
        want, want3 = want * fac, want3 * fac
    tol = 3e-5 if x3 else 1e-5  # relative to sum_k |a||b| ; x3: dropped lo*lo ~ 2^-16..2^-18
    errs = []
    detail = str(info)
    denom = scale if act != 2 else scale.clamp_min(1.0)
    if "f32" in outs or use_col:
        got = of32[:info["splits"]].sum(0).double().cpu()[:, :N]
        if use_col:
            gc = ocol[:info["splits"]].sum(0).double().cpu()
            e_col = ((gc - want[:, N - 1]).abs() / denom[:, N - 1]).max().item()
            errs.append(e_col)
            got, want_, denom_ = got[:, :N - 1], want[:, :N - 1], denom[:, :N - 1]
            # diverted column and beyond must be untouched in the fp32 output
            if not torch.isnan(of32[:, :, N - 1:]).all():   # (slabs the plan does not write stay NaN as a whole)
                errs.append(float("inf"))
                detail += " col-divert wrote into out_f32"
        else:
            want_, denom_ = want, denom
        e = ((got - want_).abs() / denom_)
        if torch.isnan(e).any():
            errs.append(float("inf"))
            detail += " NaN(f32: unwritten?)"
        else:
            errs.append(e.max().item())
            if e.max().item() > tol:
                bad = (e > tol).nonzero()
                detail += f" first bad f32 at {bad[0].tolist()} nbad={bad.shape[0]}"
    if "bf" in outs:
        got = ohi.double().cpu()[:M, :N] + (0 if no_lo else olo.double().cpu()[:M, :N])
        e = ((got - want).abs() / denom).max().item()
        errs.append(e)
        if e > tol + 2e-5:
            detail += f" bf-out err {e:.2e}"
    if "T" in outs:
        got = (othi.double().cpu()[:N, :M] + (0 if no_lo else otlo.double().cpu()[:N, :M])).t()
        e = ((got - want).abs() / denom).max().item()
        errs.append(e)
        if e > tol + 2e-5:
            detail += f" bfT-out err {e:.2e}"
    # hi/lo outputs themselves carry ~2^-17 representation error; hi alone is the value rounded to bf16 (2^-9)
    tol_eff = tol + ((2.0 ** -8 if no_lo else 2e-5) if ("bf" in outs or "T" in outs) else 0.0)
    err = max(errs) if errs else float("inf")
    # Distance to the exact value of the products the kernel forms: fp32 accumulation only, none of the error of the
    # bf16 split.  The worst-case bound n u sum|a||b| is looser than the tolerance above once K > 80, so the check is
    # statistical: roundings of n addends add up like sqrt(n).  ACC_MAX is empirical (see its definition).
    acc = None
    if ("f32" in outs or use_col) and act != 2 and mask != 2:
        scale3 = Ah.double().abs() @ Bh.double().abs().t()
        if x3:
            scale3 = scale3 + Ah.double().abs() @ Bl.double().abs().t() + Al.double().abs() @ Bh.double().abs().t()
        if bias:
            scale3 = scale3 + bvec.double().abs()[None, :]
        n = (3 if x3 else 1) * K + splits + 1
        g3 = of32[:splits].sum(0).double().cpu()[:, :N]
        if use_col:
            g3[:, N - 1] = ocol[:splits].sum(0).double().cpu()
        acc = float(((g3 - want3).abs() / (n ** 0.5 * U * scale3).clamp_min(1e-300)).max())
        detail += " acc=%.3g" % acc
        if not acc <= ACC_MAX:
            structural.append("fp32 accumulation error above ACC_MAX")
    if structural:
        return Result(name, float("inf"), tol_eff, False, detail + " " + "; ".join(structural), info, acc)
    return Result(name, err, tol_eff, bool(err <= tol_eff), detail, info, acc)


def all_cases():
    cases = []
    for (a_mn, b_mn) in [(0, 0), (0, 1), (1, 1), (1, 0)]:
        for x3 in (0, 1):
            cases.append(dict(M=128, N=128, K=64, x3=x3, a_mn=a_mn, b_mn=b_mn, tile_n=128))
            cases.append(dict(M=256, N=192, K=192, x3=x3, a_mn=a_mn, b_mn=b_mn, tile_n=64))
            cases.append(dict(M=300, N=100, K=72, x3=x3, a_mn=a_mn, b_mn=b_mn))
    # the real layer shapes (fwd K-major; dgrad b_mn; wgrad a_mn+b_mn with split-K + bias column)
    for x3 in (0, 1):
        cases += [
            dict(M=2048, N=512, K=14, x3=x3, a_mn=0, b_mn=0, act=1, outs="f32 bf"),
            dict(M=2048, N=1024, K=480, x3=x3, a_mn=0, b_mn=0, act=1, outs="f32 bf T"),
            dict(M=2048, N=128, K=257, x3=x3, a_mn=0, b_mn=0, act=2, outs="f32 bf"),
            dict(M=2048, N=479, K=1024, x3=x3, a_mn=0, b_mn=1, outs="f32"),
            dict(M=2048, N=512, K=256, x3=x3, a_mn=0, b_mn=1, mask=1, outs="bf T"),
            dict(M=2048, N=256, K=128, x3=x3, a_mn=0, b_mn=1, mask=2, outs="bf"),
            dict(M=1024, N=480, K=2048, x3=x3, a_mn=1, b_mn=1, split_k=4, outs="f32 col"),
            dict(M=512, N=14, K=2048, x3=x3, a_mn=1, b_mn=1, split_k=8, outs="f32 col"),
            dict(M=256, N=513, K=2048, x3=x3, a_mn=1, b_mn=1, split_k=2, outs="f32 col"),
        ]
    for tn in (32, 64, 128):
        cases.append(dict(M=384, N=256, K=1024, x3=1, a_mn=0, b_mn=0, tile_n=tn, outs="f32"))
    # epilogue paths: fp32 bias, ragged rows / columns, fp32 rows that are not 16-byte aligned
    cases += [
        dict(M=2048, N=512, K=13, x3=1, a_mn=0, b_mn=0, act=1, outs="f32 bf", bias=1),
        dict(M=300, N=96, K=134, x3=1, a_mn=0, b_mn=0, act=1, outs="f32 bf", bias=1),
        dict(M=2048, N=256, K=512, x3=1, a_mn=0, b_mn=0, act=2, outs="f32 bf", bias=1),
        dict(M=77, N=479, K=192, x3=1, a_mn=0, b_mn=1, outs="f32", ldf_exact=1),
        dict(M=1024, N=480, K=2048, x3=1, a_mn=1, b_mn=1, split_k=4, outs="f32 col", ldf_exact=1),
        dict(M=130, N=70, K=64, x3=1, a_mn=0, b_mn=1, mask=1, outs="f32 bf T"),
        dict(M=130, N=70, K=64, x3=0, a_mn=0, b_mn=1, mask=2, outs="bf"),
    ]
    return cases


def run_all(report=None):
    rows = []
    for c in all_cases():
        rows.append(run_case(**c))
    lines = []
    for name, err, tol, ok, detail, _, _ in rows:
        lines.append(f"{'OK  ' if ok else 'FAIL'} err={err:.3e} tol={tol:.1e}  {name}  {detail}")
    txt = "\n".join(lines)
    if report:
        with open(report, "w") as fh:
            fh.write(txt + "\n")
    return rows, txt


if __name__ == "__main__":
    rows, txt = run_all(sys.argv[1] if len(sys.argv) > 1 else None)
    print(txt)
    nbad = sum(1 for r in rows if not r[3])
    print(f"{len(rows) - nbad}/{len(rows)} cases ok")
