"""Exhaustive check of the wgmma GEMM (dlrm_b200_gemm_tc_*) against float64 references.
Usable as a CLI (full table, never stops at the first failure -- one GPU call tells everything):

    python tests/gemm_tc_check.py [report.txt]

and from pytest (tests/test_gpu_gemm_tc.py).  Test infrastructure."""
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


def pad_cols(t: torch.Tensor, mult=8):
    r, c = t.shape
    cp = (c + mult - 1) // mult * mult
    out = torch.zeros((r, cp), dtype=t.dtype, device=t.device)
    out[:, :c] = t
    return out


def run_case(M, N, K, x3, a_mn, b_mn, tile_n=0, split_k=1, act=0, mask=0, outs="f32", seed=0, bias=0, ldf_exact=0):
    """Returns (name, max_rel_err, tolerance, ok, detail)."""
    from dlrm_b200 import _lib

    name = (f"M{M} N{N} K{K} x3={x3} a_mn={a_mn} b_mn={b_mn} tn={tile_n} sk={split_k} act={act} mask={mask} {outs}"
            + (" bias" if bias else "") + (" ldf=N" if ldf_exact else ""))
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(N, K, generator=g)
    # awkward magnitudes: exercise the lo terms
    A = A * (1 + 0.01 * torch.randn(M, K, generator=g))
    if act == 2:  # keep sigmoid out of saturation so its absolute error is meaningful
        A = A * (2.0 / K ** 0.5)
    Ah, Al = split(A)
    Bh, Bl = split(B)
    # operands in the requested majorness
    def lay(h, l, mn):
        if mn:
            return pad_cols(h.t().contiguous()).to(DEV), pad_cols(l.t().contiguous()).to(DEV)
        return pad_cols(h).to(DEV), pad_cols(l).to(DEV)
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
        mh, ml = split(ymask)
        dmh, dml = pad_cols(mh).to(DEV), pad_cols(ml).to(DEV)
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
    ohi = torch.zeros((M, ldo), dtype=torch.bfloat16, device=DEV)
    olo = torch.zeros((M, ldo), dtype=torch.bfloat16, device=DEV)
    othi = torch.zeros((N, ldt), dtype=torch.bfloat16, device=DEV)
    otlo = torch.zeros((N, ldt), dtype=torch.bfloat16, device=DEV)
    use_col = "col" in outs
    if "f32" in outs or use_col:
        kw.update(out_f32=of32.data_ptr(), ld_f32=ldf, slab_stride=M * ldf)
    if use_col:
        kw.update(out_col=ocol.data_ptr(), col_index=N - 1, col_slab_stride=M)
    if "bf" in outs:
        kw.update(out_hi=ohi.data_ptr(), out_lo=olo.data_ptr(), ld_out=ldo)
    if "T" in outs:
        kw.update(outT_hi=othi.data_ptr(), outT_lo=otlo.data_ptr(), ld_outT=ldt)
    try:
        plan = _lib.GemmTcPlan(**kw)
        info = plan.info()
        plan.run(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
    except Exception as e:  # noqa: BLE001
        return name, float("inf"), 0.0, False, "EXC " + str(e)[:200]
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
        got = of32.sum(0).double().cpu()[:, :N]
        if use_col:
            gc = ocol.sum(0).double().cpu()
            e_col = ((gc - want[:, N - 1]).abs() / denom[:, N - 1]).max().item()
            errs.append(e_col)
            got, want_, denom_ = got[:, :N - 1], want[:, :N - 1], denom[:, :N - 1]
            # diverted column and beyond must be untouched in the fp32 output
            if not torch.isnan(of32[:, :, N - 1:]).all():
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
        got = ohi.double().cpu()[:, :N] + olo.double().cpu()[:, :N]
        e = ((got - want).abs() / denom).max().item()
        errs.append(e)
        if e > tol + 2e-5:
            detail += f" bf-out err {e:.2e}"
    if "T" in outs:
        got = (othi.double().cpu()[:, :M] + otlo.double().cpu()[:, :M]).t()
        e = ((got - want).abs() / denom).max().item()
        errs.append(e)
        if e > tol + 2e-5:
            detail += f" bfT-out err {e:.2e}"
    # hi/lo outputs themselves carry ~2^-17 representation error
    tol_eff = tol + (2e-5 if ("bf" in outs or "T" in outs) else 0.0)
    err = max(errs) if errs else float("inf")
    # additionally: distance to the exact 3-term value (pure fp32-accumulation error)
    return name, err, tol_eff, bool(err <= tol_eff), detail


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
    for name, err, tol, ok, detail in rows:
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
