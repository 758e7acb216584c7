"""wgmma GEMM (TMA + wgmma) vs float64 references: every majorness / precision / epilogue variant."""
import pytest

pytestmark = pytest.mark.gpu


def test_gemm_tc_all_variants():
    from gemm_tc_check import run_all

    rows, txt = run_all()
    bad = [r for r in rows if not r[3]]
    assert not bad, "wgmma GEMM mismatches:\n" + "\n".join(
        f"{n}: err={e:.3e} tol={t:.1e} {d}" for n, e, t, _, d in bad)
