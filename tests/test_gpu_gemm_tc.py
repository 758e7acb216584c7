"""wgmma GEMM (TMA + wgmma) vs float64 references: every majorness / precision / epilogue variant."""
import pytest

pytestmark = pytest.mark.gpu


def test_gemm_tc_all_variants():
    from gemm_tc_check import run_all

    rows, txt = run_all()
    bad = [r for r in rows if not r.ok]
    assert not bad, "wgmma GEMM mismatches:\n" + "\n".join(
        f"{r.name}: err={r.err:.3e} tol={r.tol:.1e} {r.detail}" for r in bad)
