"""The committed recipe for tests/golden/*.npz must keep running: regenerate two fixtures from the LIVE
reference (build container only: /root/reference is absent on the GPU box) and compare them bit for bit
with the committed files."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("DLRM_REFERENCE", "/root/reference")


@pytest.mark.skipif(not os.path.exists(os.path.join(REF, "dlrm_s_pytorch.py")), reason="live reference not present")
def test_make_goldens_regenerates_committed_fixtures(tmp_path):
    env = dict(os.environ, DLRM_GOLDEN_OUT=str(tmp_path))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "oracle", "make_goldens.py"), "tiny_default", "cfg0_cat"],
                       cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    for name in ("tiny_default", "cfg0_cat"):
        new = np.load(os.path.join(str(tmp_path), name + ".npz"))
        old = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
        assert sorted(new.files) == sorted(old.files)
        for k in old.files:
            assert np.array_equal(new[k], old[k]), (name, k)


@pytest.mark.skipif(not os.path.exists(os.path.join(REF, "dlrm_s_pytorch.py")), reason="live reference not present")
def test_make_cli_goldens_reproduces_the_recorded_reference_run(tmp_path):
    """oracle/make_cli_goldens.py runs the unmodified reference CLI; tag C (test pass + checkpoint) must give the
    committed lines again (the path inside 'Saving model ...' aside)."""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "oracle", "make_cli_goldens.py"), "--out", str(tmp_path),
                        "--tags", "C"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]

    def lines(path):
        return [("Saving model" if ln.startswith("Saving model") else ln) for ln in open(path).read().splitlines()
                if not ln.startswith("time/loss")]

    assert lines(os.path.join(str(tmp_path), "cli_cfg0_C.txt")) == lines(os.path.join(ROOT, "tests", "golden",
                                                                                     "cli_cfg0_C.txt"))
    assert os.path.getsize(os.path.join(str(tmp_path), "cli_cfg0_C_ref.pt")) > 100_000
