"""Regenerate tests/golden/cli_cfg0_Q{8,4}.txt and cli_cfg0_QW{8,4}.txt by running the UNMODIFIED reference command line
(/root/reference/dlrm_s_pytorch.py, CPU) in quantized inference: oracle/make_cli_goldens.py's common flags, the flags of
tests/golden/cli_cfg0_<tag>.flags, and --load-model of a recorded reference checkpoint (cli_cfg0_C_ref.pt for Q8 / Q4,
cli_cfg0_W1_ref.pt, with learned v_W_l, for QW8 / QW4).  Test infrastructure; needs the reference checkout, so it runs
in the build container only.

    python oracle/make_quant_cli_goldens.py [--out DIR]        # default: tests/golden

The recorded lines are the ones the tests compare: the checkpoint's 'Training state' / 'Testing state', 'Testing for
inference only' and the accuracy line.

It also records tests/golden/cli_kaggle_Q{8,4}.txt on the Kaggle fixture with --mlperf-logging, where the bit width
changes the printed metrics: the reference trains the cli_kaggle_C run for two epochs and saves cli_kaggle_Q_ref.pt
(through oracle/ref_bin_driver.py, as oracle/make_kaggle_goldens.py runs it), then tests that checkpoint quantized
with the flags of cli_kaggle_Q<bits>.flags.  The recorded lines are 'Testing state' and the 'recall ...' line."""
import argparse
import os
import re
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.make_cli_goldens import COMMON, REF, ROOT  # noqa: E402

CHECKPOINT = {"Q8": "cli_cfg0_C_ref.pt", "Q4": "cli_cfg0_C_ref.pt", "QW8": "cli_cfg0_W1_ref.pt",
              "QW4": "cli_cfg0_W1_ref.pt"}
KEEP = re.compile(r"Training state|Testing state|Testing for inference only|^ accuracy")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden"))
    args = ap.parse_args()
    env = dict(os.environ, TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD="1")    # the checkpoint holds numpy scalars
    for tag, ck in CHECKPOINT.items():
        flags = open(os.path.join(ROOT, "tests", "golden", "cli_cfg0_%s.flags" % tag)).read().split()
        ck = os.path.join(ROOT, "tests", "golden", ck)
        with tempfile.TemporaryDirectory() as tmp:        # the reference writes its TensorBoard run into the cwd
            r = subprocess.run([sys.executable, os.path.join(REF, "dlrm_s_pytorch.py")] + COMMON + flags
                               + ["--load-model=" + ck], cwd=tmp, capture_output=True, text=True, env=env)
        if r.returncode != 0:
            raise SystemExit("reference CLI failed:\n" + r.stdout[-2000:] + r.stderr[-2000:])
        lines = [ln for ln in r.stdout.splitlines() if KEEP.search(ln)]
        with open(os.path.join(args.out, "cli_cfg0_%s.txt" % tag), "w") as fh:
            fh.write("\n".join(lines) + "\n")
        print("tag %s: %d lines" % (tag, len(lines)))
    gold = os.path.join(ROOT, "tests", "golden")
    data = ["--raw-data-file=" + os.path.join(gold, "kaggle.txt"),
            "--processed-data-file=" + os.path.join(gold, "kaggle_processed.npz")]
    driver = [sys.executable, os.path.join(ROOT, "oracle", "ref_bin_driver.py")]
    base = open(os.path.join(gold, "cli_kaggle_C.flags")).read().split()
    ck = os.path.join(args.out, "cli_kaggle_Q_ref.pt")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run(driver + base + data + ["--nepochs=2", "--save-model=" + ck], cwd=tmp, capture_output=True,
                           text=True, env=env)
        if r.returncode != 0:
            raise SystemExit("reference CLI failed:\n" + r.stdout[-2000:] + r.stderr[-2000:])
        for bits in (8, 4):
            flags = open(os.path.join(gold, "cli_kaggle_Q%d.flags" % bits)).read().split()
            r = subprocess.run(driver + flags + data + ["--load-model=" + ck], cwd=tmp, capture_output=True,
                               text=True, env=env)
            if r.returncode != 0:
                raise SystemExit("reference CLI failed:\n" + r.stdout[-2000:] + r.stderr[-2000:])
            lines = [ln for ln in r.stdout.splitlines() if re.search(r"Testing state|^recall ", ln)]
            with open(os.path.join(args.out, "cli_kaggle_Q%d.txt" % bits), "w") as fh:
                fh.write("\n".join(lines) + "\n")
            print("kaggle Q%d: %s" % (bits, lines[-1]))


if __name__ == "__main__":
    main()
