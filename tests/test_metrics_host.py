"""MLPerf test metrics (dlrm_b200/metrics.py) on CPU tensors against oracle/metrics_f64.py and, when it imports,
sklearn (the reference's inference(), dlrm_s_pytorch.py:825-849)."""
import numpy as np
import pytest
import torch

from dlrm_b200 import metrics as M
from oracle import metrics_f64 as O

NAMES = ("recall", "precision", "f1", "ap", "roc_auc", "accuracy")


def _sklearn(scores, labels):
    skm = pytest.importorskip("sklearn.metrics")
    s, y = scores.astype(np.float32), labels.astype(np.float32)
    pred = np.round(s)
    return {"recall": skm.recall_score(y, pred), "precision": skm.precision_score(y, pred, zero_division=0.0),
            "f1": skm.f1_score(y, pred), "ap": skm.average_precision_score(y, s),
            "roc_auc": skm.roc_auc_score(y, s), "accuracy": skm.accuracy_score(y, pred)}


def _cases():
    rng = np.random.default_rng(7)
    n = 5000
    y = rng.integers(0, 2, n)
    yield "continuous", rng.random(n, dtype=np.float32) * 0.3 + 0.7 * y * rng.random(n, dtype=np.float32), y
    yield "heavy ties", (rng.integers(0, 12, n) / 11).astype(np.float32), y          # 12 distinct scores
    half = rng.random(n).astype(np.float32)
    half[rng.random(n) < 0.3] = 0.5
    yield "exactly 0.5", half, y
    yield "no predicted positive", (rng.random(n) * 0.5).astype(np.float32), y       # every score <= 0.5
    yield "ties at 0 and 1", rng.integers(0, 2, n).astype(np.float32), y


@pytest.mark.parametrize("name,scores,labels", list(_cases()), ids=[c[0] for c in _cases()])
def test_metrics_match_the_oracle_and_sklearn(name, scores, labels):
    got = M.mlperf_metrics(torch.from_numpy(scores), torch.from_numpy(labels.astype(np.float32)))
    want = O.mlperf_metrics(scores, labels)
    for k in NAMES:
        assert abs(got[k] - want[k]) <= 1e-12, (k, got[k], want[k])
    if name == "no predicted positive":
        assert got["precision"] == 0.0 and got["recall"] == 0.0
    sk = _sklearn(scores, labels)
    for k in NAMES:
        assert abs(got[k] - sk[k]) <= 1e-12, (k, got[k], sk[k])


def test_keys_accumulate_over_batches_and_finalize_is_repeatable():
    rng = np.random.default_rng(1)
    s = (rng.integers(0, 50, 3000) / 49).astype(np.float32)
    y = rng.integers(0, 2, 3000).astype(np.float32)
    acc = M.ScoreKeys(4000, "cpu")
    for lo in range(0, 3000, 700):                   # batches of 700, short tail
        acc.add(torch.from_numpy(s[lo:lo + 700]).view(-1, 1), torch.from_numpy(y[lo:lo + 700]).view(-1, 1))
    a, b = acc.finalize(), acc.finalize()
    assert a == b and a == M.mlperf_metrics(torch.from_numpy(s), torch.from_numpy(y))
    acc.reset()
    with pytest.raises(ValueError):
        acc.finalize()                                # no samples


@pytest.mark.parametrize("scores,labels,msg", [
    ([0.1, 0.7, 0.2], [1, 1, 1], "one class"),
    ([0.1, float("nan"), 0.2], [0, 1, 1], "NaN"),
    ([0.1, 0.7, 0.2], [0, 2, 1], "labels must be 0 or 1"),
    ([0.1, -0.5, 0.2], [0, 1, 1], "[0, 1]"),
])
def test_invalid_input_is_an_error(scores, labels, msg):
    with pytest.raises(ValueError, match=msg.replace("[", r"\[").replace("]", r"\]")):
        M.mlperf_metrics(torch.tensor(scores), torch.tensor(labels, dtype=torch.float32))
    if msg != "[0, 1]":
        with pytest.raises(ValueError):
            O.mlperf_metrics(np.array(scores), np.array(labels))
