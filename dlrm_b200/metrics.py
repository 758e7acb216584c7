"""The MLPerf test metrics of the reference's inference() (dlrm_s_pytorch.py:825-849: sklearn's recall, precision,
f1, average precision, ROC AUC and accuracy of np.round(score)) computed where the scores are.

During a test pass every sample becomes one int32 key, (float_bits(score) << 1) | label, stored at the sample's
position in a device buffer: nothing crosses to the host per batch.  Scores lie in [0, 1], so their bits are below
2^30 and the key order is (score, label).  finalize() sorts the keys once per pass and counts per group of equal
scores in int64; only the final divisions and the AP sum are float64.  The same code runs on CPU tensors.

With P positives, N negatives and the groups g of equal score:
  prediction = score > 0.5 (np.round rounds 0.5 to 0); recall = TP/P; precision = TP/(TP+FP), 0 when nothing is
  predicted positive (sklearn's zero_division); f1 = 2TP/(2TP+FP+FN); accuracy = (TP+TN)/n;
  roc_auc = sum_g neg_g (2 pos_above_g + pos_g) / (2 P N)    (the trapezoid over distinct thresholds);
  ap = sum_g (pos_g / P) tp_g / (tp_g + fp_g), tp_g / fp_g counted from the top score down to g inclusive.
"""
from __future__ import annotations

import torch

_HALF_BITS = 0x3F000000          # float_bits(0.5)
_MAX_KEY = (0x3F800000 << 1) | 1  # key of score 1.0 with label 1


class ScoreKeys:
    """Device buffer of one test pass's keys.  add() enqueues work only; finalize() is the one host sync."""

    def __init__(self, capacity: int, device):
        self.keys = torch.empty(int(capacity), dtype=torch.int32, device=device)
        self.invalid = torch.zeros((), dtype=torch.bool, device=device)
        self.n = 0

    def reset(self):
        self.invalid.zero_()
        self.n = 0

    def add(self, scores: torch.Tensor, labels: torch.Tensor):
        s = scores.detach().reshape(-1).to(torch.float32)
        y = labels.detach().reshape(-1)
        m = s.numel()
        if y.numel() != m or self.n + m > self.keys.numel():
            raise ValueError("%d scores / %d labels do not fit the key buffer (%d of %d used)"
                             % (m, y.numel(), self.n, self.keys.numel()))
        # a NaN or out-of-range score, or a label other than 0/1, would alias another key: flag it for finalize()
        bad = torch.isnan(s) | (s < 0) | (s > 1) | ((y != 0) & (y != 1))
        torch.logical_or(self.invalid, bad.any(), out=self.invalid)
        out = self.keys[self.n:self.n + m]
        torch.bitwise_left_shift(s.view(torch.int32), 1, out=out)
        out.bitwise_or_(y.to(torch.int32))
        self.n += m

    def finalize(self) -> dict:
        if bool(self.invalid):
            raise ValueError("test scores must lie in [0, 1] (no NaN) and labels must be 0 or 1")
        return metrics_from_keys(self.keys[:self.n])


def metrics_from_keys(keys: torch.Tensor) -> dict:
    """dict(recall, precision, f1, ap, roc_auc, accuracy) of the keys (any order), as Python floats."""
    n = keys.numel()
    if n == 0:
        raise ValueError("no test samples")
    if bool(((keys < 0) | (keys > _MAX_KEY)).any()):
        raise ValueError("test scores must lie in [0, 1] (no NaN)")
    k = torch.sort(keys).values
    lab = (k & 1).to(torch.int64)
    bits = k >> 1
    _, counts = torch.unique_consecutive(bits, return_counts=True)      # groups in ascending score
    ends = torch.cumsum(counts, 0) - 1
    pos_le = torch.cumsum(lab, 0)[ends]                                 # positives with score <= group
    pos_g = torch.diff(pos_le, prepend=pos_le.new_zeros(1))
    neg_g = counts - pos_g
    P = int(pos_le[-1])
    N = n - P
    if P == 0 or N == 0:
        raise ValueError("only one class present in the test labels: ROC AUC is not defined")
    above = bits > _HALF_BITS
    TP = int((lab * above).sum())
    FP = int(above.sum()) - TP
    FN, TN = P - TP, N - FP
    two_u = int((neg_g * (2 * (P - pos_le) + pos_g)).sum())
    tp_top = P - pos_le + pos_g                                         # from the top down to g inclusive
    all_top = n - (ends + 1) + counts
    ap = float((pos_g.to(torch.float64) / P * (tp_top.to(torch.float64) / all_top.to(torch.float64))).sum())
    return {"recall": TP / P,
            "precision": TP / (TP + FP) if TP + FP else 0.0,
            "f1": 2 * TP / (2 * TP + FP + FN),
            "ap": ap,
            "roc_auc": two_u / (2 * P * N),
            "accuracy": (TP + TN) / n}


def mlperf_metrics(scores: torch.Tensor, labels: torch.Tensor) -> dict:
    """The metrics of one set of scores and 0/1 labels (on any device)."""
    acc = ScoreKeys(scores.numel(), scores.device)
    acc.add(scores, labels)
    return acc.finalize()
