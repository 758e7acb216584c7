"""numpy restatement of the MLPerf test metrics (dlrm_s_pytorch.py:825-849: sklearn recall_score, precision_score,
f1_score, average_precision_score, roc_auc_score and accuracy_score with y_pred = np.round(score)): the checker of
dlrm_b200/metrics.py.  Independent of it: a walk down the distinct thresholds (sklearn's _binary_clf_curve) with
exact integer counts, the AUC numerator as an exact integer and the AP as a correctly rounded sum (math.fsum)."""
import math

import numpy as np


def mlperf_metrics(scores, labels):
    s = np.asarray(scores, dtype=np.float64).reshape(-1)
    y = np.asarray(labels).reshape(-1)
    if np.isnan(s).any() or not np.isin(y, (0, 1)).all():
        raise ValueError("NaN score or label other than 0/1")
    y = y.astype(np.int64)
    n = s.size
    P = int(y.sum())
    N = n - P
    if P == 0 or N == 0:
        raise ValueError("one class only")
    pred = np.round(s) > 0                        # half to even: 0.5 -> 0
    TP = int((pred & (y == 1)).sum())
    FP = int((pred & (y == 0)).sum())
    FN, TN = P - TP, N - FP
    order = np.argsort(-s, kind="stable")
    ss, yy = s[order], y[order]
    last = np.r_[np.nonzero(np.diff(ss))[0], n - 1]  # last position of every distinct threshold, descending
    tps = np.cumsum(yy)[last]
    fps = last + 1 - tps
    dt = np.diff(np.r_[0, tps])
    df = np.diff(np.r_[0, fps])
    # trapezoid: sum over thresholds of dfps * (tps_prev + tps), exact in Python ints
    auc_num = sum(int(a) * (int(b) + int(c)) for a, b, c in zip(df, np.r_[0, tps[:-1]], tps))
    ap = math.fsum(float(d) / P * (float(t) / float(t + f)) for d, t, f in zip(dt, tps, fps) if d)
    return {"recall": TP / P, "precision": TP / (TP + FP) if TP + FP else 0.0,
            "f1": 2 * TP / (2 * TP + FP + FN), "ap": ap, "roc_auc": auc_num / (2 * P * N),
            "accuracy": (TP + TN) / n}
