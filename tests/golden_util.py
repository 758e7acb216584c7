"""Loader for tests/golden/*.npz (written by oracle/make_goldens.py from the live reference; the storage of the
larger cases is described in oracle/golden_format.py)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import dlrm_numpy as O  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
ALL_CASES = ["tiny_default", "cfg0", "cfg0_itself_thr", "cfg0_cat", "cfg0_weighted", "mini_cfg1"]


class Golden:
    def __init__(self, name):
        self.name = name
        z = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))
        for part in ("_sgd", "_rwsadagrad"):      # optimizer-step records stored beside the case
            path = os.path.join(GOLDEN_DIR, name + part + ".npz")
            if os.path.exists(path):
                z.update(np.load(path))
        self.z = z
        self.m_spa = int(z["m_spa"])
        self.ln_emb = [int(v) for v in z["ln_emb"]]
        self.ln_bot = [int(v) for v in z["ln_bot"]]
        self.ln_top = [int(v) for v in z["ln_top"]]
        self.B = int(z["B"])
        self.loss = str(z["loss"])
        self.lr = float(z["lr"])
        self.nsteps = int(z["nsteps"])
        self.itself = bool(int(z["itself"]))
        self.thr = float(z["thr"])
        self.op = str(z["op"])
        self.weighted = str(z["weighted"]) or None
        self.T = len(self.ln_emb)

    def params(self):
        """Fresh copy of the initial weights (stored, or regenerated from the seed)."""
        z = self.z
        if int(z["store_params"]):
            p = dict(
                emb=[z[f"emb{k}"].copy() for k in range(self.T)],
                bot=[(z[f"botW{i}"].copy(), z[f"botb{i}"].copy()) for i in range(len(self.ln_bot) - 1)],
                top=[(z[f"topW{i}"].copy(), z[f"topb{i}"].copy()) for i in range(len(self.ln_top) - 1)],
                v_W_l=None,
            )
        else:
            rng = np.random.default_rng(int(z["seed"]))
            p = O.random_params(rng, self.m_spa, self.ln_emb, self.ln_bot, self.ln_top)
        if self.weighted:
            p["v_W_l"] = [z[f"vW{k}"].copy() for k in range(self.T)]
        return p

    def batch(self, s):
        z = self.z
        X = z[f"b{s}_X"]
        off = z[f"b{s}_off"]
        idx = [z[f"b{s}_idx{k}"] for k in range(self.T)]
        T = z[f"b{s}_T"]
        return X, [off[k] for k in range(self.T)], idx, T

    def kw(self):
        return dict(op=self.op, itself=self.itself, loss_threshold=self.thr)

    def has(self, key):
        return key in self.z

    def dense_grad(self, key, got):
        """(got, want) for the dense gradient `key`: whole arrays, or both at the stored sample of entries."""
        if key in self.z:
            return got, self.z[key]
        return np.asarray(got).ravel()[self.z[key + "_idx"]], self.z[key + "_val"]

    def __getitem__(self, key):
        return self.z[key]
