"""How a large golden case is stored (every file under tests/golden stays below 1 MB).  TEST INFRASTRUCTURE.

`shrink(d)` takes the full record of a case (oracle/make_goldens.py) and returns {file suffix: arrays}:
  * the initial weights are dropped: they are oracle.dlrm_numpy.random_params(default_rng(seed)) and the loader
    (tests/golden_util.py) regenerates them;
  * a dense weight gradient of more than GRAD_SAMPLE entries keeps a fixed, seeded sample of them:
    g_<layer>_idx (flat indices) and g_<layer>_val -- unless the layer's weights after the first optimizer step
    are recorded (the optimizer check feeds it the whole gradient);
  * an embedding snapshot after optimizer steps keeps a fixed, seeded sample of its touched rows (the per-table
    checksum of the whole table is kept);
  * the records of the SGD and RWSAdagrad steps go to files of their own ("_sgd", "_rwsadagrad").
"""
import numpy as np

GRAD_SAMPLE = 4096
SNAPSHOT_VALUES = 8192      # embedding values kept per snapshot (rows = this / dim, at least 32)


def _sample(n, k):
    return np.sort(np.random.default_rng(0).choice(n, k, replace=False))


def shrink(d):
    d = dict(d)
    if int(d["store_params"]):
        for key in [k for k in d if k.startswith(("emb", "botW", "botb", "topW", "topb"))]:
            del d[key]
        d["store_params"] = 0
    nrows = max(32, SNAPSHOT_VALUES // int(d["m_spa"]))
    for key in list(d):
        if key.startswith("g_") and "W" in key and np.asarray(d[key]).size > GRAD_SAMPLE and "sgd1_" + key[2:] not in d:
            g = np.asarray(d.pop(key)).ravel()
            sel = _sample(g.size, GRAD_SAMPLE)
            d[key + "_idx"], d[key + "_val"] = sel.astype(np.int32), g[sel]
        elif key.endswith("_rows") and not key.startswith("g_") and np.asarray(d[key]).size > nrows:
            sel = _sample(np.asarray(d[key]).size, nrows)
            vals = key[:-5] + "_vals"
            d[key], d[vals] = np.asarray(d[key])[sel], np.asarray(d[vals])[sel]
    out = {"": {}, "_sgd": {}, "_rwsadagrad": {}}
    for key, v in d.items():
        part = "_sgd" if key.startswith("sgd") else "_rwsadagrad" if key.startswith("rwsadagrad") else ""
        out[part][key] = v
    return out
