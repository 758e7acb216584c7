"""Preprocessed Criteo Kaggle / Terabyte data (the reference's `CriteoDataset`, dlrm_data_pytorch.py:50-337, the
non-memory-map branch) with the chosen split resident in device memory.

The reference loads `<processed>.npz` (`X_int [N, 13]`, `X_cat [N, 26]`, `y [N]`, all int32, and `counts`), splits it
by the day counts of `<raw dir>/<raw stem>_day_count.npz` (train = days 0..D-2; the last day halved by
np.array_split: test the first half, val the second), optionally shuffles it with numpy's GLOBAL RNG, and builds
every mini-batch on the host from a Python list of per-sample rows (collate_wrapper_criteo_offset).

`CriteoDataset` keeps that surface and those semantics: the same files and printed lines, the same split and sample
order, numpy's global RNG consumed by exactly the same draws (so the model built afterwards gets the reference's
initial weights for the same seed), `len()`, `[i]` -> `(X_int[i], X_cat[i] % max_ind_range, y[i])` and `collate`,
which together are the host oracle.  The split is not copied: it is an int64 order vector into the three arrays.
`to_device()` uploads the arrays once (shared with another split of the same file) and the order vector, and
`DeviceBatches` assembles batch j on the GPU with dlrm_b200_gather_records, so a training step does no host data
work and no host-to-device copy.
"""
from __future__ import annotations

import os

import numpy as np
import torch

DEN_FEA, SPA_FEA = 13, 26
DAYS = {"kaggle": 7, "terabyte": 24}


def data_files(dataset, raw_path, pro_data):
    """The files the reference reads once preprocessing has run: (processed npz, day-count npz)."""
    lstr = raw_path.split("/")
    d_path = "/".join(lstr[0:-1]) + "/"
    d_file = lstr[-1].split(".")[0] if dataset == "kaggle" else lstr[-1]
    return str(pro_data), d_path + d_file + "_day_count.npz"


def split_order(n, total_per_file, randomize, split):
    """Sample order of `split` (dlrm_data_pytorch.py:212-259): positions into the processed arrays.  Draws from
    numpy's global RNG exactly as the reference does."""
    days = len(total_per_file)
    offset_per_file = np.cumsum(np.concatenate([[0], np.asarray(total_per_file, dtype=np.int64)]))
    if int(offset_per_file[-1]) != n:
        raise ValueError("the day counts add up to %d samples, the processed file holds %d"
                         % (int(offset_per_file[-1]), n))
    indices = np.arange(n)
    if split == "none":
        if randomize == "total":
            indices = np.random.permutation(indices)
            print("Randomized indices...")
        # X[indices] = X moves row i to position indices[i]: position p holds row argsort(indices)[p]
        order = np.argsort(indices, kind="stable")
    else:
        indices = np.array_split(indices, offset_per_file[1:-1])
        if randomize == "day":
            for i in range(days - 1):
                indices[i] = np.random.permutation(indices[i])
            print("Randomized indices per day ...")
        train_indices = np.concatenate(indices[:-1])
        test_indices, val_indices = np.array_split(indices[-1], 2)
        print("Defined %s indices..." % (split))
        if randomize == "total":
            train_indices = np.random.permutation(train_indices)
            print("Randomized indices across days ...")
        order = {"train": train_indices, "val": val_indices, "test": test_indices}.get(split)
        if order is None:
            raise ValueError("dataset split is neither none, nor train, test or val: %r" % (split,))
    print("Split data according to indices...")
    return np.ascontiguousarray(order, dtype=np.int64)


class CriteoDataset(torch.utils.data.Dataset):
    """One item = one sample of `split`, as in the reference.  `data=` another CriteoDataset of the same processed
    file shares its arrays (host and device) instead of loading them again."""

    def __init__(self, dataset, max_ind_range, sub_sample_rate, randomize, split="train", raw_path="", pro_data="",
                 memory_map=False, dataset_multiprocessing=False, *, data=None):
        # sub_sample_rate and dataset_multiprocessing only act while preprocessing raw text
        if dataset not in DAYS:
            raise ValueError("Data set option is not supported: %r (kaggle | terabyte)" % (dataset,))
        if memory_map:
            raise ValueError("memory_map: the per-day _reordered.npz files are not supported (the processed .npz is "
                             "read whole)")
        self.max_ind_range = max_ind_range
        self.memory_map = False
        self.split = split
        pro, total_file = data_files(dataset, raw_path, pro_data)
        for f in (pro, total_file):
            if not os.path.exists(f):
                raise FileNotFoundError("%s does not exist (preprocessing raw Criteo text is not provided: make the "
                                        "processed files with the reference's data_utils.getCriteoAdData)" % f)
        print("Reading pre-processed data=%s" % pro)
        with np.load(total_file) as d:
            total_per_file = d["total_per_file"]
        if len(total_per_file) != DAYS[dataset]:
            raise ValueError("%s: %d days, %s has %d" % (total_file, len(total_per_file), dataset, DAYS[dataset]))
        if data is not None:
            self.X_int, self.X_cat, self.y, self.counts = data.X_int, data.X_cat, data.y, data.counts
            self._shared = data
        else:
            with np.load(pro) as d:
                self.X_int = np.ascontiguousarray(d["X_int"], dtype=np.int32)
                X_cat = d["X_cat"]
                self.y = np.ascontiguousarray(d["y"], dtype=np.int32)
                self.counts = d["counts"]
            # the reference's preprocessing stores the categorical ids as float64: keep them as int32, exactly
            self.X_cat = np.ascontiguousarray(X_cat, dtype=np.int32)
            if X_cat.dtype != np.int32 and not np.array_equal(self.X_cat, X_cat):
                raise ValueError("%s: X_cat holds values that are not int32 integers" % pro)
            del X_cat
            self._shared = None
        self.m_den = self.X_int.shape[1]
        self.n_emb = len(self.counts)
        if self.m_den != DEN_FEA or self.X_cat.shape[1] != self.n_emb or self.n_emb != SPA_FEA or \
                not (self.X_int.shape[0] == self.X_cat.shape[0] == self.y.shape[0]):
            raise ValueError("%s: expected X_int [N, 13], X_cat [N, 26], y [N] and 26 counts" % pro)
        print("Sparse fea = %d, Dense fea = %d" % (self.n_emb, self.m_den))
        self.order = split_order(len(self.y), total_per_file, randomize, split)
        self.dev = None         # to_device(): (X_int, X_cat, y, order) on the GPU

    def __len__(self):
        return len(self.order)

    def __getitem__(self, index):
        if isinstance(index, slice):
            return [self[i] for i in range(index.start or 0, index.stop or len(self), index.step or 1)]
        r = self.order[index]
        if self.max_ind_range > 0:
            return self.X_int[r], self.X_cat[r] % self.max_ind_range, self.y[r]
        return self.X_int[r], self.X_cat[r], self.y[r]

    def resident_bytes(self):
        """Device bytes of to_device(): the three arrays (counted once per processed file) and this order."""
        own = self.order.nbytes
        return own if self._shared is not None else own + self.X_int.nbytes + self.X_cat.nbytes + self.y.nbytes

    def to_device(self, device):
        """Upload the arrays (once per processed file) and this split's order.  Refused before any allocation if
        the device does not have the room."""
        if self.dev is not None:
            return self
        n = len(self.y)
        if len(self.order) and (int(self.order.min()) < 0 or int(self.order.max()) >= n):
            raise ValueError("split order out of range [0, %d)" % n)   # checked once here: the kernel trusts it
        shared = self._shared.to_device(device).dev if self._shared is not None else None
        need = self.resident_bytes()
        free, _ = torch.cuda.mem_get_info(torch.device(device))
        if need > free:
            raise RuntimeError("the %s split needs %d bytes of device memory (%.2f GB) on %s, %d are free"
                               % (self.split, need, need / 1e9, device, free))
        if shared is None:
            shared = tuple(torch.from_numpy(a).to(device) for a in (self.X_int, self.X_cat, self.y))
        self.dev = shared[:3] + (torch.from_numpy(self.order).to(device),)
        return self

    @staticmethod
    def collate(list_of_tuples):
        """collate_wrapper_criteo_offset (dlrm_data_pytorch.py:324-337): (X, lS_o, lS_i, T) of a list of items."""
        transposed_data = list(zip(*list_of_tuples))
        X_int = torch.log(torch.tensor(np.stack(transposed_data[0]), dtype=torch.float) + 1)
        X_cat = torch.tensor(np.stack(transposed_data[1]), dtype=torch.long)
        T = torch.tensor(np.asarray(transposed_data[2]), dtype=torch.float32).view(-1, 1)
        batchSize, featureCnt = X_cat.shape
        lS_i = [X_cat[:, i] for i in range(featureCnt)]
        lS_o = [torch.tensor(range(batchSize)) for _ in range(featureCnt)]
        return X_int, torch.stack(lS_o), torch.stack(lS_i), T


class DeviceBatches:
    """Item j = samples [j*B, min((j+1)*B, len)) of `ds` assembled on `device` (the tail batch is kept), in the
    reference's format (X, lS_o, lS_i, T) as views of one DeviceBatch per batch size: lS_i = indices[:26n].view(26, n)
    and lS_o a static arange(n) per table.  The views are rewritten by the next item of the same size."""

    def __init__(self, ds, batch_size, device):
        self.ds, self.batch_size, self.device, self.batches = ds.to_device(device), int(batch_size), device, {}

    def __len__(self):
        return -(-len(self.ds) // self.batch_size)

    def __getitem__(self, j):
        from .data import DeviceBatch, PackedLayout

        lo = j * self.batch_size
        n = min(self.batch_size, len(self.ds) - lo)
        if not 0 <= j < len(self):
            raise IndexError(j)
        if n not in self.batches:
            self.batches[n] = (DeviceBatch(PackedLayout(n, SPA_FEA, DEN_FEA, n * SPA_FEA), self.device),
                               torch.arange(n, device=self.device).expand(SPA_FEA, n))
        db, lS_o = self.batches[n]
        gather_records(self.ds, self.ds.dev[3][lo:lo + n], db)
        return db.X, lS_o, db.indices[:n * SPA_FEA].view(SPA_FEA, n), db.target


def gather_records(ds, ids, db):
    """Rows `ids` (int64 device tensor [n], a slice of a checked order) of the resident arrays of `ds` -> DeviceBatch
    `db` (layout B == n), on the current stream."""
    from . import _lib

    X_int, X_cat, y = ds.dev[:3]
    n = ids.shape[0]
    L = db.layout
    if ids.dtype != torch.int64 or ids.dim() != 1 or not ids.is_contiguous() or ids.device != X_int.device:
        raise ValueError("ids must be a contiguous int64 vector on the arrays' device")
    if n != L.B or L.T != SPA_FEA or L.m_den != DEN_FEA or n * SPA_FEA > L.cap_nnz:
        raise ValueError("%d samples do not match the device layout (B=%d, T=%d, m_den=%d, cap_nnz=%d)"
                         % (n, L.B, L.T, L.m_den, L.cap_nnz))
    _lib.check(_lib.lib().dlrm_b200_gather_records(
        X_int.data_ptr(), X_cat.data_ptr(), y.data_ptr(), ids.data_ptr(), n, DEN_FEA, SPA_FEA,
        int(ds.max_ind_range), db.X.data_ptr(), db.target.data_ptr(), db.offsets.data_ptr(), db.indices.data_ptr(),
        torch.cuda.current_stream(ids.device).cuda_stream), "gather_records")
    db.nnz = n * SPA_FEA
    return db
