"""MLPerf binary record reader at the boundary of the hot path (SURVEY.md section 8f, row 4).

The reference's `CriteoBinDataset` (data_loader_terabyte.py:197-249) reads one mini-batch per item from
a flat file of int32 records `[label | 13 dense counts | 26 categorical ids]`, then `_transform_features`
(:74-93) turns it into the model's inputs: dense = log(x + 1) as fp32, ids optionally folded by
`max_ind_range`, one id per (table, sample) so the offsets of every table are 0..B-1.

This module keeps that surface (`CriteoBinDataset(data_file, counts_file, batch_size, max_ind_range,
bytes_per_feature)`, `len()`, `[idx]` -> `(x_int, lS_o, x_cat.t(), y)`) over a read-only memory map,
and adds `fill(idx, host_batch)`, which writes the batch straight into the packed pinned buffer of
dlrm_b200/data.py (one host-to-device copy per step), and `load(idx, device_batch)`, which ships the raw
records and decodes them on the GPU (the CLI's per-step path; `__getitem__` and `fill` are its host
oracle).  `numpy_to_binary` writes such a file from arrays (the train-split branch of
data_loader_terabyte.py:252-290).
"""
from __future__ import annotations

import math
import os

import numpy as np
import torch

TAR_FEA, DEN_FEA, SPA_FEA = 1, 13, 26
TOT_FEA = TAR_FEA + DEN_FEA + SPA_FEA


class CriteoBinDataset(torch.utils.data.Dataset):
    """One item = one mini-batch of `batch_size` records (the last one may be short)."""

    def __init__(self, data_file, counts_file=None, batch_size=1, max_ind_range=-1, bytes_per_feature=4):
        if bytes_per_feature != 4:
            raise ValueError("records are int32: bytes_per_feature must be 4")
        self.tar_fea, self.den_fea, self.spa_fea = TAR_FEA, DEN_FEA, SPA_FEA
        self.tad_fea = TAR_FEA + DEN_FEA
        self.tot_fea = TOT_FEA
        self.batch_size = int(batch_size)
        self.max_ind_range = max_ind_range
        self.bytes_per_entry = bytes_per_feature * TOT_FEA * self.batch_size
        nbytes = os.path.getsize(data_file)
        if nbytes % (bytes_per_feature * TOT_FEA):
            raise ValueError("%s: %d bytes is not a whole number of %d-byte records" %
                             (data_file, nbytes, bytes_per_feature * TOT_FEA))
        self.num_entries = math.ceil(nbytes / self.bytes_per_entry)
        self.num_records = nbytes // (bytes_per_feature * TOT_FEA)
        print("data file:", data_file, "number of batches:", self.num_entries)
        self.records = np.memmap(data_file, dtype=np.int32, mode="r",
                                 shape=(self.num_records, TOT_FEA)) if self.num_records else \
            np.zeros((0, TOT_FEA), dtype=np.int32)
        self.counts = None
        if counts_file is not None:
            with np.load(counts_file) as data:
                self.counts = data["counts"]
        self.m_den = DEN_FEA
        self._stage = self._raw = self._copied = None     # load(): pinned staging / device records / copy event

    def __len__(self):
        return self.num_entries

    def _rows(self, idx):
        lo = idx * self.batch_size
        return self.records[lo:min(lo + self.batch_size, self.num_records)]

    def __getitem__(self, idx):
        rec = torch.from_numpy(np.array(self._rows(idx)))          # private copy, like file.read()
        cat = rec[:, self.tad_fea:]
        if self.max_ind_range > 0:
            cat = cat % self.max_ind_range
        x_int = torch.log(rec[:, TAR_FEA:self.tad_fea].to(torch.float) + 1)
        y = rec[:, 0].to(torch.float32).view(-1, 1)
        n = rec.shape[0]
        lS_o = torch.arange(n).reshape(1, -1).repeat(SPA_FEA, 1)
        return x_int, lS_o, cat.to(torch.long).t(), y

    def fill(self, idx, hb):
        """Batch `idx` into a packed HostBatch: X = log(dense + 1), target, offsets [26, B+1] as global
        positions (table k owns positions k*B .. k*B+B), ids table-major."""
        rec = self._rows(idx)
        L = hb.layout
        n = rec.shape[0]
        if n != L.B or L.T != SPA_FEA or L.m_den != DEN_FEA:
            raise ValueError("record batch (%d x 13 dense x 26 ids) does not match the packed layout "
                             "(B=%d, T=%d, m_den=%d)" % (n, L.B, L.T, L.m_den))
        if n * SPA_FEA > L.cap_nnz:
            raise RuntimeError("packed batch capacity %d exceeded" % L.cap_nnz)
        dense = torch.from_numpy(np.ascontiguousarray(rec[:, TAR_FEA:TAR_FEA + DEN_FEA]))
        torch.log(dense.to(torch.float) + 1, out=hb.X)
        hb.target.numpy()[:, 0] = rec[:, 0]
        cat = rec[:, TAR_FEA + DEN_FEA:].astype(np.int64)
        if self.max_ind_range > 0:
            cat = cat % self.max_ind_range
        hb.indices_t.numpy()[:n * SPA_FEA].reshape(SPA_FEA, n)[...] = cat.T
        hb.offsets[...] = (np.arange(SPA_FEA, dtype=np.int64) * n)[:, None] + np.arange(n + 1, dtype=np.int64)[None, :]
        hb.nnz = n * SPA_FEA
        return hb

    def load(self, idx, db):
        """Batch `idx` into a DeviceBatch of its own size (the last batch may be short), decoded on the GPU: the
        records go from the memory map into a pinned staging buffer, cross in ONE non-blocking copy (160 B per
        sample instead of the 472 B of a packed batch) and dlrm_b200_decode_records writes what fill() writes.
        The host does no arithmetic.  Asynchronous on the current stream."""
        rec = self._rows(idx)
        n = rec.shape[0]
        if self._stage is None:
            self._stage = torch.empty((self.batch_size, TOT_FEA), dtype=torch.int32).pin_memory()
            self._raw = torch.empty((self.batch_size, TOT_FEA), dtype=torch.int32, device=db.buf.device)
            self._copied = torch.cuda.Event()
        else:
            self._copied.synchronize()      # the previous batch has left the staging buffer
        self._stage.numpy()[:n] = rec
        self._raw[:n].copy_(self._stage[:n], non_blocking=True)
        self._copied.record()
        decode_records(self._raw[:n], self.max_ind_range, db)
        return db


class DeviceBatches:
    """Item j = batch j of `ds` decoded on `device` (CriteoBinDataset.load), in the reference's format
    (X, lS_o, lS_i, T) as views of one DeviceBatch per batch size: lS_i = indices[:26n].view(26, n) and lS_o a
    static arange(n) per table, which the DLRM_Net facade consumes without a copy.  The views are rewritten by
    the next item of the same size."""

    def __init__(self, ds, device):
        self.ds, self.device, self.batches = ds, device, {}

    def __len__(self):
        return len(self.ds)

    def __getitem__(self, j):
        from .data import DeviceBatch, PackedLayout

        n = min(self.ds.batch_size, self.ds.num_records - j * self.ds.batch_size)
        if n not in self.batches:
            self.batches[n] = (DeviceBatch(PackedLayout(n, SPA_FEA, DEN_FEA, n * SPA_FEA), self.device),
                               torch.arange(n, device=self.device).expand(SPA_FEA, n))
        db, lS_o = self.batches[n]
        self.ds.load(j, db)
        return db.X, lS_o, db.indices[:n * SPA_FEA].view(SPA_FEA, n), db.target


def decode_records(raw, max_ind_range, db):
    """raw: int32 device tensor [n, 40] of records -> DeviceBatch `db` (layout B == n), on the current stream."""
    from . import _lib

    n = raw.shape[0]
    L = db.layout
    if raw.dtype != torch.int32 or raw.dim() != 2 or raw.shape[1] != TOT_FEA or not raw.is_contiguous():
        raise ValueError("records must be a contiguous int32 tensor [n, %d]" % TOT_FEA)
    if n != L.B or L.T != SPA_FEA or L.m_den != DEN_FEA or n * SPA_FEA > L.cap_nnz:
        raise ValueError("%d records do not match the device layout (B=%d, T=%d, m_den=%d, cap_nnz=%d)"
                         % (n, L.B, L.T, L.m_den, L.cap_nnz))
    _lib.check(_lib.lib().dlrm_b200_decode_records(
        raw.data_ptr(), n, DEN_FEA, SPA_FEA, int(max_ind_range), db.X.data_ptr(), db.target.data_ptr(),
        db.offsets.data_ptr(), db.indices.data_ptr(), torch.cuda.current_stream(raw.device).cuda_stream),
        "decode_records")
    db.nnz = n * SPA_FEA
    return db


def numpy_to_binary(y, x_int, x_cat, output_file_path):
    """Write records `[y | x_int | x_cat]` as int32 (all values must fit into int32)."""
    y = np.asarray(y).reshape(-1, 1)
    rec = np.concatenate([y, np.asarray(x_int), np.asarray(x_cat)], axis=1).astype(np.int32)
    if rec.shape[1] != TOT_FEA:
        raise ValueError("expected 1 + 13 + 26 columns, got %d" % rec.shape[1])
    with open(output_file_path, "wb") as f:
        f.write(rec.tobytes())
