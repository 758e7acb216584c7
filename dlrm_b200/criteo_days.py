"""Per-day preprocessed Criteo files (the reference's `--memory-map` path: CriteoDataset(memory_map=True),
dlrm_data_pytorch.py:93-199, :270-289, and data_loader_terabyte.DataLoader, :22-170) streamed through device
memory.

The reference's preprocessing writes one `savez_compressed` zip per day, `X_int [n, 13]`, `X_cat [n, 26]` and
`y [n]`, all float64 (a Terabyte day is about 60 GB inflated).  Both reference loaders give the same batches:
consecutive chunks of `batch` samples over days 0..D-2 in file order for train (batches cross day boundaries, the
tail batch is kept), and the first ceil(n/2) samples of day D-1 for test.  Nothing is shuffled at read time.

Here the days are never loaded whole:
  * `MemberReader` reads one member of a day's zip as a stream of rows (zipfile + the .npy header), inflating
    straight into a caller's buffer; stored and deflated members and zip64 are accepted.
  * `_Producer` is one worker thread doing only file I/O and inflate.  It fills pinned host chunks of at most
    `chunk_rows` samples of one day, inflating the three members of a chunk concurrently (zlib releases the GIL),
    and runs ahead across day boundaries.  It makes no CUDA call.
  * `DayBatches` (the caller's thread) copies each chunk to a device staging buffer on its own copy stream and
    converts it there with dlrm_b200_ingest_records into int32 rows of a device ring of `ring_rows` samples; every
    value is checked on the device.  Batch j is then assembled by dlrm_b200_gather_records from the ring, through a
    resident int64 vector arange(2C) % C whose slice [s mod C, s mod C + n) names ring rows [s, s + n).

Device memory is the ring, the staging buffer and the id vector, whatever the size of a day; host memory is the
pinned chunks.
"""
from __future__ import annotations

import concurrent.futures
import os
import queue
import threading
import zipfile

import numpy as np
import torch

from .criteo import DAYS, DEN_FEA, SPA_FEA

MEMBERS = (("X_int", DEN_FEA), ("X_cat", SPA_FEA), ("y", 1))
DTYPE_CODES = {np.dtype("<f8"): 0, np.dtype("<i8"): 1, np.dtype("<i4"): 2}    # dlrm_b200_ingest_records' codes
# 65,536 samples per chunk: 21 MB of float64 rows (320 bytes each) per pinned slot and in the device staging buffer
CHUNK_ROWS = 1 << 16
SLOTS = 3                  # pinned chunks: one being filled, one being copied, one waiting
LOOKAHEAD_CHUNKS = 4       # ring = batch + 4 chunks: 42 MB of int32 rows (160 bytes each) beyond the batch
_ALIGN = 16
_PIECE = 1 << 20


def day_files(dataset, raw_path):
    """(day files, day-count file, feature-count file) that the reference's --memory-map path reads
    (dlrm_data_pytorch.py:80-89, :125, :188): `<dir>/<stem>_day_{d}_reordered.npz` for Kaggle,
    `<dir>/<stem>_{d}_reordered.npz` for Terabyte."""
    if dataset not in DAYS:
        raise ValueError("Data set option is not supported: %r (kaggle | terabyte)" % (dataset,))
    lstr = raw_path.split("/")
    d_path = "/".join(lstr[0:-1]) + "/"
    d_file = lstr[-1].split(".")[0] if dataset == "kaggle" else lstr[-1]
    npz = d_path + (d_file + "_day" if dataset == "kaggle" else d_file)
    days = [npz + "_%d_reordered.npz" % d for d in range(DAYS[dataset])]
    return days, d_path + d_file + "_day_count.npz", d_path + d_file + "_fea_count.npz"


def split_segments(total_per_file, split):
    """The samples of `split` in order, as (day, first row, end row) per day."""
    n = [int(v) for v in total_per_file]
    if split == "train":
        return [(d, 0, n[d]) for d in range(len(n) - 1)]
    if split == "test":
        return [(len(n) - 1, 0, -(-n[-1] // 2))]
    raise ValueError("split %r: the per-day files are read for train and test only" % (split,))


def plan(total_per_file, split, batch):
    """Batch j of `split` as a list of (day, first row, end row): consecutive chunks of `batch` samples over the
    split's days, the tail batch kept."""
    out, cur, room = [], [], batch
    for d, lo, hi in split_segments(total_per_file, split):
        while lo < hi:
            take = min(room, hi - lo)
            cur.append((d, lo, lo + take))
            lo += take
            room -= take
            if room == 0:
                out.append(cur)
                cur, room = [], batch
    if cur:
        out.append(cur)
    return out


class MemberReader:
    """Member `name` (`name.npy`) of the day file `path`, read as a stream of rows without loading it."""

    def __init__(self, path, name, cols):
        self.path, self.name = path, name
        try:
            self._zip = zipfile.ZipFile(path)
        except zipfile.BadZipFile as e:
            raise ValueError("%s: %s" % (path, e)) from None
        try:
            self._f = self._zip.open(name + ".npy")
            version = np.lib.format.read_magic(self._f)
            read = np.lib.format.read_array_header_1_0 if version == (1, 0) else np.lib.format.read_array_header_2_0
            shape, fortran, dtype = read(self._f)
        except KeyError:
            self.close()
            raise ValueError("%s: member %s.npy is missing" % (path, name)) from None
        except ValueError as e:
            self.close()
            raise ValueError("%s: member %s.npy: %s" % (path, name, e)) from None
        if fortran and len(shape) > 1:
            self.close()
            raise ValueError("%s: member %s is stored in Fortran order (C order is read)" % (path, name))
        if dtype not in DTYPE_CODES:
            self.close()
            raise ValueError("%s: member %s has dtype %s (little-endian float64, int64 or int32 are read)"
                             % (path, name, dtype.str))
        want = (shape[0],) if cols == 1 else (shape[0], cols) if len(shape) else None
        if len(shape) == 0 or tuple(shape) != want:
            self.close()
            raise ValueError("%s: member %s has shape %s, expected [n%s]" % (path, name, tuple(shape),
                                                                             "" if cols == 1 else ", %d" % cols))
        self.rows, self.dtype, self.code = int(shape[0]), dtype, DTYPE_CODES[dtype]
        self.row_bytes = cols * dtype.itemsize

    def readinto(self, buf, rows):
        """Inflate the next `rows` rows into the writable buffer `buf` (at least rows * row_bytes bytes)."""
        mv = memoryview(buf).cast("B")[:rows * self.row_bytes]
        got = 0
        while got < len(mv):
            # zipfile copies what it inflates while holding the GIL: pieces of 1 MiB keep each copy short, so the
            # training loop on the caller's thread is not held up behind it
            k = self._f.readinto(mv[got:got + _PIECE])
            if not k:
                raise ValueError("%s: member %s ends after %d of %d bytes" % (self.path, self.name, got, len(mv)))
            got += k

    def skip(self, rows):
        """Inflate and discard `rows` rows (DEFLATE cannot seek)."""
        left = rows * self.row_bytes
        while left > 0:
            k = len(self._f.read(min(left, _PIECE)))
            if not k:
                raise ValueError("%s: member %s ends %d bytes early" % (self.path, self.name, left))
            left -= k

    def close(self):
        f = getattr(self, "_f", None)
        if f is not None:
            f.close()
        self._zip.close()


def open_day(path, count):
    """The three member readers of one day, checked against each other and against the day count."""
    readers = []
    try:
        for name, cols in MEMBERS:
            readers.append(MemberReader(path, name, cols))
        if len({r.rows for r in readers}) > 1:
            raise ValueError("%s: members X_int, X_cat, y hold %s samples (they must agree)"
                             % (path, ", ".join(str(r.rows) for r in readers)))
        for r in readers:
            if r.rows != count:
                raise ValueError("%s: member %s holds %d samples, the day count says %d"
                                 % (path, r.name, r.rows, count))
    except Exception:
        for r in readers:
            r.close()
        raise
    return readers


class _Chunk:
    __slots__ = ("slot", "path", "pos", "row0", "n", "offsets", "codes", "nbytes")


def _layout(n, readers):
    """Byte offsets of the three members of an n-row chunk in a slot (each 16-byte aligned) and its size."""
    offsets, at = [], 0
    for r in readers:
        offsets.append(at)
        at += -(-n * r.row_bytes // _ALIGN) * _ALIGN
    return offsets, at


def slot_bytes(chunk_rows):
    return sum(-(-chunk_rows * cols * 8 // _ALIGN) * _ALIGN for _, cols in MEMBERS)


class _Producer:
    """The worker thread: fills free slots with consecutive chunks of the split from sample `start` on and hands
    them over in `ready`; ends with None, or with the exception that stopped it."""

    def __init__(self, files, counts, segments, start, chunk_rows, buffers):
        self.ready, self.free, self.stop = queue.Queue(), queue.Queue(), threading.Event()
        for k in range(len(buffers)):
            self.free.put(k)
        self.args = files, counts, segments, start, chunk_rows, buffers
        self.thread = threading.Thread(target=self._run, name="criteo-days-inflate", daemon=True)
        self.thread.start()

    def _slot(self):
        while not self.stop.is_set():
            try:
                return self.free.get(timeout=0.05)
            except queue.Empty:
                pass
        return None

    def _run(self):
        files, counts, segments, start, chunk_rows, buffers = self.args
        try:
            with concurrent.futures.ThreadPoolExecutor(2, thread_name_prefix="criteo-days-member") as pool:
                pos = 0
                for d, lo, hi in segments:
                    if pos + (hi - lo) <= start:           # whole days before the start are not opened
                        pos += hi - lo
                        continue
                    readers = open_day(files[d], int(counts[d]))
                    try:
                        row = lo + max(0, start - pos)
                        pos += row - lo
                        if row > 0:
                            for r in readers:
                                r.skip(row)
                        while row < hi:
                            slot = self._slot()
                            if slot is None:
                                return
                            c = _Chunk()
                            c.slot, c.path, c.pos, c.row0, c.n = slot, files[d], pos, row, min(chunk_rows, hi - row)
                            c.offsets, c.nbytes = _layout(c.n, readers)
                            c.codes = [r.code for r in readers]
                            buf = buffers[slot]
                            jobs = [pool.submit(readers[m].readinto, buf[c.offsets[m]:], c.n) for m in (0, 2)]
                            readers[1].readinto(buf[c.offsets[1]:], c.n)
                            for f in jobs:
                                f.result()
                            self.ready.put(c)
                            row += c.n
                            pos += c.n
                    finally:
                        for r in readers:
                            r.close()
            self.ready.put(None)
        except BaseException as e:          # handed to the caller's thread, which raises it
            self.ready.put(e)

    def close(self):
        self.stop.set()
        self.thread.join()


class DayBatches:
    """Batches of one split of the per-day files, in the reference's format and order.

    `batches[j]` is `(X, lS_o, lS_i, T)` as views of one DeviceBatch per batch size, exactly as
    criteo.DeviceBatches returns them (rewritten by the next item of the same size); `len()` counts the tail batch.
    Access is sequential: j is the next batch, a later one (the stream seeks there) or 0 (the stream restarts).
    `chunk_rows` / `ring_rows` size the stream (defaults CHUNK_ROWS and batch + LOOKAHEAD_CHUNKS chunks); the ring
    must hold a batch and a chunk."""

    def __init__(self, dataset, raw_path, split, batch_size, max_ind_range, device, *, chunk_rows=None,
                 ring_rows=None):
        self.files, count_file, fea_file = day_files(dataset, raw_path)
        for f in self.files + [count_file, fea_file]:
            if not os.path.exists(f):
                raise FileNotFoundError(f)
        with np.load(count_file) as z:
            self.counts = np.asarray(z["total_per_file"], dtype=np.int64)
        if len(self.counts) != len(self.files):
            raise ValueError("%s: %d days, %s has %d" % (count_file, len(self.counts), dataset, len(self.files)))
        for d, f in enumerate(self.files):                  # headers only: a bad file is refused before training
            for r in open_day(f, int(self.counts[d])):
                r.close()
        self.split, self.batch_size, self.max_ind_range = split, int(batch_size), int(max_ind_range)
        self.segments = split_segments(self.counts, split)
        self.num_samples = sum(hi - lo for _, lo, hi in self.segments)
        self.chunk_rows = int(chunk_rows or CHUNK_ROWS)
        self.ring_rows = int(ring_rows or self.batch_size + LOOKAHEAD_CHUNKS * self.chunk_rows)
        if self.batch_size <= 0 or self.chunk_rows <= 0 or self.ring_rows < self.batch_size + self.chunk_rows:
            raise ValueError("ring of %d rows for batches of %d and chunks of %d (it must hold a batch and a chunk)"
                             % (self.ring_rows, self.batch_size, self.chunk_rows))
        self.device = torch.device(device)
        C = self.ring_rows
        i32 = dict(dtype=torch.int32, device=self.device)
        # ring (X_int, X_cat, y): the arrays criteo.gather_records reads, indexed through `ids`
        self.dev = (torch.empty(C, DEN_FEA, **i32), torch.empty(C, SPA_FEA, **i32), torch.empty(C, **i32))
        self.ids = torch.arange(2 * C, dtype=torch.int64, device=self.device) % C
        self.staging = torch.empty(slot_bytes(self.chunk_rows), dtype=torch.uint8, device=self.device)
        self.bad = torch.empty(1, dtype=torch.int64, device=self.device)
        self.pinned = [torch.empty(slot_bytes(self.chunk_rows), dtype=torch.uint8, pin_memory=True)
                       for _ in range(SLOTS)]
        self.bad_host = torch.empty(SLOTS, dtype=torch.int64, pin_memory=True)
        self.copy_stream = torch.cuda.Stream(self.device)
        self.batches = {}
        self._producer = None
        self._gather_ev = None
        self._next_j = None

    def device_bytes(self):
        """Device memory the stream holds: ring, id vector, staging buffer and the error word."""
        return sum(t.numel() * t.element_size() for t in self.dev + (self.ids, self.staging, self.bad))

    def host_bytes(self):
        return sum(t.numel() for t in self.pinned) + self.bad_host.numel() * 8

    def __len__(self):
        return -(-self.num_samples // self.batch_size)

    # -- the stream ------------------------------------------------------------------------------------------
    def _start(self, pos):
        self._stop()
        self._producer = _Producer(self.files, self.counts, self.segments, pos, self.chunk_rows,
                                   [p.numpy() for p in self.pinned])
        self._pending = []          # (chunk, event) uploaded, slot not yet returned
        self._peeked = None
        self._ingested = pos        # samples [.., _ingested) are in the ring (or on their way, in copy-stream order)
        self._ingest_ev = None
        self._done = False

    def _stop(self):
        if self._producer is not None:
            self._producer.close()
            self._producer = None
            self._retire(len(self._pending))

    def close(self):
        """Stop the worker thread (also done by exhaustion, restart and garbage collection)."""
        self._stop()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _retire(self, count):
        """Wait for the first `count` pending chunks (the rest as far as they have completed), check their error
        words, and hand their slots back to the worker."""
        while self._pending and (count > 0 or self._pending[0][1].query()):
            c, ev = self._pending.pop(0)
            ev.synchronize()
            count -= 1
            v = int(self.bad_host[c.slot])
            if v >= 0:
                self._stop_quietly()
                raise ValueError("%s: row %d: %s holds a value that is not an integer in int32 range%s"
                                 % (c.path, c.row0 + v // 4, MEMBERS[v % 4][0],
                                    ("", " or a negative id", " or a label outside {0, 1}")[v % 4]))
            if self._producer is not None:
                self._producer.free.put(c.slot)

    def _stop_quietly(self):
        if self._producer is not None:
            self._producer.close()
            self._producer = None
        self._pending = []
        self._next_j = None         # after an error the next request starts the stream afresh

    def _peek(self, block):
        if self._peeked is None and not self._done:
            if not block and self._producer.ready.empty():
                return None
            if block and self._producer.ready.empty() and self._pending:
                self._retire(len(self._pending))           # the worker may be waiting for a slot
            item = self._producer.ready.get()
            if item is None:
                self._done = True
                self._producer.thread.join()
            elif isinstance(item, BaseException):
                self._stop_quietly()
                raise item
            else:
                self._peeked = item
        return self._peeked

    def _upload(self, c):
        """Chunk c: pinned slot -> staging (copy stream) -> ingest into ring rows [c.pos, c.pos + n) mod C."""
        from . import _lib

        self._peeked = None
        C = self.ring_rows
        with torch.cuda.stream(self.copy_stream):
            if self._gather_ev is not None:     # ring rows are overwritten only after the gathers that read them
                self.copy_stream.wait_event(self._gather_ev)
            self.staging[:c.nbytes].copy_(self.pinned[c.slot][:c.nbytes], non_blocking=True)
            self.bad.fill_(-1)
            base = self.staging.data_ptr()
            ri, rc, ry = self.dev
            _lib.check(_lib.lib().dlrm_b200_ingest_records(
                base + c.offsets[0], c.codes[0], base + c.offsets[1], c.codes[1], base + c.offsets[2], c.codes[2],
                c.n, DEN_FEA, SPA_FEA, ri.data_ptr(), rc.data_ptr(), ry.data_ptr(), C, c.pos % C,
                self.bad.data_ptr(), self.copy_stream.cuda_stream), "ingest_records")
            self.bad_host[c.slot:c.slot + 1].copy_(self.bad, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self._pending.append((c, ev))
        self._ingest_ev = ev
        self._ingested = c.pos + c.n

    def __getitem__(self, j):
        from . import criteo
        from .data import DeviceBatch, PackedLayout

        if not 0 <= j < len(self):
            raise IndexError(j)
        if j == 0 or self._next_j is None or j > self._next_j:
            self._start(j * self.batch_size)
        elif j != self._next_j:
            raise IndexError("batch %d requested after batch %d: the per-day stream moves forward or restarts at 0"
                             % (j, self._next_j - 1))
        lo = j * self.batch_size
        n = min(self.batch_size, self.num_samples - lo)
        # chunks that began before this batch were read by earlier batches: their errors surface now at the latest
        self._retire(sum(1 for c, _ in self._pending if c.pos < lo))
        while self._ingested < lo + n:
            c = self._peek(True)
            assert c is not None and c.pos + c.n <= lo + self.ring_rows
            self._upload(c)
        if n not in self.batches:
            self.batches[n] = (DeviceBatch(PackedLayout(n, SPA_FEA, DEN_FEA, n * SPA_FEA), self.device),
                               torch.arange(n, device=self.device).expand(SPA_FEA, n))
        db, lS_o = self.batches[n]
        stream = torch.cuda.current_stream(self.device)
        stream.wait_event(self._ingest_ev)
        s = lo % self.ring_rows
        criteo.gather_records(self, self.ids[s:s + n], db)
        self._gather_ev = torch.cuda.Event()
        self._gather_ev.record(stream)
        # run ahead: chunks whose ring rows only held samples this and earlier batches have read
        while True:
            c = self._peek(False)
            if c is None or c.pos + c.n > lo + n + self.ring_rows:
                break
            self._upload(c)
        self._next_j = j + 1
        if j == len(self) - 1:           # the last batch: its data is checked before it is used
            self._retire(len(self._pending))
            self._stop()
        return db.X, lS_o, db.indices[:n * SPA_FEA].view(SPA_FEA, n), db.target
