"""The row cache of host embedding tables (`--emb-host-cache`, csrc/host_tables.cu), restated on the CPU.

A cache of N rows (a multiple of 32) has N / 32 sets of 32 ways; way w of set s is cache slot 32 s + w.  A row is
named by (t, row), t the host table's index in the engine's list of host tables, and its tag is row * 64 + t.  Its set
is splitmix64(tag) mod (N / 32).

A training step (the step counter advances first, so the first step is 1):
  * every distinct row of the batch that is resident is a hit; its way's last use becomes the step;
  * every other distinct row is a miss.  Per set, the misses in ascending (t, row) order take the ways whose last use
    is not the step, ordered by (last use, way) -- an empty way has last use 0, so empty ways go first, lower way
    first.  An occupied way taken is an eviction.  Misses left without a way are staged: they go back to host memory.
A forward-only pass changes nothing.  flush() empties the cache; counters and the step stay.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Tuple

_M64 = (1 << 64) - 1

Row = Tuple[int, int]      # (host table index, row)


def splitmix64(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def tag_of(t: int, row: int) -> int:
    return int(row) * 64 + int(t)


def set_of(t: int, row: int, n_sets: int) -> int:
    return splitmix64(tag_of(t, row)) % n_sets


class HostCacheModel:
    def __init__(self, rows: int):
        self.N = (int(rows) + 31) // 32 * 32
        if self.N <= 0:
            raise ValueError("a cache needs at least one row")
        self.S = self.N // 32
        self.tag = [-1] * self.N           # row * 64 + t of the resident row, -1 = empty
        self.used = [0] * self.N           # last training step that used the slot, 0 = empty
        self.where: Dict[Row, int] = {}    # resident row -> slot
        self.step = 0
        self.hits = self.inserts = self.evictions = self.staged = 0

    def stats(self) -> Dict[str, int]:
        return dict(hits=self.hits, inserts=self.inserts, evictions=self.evictions, staged=self.staged)

    def train_step(self, rows: Iterable[Row]) -> Dict[str, List]:
        """One training step over the (t, row) pairs of a batch (duplicates allowed).  Returns what happened to each
        distinct row: hits, inserted (row, slot), evicted (row, slot), staged (rows back to host memory)."""
        self.step += 1
        distinct = sorted({(int(t), int(r)) for t, r in rows})
        hits = [k for k in distinct if k in self.where]
        for k in hits:
            self.used[self.where[k]] = self.step
        by_set: Dict[int, List[Row]] = {}
        for k in distinct:
            if k not in self.where:
                by_set.setdefault(set_of(k[0], k[1], self.S), []).append(k)
        inserted, evicted, staged = [], [], []
        for s in sorted(by_set):
            misses = sorted(by_set[s])                       # ascending (t, row)
            ways = sorted((w for w in range(32) if self.used[32 * s + w] != self.step),
                          key=lambda w: (self.used[32 * s + w], w))
            for k, w in zip(misses, ways):
                slot = 32 * s + w
                if self.tag[slot] >= 0:
                    old = (self.tag[slot] & 63, self.tag[slot] >> 6)
                    del self.where[old]
                    evicted.append((old, slot))
                self.tag[slot], self.used[slot] = tag_of(*k), self.step
                self.where[k] = slot
                inserted.append((k, slot))
            staged += misses[len(ways):]
        self.hits += len(hits)
        self.inserts += len(inserted)
        self.evictions += len(evicted)
        self.staged += len(staged)
        return dict(hits=hits, inserted=inserted, evicted=evicted, staged=sorted(staged))

    def forward_pass(self, rows: Iterable[Row]) -> Dict[str, List]:
        """A pass without an update: hits are read from the cache, misses staged and released; no state changes."""
        distinct = sorted({(int(t), int(r)) for t, r in rows})
        return dict(hits=[k for k in distinct if k in self.where], staged=[k for k in distinct if k not in self.where])

    def flush(self) -> List[Tuple[Row, int]]:
        """Every resident row goes home; the cache is empty afterwards.  Returns the (row, slot) pairs written."""
        out = sorted(((k, s) for k, s in self.where.items()), key=lambda x: x[1])
        self.where.clear()
        self.tag = [-1] * self.N
        self.used = [0] * self.N
        return out

    def device_map(self, t: int, rows: int) -> List[int]:
        """The int32 slot map of host table t between steps: slot + 1 of a resident row, else 0."""
        m = [0] * int(rows)
        for (tt, r), s in self.where.items():
            if tt == t:
                m[r] = s + 1
        return m
