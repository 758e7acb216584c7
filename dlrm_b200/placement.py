"""Where every embedding table lives on an N-GPU box: the host-side logic that replaces the reference's
contiguous table slices (`extend_distributed.get_my_slice`, extend_distributed.py:47-51).

The reference gives rank r tables [r*T/N, (r+1)*T/N).  With the MLPerf sizes (dlrm_b200/mlperf.py) that puts
tables 20-22 (L = 100 + 27 + 10 of 214 lookups per sample) on one rank: 64 % of all gather bytes.  Here

  * the cost of a table is its lookups per sample L_k (gather bytes per sample = L_k * dim * 4);
  * a table whose cost exceeds `split_above` x (total cost / N) is ROW-SPLIT over all N ranks: rank r owns the
    contiguous row range [r*ceil(R/N), ...); every rank pools the rows of its range for the whole global batch
    (a partial sum per sample) and the N partials are added on the rank that owns the sample -- the same
    mechanism that serves a table too large for one GPU (BASELINE.json configs[4], 2e9 rows);
  * the remaining tables are placed whole, largest first, each on the currently least-loaded rank that still has
    memory for it (LPT greedy), so max load / mean load stays within a few percent.

Pure host logic (no torch, no CUDA): covered by tests/test_placement.py on CPU.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Sequence


@dataclass(frozen=True)
class Shard:
    table: int        # global table index
    rank: int         # owner
    row_lo: int       # first row of the table stored on `rank`
    row_hi: int       # one past the last
    rows: int         # rows of the whole table
    part: int         # index of this shard among the table's shards (0 for a whole table)
    nparts: int       # 1 = whole table

    @property
    def whole(self) -> bool:
        return self.nparts == 1

    @property
    def local_rows(self) -> int:
        return self.row_hi - self.row_lo


@dataclass
class Placement:
    world: int
    shards: List[Shard]
    cost: List[float]          # per table (lookups per sample)

    def of_rank(self, rank: int) -> List[Shard]:
        """Shards stored on `rank`, ordered by (table, part): the order of the rank's local table arena."""
        return sorted((s for s in self.shards if s.rank == rank), key=lambda s: (s.table, s.part))

    def of_table(self, table: int) -> List[Shard]:
        return sorted((s for s in self.shards if s.table == table), key=lambda s: s.part)

    def split_tables(self) -> List[int]:
        return sorted({s.table for s in self.shards if not s.whole})

    def load(self) -> List[float]:
        """Expected lookups per (global) sample served by every rank (a row-split table spreads evenly)."""
        out = [0.0] * self.world
        for s in self.shards:
            out[s.rank] += self.cost[s.table] * (s.local_rows / max(s.rows, 1) if not s.whole else 1.0)
        return out

    def rows_per_rank(self) -> List[int]:
        out = [0] * self.world
        for s in self.shards:
            out[s.rank] += s.local_rows
        return out

    def imbalance(self) -> float:
        ld = self.load()
        return max(ld) / (sum(ld) / len(ld)) if sum(ld) > 0 else 1.0


def contiguous(rows: Sequence[int], world: int) -> Placement:
    """The reference's placement (extend_distributed.py:47-51): contiguous slices, nothing split."""
    T = len(rows)
    k, m = divmod(T, world)
    shards = []
    for r in range(world):
        for t in range(r * k + min(r, m), (r + 1) * k + min(r + 1, m)):
            shards.append(Shard(t, r, 0, int(rows[t]), int(rows[t]), 0, 1))
    return Placement(world, shards, [1.0] * T)


def row_bytes(dim: int, emb_dtype: str = "fp32") -> int:
    """Bytes a table row takes in HBM: an fp32 row counted as its weights (dim * 4; `plan` defaults to 512, the
    dim-128 value); an fp16 row is its halves plus the fp32 accumulator and int32 list head, padded to 16 bytes
    (272 bytes at dim 128)."""
    if emb_dtype == "fp16":
        return (2 * int(dim) + 8 + 15) // 16 * 16
    if emb_dtype == "fp32":
        return 4 * int(dim)
    raise ValueError("emb_dtype must be fp32 or fp16")


def plan(rows: Sequence[int], cost: Sequence[float], world: int, *, split_above: float = 0.6,
         bytes_per_row: int = 512, mem_budget_bytes: float = 150e9, force_split: Sequence[int] = (),
         target_imbalance: float = 1.06, max_extra_splits: int = 4) -> Placement:
    """Cost-balanced placement.  rows[k], cost[k] (lookups per sample) per table.  After the first pass, while
    max load / mean load exceeds `target_imbalance`, the cheapest whole table of the most loaded rank is row-split
    too (e.g. 26 equal tables on 8 ranks: 24 whole + 2 split = 3.25 each instead of 4/3/3/...)."""
    best = cur = _plan_once(rows, cost, world, split_above, bytes_per_row, mem_budget_bytes, force_split)
    extra = list(force_split)
    for _ in range(max_extra_splits if world > 1 else 0):
        if best.imbalance() <= target_imbalance:
            break
        ld = cur.load()
        hot = max(range(world), key=lambda r: ld[r])
        cands = [s for s in cur.of_rank(hot) if s.whole and s.rows >= world * world]   # no empty parts (ceil split)
        if not cands:
            break
        extra = extra + [min(cands, key=lambda s: (cur.cost[s.table], s.table)).table]
        cur = _plan_once(rows, cost, world, split_above, bytes_per_row, mem_budget_bytes, extra)
        if cur.imbalance() < best.imbalance() - 1e-9:     # one more split may not help, two may
            best = cur
    if world > 1 and not force_split:
        # The split heuristic is tuned for tens of tables; on degenerate inputs (two tables, two ranks) a plain
        # table-wise placement can be better balanced: keep whichever of {heuristic, LPT without hot-table splits,
        # the reference's contiguous slices when they fit} is best (the heuristic on a tie).
        cands = [best, _plan_once(rows, cost, world, float("inf"), bytes_per_row, mem_budget_bytes, ())]
        if len(rows) >= world:
            ref = contiguous(rows, world)
            ref.cost = [float(c) for c in cost]
            if max(ref.rows_per_rank()) * bytes_per_row <= mem_budget_bytes:
                cands.append(ref)
        best = min(enumerate(cands), key=lambda ip: (round(ip[1].imbalance(), 3), ip[0]))[1]    # ties: the heuristic
    return best


def _plan_once(rows, cost, world, split_above, bytes_per_row, mem_budget_bytes, force_split) -> Placement:
    T = len(rows)
    rows = [int(r) for r in rows]
    cost = [float(c) for c in cost]
    if world == 1:
        shards = [Shard(t, 0, 0, rows[t], rows[t], 0, 1) for t in range(T)]
        for t in force_split:      # single-GPU exercise of the row-split machinery (tests)
            half = (rows[t] + 1) // 2
            shards = [s for s in shards if s.table != t] + [Shard(t, 0, 0, half, rows[t], 0, 2),
                                                            Shard(t, 0, half, rows[t], rows[t], 1, 2)]
        return Placement(1, shards, cost)
    mean = sum(cost) / world
    split = set(int(t) for t in force_split)
    for t in split:
        if rows[t] < world * world:
            raise ValueError("table %d has %d rows: too few to split over %d ranks" % (t, rows[t], world))
    for t in range(T):
        too_hot = cost[t] > split_above * mean
        too_big = rows[t] * bytes_per_row > mem_budget_bytes
        if (too_hot or too_big) and rows[t] >= world * world:     # ceil(rows / world) per part: no part is empty
            split.add(t)
    shards: List[Shard] = []
    load = [0.0] * world
    mem = [0.0] * world
    for t in sorted(split):
        per = -(-rows[t] // world)
        for r in range(world):
            lo, hi = min(r * per, rows[t]), min((r + 1) * per, rows[t])
            shards.append(Shard(t, r, lo, hi, rows[t], r, world))
            load[r] += cost[t] * (hi - lo) / rows[t]
            mem[r] += (hi - lo) * bytes_per_row
    # LPT: biggest cost first (ties: more rows first), onto the least-loaded rank with room
    for t in sorted((t for t in range(T) if t not in split), key=lambda t: (-cost[t], -rows[t], t)):
        need = rows[t] * bytes_per_row
        cands = [r for r in range(world) if mem[r] + need <= mem_budget_bytes] or list(range(world))
        r = min(cands, key=lambda r: (load[r], mem[r], r))
        shards.append(Shard(t, r, 0, rows[t], rows[t], 0, 1))
        load[r] += cost[t]
        mem[r] += need
    return Placement(world, shards, cost)
