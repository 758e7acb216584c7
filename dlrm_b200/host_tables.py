"""Which embedding tables live in pinned host memory (`--emb-host-tables`, `Engine(host_tables=...)`).

A host table keeps its rows, accumulators and list heads in page-locked host memory; the rows a batch touches are
staged through HBM every step (csrc/host_tables.cu).  On the device it costs its slot map, 4 bytes per row.

An optional row cache (`--emb-host-cache`, `Engine(host_cache_rows=...)`) keeps up to N rows of the host tables in
HBM between steps: 32-way sets, least recently used way replaced, misses inserted in (table, row) order.  A row that
stays hot then crosses the host link once instead of twice per step.  oracle/host_cache_model.py restates the policy.
"""
from __future__ import annotations

from typing import List, Sequence, Union

# largest cache rows + staging positions: slot + 1 must be a positive int32 in the slot map
MAP_LIMIT = 0x7ffffffe


def parse(value: str, num_tables: int) -> object:
    """The flag's value: "" (no host tables), "auto", or dash-separated table ids such as "0-9-19-20-21"."""
    value = (value or "").strip()
    if value in ("", "auto"):
        return value
    try:
        ids = [int(v) for v in value.split("-")]
    except ValueError:
        raise ValueError("--emb-host-tables=%s: expected auto or dash-separated table ids" % value) from None
    bad = [k for k in ids if not 0 <= k < num_tables]
    if bad:
        raise ValueError("--emb-host-tables: table %d does not exist (%d tables)" % (bad[0], num_tables))
    return sorted(set(ids))


def auto_host_tables(rows: Sequence[int], row_bytes: int, free_bytes: int, reserve_bytes: int,
                     small_rows_max: int = 256) -> List[int]:
    """Move the largest tables (ties: the lower table id first) to host memory until the tables left on the device,
    plus 4 bytes per host row of slot map, fit into free_bytes - reserve_bytes.  Tiny tables (<= small_rows_max rows)
    never move.  [] when everything fits; ValueError when nothing that may move makes it fit."""
    rows = [int(r) for r in rows]
    budget = int(free_bytes) - int(reserve_bytes)
    need = sum(rows) * int(row_bytes)
    order = sorted((k for k, r in enumerate(rows) if r > small_rows_max), key=lambda k: (-rows[k], k))
    host: List[int] = []
    for k in order:
        if need <= budget:
            break
        need -= rows[k] * (int(row_bytes) - 4)
        host.append(k)
    if need > budget:
        raise ValueError("the embedding tables need %d bytes of device memory even with every table of more than %d "
                         "rows in host memory, and %d are free beyond the %d-byte reserve"
                         % (need, small_rows_max, max(budget, 0), int(reserve_bytes)))
    return sorted(host)


def parse_cache(value: str) -> Union[int, str]:
    """--emb-host-cache's value: "" (no cache: 0), "auto", or a row count (rounded up to a multiple of 32)."""
    value = (value or "").strip()
    if value == "":
        return 0
    if value == "auto":
        return value
    try:
        rows = int(value)
    except ValueError:
        raise ValueError("--emb-host-cache=%s: expected auto or a number of rows" % value) from None
    if rows < 0:
        raise ValueError("--emb-host-cache=%d: expected a number of rows >= 0" % rows)
    return (rows + 31) // 32 * 32


def check_cache_size(rows: int, positions: int) -> None:
    """A cache of `rows` beside a staging arena of `positions` must fit the int32 slot map."""
    if int(rows) + int(positions) > MAP_LIMIT:
        raise ValueError("--emb-host-cache=%d: cache rows + %d staging positions per batch exceed the int32 slot map "
                         "(at most %d)" % (int(rows), int(positions), MAP_LIMIT))


def auto_cache_rows(free_bytes: int, reserve_bytes: int, row_bytes: int, host_rows: int) -> int:
    """Rows of an "auto" cache: the device memory left free beyond the reserve, divided by the bytes of one cache row,
    rounded down to 32 and capped at the host rows rounded up to 32.  0 when nothing is left."""
    rows = max(int(free_bytes) - int(reserve_bytes), 0) // int(row_bytes)
    rows = min(rows, (int(host_rows) + 31) // 32 * 32, MAP_LIMIT // 2)
    return rows // 32 * 32
