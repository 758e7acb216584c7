"""Host row cache, host side: the policy model on hand-built sequences, the `--emb-host-cache` flag, "auto" sizing and
the refusals in the CLI's control flow, and the extended staging struct against include/dlrm_b200.h.  No GPU."""
import ctypes as C

import pytest
import torch

from dlrm_b200 import _lib
from dlrm_b200.host_tables import MAP_LIMIT, auto_cache_rows, check_cache_size, parse_cache
from oracle.host_cache_model import HostCacheModel, set_of


def _rows_in_set(m, s, n, t=0, start=0):
    """The first n rows of table t (from `start`) whose set is s."""
    out, r = [], start
    while len(out) < n:
        if set_of(t, r, m.S) == s:
            out.append((t, r))
        r += 1
    return out


def test_geometry_rounds_up_to_whole_sets():
    assert HostCacheModel(1).N == 32 and HostCacheModel(64).N == 64 and HostCacheModel(65).N == 96
    m = HostCacheModel(64)
    assert {set_of(t, r, m.S) for t in range(3) for r in range(200)} == {0, 1}


def test_33_new_rows_of_one_set_leave_exactly_one_staged():
    m = HostCacheModel(64)
    rows = _rows_in_set(m, 1, 33)
    got = m.train_step(rows[::-1] + rows[:5])          # order and duplicates do not matter
    assert got["staged"] == [max(rows)]                 # the largest (table, row) finds no way
    assert [k for k, _ in got["inserted"]] == sorted(rows)[:32]
    assert [s for _, s in got["inserted"]] == list(range(32, 64))   # empty ways, lower way first
    assert m.stats() == dict(hits=0, inserts=32, evictions=0, staged=1)


def test_eviction_follows_last_use_with_ties_to_the_lower_way():
    m = HostCacheModel(32)
    a = _rows_in_set(m, 0, 40)
    m.train_step(a[:16])                                # step 1: ways 0..15
    m.train_step(a[16:32])                              # step 2: ways 16..31
    m.train_step([a[3], a[20]])                         # step 3: hits renew ways 3 and 20
    got = m.train_step(a[32:35])                        # step 4: oldest are the step-1 ways, lowest first
    assert [s for _, s in got["evicted"]] == [0, 1, 2]
    assert [k for k, _ in got["evicted"]] == a[:3]
    got = m.train_step(a[35:40])                        # step 5: ways 4..8 (3 was used in step 3)
    assert [s for _, s in got["evicted"]] == [4, 5, 6, 7, 8]
    assert m.where[a[3]] == 3 and m.where[a[20]] == 20


def test_a_row_used_in_the_current_step_is_never_evicted():
    m = HostCacheModel(32)
    a = _rows_in_set(m, 0, 64)
    m.train_step(a[:32])                                # full
    got = m.train_step(a[:32] + a[32:40])              # every way is a hit of this step: nothing can go
    assert got["evicted"] == [] and got["inserted"] == [] and got["staged"] == a[32:40]
    got = m.train_step(a[:20] + a[32:64])               # 12 ways are free: the 12 smallest misses take them
    assert [k for k, _ in got["inserted"]] == a[32:44]
    assert sorted(s for _, s in got["evicted"]) == list(range(20, 32))
    assert all(m.where[k] == i for i, k in enumerate(a[:20]))


def test_a_forward_only_pass_changes_nothing():
    m = HostCacheModel(64)
    rows = [(t, r) for t in range(2) for r in range(0, 300, 7)]
    m.train_step(rows)
    before = (list(m.tag), list(m.used), dict(m.where), m.step, m.stats())
    got = m.forward_pass(rows + [(0, 5000)])
    assert (list(m.tag), list(m.used), dict(m.where), m.step, m.stats()) == before
    assert set(got["hits"]) | set(got["staged"]) == set(rows) | {(0, 5000)}


@pytest.mark.parametrize("n", [32, 64, 1024])
def test_counters_add_up(n):
    import numpy as np

    rng = np.random.default_rng(n)
    m = HostCacheModel(n)
    distinct = 0
    for step in range(20):
        rows = [(int(t), int(r)) for t, r in zip(rng.integers(0, 3, 500), rng.zipf(1.2, 500) % 3000)]
        got = m.train_step(rows)
        distinct += len(set(rows))
        assert len(got["hits"]) + len(got["inserted"]) + len(got["staged"]) == len(set(rows))
        assert len(m.where) <= m.N and len(m.where) == sum(t >= 0 for t in m.tag)
        s = m.stats()
        assert s["hits"] + s["inserts"] + s["staged"] == distinct
        assert s["evictions"] <= s["inserts"]
    assert m.stats()["hits"] > 0
    flushed = m.flush()
    assert len(flushed) == m.stats()["inserts"] - m.stats()["evictions"]
    assert not m.where and m.tag == [-1] * m.N and m.used == [0] * m.N


def test_parse_and_size_checks():
    assert parse_cache("") == 0 and parse_cache("auto") == "auto"
    assert parse_cache("64") == 64 and parse_cache("65") == 96 and parse_cache("1") == 32
    with pytest.raises(ValueError, match="number of rows"):
        parse_cache("lots")
    with pytest.raises(ValueError, match=">= 0"):
        parse_cache("-32")
    check_cache_size(MAP_LIMIT - 1000, 1000)
    with pytest.raises(ValueError, match="int32 slot map"):
        check_cache_size(MAP_LIMIT - 999, 1000)


def test_auto_sizing_from_free_and_reserve_bytes():
    row = 4 * 132 + 13
    assert auto_cache_rows(10 ** 9, 10 ** 9, row, 10 ** 7) == 0                        # nothing beyond the reserve
    assert auto_cache_rows(10 ** 9, 2 * 10 ** 9, row, 10 ** 7) == 0
    assert auto_cache_rows(3 * 10 ** 9, 2 * 10 ** 9, row, 10 ** 7) == 10 ** 9 // row // 32 * 32    # 1_848_416
    assert auto_cache_rows(3 * 10 ** 9, 2 * 10 ** 9, row, 10 ** 7) == 1_848_416
    assert auto_cache_rows(80 * 10 ** 9, 0, row, 1000) == 1024                         # capped at the host rows
    assert auto_cache_rows(row * 100, 0, row, 10 ** 6) == 96                           # whole sets only


@pytest.fixture
def cli_on_cpu(monkeypatch):
    """The CLI's control flow with a stand-in model that records what it is given."""
    import dlrm_b200.cli as cli
    import dlrm_b200.dlrm_net as dn
    import dlrm_b200.optim as fo

    got = {}

    class StandIn(torch.nn.Module):
        def __init__(self, m_spa, ln_emb, ln_bot, ln_top, **kw):
            super().__init__()
            got.update(kw)
            self.lin = torch.nn.Linear(int(ln_bot[0]), 1)
            self.loss_fn = torch.nn.MSELoss()

        def forward(self, X, lS_o, lS_i):
            return torch.sigmoid(self.lin(X))

    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)
    monkeypatch.setattr(dn, "DLRM_Net", StandIn)
    monkeypatch.setattr(fo, "SGD", torch.optim.SGD)
    return cli, got


BASE = ["--arch-sparse-feature-size=16", "--arch-embedding-size=640-16-1000", "--arch-mlp-bot=5-16",
        "--arch-mlp-top=8-1", "--mini-batch-size=8", "--print-freq=1", "--use-gpu", "--num-batches=1"]


def test_flag_reaches_the_model(cli_on_cpu):
    cli, got = cli_on_cpu
    cli.run(BASE + ["--emb-host-tables=0-2"])
    assert got["emb_host_cache"] is None                          # default: no cache
    cli.run(BASE + ["--emb-host-tables=0-2", "--emb-host-cache=100"])
    assert got["emb_host_cache"] == 128
    cli.run(BASE + ["--emb-host-tables=auto", "--emb-host-cache=auto"])
    assert got["emb_host_cache"] == "auto"


@pytest.mark.parametrize("flags,msg", [
    (["--emb-host-cache=64"], "needs --emb-host-tables"),
    (["--emb-host-tables=0", "--emb-host-cache=many"], "expected auto or a number of rows"),
    (["--emb-host-tables=0", "--emb-host-cache=%d" % (MAP_LIMIT - 10)], "int32 slot map"),
    (["--emb-host-tables=0", "--emb-host-cache=64", "--emb-dtype=fp16"], "needs --emb-dtype=fp32"),
])
def test_refusals_name_the_reason(cli_on_cpu, flags, msg):
    cli, _ = cli_on_cpu
    with pytest.raises(SystemExit) as e:
        cli.run(BASE + flags)
    assert msg in str(e.value)


def test_flush_symbol_and_argument_errors():
    lib = _lib.lib()
    assert "dlrm_b200_host_cache_flush" in _lib.SYMBOLS and hasattr(lib, "dlrm_b200_host_cache_flush")
    st = _lib.HostStage(head_col=-1)
    assert st.cache_rows == 0 and not st.cache_tag and st.forward_only == 0      # zero: no cache
    arr = (_lib.HostTable * 1)()
    buf = (C.c_int64 * 64)()
    p = C.addressof(buf)
    arr[0].weight, arr[0].map, arr[0].offsets, arr[0].rows = p, p, p, 10
    st.weight = st.slot_idx = st.list = st.key = st.count = p
    st.capacity = 16
    assert lib.dlrm_b200_host_cache_flush(arr, 1, C.byref(st), 16, None) != 0
    assert b"no cache" in lib.dlrm_b200_last_error()
    st.cache_rows = 48
    assert lib.dlrm_b200_host_cache_flush(arr, 1, C.byref(st), 16, None) != 0
    assert b"multiple of 32" in lib.dlrm_b200_last_error()
    st.cache_rows = 64
    assert lib.dlrm_b200_host_stage_in(arr, 1, C.byref(st), 16, 8, 8, 1, None) != 0
    assert b"NULL cache pointer" in lib.dlrm_b200_last_error()
    st.cache_rows, st.capacity = MAP_LIMIT // 32 * 32, 64
    assert lib.dlrm_b200_host_write_back(arr, 1, C.byref(st), 16, None) != 0
    assert b"int32 slot map" in lib.dlrm_b200_last_error()
