"""Host embedding tables, host side: the auto placement policy, the `--emb-host-tables` flag and its refusals in the
CLI's control flow, and the new ABI entry points and structs against include/dlrm_b200.h.  No GPU needed."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from dlrm_b200 import _lib
from dlrm_b200.host_tables import auto_host_tables, parse
from dlrm_b200.mlperf import TABLE_ROWS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GB = 10 ** 9
ROW = 4 * 128 + 8              # fp32 D = 128 row + separate accumulator + list head (DLRM_Net's layout)
ROW_ADAGRAD = ROW + 4 * 128    # + the element-wise Adagrad accumulators


def test_auto_policy_on_the_terabyte_40m_cap_sizes():
    assert sum(TABLE_ROWS) == 204_184_588
    assert auto_host_tables(TABLE_ROWS, ROW, 200 * GB, 0) == []                   # everything fits
    assert auto_host_tables(TABLE_ROWS, ROW, 80 * GB, 4 * GB) == [0, 9]
    assert auto_host_tables(TABLE_ROWS, ROW, 80 * GB, 22 * GB) == [0, 9, 19]      # a 40 M x 128 draw kept free
    assert auto_host_tables(TABLE_ROWS, ROW_ADAGRAD, 80 * GB, 4 * GB) == [0, 9, 19, 20]
    assert auto_host_tables(TABLE_ROWS, ROW_ADAGRAD, 60 * GB, 22 * GB) == [0, 9, 19, 20, 21]
    assert auto_host_tables(TABLE_ROWS, ROW, 20 * GB, 4 * GB) == [0, 9, 19, 20, 21]
    assert auto_host_tables(TABLE_ROWS, ROW, 4 * GB, 1 * GB) == [0, 9, 19, 20, 21]
    # then the next largest: 10 (3.07 M rows), 22 (590 k), 11 (405 k)
    assert auto_host_tables(TABLE_ROWS, ROW, 2 * GB, 1 * GB) == [0, 9, 10, 11, 19, 20, 21, 22]
    with pytest.raises(ValueError, match="even with every table"):
        auto_host_tables(TABLE_ROWS, ROW, 1 * GB, 1 * GB)


def test_auto_policy_ties_slot_map_and_tiny_tables():
    # equal sizes: the lower table id moves first; the device keeps 4 bytes per host row (slot map)
    assert auto_host_tables([1000, 1000, 1000], 100, 204_000, 0) == [0]
    assert auto_host_tables([1000, 1000, 1000], 100, 108_000, 0) == [0, 1]
    assert auto_host_tables([1000, 1000, 1000], 100, 107_999, 0) == [0, 1, 2]
    with pytest.raises(ValueError):
        auto_host_tables([1000, 1000, 1000], 100, 11_999, 0)
    # tables of <= small_rows_max rows never move, however tight the budget
    with pytest.raises(ValueError):
        auto_host_tables([200, 5000], 100, 20_000 + 4 * 5000 - 1, 0)
    assert auto_host_tables([200, 5000], 100, 20_000 + 4 * 5000, 0) == [1]


def test_parse():
    assert parse("", 26) == "" and parse("auto", 26) == "auto"
    assert parse("21-0-9-9", 26) == [0, 9, 21]
    with pytest.raises(ValueError, match="does not exist"):
        parse("0-26", 26)
    with pytest.raises(ValueError, match="dash-separated"):
        parse("0,9", 26)


@pytest.fixture
def cli_on_cpu(monkeypatch):
    """The CLI's control flow with a stand-in model that records the host tables it is given."""
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
    cli.run(BASE)
    assert got["emb_host_tables"] is None                        # default: nothing changes
    cli.run(BASE + ["--emb-host-tables=2-0"])
    assert got["emb_host_tables"] == [0, 2]
    cli.run(BASE + ["--emb-host-tables=auto"])
    assert got["emb_host_tables"] == "auto"


@pytest.mark.parametrize("flags,msg", [
    (["--emb-host-tables=0", "--emb-dtype=fp16"], "needs --emb-dtype=fp32"),
    (["--emb-host-tables=0", "--weighted-pooling=fixed"], "weighted pooling"),
    (["--emb-host-tables=0-1"], "table 1 has 16 rows: tiny tables"),
    (["--emb-host-tables=3"], "table 3 does not exist"),
    (["--emb-host-tables=first"], "dash-separated"),
])
def test_refusals_name_the_reason(cli_on_cpu, flags, msg):
    cli, _ = cli_on_cpu
    with pytest.raises(SystemExit) as e:
        cli.run(BASE + flags)
    assert msg in str(e.value)


def test_sharded_runs_are_refused(cli_on_cpu, monkeypatch):
    cli, _ = cli_on_cpu
    import dlrm_b200.dist as ddist

    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setattr(ddist, "init_distributed", lambda backend: (0, 2))
    monkeypatch.setattr(torch.cuda, "set_device", lambda *a: None)
    with pytest.raises(SystemExit) as e:
        cli.run(BASE + ["--emb-host-tables=0"])
    assert "sharded runs" in str(e.value)


def test_abi_symbols_and_struct_layouts(tmp_path):
    lib = _lib.lib()
    for s in ("dlrm_b200_host_stage_in", "dlrm_b200_host_write_back", "dlrm_b200_host_release",
              "dlrm_b200_host_register", "dlrm_b200_host_unregister"):
        assert s in _lib.SYMBOLS and hasattr(lib, s)
    assert lib.dlrm_b200_abi_version() == 1
    pairs = {"dlrm_host_table_t": _lib.HostTable, "dlrm_host_stage_t": _lib.HostStage}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "dlrm_b200.h"', "int main(void) {"]
    for cname, cls in pairs.items():
        lines.append('printf("%s %%zu\\n", sizeof(%s));' % (cname, cname))
        for fname, _ in cls._fields_:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
    lines += ["return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe], check=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines()
    got = dict(ln.split() for ln in out)
    for cname, cls in pairs.items():
        assert int(got[cname]) == C.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert int(got[cname + "." + fname]) == getattr(cls, fname).offset, cname + "." + fname


def test_argument_errors_before_any_cuda_call():
    lib = _lib.lib()
    st = _lib.HostStage(head_col=-1)
    assert lib.dlrm_b200_host_stage_in(None, 0, C.byref(st), 16, 8, 8, 1, None) != 0
    assert b"num_tables" in lib.dlrm_b200_last_error()
    arr = (_lib.HostTable * 1)()
    assert lib.dlrm_b200_host_write_back(arr, 1, C.byref(st), 16, None) != 0
    assert b"capacity" in lib.dlrm_b200_last_error()
    assert lib.dlrm_b200_host_register(None, 16) != 0
