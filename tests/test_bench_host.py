"""bench.py host logic that runs without a GPU: the stage watchdog and the control flow on fakes."""
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SCRIPT = r"""
import sys, time
sys.path.insert(0, %r)
import bench
p = bench.Progress(0)
p.stage("setup")
if %d:
    p.line = {"metric": "m", "value": 123.0, "e2e": None}
    p.extra["parity_check"] = {"ok": True}
p.stage("a stage that never ends")
time.sleep(30)
print("NOT REACHED")
"""


def _run(with_value):
    env = dict(os.environ, DLRM_BENCH_STAGE_LIMIT="1", DLRM_BENCH_SETUP_LIMIT="1")
    return subprocess.run([sys.executable, "-c", _SCRIPT % (ROOT, with_value)], capture_output=True, text=True, timeout=60,
                          env=env)


def test_watchdog_prints_the_partial_line_and_leaves():
    r = _run(1)
    assert r.returncode == 0 and "NOT REACHED" not in r.stdout
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["value"] == 123.0 and line["parity_check"] == {"ok": True}
    assert "stalled in stage 'a stage that never ends'" in line["error"]
    assert "WATCHDOG" in r.stderr and "[bench r0" in r.stderr


def test_watchdog_without_a_measurement_exits_nonzero_with_an_error_line():
    r = _run(0)
    assert r.returncode == 3
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["value"] is None and "stalled" in line["error"]


def test_bench_flow_on_fakes(monkeypatch, capsys, tmp_path):
    """The whole `ours()` control flow (stages, timed loops, end-to-end loop, optional stages, line assembly, phase
    timeline) on fake engines: no kernels, but every name, ordering and JSON field of the real flow."""
    import contextlib
    import types

    import numpy as np
    import torch
    import torch.distributed as dist

    sys.path.insert(0, ROOT)
    import bench
    from dlrm_b200 import dist as ddist, engine as eng_mod

    class Ev:
        def __init__(self, *a, **k):
            pass

        def record(self, *a):
            pass

        def elapsed_time(self, other):
            return 2.0

    class St:
        def wait_event(self, e):
            pass

        def synchronize(self):
            pass

    monkeypatch.setattr(torch.cuda, "Event", Ev)
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: St())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: St())
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "set_device", lambda *a, **k: None)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    monkeypatch.setenv("DLRM_BENCH_TEST_DEVICE", "cpu")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)

    def init(backend=None):
        if not dist.is_initialized():
            dist.init_process_group("gloo", rank=0, world_size=1)
        return 0, 1

    monkeypatch.setattr(ddist, "init_distributed", init)

    class FakeEng:
        def __init__(self):
            self.n_launch, self._marks, self.D = 0, None, 128
            self.dT, self.head = torch.zeros(4), torch.zeros(4, dtype=torch.int32)

        def init_params(self, seed):
            pass

        def ensure_optimizer_state(self, o):
            pass

        def _mark(self, name):
            if self._marks is not None:
                self._marks.append((name, Ev()))

        def train_step(self, X, sp, T, lr, opt):
            self.n_launch += 30
            self._mark("begin")
            self._mark("emb:update")
            return torch.zeros(1)

        def forward(self, X, sp):
            return torch.zeros(1)

    class FakeDE:
        def __init__(self, D, rows, ln_bot, ln_top, local_batch, **kw):
            self.eng, self.B, self.Bg, self.world, self.rank = FakeEng(), local_batch, local_batch, 1, 0
            self.mine = []

        def gather_bytes_per_step(self, cost):
            return 1e9

        def nvlink_bytes_per_step(self, *a):
            return {"total_bytes_per_rank_per_step": 0.0}

        def sync_dense_params_from_rank0(self):
            pass

    class FakeMH:
        nbytes = 1024

        def __init__(self, de, hot, m_den, nsets):
            self.stage = [torch.zeros(8) for _ in range(nsets)]
            self.sparse = [object()] * nsets
            self.X = [torch.zeros(2, 13)] * nsets
            self.target = [torch.zeros(2, 1)] * nsets

        def host_buffer(self):
            return torch.zeros(8)

        def fill_host(self, buf, seed, i, rows):
            return buf

        def upload(self, k, buf):
            return 1024

        def exchange(self, k):
            pass

    class FakeGraph:
        def __init__(self, eng, stage, lr, opt, train=True, pre=None):
            self.eng = eng

        def replay(self):
            self.eng.n_launch += 1
            return torch.zeros(1)

    class FakeSampler:
        def __init__(self, local):
            pass

        def start(self):
            pass

        def stop(self, t0, t1):
            return {"sm_mhz": 1965.0, "sm_max_mhz": 1965.0, "reasons": [], "samples": 1}

    monkeypatch.setattr(ddist, "DistEngine", FakeDE)
    monkeypatch.setattr(ddist, "MultiHotExchange", FakeMH)
    monkeypatch.setattr(eng_mod, "GraphedTrainStep", FakeGraph)
    monkeypatch.setattr(bench, "ClockSampler", FakeSampler)
    monkeypatch.setattr(bench, "parity_check", lambda cls, dev, gemm: {"ok": True, "loss": 1e-6})
    monkeypatch.setattr(bench, "measure_rooflines", lambda *a: ({"bound": "hbm", "frac": 0.7}, {"bound": "hbm", "frac": 0.3}))
    monkeypatch.setattr(bench, "cpu_arm", lambda args, W, budget_s=0: {"value": 7000.0, "kind": "reference"})
    out = tmp_path / "phases.json"
    args = types.SimpleNamespace(workload="cfg3", gemm="tc", split_forward="partial", ring=2, steps=4, warmup=3,
                                 no_graph=False, no_check=False, no_cpu=False, cpu_budget=1.0, phases=2,
                                 phases_out=str(out), gpus=1, impl="ours", dump_outputs=None)
    bench.ours(args, bench.workload("cfg3", 1))
    cap = capsys.readouterr()
    lines = [ln for ln in cap.out.splitlines() if ln.startswith("{")]
    assert len(lines) == 1                                # exactly one bench line on stdout
    d = json.loads(lines[0])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "roofline", "roofline_update", "cpu_baseline", "e2e", "gpu_launches",
              "parity_check", "clocks", "placement", "nvlink"):
        assert k in d, k
    assert d["value"] == 8192 / 0.5e-3 and d["ms_per_step"] == 0.5 and d["e2e"]["ms_per_step"] == 0.5
    assert d["parity_check"]["ok"] and d["roofline"]["frac"] == 0.7 and d["cpu_baseline"]["value"] == 7000.0
    assert d["gpu_launches"] == 4 and "error" not in d
    assert "parity check" in cap.err and "teardown" in cap.err and "phases {" in cap.err
    ph = json.loads(out.read_text())
    assert [m[0] for m in ph["marks"]] == ["index_exchange", "begin", "emb:update", "step_end"]


def test_dump_outputs_writes_the_step_arrays(tmp_path):
    """bench.dump_outputs on a CPU stand-in of the engine: one float32 / float64 .npy per array, the fixed row
    sample, and well under the 64 MB cap at the cfg3 model's size."""
    import numpy as np
    import torch

    sys.path.insert(0, ROOT)
    import bench

    D, rows, B = 128, 1000, 8192
    eng = types.SimpleNamespace(D=D, total_rows=rows, top_act=[torch.rand(B, 1)], dense=torch.rand(2368900),
                                tables=torch.rand(rows, D + 4))
    eng.momentum = eng.tables[:, D]
    bench.dump_outputs(str(tmp_path), eng, torch.tensor([0.5]), B, True)
    files = sorted(p.name for p in tmp_path.iterdir())
    assert files == ["dense_params.npy", "emb_accumulator.npy", "emb_row_index.npy", "emb_rows.npy", "loss.npy", "p.npy"]
    total = 0
    for f in files:
        a = np.load(tmp_path / f)
        assert a.dtype in (np.float32, np.float64), (f, a.dtype)
        total += a.nbytes
    assert total < 64 << 20
    idx = np.load(tmp_path / "emb_row_index.npy").astype(np.int64)
    assert idx.shape == (bench.DUMP_ROWS,)
    np.testing.assert_array_equal(np.load(tmp_path / "emb_rows.npy"), eng.tables[torch.from_numpy(idx), :D].numpy())
    bench.dump_outputs(str(tmp_path / "again"), eng, torch.tensor([0.5]), B, True)
    np.testing.assert_array_equal(np.load(tmp_path / "again" / "emb_row_index.npy"), idx)   # the same sample every run


def test_bench_rejects_zero_steps_and_dumps_without_the_gpu_path():
    for extra in (["--steps", "0"], ["--impl", "reference", "--dump-outputs", "x"]):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + extra, capture_output=True, text=True,
                           timeout=120)
        assert r.returncode == 2 and "error" in r.stderr, (extra, r.stderr[-500:])
