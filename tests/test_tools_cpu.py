"""The measurement tools under tools/ without a GPU: they import without touching CUDA, answer --help, refuse to run
without a device before doing anything else, and leave timing, peak memory and the card record to tools/harness.py."""
import glob
import importlib
import inspect
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch

from tools import harness

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(ROOT, "tools", "*.py")))
MEASURING = [t for t in TOOLS if t != "harness"]
WITH_ARGS = [t for t in MEASURING if "argparse" in open(os.path.join(ROOT, "tools", t + ".py")).read()]
PYTHON = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])


def forbid_cuda(patch=setattr, allow=()):
    """Replace every public torch.cuda callable, and the lazy initialisation that creating a tensor on a CUDA device goes
    through, by one that raises."""
    def forbidden(name):
        def call(*args, **kwargs):
            raise AssertionError(f"torch.cuda.{name} called")
        return call
    for name in [n for n in dir(torch.cuda) if not n.startswith("_")] + ["_lazy_init"]:
        obj = getattr(torch.cuda, name)
        if callable(obj) and name not in allow and not (isinstance(obj, type) and issubclass(obj, BaseException)):
            patch(torch.cuda, name, forbidden(name))


@pytest.fixture(scope="module")
def import_report():
    """Import every tool in a fresh interpreter with CUDA forbidden; {tool: None or the error}."""
    script = "import torch\n" + inspect.getsource(forbid_cuda) + f"""
import importlib, json, sys
sys.path.insert(0, {ROOT!r})
forbid_cuda()
report = {{}}
for name in {TOOLS!r}:
    try:
        importlib.import_module("tools." + name)
        report[name] = None
    except BaseException as exc:
        report[name] = f"{{type(exc).__name__}}: {{exc}}"
print(json.dumps(report))
"""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run(PYTHON + ["-c", script], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("tool", TOOLS)
def test_imports_without_cuda(tool, import_report):
    assert import_report[tool] is None, import_report[tool]


@pytest.fixture(scope="module")
def help_runs():
    procs = {t: subprocess.Popen(PYTHON + [os.path.join("tools", t + ".py"), "--help"], cwd=ROOT, stdout=subprocess.PIPE,
                                 stderr=subprocess.PIPE, text=True) for t in WITH_ARGS}
    return {t: (*p.communicate(timeout=600), p.returncode) for t, p in procs.items()}


@pytest.mark.parametrize("tool", WITH_ARGS)
def test_help_exits_zero(tool, help_runs):
    out, err, code = help_runs[tool]
    assert code == 0, err
    assert "usage:" in out


@pytest.mark.parametrize("tool", MEASURING)
def test_main_refuses_without_gpu(tool, monkeypatch):
    module = importlib.import_module("tools." + tool)
    forbid_cuda(monkeypatch.setattr, allow=("is_available",))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    monkeypatch.setattr(sys, "argv", [tool + ".py"])
    with pytest.raises(SystemExit) as exc:
        module.main()
    assert exc.value.code == harness.NO_GPU


@pytest.mark.parametrize("tool", MEASURING)
def test_timing_and_card_only_in_harness(tool):
    src = open(os.path.join(ROOT, "tools", tool + ".py")).read()
    for needle in ("torch.cuda.Event(", "nvidia-smi", "reset_peak_memory_stats", "max_memory_allocated"):
        assert needle not in src, needle


def _fake_smi(monkeypatch, result):
    calls = []

    def run(argv, **kwargs):
        calls.append((argv, kwargs))
        if isinstance(result, BaseException):
            raise result
        return result
    monkeypatch.setattr(harness.subprocess, "run", run)
    return calls


def test_card_reads_one_query(monkeypatch):
    monkeypatch.setattr(torch.cuda, "get_device_name", lambda index=0: f"NVIDIA H100 80GB HBM3 #{index}")
    calls = _fake_smi(monkeypatch, SimpleNamespace(returncode=0, stdout="700.00, 1980, 1755\n", stderr=""))
    assert harness.card(1) == {"name": "NVIDIA H100 80GB HBM3 #1", "power_limit_w": 700.0, "max_sm_mhz": 1980,
                               "sm_mhz": 1755}
    (argv, kwargs), = calls
    assert argv == ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader,nounits",
                    "-i", "1"]
    assert kwargs.get("timeout")


@pytest.mark.parametrize("result", [
    SimpleNamespace(returncode=0, stdout="", stderr=""),
    SimpleNamespace(returncode=9, stdout="", stderr="NVIDIA-SMI has failed"),
    subprocess.TimeoutExpired(["nvidia-smi"], 30),
    FileNotFoundError("nvidia-smi"),
    SimpleNamespace(returncode=0, stdout="[N/A], [N/A], [N/A]\n", stderr=""),
], ids=["empty", "nonzero", "timeout", "missing", "not-available"])
def test_card_unreadable_fields_are_none(monkeypatch, result):
    def no_device(index=0):
        raise RuntimeError("no CUDA device")
    monkeypatch.setattr(torch.cuda, "get_device_name", no_device)
    _fake_smi(monkeypatch, result)
    assert harness.card() == {"name": None, "power_limit_w": None, "max_sm_mhz": None, "sm_mhz": None}


class _Clock:
    """Stub CUDA events on a fake device clock that each call of `fn` advances by its next duration."""

    def __init__(self, monkeypatch, durations):
        self.now, self.log, self.durations = 0.0, [], iter(durations)
        clock = self

        class Event:
            def __init__(self, enable_timing=False):
                assert enable_timing

            def record(self):
                clock.log.append("record")
                self.at = clock.now

            def elapsed_time(self, end):
                return end.at - self.at
        monkeypatch.setattr(torch.cuda, "Event", Event)
        monkeypatch.setattr(torch.cuda, "synchronize", lambda: self.log.append("sync"))

    def fn(self):
        self.log.append("fn")
        self.now += next(self.durations)

    def zero_(self):
        self.log.append("flush")


def test_median_ms_flushes_before_every_timed_call(monkeypatch):
    c = _Clock(monkeypatch, [100, 100, 100, 5, 1, 9, 3, 4])
    assert harness.median_ms(c.fn, 5, 3, flush=c) == 4
    assert c.log == ["fn"] * 3 + ["flush", "record", "fn", "record", "sync"] * 5


def test_window_ms_is_the_mean_after_warmup(monkeypatch):
    c = _Clock(monkeypatch, [100, 100, 5, 1, 9])
    assert harness.window_ms(c.fn, 3, 2) == 5
    assert c.log == ["fn"] * 2 + ["sync", "record"] + ["fn"] * 3 + ["record", "sync"]
