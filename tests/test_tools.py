"""The timing tools under tools/ on the CPU: they import without a device and share one measurement module."""
import glob
import os
import subprocess
import sys

import pytest

REPO = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
TOOLS = os.path.join(REPO, "tools")
NAMES = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(TOOLS, "*.py")))
NOT_TIMING = {"_measure", "rpn_band_bytes", "show_bench"}

# imports every tool in a fresh interpreter with subprocess.Popen disabled and stdout captured; prints the tools that
# have a main()
IMPORT_ALL = """
import importlib, io, subprocess, sys
def refuse(*a, **k):
    raise AssertionError("a subprocess was started at import: %r" % (a,))
subprocess.Popen = refuse
sys.path.insert(0, {tools!r})
out, sys.stdout = sys.stdout, io.StringIO()
mains = [n for n in {names!r} if callable(getattr(importlib.import_module(n), "main", None))]
printed, sys.stdout = sys.stdout.getvalue(), out
assert printed == "", "importing a tool printed %r" % printed
import torch
assert not torch.cuda.is_initialized(), "importing a tool initialised CUDA"
print(",".join(mains))
"""


@pytest.fixture(scope="module")
def measure():
    if TOOLS not in sys.path:
        sys.path.insert(0, TOOLS)
    import _measure
    return _measure


def test_tools_import_quietly_and_expose_main():
    code = IMPORT_ALL.format(tools=TOOLS, names=NAMES)
    r = subprocess.run([sys.executable, "-c", code], cwd=REPO, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    mains = set(r.stdout.strip().split(","))
    assert set(NAMES) - NOT_TIMING <= mains


def test_one_measurement_module():
    for name in NAMES:
        if name == "_measure":
            continue
        with open(os.path.join(TOOLS, name + ".py")) as f:
            text = f.read()
        for needle in ("torch.cuda.Event(", "nvidia-smi", "sys.path.insert"):
            assert needle not in text, "%s.py contains %s: measurement code belongs in _measure.py" % (name, needle)


def test_no_cpu_fallback(measure, monkeypatch):
    monkeypatch.setattr(measure.torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="CUDA device"):
        measure.require_gpu("a tool")
    with pytest.raises(RuntimeError, match="CUDA device"):
        measure.timed(lambda: None, 1)


def test_card_fields(measure, monkeypatch):
    assert measure.parse_card("NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz\n") == {
        "device": "NVIDIA H100 80GB HBM3", "power_limit": "700.00 W", "sm_clock_max": "1980 MHz"}
    assert measure.parse_card("NVIDIA H100 80GB HBM3, [N/A], 1980 MHz\n") == {
        "device": "NVIDIA H100 80GB HBM3", "power_limit": "unavailable", "sm_clock_max": "1980 MHz"}
    unavailable = {"device": "unavailable", "power_limit": "unavailable", "sm_clock_max": "unavailable"}
    assert measure.parse_card("") == unavailable
    monkeypatch.setenv("PATH", "")                          # no nvidia-smi to run
    monkeypatch.setattr(measure.torch.cuda, "current_device", lambda: 0)
    assert measure.card() == unavailable
