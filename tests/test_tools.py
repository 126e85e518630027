"""The measurement tools under tools/ (no GPU): every module imports without touching a GPU or running a measurement, every argparse tool
answers --help, and the harness they share (tools/measure.py) alternates arms, summarises and names the card as the tools rely on."""
import glob
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
sys.path.insert(0, TOOLS)

import measure  # noqa: E402

MODULES = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(TOOLS, "*.py")))
ARGPARSE = [m for m in MODULES if "import argparse" in open(os.path.join(TOOLS, m + ".py")).read()]

# One fresh interpreter imports every module, then runs main() of each argparse tool with --help.  Per module it records whether the import
# initialised CUDA or changed an NSB_* variable (NSB_LIB picks the library every later import of the package loads), and the exit code and
# output of --help.
PROBE = r"""
import contextlib, importlib, io, json, os, sys
sys.path.insert(0, sys.argv[1])
import torch
nsb = lambda: {k: v for k, v in os.environ.items() if k.startswith("NSB_")}
out = {}
for name in sys.argv[2:]:
    env = nsb()
    m = importlib.import_module(name)
    r = out[name] = dict(cuda=torch.cuda.is_initialized(), env_changed=nsb() != env, help=None)
    if "import argparse" in open(m.__file__).read():
        sys.argv[1:] = ["--help"]
        buf = io.StringIO()
        try:
            with contextlib.redirect_stdout(buf):
                m.main()
            r["help"] = "returned without exiting"
        except SystemExit as e:
            r["help"] = dict(code=e.code, usage="usage:" in buf.getvalue())
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def probed():
    r = subprocess.run([sys.executable, "-c", PROBE, TOOLS] + MODULES, capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name", MODULES)
def test_tool_imports_without_touching_the_gpu(probed, name):
    assert not probed[name]["cuda"], "importing tools/%s.py initialised CUDA" % name
    assert not probed[name]["env_changed"], "importing tools/%s.py changed an NSB_* variable" % name


@pytest.mark.parametrize("name", ARGPARSE)
def test_argparse_tool_answers_help(probed, name):
    assert probed[name]["help"] == dict(code=0, usage=True), probed[name]["help"]


def test_alternate_reverses_the_order_on_odd_rounds():
    calls = []

    def run(arm):
        calls.append(arm)
        return "%s%d" % (arm, len(calls))
    got = measure.alternate(("a", "b", "c"), 3, run)
    assert calls == ["a", "b", "c", "c", "b", "a", "a", "b", "c"]
    assert got == {"a": ["a1", "a6", "a7"], "b": ["b2", "b5", "b8"], "c": ["c3", "c4", "c9"]}
    calls.clear()
    assert measure.alternate([1, 2], 2, run, reverse=False) == {1: ["11", "13"], 2: ["22", "24"]}
    assert calls == [1, 2, 1, 2]


def test_stats():
    assert measure.stats([2.0, 0.5, 4.0, 1.5]) == dict(mean=2.0, min=0.5, max=4.0)
    assert measure.stats([3.25]) == dict(mean=3.25, min=3.25, max=3.25)
    assert measure.median_spread([2.0, 0.5, 4.0, 1.5]) == dict(median=1.75, spread=3.5)
    assert measure.median_spread([5.0, 1.0, 2.0]) == dict(median=2.0, spread=4.0)


def test_card_without_nvidia_smi(monkeypatch):
    monkeypatch.setenv("PATH", "")
    line = measure.card()
    assert isinstance(line, str) and line.endswith(", power limit and clocks unknown")
