"""What every solve entry point reports around its loop, on the device stand-in of tests/hostsim, against
tests/golden/entry_frame.json: return codes, iterations, norms, every counter of struct acgsolvercuda, launch counts
and the solver-specific fields of acgsolvercuda_info, for converged, maxits-bound and maxits = 0 solves with and
without warm-up, and every refused call with the counters after it (see tests/hostsim/run_frame_sim.py).  Integers
must match exactly, floats to 1e-12 relative (another compiler may round the stand-in's sums differently)."""
import json
import math
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "hostsim")
GOLDEN = os.path.join(ROOT, "tests", "golden", "entry_frame.json")


@pytest.fixture(scope="module")
def frame():
    p = subprocess.run(["make", "-C", SIM, "-f", "Makefile.refresh"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    p = subprocess.run([sys.executable, os.path.join(SIM, "run_frame_sim.py")], capture_output=True, text=True,
                       timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    return json.loads(p.stdout)


def _same(got, want, where):
    if isinstance(want, dict):
        assert isinstance(got, dict) and sorted(got) == sorted(want), where
        for k in want:
            _same(got[k], want[k], f"{where}.{k}")
    elif isinstance(want, list):
        assert isinstance(got, list) and len(got) == len(want), where
        for i, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f"{where}[{i}]")
    elif isinstance(want, float):
        assert isinstance(got, float), (where, got, want)
        ok = got == want or (math.isnan(got) and math.isnan(want)) or abs(got - want) <= 1e-12 * max(abs(got), abs(want))
        assert ok, (where, got, want)
    else:
        assert type(got) is type(want) and got == want, (where, got, want)


def _records(frame, part):
    with open(GOLDEN) as f:
        want = json.load(f)
    assert frame["fields"] == want["fields"]
    keys = sorted(k for k in want if k.split("/")[1:2] == [part])
    assert keys and keys == sorted(k for k in frame if k.split("/")[1:2] == [part])
    return [(k, frame[k], want[k]) for k in keys]


def _check(frame, part):
    fields = frame["fields"]
    for key, got, want in _records(frame, part):
        _same({k: v for k, v in got.items() if k != "state"}, {k: v for k, v in want.items() if k != "state"}, key)
        assert len(got.get("state", [])) == len(want.get("state", [])) == (len(fields) if "state" in want else 0), key
        for name, g, w in zip(fields, got.get("state", []), want.get("state", [])):
            _same(g, w, f"{key}.{name}")


def test_solves_match_the_golden_frame(frame):
    _check(frame, "solves")


def test_refusals_match_the_golden_frame(frame):
    _check(frame, "refusals")


def test_products_and_chebyshev_diagonal_refusal_match_the_golden_frame(frame):
    _check(frame, "products")
    _check(frame, "cheb_baddiag")
