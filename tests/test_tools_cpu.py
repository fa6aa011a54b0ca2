"""tools/timing.py, the benchmark scripts' shared measurement code, and the scripts' command lines, without a GPU."""
import glob
import os
import subprocess
import sys

import pytest

from tools import timing

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMES = ([2.5], [3.0, 1.0], [0.5, 0.25, 1.75], [4.0, 1.0, 3.0, 2.0], [9.5, 0.125, 7.25, 3.0, 3.0, 1.5, 8.0],
         [float(x % 11) + 0.0625 * x for x in range(30)], [float(x) for x in range(20, 0, -1)])


def old_pct(t, q):      # the percentile the scripts shared before timing.py
    t = sorted(t)
    return t[min(len(t) - 1, int(q * len(t)))]


@pytest.mark.parametrize("t", TIMES, ids=lambda t: f"n{len(t)}")
def test_summary_matches_the_old_statistics(t):
    s = timing.summary(t)
    assert (s["median_ms"], s["p10_ms"], s["p90_ms"]) == (old_pct(t, 0.5), old_pct(t, 0.1), old_pct(t, 0.9))
    ts = sorted(t)
    assert (s["median_ms"], s["min_ms"], s["max_ms"]) == (ts[len(ts) // 2], ts[0], ts[-1])


def test_summary_rounds_to_four_places():
    assert timing.summary([1.23456789]) == dict.fromkeys(("median_ms", "p10_ms", "p90_ms", "min_ms", "max_ms"), 1.2346)


def test_card_is_unknown_without_nvidia_smi(monkeypatch, tmp_path):
    monkeypatch.setenv("PATH", str(tmp_path))
    assert timing.card() == {"name": "unknown", "power_limit": "unknown", "max_sm_clock": "unknown"}


SCRIPTS = sorted(p for p in glob.glob(os.path.join(ROOT, "tools", "*.py")) if "argparse" in open(p).read())


def test_every_timing_script_has_a_command_line():
    names = {os.path.basename(p) for p in SCRIPTS}
    assert {"knn_bench.py", "sugar_dn_bench.py", "sugar_reg_bench.py", "texture_bench.py", "frosting_bg_bench.py",
            "frosting_edit_bench.py"} <= names


@pytest.mark.parametrize("script", SCRIPTS, ids=os.path.basename)
def test_help_exits_zero(script):
    r = subprocess.run([sys.executable, script, "--help"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert "usage:" in r.stdout
