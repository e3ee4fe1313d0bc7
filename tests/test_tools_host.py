"""The benchmark scripts under tools/ without a GPU: their usage text, the shared summary and the one no-device message."""
import importlib.util
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
BENCH = ["bench_align", "bench_cli", "bench_losses", "bench_mesh", "bench_metrics", "bench_panorama", "bench_panorama_batch",
         "bench_panorama_mesh", "bench_v1"]
CALLS = [(name, "--help") for name in BENCH + ["prof_gemm"]] + [(name,) for name in BENCH]


@pytest.fixture(scope="module")
def results():
    """(exit code, stdout, stderr) of every call in CALLS, run side by side: each one spends seconds importing torch."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")           # no device, also on a machine that has one
    procs = {c: subprocess.Popen([sys.executable, os.path.join(TOOLS, f"{c[0]}.py"), *c[1:]], stdout=subprocess.PIPE,
                                 stderr=subprocess.PIPE, text=True, env=env) for c in CALLS}
    out = {}
    for c, p in procs.items():
        stdout, stderr = p.communicate(timeout=300)
        out[c] = (p.returncode, stdout, stderr)
    return out


@pytest.mark.parametrize("name", BENCH + ["prof_gemm"])
def test_help_without_gpu_or_library(results, name):
    code, stdout, stderr = results[(name, "--help")]
    assert code == 0, stderr
    assert "usage:" in stdout


@pytest.mark.parametrize("name", BENCH)
def test_no_device_exits_with_one_message(results, name):
    code, stdout, stderr = results[(name,)]
    assert code != 0
    assert "Traceback" not in stderr, stderr
    assert stderr.strip().splitlines()[-1] == f"{name}.py measures on an H100; no CUDA device is visible"
    assert stdout == ""


def test_summary():
    spec = importlib.util.spec_from_file_location("measure", os.path.join(TOOLS, "measure.py"))
    measure = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(measure)
    assert measure.summary([4.0, 1.0, 3.0, 2.0]) == {"median": 3.0, "min": 1.0, "max": 4.0, "samples": 4}
    assert measure.summary([6.0, 2.0, 4.0], per=2) == {"median": 2.0, "min": 1.0, "max": 3.0, "samples": 3}
