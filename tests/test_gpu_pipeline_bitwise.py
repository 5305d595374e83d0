"""The bitwise accumulators through the TMA-staged tile pipeline (B200SQL_PIPELINE=1, read once per process, so
in a child process): the dense, hash, star and scan_agg checks of tests/test_gpu_bitwise.py at sizes that take
the staged kernel instances."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_staged_pipeline_bitwise():
    env = dict(os.environ, B200SQL_PIPELINE="1")
    res = subprocess.run(
        [sys.executable, "-m", "pytest", "tests/test_gpu_bitwise.py", "-m", "gpu", "-x", "-q", "-k",
         "dense_family or hash1 or hashk or star_agg or scan_agg"],
        cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-2000:]
    assert " passed" in res.stdout
