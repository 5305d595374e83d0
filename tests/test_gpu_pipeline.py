"""The TMA-staged tile pipeline (csrc/pipeline.cuh: cp.async.bulk + mbarrier ring) is opt-in
(B200SQL_PIPELINE=1, read once per process), so its parity run happens in a child process:
the same frame-level parity tests, with every aggregation kernel taking the staged path, the exact
predicate-term checks of b2_scan_agg (tests/test_gpu_rowwise.py) and the word-for-word group-by, star and
scan_agg checks (tests/test_gpu_groupagg.py) at sizes that take it too."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_staged_pipeline_parity():
    env = dict(os.environ, B200SQL_PIPELINE="1")
    res = subprocess.run(
        [sys.executable, "-m", "pytest", "tests/test_gpu_frame.py", "tests/test_gpu_rowwise.py",
         "tests/test_gpu_groupagg.py", "-m", "gpu", "-x",
         "-q", "-k", "global_aggregates or groupby_dense or groupby_hash or star_fused or two_keys or null_keys "
         "or terms_every_op_and_literal or terms_conjunctions_scan_agg or star_bitmap or star_dense_lookup "
         "or star_hash_lookup or scan_agg_sums"],
        cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-2000:]
    assert " passed" in res.stdout
