"""The radix-select reference of tests/select_ref.py checked on its own (no GPU, no library): its order
statistics against np.partition on seeded int64 / float64 data and at the edges -- INT64_MIN / MAX, +-inf,
-0.0 and +0.0, subnormals, all-equal, n = 1, duplicates straddling a quantile -- and its pass count."""
import numpy as np
import pytest

from tests import select_ref as R

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


def _quantile_ranks(n):
    out = set()
    for q in (0.25, 0.5, 0.75):
        lo = int(np.floor(q * (n - 1)))
        out |= {lo, min(lo + 1, n - 1)}
    return sorted(out)


def _check(values, ranks=None):
    u = R.images(values)
    n = u.shape[0]
    ranks = _quantile_ranks(n) if ranks is None else ranks
    got, npass = R.select(u, ranks)
    assert npass == R.passes(int(u.min()), int(u.max()))
    clean = values[~np.isnan(values)] if values.dtype == np.float64 else values
    part = np.partition(clean, ranks)
    for k in ranks:
        v = R.value_of(got[k], values.dtype)
        assert v == part[k], (k, v, part[k])
        assert got[k] == int(np.sort(u)[k])      # exact image, so -0.0 / +0.0 are told apart too
    return npass


def _edge_sets():
    rng = np.random.default_rng(7)
    yield "int64_extremes", np.array([I64_MIN, I64_MAX, 0, -1, 1, I64_MIN + 1, I64_MAX - 1], np.int64)
    yield "float_edges", np.array([-np.inf, np.inf, -0.0, 0.0, 5e-324, -5e-324, 2.2250738585072014e-308,
                                   -1.0, 1.0, np.nan, 1e308, -1e308], np.float64)
    yield "zeros", np.array([-0.0, 0.0, -0.0, 0.0, 0.0], np.float64)
    yield "subnormals", (rng.random(257) * 1e-310).astype(np.float64)
    yield "all_equal_i", np.full(100, 42, np.int64)
    yield "all_equal_f", np.full(33, -2.5)
    yield "n1", np.array([17], np.int64)
    yield "n1_f", np.array([np.nan, -3.0])
    # 9 rows: the 25 % quantile sits at index 2, between duplicates 5, 5 and 6
    yield "straddle", np.array([1, 5, 5, 5, 6, 6, 9, 9, 9], np.int64)
    yield "dups_f", np.repeat(np.array([0.5, 0.25, 0.75, 1.5]), [3, 5, 2, 7])


@pytest.mark.parametrize("name,values", list(_edge_sets()))
def test_edges_match_np_partition(name, values):
    _check(values)


@pytest.mark.parametrize("seed", range(4))
def test_random_int64_and_float64(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 5000))
    _check(rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True))
    _check(rng.integers(-1000, 1000, n).astype(np.int64))
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-300, 300)
    x[rng.random(n) < 0.1] = np.nan
    if not np.isnan(x).all():
        _check(x)
    ks = sorted(set(rng.integers(0, n, 8).tolist()))
    _check(rng.integers(0, 50, n).astype(np.int64), ks)


def test_pass_count_follows_the_min_max_images():
    # a 20-bit int64 range takes 2 passes, the full int64 range 6, one value none
    assert _check(np.arange(1 << 20, dtype=np.int64) * 1 + 123) == 2
    assert _check(np.array([I64_MIN, I64_MAX], np.int64)) == 6
    assert _check(np.array([3, 3, 3], np.int64)) == 0
    assert R.passes(0, 1) == 1 and R.passes(0, (1 << 11) - 1) == 1 and R.passes(0, 1 << 11) == 2


def test_hist_pass_counts_only_rows_under_the_prefix():
    u = np.array([0x10, 0x11, 0x1F, 0x20, 0x2F], np.uint64)
    h = R.hist_pass(u, [1, 2], 0, 4)
    assert h[:16].tolist() == [1, 1] + [0] * 13 + [1]
    assert h[16:].tolist() == [1] + [0] * 14 + [1]
    # shift + bits == 64: every row, prefix 0
    h = R.hist_pass(np.array([1 << 63, 5], np.uint64), [0], 53, 11)
    assert h[1 << 10] == 1 and h[0] == 1
