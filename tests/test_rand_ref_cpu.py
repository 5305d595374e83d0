"""The NumPy restatement of the random-number contract (tests/rand_ref.py) checked on its own: Philox's
known-answer vectors, the counter carry, the threshold edges, RAND_INTEGER's range and the statistics."""
import numpy as np
import pytest
from scipy import stats

from tests import rand_ref as R

# Random123 kat_vectors for philox4x32_10: counter ; key -> output
KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_known_answer_vectors(ctr, key, want):
    got = R.philox(*ctr, key[0] | key[1] << 32)
    assert [int(w) for w in got] == list(want)


def test_host_module_matches_the_reference():
    import dask_sql_b200.rand as H
    for ctr, key, want in KAT:
        assert H.philox4x32_10(ctr, key[0] | key[1] << 32) == list(want)
    assert H.key_of(-1) == R.key_of(-1) == -1
    assert H.key_of(2 ** 64 + 5) == 5
    for p in (0, 1e-7, 10, 99.9999, 100):
        assert H.threshold(p) == R.threshold(p)
    keep = R.system_keep(50, 12345, 3, 30)
    assert [H.system_keeps(k, 12345, 3, 30) for k in range(50)] == keep.tolist()
    assert H.row_bases([5, 0, 7], 100) == [100, 105, 105]


def test_counter_carries_into_the_high_word():
    r = np.array([2 ** 32 - 1, 2 ** 32], dtype=np.int64)
    lo, hi = r.astype(np.uint64) & R.M32, r.astype(np.uint64) >> np.uint64(32)
    assert lo.tolist() == [2 ** 32 - 1, 0] and hi.tolist() == [0, 1]
    w0, w1, _, _ = R.philox(lo, hi, 1, 0, 7)
    u = R.rand_u64(r, 7, 1)
    assert u.tolist() == (w0 | (w1 << np.uint64(32))).tolist()
    assert u[0] != u[1]
    assert R.rand_u64(np.array([0]), 7, 1)[0] != u[1]          # 2^32 does not wrap back onto row 0


def test_threshold_edges():
    rows = np.arange(100_003)
    assert not R.bernoulli_mask(rows, 1, 1, 0).any()
    assert R.bernoulli_mask(rows, 1, 1, 100).all()
    assert R.threshold(1e-7) == 4                  # 1e-9 * 2^32 = 4.29
    assert R.threshold(99.9999) == 2 ** 32 - 4295
    assert R.bernoulli_mask(rows, 1, 1, 1e-7).sum() <= 5
    assert (~R.bernoulli_mask(rows, 1, 1, 99.9999)).sum() <= 10
    assert R.system_keep(10, 1, 1, 100).all() and not R.system_keep(10, 1, 1, 0).any()


def test_mask_groups_rows_in_fours():
    """rows 4g .. 4g+3 read the four words of one draw"""
    rows = np.arange(64)
    g = rows >> 2
    w = np.stack(R.philox(g, 0, 5, 1, 99))
    t = R.threshold(40)
    assert (R.bernoulli_mask(rows, 99, 5, 40) == (w[rows & 3, rows] < t)).all()


def test_rand_integer_range():
    rows = np.arange(10_000)
    assert (R.rand_integer(rows, 3, 1, 1) == 0).all()
    big = R.rand_integer(rows, 3, 1, 2 ** 63 - 1)
    assert (big >= 0).all() and big.max() > 2 ** 62
    u = R.rand_u64(rows, 3, 1)              # (u * (2^63 - 1)) >> 64 is u >> 1 or one less
    assert np.abs(big - (u >> np.uint64(1)).astype(np.int64)).max() <= 1
    r10 = R.rand_integer(rows, 3, 1, 10)
    assert r10.min() == 0 and r10.max() == 9


def test_rand_is_in_unit_interval():
    x = R.rand(np.arange(100_000), -5, 2)
    assert x.dtype == np.float64 and (x >= 0).all() and (x < 1).all()
    assert (x * 2.0 ** 53 == np.floor(x * 2.0 ** 53)).all()


def test_uniformity_chi2_and_bernoulli_bound():
    n = 1_000_000
    rows = np.arange(n)
    counts = np.bincount(R.rand_integer(rows, 20261018, 1, 100), minlength=100)
    assert stats.chisquare(counts).pvalue > 1e-6
    hist = np.histogram(R.rand(rows, 20261018, 2), bins=64, range=(0, 1))[0]
    assert stats.chisquare(hist).pvalue > 1e-6
    for p in (1, 10, 50):
        kept = int(R.bernoulli_mask(rows, 20261018, 3, p).sum())
        q = p / 100
        assert abs(kept - n * q) <= 6 * np.sqrt(n * q * (1 - q))
