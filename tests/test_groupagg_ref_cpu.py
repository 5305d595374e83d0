"""The group-by reference (tests/groupagg_ref.py) against hand-computed cases, on a machine without a GPU:
int64 SUM wrap, -0.0 / NaN / sentinel keys, all-NULL groups, MIN / MAX of +-0.0, the float-sum bound on a
cancelling example, a star build and one range partition."""
import math

import numpy as np
import pytest

from tests import groupagg_ref as G
from tests import rowwise_ref as R

MIN, MAX = R.INT64_MIN, R.INT64_MAX


def col(vals, dtype, null=None):
    dt = {R.I64: np.int64, R.F64: np.float64, R.U8: np.uint8}[dtype]
    return R.Column(np.array(vals, dtype=dt), None if null is None else np.array(null, bool), dtype)


def test_int_sum_wraps_per_group_and_untouched_slots_keep_their_initial_words():
    v = col([MAX, 1, MIN, -1, 5], R.I64)
    ex = G.aggregate([v, v, v, None], [G.AGG_SUM, G.AGG_MIN, G.AGG_MAX, G.AGG_COUNT], [0, 0, 1, 1, -1], 4)
    assert ex.acc[0].tolist() == [MIN, MAX, 0, 0]              # MAX + 1 wraps; MIN - 1 wraps
    assert ex.acc[1].tolist() == [1, MIN, MAX, MAX]
    assert ex.acc[2].tolist() == [MAX, -1, MIN, MIN]
    assert ex.rows.tolist() == [2, 2, 0, 0] and ex.cnt[3].tolist() == [2, 2, 0, 0]
    assert ex.present.tolist() == [True, True, False, False]
    assert G.pack_bits(ex.present).tolist() == [3]


def test_all_null_group_leaves_the_accumulator_untouched():
    v = col([1.0, math.nan, 2.0, 3.0], R.F64, [False, False, True, True])
    ex = G.aggregate([v, v, v], [G.AGG_SUM, G.AGG_MIN, G.AGG_COUNT], [0, 1, 1, 1], 2, indicator=0)
    assert ex.touched[0].tolist() == [True, False]             # slot 1: NaN and two bitmap NULLs
    assert ex.acc[1].tolist() == [int(R.ordered(R.f2bits(1.0))), MAX]
    assert ex.cnt[0].tolist() == [1, 0] and ex.rows.tolist() == [1, 3]
    assert G.initial_word(G.AGG_SUM, R.F64, indicator=True) == G.NEG_ZERO_BITS
    G.check_float_sum(np.array([R.f2bits(1.0), G.NEG_ZERO_BITS]), ex.exact[0], ex.bound[0], ex.touched[0],
                      G.NEG_ZERO_BITS, True)
    with pytest.raises(AssertionError):   # a group that appeared although all its inputs are NULL
        G.check_float_sum(np.array([R.f2bits(1.0), 0]), ex.exact[0], ex.bound[0], ex.touched[0], G.NEG_ZERO_BITS, True)


def test_min_max_of_signed_zeros_and_a_touched_sum_is_never_negative_zero():
    v = col([0.0, -0.0, -0.0], R.F64)
    ex = G.aggregate([v, v, v], [G.AGG_MIN, G.AGG_MAX, G.AGG_SUM], [0, 0, 1], 2)
    assert R.ordered(ex.acc[0][0]) == R.f2bits(-0.0) and R.ordered(ex.acc[1][0]) == R.f2bits(0.0)
    assert np.float64(ex.exact[2][1]).view(np.int64) == 0      # -0.0 + 0.0 = +0.0
    with pytest.raises(AssertionError):
        G.check_float_sum(np.array([0, G.NEG_ZERO_BITS]), ex.exact[2], ex.bound[2], ex.touched[2], 0, True)


def test_sumf_rounds_each_int_then_adds():
    v = col([2 ** 53 + 1, 2 ** 53 + 1, -(2 ** 53)], R.I64)
    ex = G.aggregate([v], [G.AGG_SUMF], [0, 0, 0], 1)
    assert ex.exact[0][0] == 2.0 ** 53                           # each 2^53 + 1 rounds to 2^53 first


def test_float_sum_bound_on_a_cancelling_example():
    x = [1e16, 1.0, -1e16, 1.0]
    assert G.exact_sum(x) == 2.0
    b = G.sum_bound(x)
    assert abs(b - 3 * 2.0 ** -53 / (1 - 3 * 2.0 ** -53) * (2e16 + 2)) < 1e-6
    naive = ((1e16 + 1.0) - 1e16) + 1.0                          # 1.0: one order loses a unit
    assert naive != 2.0 and abs(naive - 2.0) <= b
    G.check_float_sum(np.array([R.f2bits(naive)]), [2.0], [b], np.array([True]), 0, False)
    with pytest.raises(AssertionError):                          # but a dropped partial is not within it
        G.check_float_sum(np.array([R.f2bits(2.0 - 1e16 * 1e-15)]), [2.0], [b * 1e-3], np.array([True]), 0, False)
    assert G.exact_sum([math.inf, 1.0]) == math.inf and math.isnan(G.exact_sum([math.inf, -math.inf]))
    assert G.exact_sum([1e308] * 4) == math.inf
    assert G.gamma(1) == 0.0


def test_hash1_identity_of_edge_keys():
    nan2 = np.array([0x7FF8000000000001], np.int64).view(np.float64)[0]
    f = col([0.0, -0.0, math.nan, nan2, 1.5, 2.0], R.F64, [0, 0, 0, 0, 0, 1])
    assert G.hash1_identity(f) == [0, 0, G.NULL_GROUP, G.NULL_GROUP, int(R.f2bits(1.5)), G.NULL_GROUP]
    i = col([MIN, 0, MIN + 1, 7], R.I64, [0, 0, 0, 1])
    assert G.hash1_identity(i) == [G.EMPTY_GROUP, 0, MIN + 1, G.NULL_GROUP]
    gid, groups = G.codes(G.hash1_identity(i), np.array([True, True, False, True]))
    assert gid.tolist() == [0, 1, -1, 2] and groups == [G.EMPTY_GROUP, 0, G.NULL_GROUP]


def test_hashk_null_masks_make_distinct_groups():
    a = col([0, 0, 0], R.I64, [1, 0, 0])
    b = col([0.0, -0.0, -0.0], R.F64, [0, 1, 0])
    u = col([1, 1, 1], R.U8)
    ident = G.hashk_identity([a, b, u])
    assert ident == [(0, 0, 1, 1), (0, 0, 1, 2), (0, 0, 1, 0)]


def test_dense_slots_in_uint64_arithmetic():
    k = col([MAX, MAX - 3, MAX - 4, 5, 0], R.I64, [0, 0, 0, 0, 1])
    s = G.dense_slots(k, np.array([True, True, True, True, True]), MAX - 3, 5)
    assert s.tolist() == [3, 0, -1, -1, 4]
    s = G.dense_slots(col([MIN, MIN + 2, MAX], R.I64), np.array([True, False, True]), MIN, 4)
    assert s.tolist() == [0, -1, -1]
    u8 = col([0, 1, 1], R.U8, [0, 0, 1])
    assert G.dense_slots(u8, np.ones(3, bool), 0, 3).tolist() == [0, 1, 2]


def test_star_builds():
    pk = col([12, 10, 14, 10, 11], R.I64, [0, 0, 0, 0, 1])
    grp = col([100, 101, 102, 103, 104], R.I64, [0, 0, 1, 0, 0])
    flag = col([0, 0, 0, 9, 0], R.I64)
    ok = R.eval_terms([flag], [(0, R.LT, 0, 5, 0.0)], 5)
    dirw, slots, dup = G.star_build_bitmap([[flag, pk, grp]], [ok], 1, 2, 10, 40, 100, 7)
    assert not dup                                   # the second 10 is filtered out
    assert dirw[0] == 0b10101 and dirw[1] == 3 << 32
    assert slots.tolist() == [1, 0, 7]               # keys 10, 12, 14 in key order; 14's grp is NULL
    lk, dup = G.star_build_dense(pk, [3, 0, 2], [5, 6, 7], 10, 4)      # pk 14 is outside [10, 14)
    assert lk.tolist() == [5, -1, 6, -1] and not dup
    _, dup = G.star_build_dense(pk, [1, 3], [0, 1], 10, 4)
    assert dup
    m, dup = G.star_map(pk, [0, 1, 4], [1, 2, 3])
    assert m == {12: 1, 10: 2} and not dup
    assert G.star_slots(col([10, 11, 12, 10], R.I64, [0, 0, 0, 1]), np.array([1, 1, 0, 1], bool), m).tolist() == \
        [2, -1, -1, -1]


def test_join_agg_values():
    p = col([3, MAX, 2, 5], R.I64, [0, 0, 0, 1])
    b = col([2, 2, math.nan, 1.5], R.F64)
    matched = np.array([True, True, True, True])
    v = G.join_agg_values(p, b, G.JA_MUL, matched)
    assert v.dtype == R.F64 and v.values[0] == 6.0 and v.values[1] == 2.0 ** 64
    assert v.null.tolist() == [False, False, True, True]
    bi = col([2, 2, 3, 4], R.I64)
    w = G.join_agg_values(p, bi, G.JA_MUL, np.array([True, True, False, True]))
    assert w.values[1] == -2 and w.null.tolist() == [False, False, True, True]      # MAX * 2 wraps
    assert G.join_agg_values(p, bi, G.JA_RSUB, matched).values[0] == -1


def test_range_partition():
    key = col([5, 1, 9, 3, 7, 2], R.I64, [0, 0, 0, 0, 0, 1])
    val = col([50, 10, 90, 30, 70, 20], R.I64)
    ok = np.array([True, True, True, False, True, True])
    starts, buckets = G.range_partition([[key, val]], [ok], 0, 1, 10, 2, 3, [1])
    # slots: 4, 0, 8, -, 6, NULL -> 9;  buckets (slot >> 2): 1, 0, 2, -, 1, 2
    assert starts.tolist() == [0, 1, 3, 5]
    assert buckets[0].tolist() == [[1, 10]]
    assert buckets[1].tolist() == [[5, 50], [7, 70]]
    assert buckets[2].tolist() == [[9, 90], [10, 20]]       # the NULL key comes out as kmin + nslots - 1
