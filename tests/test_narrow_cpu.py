"""Which int64 columns a star scan streams as 32-bit images, and from which base (device.narrow_base): every
non-NULL value in [vmin, vmin + 2^32), decided exactly at the ends of int64."""
import pytest

from dask_sql_b200.device import F64, I64, Stats, narrow_base

I64_MAX, I64_MIN = 2 ** 63 - 1, -(2 ** 63)


@pytest.mark.parametrize("lo,hi,base", [
    (0, 2 ** 32 - 1, 0),                         # span 2^32 - 1: the widest that fits
    (0, 2 ** 32, None),                          # span 2^32: one value too many
    (-(2 ** 31), 2 ** 31 - 1, -(2 ** 31)),
    (I64_MIN, I64_MIN + 2 ** 32 - 1, I64_MIN),
    (I64_MIN, I64_MIN + 2 ** 32, None),
    (I64_MAX - (2 ** 32 - 1), I64_MAX, I64_MAX - (2 ** 32 - 1)),
    (I64_MAX - 2 ** 32, I64_MAX, None),
    (I64_MIN, I64_MAX, None),
    (-5, -5, -5),
])
def test_narrow_base(lo, hi, base):
    assert narrow_base(Stats(lo, hi, 0), I64) == base


def test_no_image_without_values_or_for_floats():
    assert narrow_base(Stats(None, None, 10), I64) is None
    assert narrow_base(Stats(0.0, 1.0, 0), F64) is None

