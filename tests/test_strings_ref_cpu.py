"""The host reference of the VARCHAR rules (tests/strings_ref.py) reproduces the reference project's
known answers (tests/golden/reference_strings.py)."""
import re

import pytest

from tests import strings_ref as R
from tests.golden import reference_strings as G


def _parse_like(pred):
    m = re.fullmatch(r"a (NOT )?(I?LIKE) '(.*?)'(?: ESCAPE '(.)')?", pred, re.S)
    return bool(m.group(1)), m.group(2) == "ILIKE", m.group(3), m.group(4) or "\\"


@pytest.mark.parametrize("pred,rows", G.LIKE_CASES)
def test_like_reference_answers(pred, rows):
    neg, ilike, pattern, escape = _parse_like(pred)
    got = [i for i, s in enumerate(G.STRING_TABLE) if R.like(s, pattern, escape, ilike) != neg]
    assert got == rows


def test_sort_reference_answer():
    assert R.dictionary(G.SORT_TABLE) == G.SORT_ASC


def test_filter_reference_answers():
    for pred, rows in G.FILTER_CASES:
        lit = re.fullmatch(r"a = '(.*)'", pred).group(1)
        assert [i for i, s in enumerate(G.STRING_TABLE) if s == lit] == rows


def test_lower_bound_modes():
    a = ["", "a", "ab", "b", "é", "😀"]
    b = ["", "aa", "b", "zz", "é", "😀😀", "\x00"]
    assert R.lb_match(a, b) == [0, None, 3, None, 4, None, None]
    assert R.lb_order(a, b) == [0, 3, 6, 7, 8, 11, 1]


def test_trailing_newline_is_not_dropped():
    # `$` in the reference's re.match('^...$') matches before a trailing newline; a full match does not
    assert not R.like("abc\n", "abc")
    assert R.like("abc\n", "abc%")
    assert R.like("a\nb", "a_b")
