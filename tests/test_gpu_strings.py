"""The VARCHAR device pieces through the C-ABI, entry for entry against tests/strings_ref.py:
b2_str_like over a seeded corpus (ASCII, 2- / 3- / 4-byte code points, wildcards and escape characters in
the data, newlines, the empty string, entries over 1 KB, dictionaries of 0 and 1 entries) in LIKE and ILIKE,
b2_str_lower_bound in both modes, and B2_OP_MAP on NULL, out-of-range and cleared entries with both table
dtypes."""
import random

import numpy as np
import pyarrow as pa
import pytest

from tests import strings_ref as R

pytestmark = pytest.mark.gpu

ALPHABET = list("abcAB%_\\!\n ") + ["é", "Ä", "ß", "中", "€", "😀", "𝄞"]


def _dev():
    import torch
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _dictionary(strings):
    from dask_sql_b200 import strings as S
    d = S.Dictionary(pa.array(R.dictionary(strings), type=pa.large_string()))
    assert d.to_list() == R.dictionary(strings)
    return d


def _corpus(seed, n=600):
    rnd = random.Random(seed)
    out = {"", "a", "A", "%", "_", "\\", "abc\n", "\n", "😀", "a\nb"}
    while len(out) < n:
        k = rnd.choice([1, 2, 3, 5, 8, 13])
        out.add("".join(rnd.choice(ALPHABET) for _ in range(k)))
    for k in (1100, 1500):                        # entries longer than 1 KB
        out.add("".join(rnd.choice(ALPHABET) for _ in range(k)))
        out.add("x" * k + "abc")
    return sorted(out)


def _patterns(seed, n=120):
    rnd = random.Random(seed)
    pats = ["%", "", "_", "%%", "a%", "%a", "%a%", "a_c", "%\\%%", "\\_", "%\\\\%", "___", "%_%_%", "abc",
            "é%", "%😀", "_😀%", "%\n%", "%ß_", "x%abc", "%abc", "A%", "%b%c%", "%%_%%"]
    while len(pats) < n:
        k = rnd.choice([1, 2, 3, 4, 6])
        pats.append("".join(rnd.choice(ALPHABET + ["%", "_", "%"]) for _ in range(k)))
    return pats


def _like_table(d, pattern, escape, ilike):
    from dask_sql_b200 import strings as S
    col = S.like_table(d, pattern, escape, ilike, _dev())
    return col.data.cpu().numpy().astype(bool).tolist()


@pytest.mark.parametrize("ilike", [False, True])
def test_str_like_matches_reference_entry_for_entry(ilike):
    words = _corpus(7)
    d = _dictionary(words)
    for pattern in _patterns(11):
        got = _like_table(d, pattern, "\\", ilike)
        want = [R.like(w, pattern, "\\", ilike) for w in words]
        assert got == want, pattern


def test_str_like_escape_characters():
    words = _corpus(3, 200) + ["a%b", "a!%b", "Ä%", "ÄÄ", "Ä_x", "!"]
    d = _dictionary(words)
    words = d.to_list()
    for pattern, escape in [("a!%b", "!"), ("%!_%", "!"), ("Ä%Ä_%", "Ä"), ("!!", "!"), ("a%b", None),
                            ("%\\%", None), ("x!", "!"), ("Ä%", "Ä"), ("😀%", "😀"), ("%😀_", "😀")]:
        got = _like_table(d, pattern, escape, False)
        assert got == [R.like(w, pattern, escape) for w in words], (pattern, escape)
    # ILIKE with a letter escape: the escape is recognised as written, only literals fold
    d = _dictionary(words + ["xR", "xr%", "XR%", "x%", "X%a", "xRa", "r", "R"])
    words = d.to_list()
    for pattern, escape in [("xR%", "r"), ("xr%", "r"), ("Xr%", "r"), ("R%", "r"), ("rr", "r"), ("ä%", "Ä")]:
        got = _like_table(d, pattern, escape, True)
        assert got == [R.like(w, pattern, escape, True) for w in words], (pattern, escape)


@pytest.mark.parametrize("words", [[], ["only"], [""]])
def test_str_like_tiny_dictionaries(words):
    d = _dictionary(words)
    for p in ["%", "", "o%", "_", "only"]:
        assert _like_table(d, p, "\\", False) == [R.like(w, p) for w in d.to_list()]


def test_str_lower_bound_both_modes():
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import strings as S
    a_words = _corpus(21, 500)
    b_words = _corpus(22, 700) + a_words[::3] + ["\x00", "\U0010ffff"]
    for aw, bw in [(a_words, b_words), ([], b_words), (a_words, []), (a_words[:1], b_words)]:
        a, b = _dictionary(aw), _dictionary(bw)
        m = S.lower_bound_table(a, b, L.STR_LB_MATCH, _dev())
        o = S.lower_bound_table(a, b, L.STR_LB_ORDER, _dev())
        bl = b.to_list()
        want_m = R.lb_match(a.to_list(), bl)
        want_o = R.lb_order(a.to_list(), bl)
        if not bl:
            continue
        codes = m.data.cpu().numpy()
        bits = np.unpackbits(m.valid.cpu().numpy().view(np.uint8), bitorder="little")[: len(bl)].astype(bool)
        assert bits.tolist() == [x is not None for x in want_m]
        assert codes[bits].tolist() == [x for x in want_m if x is not None]
        assert o.valid is None and o.data.cpu().numpy().tolist() == want_o


@pytest.mark.parametrize("dtype", ["i64", "u8"])
def test_op_map_nulls_ranges_and_cleared_entries(dtype):
    import torch
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import device as D
    from dask_sql_b200.device import DeviceColumn, _pack_valid
    dev = _dev()
    rng = np.random.default_rng(5)
    ntab = 37
    if dtype == "i64":
        tab = rng.integers(-2**62, 2**62, ntab)
        tcol = DeviceColumn(torch.from_numpy(tab).to(dev), None, L.I64)
    else:
        tab = rng.integers(0, 2, ntab).astype(np.uint8)
        tcol = DeviceColumn(torch.from_numpy(tab).to(dev), None, L.U8)
    cleared = rng.random(ntab) < 0.2
    tcol.valid = torch.from_numpy(_pack_valid(cleared)).to(dev)
    n = 5000
    x = rng.integers(-5, ntab + 5, n)
    x[:4] = [-(1 << 63), (1 << 63) - 1, ntab, -1]
    xnull = rng.random(n) < 0.1
    xcol = DeviceColumn(torch.from_numpy(x).to(dev), torch.from_numpy(_pack_valid(xnull)).to(dev), L.I64)
    for imm in (ntab, 10, 0):
        p = L.Prog()
        p.n, p.out_dtype = 2, L.I64
        p.code[0].op, p.code[0].a = L.OP_LOAD, 0
        p.code[1].op, p.code[1].a, p.code[1].imm_i = L.OP_MAP, 1, imm
        out = D.expr_eval(p, [xcol, tcol], n, True)
        got = out.data.cpu().numpy()
        valid = np.unpackbits(out.valid.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)
        inr = (x >= 0) & (x < imm)
        want_valid = ~xnull & inr
        want_valid[inr] &= ~cleared[x[inr]]
        assert valid.tolist() == want_valid.tolist()
        np.testing.assert_array_equal(got[valid], tab[x[valid]].astype(np.int64))
    bad = L.Prog()
    bad.n, bad.out_dtype = 2, L.I64
    bad.code[0].op = L.OP_LOAD
    bad.code[1].op, bad.code[1].a, bad.code[1].imm_i = L.OP_MAP, 2, 1      # no such column
    with pytest.raises(L.B200SqlError):
        D.expr_eval(bad, [xcol, tcol], n, True)
