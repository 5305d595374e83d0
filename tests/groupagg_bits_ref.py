"""The AND / OR / XOR accumulators of include/b200sql.h on top of the group-by reference of tests/groupagg_ref.py:
AND / OR / XOR fold the 64-bit words of int64 inputs, or the 0 / 1 of U8 inputs; AND starts at all ones, OR and
XOR at 0; a slot no row reaches, and an accumulator whose inputs in the slot are all NULL, keep that initial word.
Every other op is left to groupagg_ref.  No GPU and no package import."""
import numpy as np

from tests import groupagg_ref as G

AGG_AND, AGG_OR, AGG_XOR = 5, 6, 7
BIT_UFUNC = {AGG_AND: np.bitwise_and, AGG_OR: np.bitwise_or, AGG_XOR: np.bitwise_xor}

# groupagg_ref's own functions, whatever later stands in for them (see install())
_aggregate, _initial_word = G.aggregate, G.initial_word


def initial_word(op, dtype, indicator=False):
    """groupagg_ref.initial_word, and -1 for AND, 0 for OR / XOR"""
    if op in BIT_UFUNC:
        return -1 if op == AGG_AND else 0
    return _initial_word(op, dtype, indicator)


def aggregate(inputs, ops, gid, nslots, indicator=None) -> G.Expected:
    """groupagg_ref.aggregate with the bitwise ops: their counts come from it (as COUNT), their words from here"""
    ex = _aggregate(inputs, [G.AGG_COUNT if op in BIT_UFUNC else op for op in ops], gid, nslots, indicator)
    gid = np.asarray(gid, np.int64)
    for a, (col, op) in enumerate(zip(inputs, ops)):
        if op not in BIT_UFUNC:
            continue
        ok = (gid >= 0) & ~G.null_of(col)
        words = np.full(nslots, initial_word(op, col.dtype), np.int64)
        BIT_UFUNC[op].at(words, gid[ok], col.raw()[ok])
        ex.acc[a] = words
    return ex


def permute(ex: G.Expected, slot_of_group, nslots, indicator=None, inputs=None, ops=None) -> G.Expected:
    """groupagg_ref.permute; slots no group moves to keep the bitwise ops' initial words"""
    ops = list(ops or [])
    out = G.permute(ex, slot_of_group, nslots, indicator, inputs, [G.AGG_SUM if op in BIT_UFUNC else op for op in ops])
    moved = np.zeros(nslots, bool)
    moved[np.asarray(slot_of_group, np.int64)] = True
    for a, op in enumerate(ops):
        if op == AGG_AND and out.acc[a] is not None:
            out.acc[a][~moved] = -1
    return out


def global_words(ex, ops, inputs):
    """b2_scan_agg / b2_join_agg outputs; an output with no row is the op's identity (-1 for AND)"""
    return G.global_words(ex, ops, inputs)


def install(monkeypatch):
    """let the kernel-checking helpers of tests/test_gpu_groupagg.py, which read the reference through
    groupagg_ref, see the bitwise ops for the duration of one test"""
    monkeypatch.setattr(G, "aggregate", aggregate)
    monkeypatch.setattr(G, "initial_word", initial_word)
