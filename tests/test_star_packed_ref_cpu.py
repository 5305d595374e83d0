"""The packed slot layout of the ranked-bitmap star lookup, on the CPU: the width rule at its class
edges (reference and executor agree), hand-packed words, and the 32-bit case as the int32 array's bytes."""
import numpy as np
import pytest

from tests import star_packed_ref as S


@pytest.mark.parametrize("null_slot,bits", [(0, 16), (2 ** 16 - 1, 16), (2 ** 16, 21), (2 ** 21 - 1, 21),
                                            (2 ** 21, 32), (2 ** 31 - 1, 32)])
def test_width_at_the_class_edges(null_slot, bits):
    from dask_sql_b200 import executor
    assert S.slot_bits(null_slot) == bits
    assert executor._star_slot_bits(null_slot) == bits


def test_hand_packed_k4():
    words = S.pack_slots([1, 2, 0xFFFF, 0x8000, 7], 16)
    assert words.tolist() == [0x8000_FFFF_0002_0001, 7]


def test_hand_packed_k3():
    m = (1 << 21) - 1
    words = S.pack_slots([m, 1, 5, 2 ** 20, 3], 21, nentries=9)
    assert words.tolist() == [m | (1 << 21) | (5 << 42), (2 ** 20) | (3 << 21), 0]
    assert int(words[0]) >> 63 == 0                       # the 64th bit is never used


def test_32_bits_is_the_int32_array():
    rng = np.random.default_rng(0)
    for n in (1, 2, 5, 1000):
        slots = rng.integers(0, 2 ** 31, n).astype(np.int32)
        words = S.pack_slots(slots, 32)
        assert words.tobytes()[:4 * n] == slots.tobytes()
        assert words.tobytes()[4 * n:] == b"\0" * (len(words) * 8 - 4 * n)


@pytest.mark.parametrize("bits", [16, 21, 32])
def test_unpack_inverts_pack(bits):
    rng = np.random.default_rng(bits)
    slots = rng.integers(0, 2 ** bits, 1001)
    assert (S.unpack_slots(S.pack_slots(slots, bits), bits, len(slots)) == slots).all()


@pytest.mark.parametrize("bits", [16, 21, 32])
def test_buffer_layout_keeps_slots_8_byte_aligned(bits):
    """_star_bitmap_words: the slots start at an even int32 offset, hold every entry at their width and end
    on a 64-bit word"""
    from dask_sql_b200 import executor
    for prange, dn in [(1, 1), (31, 7), (33, 100), (10_000_000, 5_000_000), (10_000_001, 5_000_001)]:
        slots, flags, total = executor._star_bitmap_words(prange, dn, bits)
        assert slots % 2 == 0 and flags % 2 == 0 and total == flags + 4
        assert slots == 2 * ((prange + 31) // 32)
        assert (flags - slots) * 32 >= min(dn, prange) * bits
        assert len(S.pack_slots(np.zeros(min(dn, prange)), bits)) * 2 == flags - slots
