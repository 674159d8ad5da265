"""CPU tests of tests/train_ref.py: the special-frame layout of the training sequence and the rulebook comparison."""
import numpy as np
import pytest

import train_ref as tr


@pytest.mark.parametrize("B", [2, 3, 4, 5, 8, 12])
def test_every_special_frame_appears(B):
    lay = dict(tr.special_layout(B))
    assert set(lay) == {1, 2}
    shown = set(lay[1].values()) | set(lay[2].values())
    assert shown == set(tr.SPECIALS)
    for where in lay.values():
        assert all(0 <= p < B for p in where) and len(set(where.values())) == len(where)
    assert {0, B - 1} <= set(lay[2])


def _table():
    """two frames of a toy strided conv: inputs, outputs in an order of their own, and the oracle's view of frame 1"""
    cin = np.array([[0, 0, 0, 0], [1, 0, 0, 1], [1, 0, 1, 1], [1, 0, 2, 2]], np.int32)
    cout = np.array([[0, 0, 0, 0], [1, 0, 1, 1], [1, 0, 0, 0]], np.int32)
    nbr = np.array([[0, -1], [2, 3], [1, -1]], np.int32)
    o_out = np.array([[0, 0, 0, 0], [0, 0, 1, 1]], np.int32)            # oracle order differs from ours
    pairs = np.full((2, 2, 3), -1, np.int32)
    pairs[0, :, :2] = [[0, 1], [0, 1]]                                   # offset 0: in 0 -> out 0, in 1 -> out 1
    pairs[1, :, :1] = [[2], [1]]                                         # offset 1: in 2 -> out 1
    pnum = np.array([2, 1], np.int32)
    return cin, cout, nbr, o_out, pairs, pnum


def test_rulebook_comparison_accepts_a_reordered_frame_and_rejects_a_wrong_neighbour():
    cin, cout, nbr, o_out, pairs, pnum = _table()
    assert tr.compare_rulebook(cin, cout, nbr, 1, o_out, pairs, pnum) is None
    bad = nbr.copy()
    bad[1, 1] = 1
    assert "row 1 offset 1" in tr.compare_rulebook(cin, cout, bad, 1, o_out, pairs, pnum)
    moved = cout.copy()
    moved[1, 3] = 2
    assert "coordinates" in tr.compare_rulebook(cin, moved, nbr, 1, o_out, pairs, pnum)
