"""CPU side of the natural-collision test (tests/test_gpu_wl_collisions.py): the birthday search over the NumPy
restatement of wl_fused2's level-1 key finds two distinct signatures that share a tag and a start slot, deterministically
and quickly; and the twin fixtures split where the collision tests expect them to."""
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import wl_hash_ref as hr  # noqa: E402
import wl_twins as tw  # noqa: E402
from oracle.gk_oracle import WLOracle, wl_partitions  # noqa: E402


def test_birthday_search_finds_a_tag_and_slot_clash():
    t0 = time.time()
    pair = hr.find_colliding_pair()
    assert time.time() - t0 < 60
    assert pair == hr.find_colliding_pair()  # seeded: the GPU test packs the same two stars
    (oa, na), (ob, nb) = pair
    assert (oa, na) != (ob, nb) and na == sorted(na) and nb == sorted(nb) and max([oa, ob] + na + nb) < 64
    k = hr.key_level1(np.array([oa, ob]), np.array([na, nb]))
    assert k[0] != k[1]
    assert hr.tag(k[0]) == hr.tag(k[1]) and hr.start_slot(k[0], 1024) == hr.start_slot(k[1], 1024)


def test_key_restatement_is_a_63_bit_value():
    k = hr.key_level1(np.arange(5), np.tile(np.arange(8), (5, 1)))
    assert np.all(k < np.uint64(1 << 63)) and len(set(k.tolist())) == 5


def test_twins_differ_in_one_sorted_position():
    for d in tw.DEGREES:
        for pos in tw.POSITIONS:
            a, b = tw.leaf_labels(d, pos, False), tw.leaf_labels(d, pos, True)
            assert a == sorted(a) and b == sorted(b)
            diff = [j for j in range(d) if a[j] != b[j]]
            assert diff == [{"first": 0, "middle": d // 2, "last": d - 1}[pos]]


def test_twin_centres_split_at_their_depth():
    d = 7
    for depth in (1, 3):
        same = tw.twin_pairs(d, "last", depth)[0]  # both centres in one graph: vertex 0 and the first of the second twin
        c2 = 1 + depth * d
        assert same[1][0] == same[1][c2] == tw.CENTRE
        _, levels = WLOracle(n_iter=3).fit_transform([same], return_levels=True)
        split = [levels[lv][0][0] != levels[lv][0][c2] for lv in range(4)]
        assert split == [lv >= depth for lv in range(4)]


def test_filler_never_splits_a_label_degree_group():
    X = tw.filler(4)
    _, levels = WLOracle(n_iter=3).fit_transform(X, return_levels=True)
    assert tw.first_split_level(wl_partitions(levels), tw.degrees_of(X), 1) is None


def test_degree_mixes_pick_each_group_width():
    for width in (8, 16, 32):
        chosen, n_large = tw.group_width(tw.degrees_of(tw.degree_mix(width)))
        assert chosen == width and n_large > 0
