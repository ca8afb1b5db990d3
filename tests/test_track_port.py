"""CPU: the tracking port (oracle/track_port.py) on hand-built frames -- exact ties, the threshold, ageing and dropping,
eviction from a full table, unobserved frames, non-finite joints, the area clamp and per-stream id counters."""
import math

import numpy as np
import pytest

from improved_body_parts_b200 import wire
from oracle import track_port as tp

# a standing skeleton of 17 joints, about 40 x 100 pixels
BASE = np.array([[20, 10], [18, 8], [22, 8], [15, 9], [25, 9], [10, 25], [30, 25], [8, 45], [32, 45], [6, 60], [34, 60],
                 [14, 60], [26, 60], [13, 80], [27, 80], [12, 100], [28, 100]], np.float64)
ALL = (1 << 17) - 1


def person(dx=0.0, dy=0.0, drop=()):
    """process()-style person: BASE moved by (dx, dy), the joints in ``drop`` absent (integer (0, 0))."""
    pts = [(0, 0) if g in drop else (np.float64(x + dx), np.float64(y + dy)) for g, (x, y) in enumerate(BASE)]
    return pts, np.float64(0.9)


def test_same_pose_has_oks_one_and_a_far_pose_zero():
    tr = tp.Track(0, BASE, ALL)
    assert tp.oks(tr, BASE, ALL) == 1.0
    assert tp.oks(tr, BASE + 1000.0, ALL) == 0.0


def test_oks_follows_cocoeval_formula_joint_by_joint():
    tr = tp.Track(0, BASE, ALL)
    moved = BASE + np.array([3.0, -2.0])
    area = (BASE[:, 0].max() - BASE[:, 0].min()) * (BASE[:, 1].max() - BASE[:, 1].min())
    want = np.float64(0.0)
    for g in range(17):
        want = want + np.exp(-((3.0 * 3.0 + 2.0 * 2.0) / tp.VARS[g] / area / 2.0))
    assert tp.oks(tr, moved, ALL) == want / 17.0


def test_exact_tie_goes_to_the_lower_track_id():
    """Two tracks with identical poses: OKS exactly 1.0 with the person on both sides; the lower id takes it."""
    tk = tp.Tracker()
    assert tk.step_people(0, [person(), person()]) == [0, 1]
    assert tk.step_people(0, [person()]) == [0]
    assert tk.last_oks[(0, 0)] == 1.0 and tk.last_oks[(1, 0)] == 1.0
    assert tk.slots[0][1].age == 1


def test_exact_tie_goes_to_the_lower_person_row():
    tk = tp.Tracker()
    assert tk.step_people(0, [person()]) == [0]
    assert tk.step_people(0, [person(), person()]) == [0, 1]


def test_greedy_takes_the_highest_oks_first():
    """Track 0 is closer to person 1 than to person 0: the pair (0, 1) is taken first, track 1 gets person 0."""
    tk = tp.Tracker(oks_threshold=0.1)
    tk.step_people(0, [person(0.0), person(6.0)])
    assert tk.step_people(0, [person(3.5), person(0.5)]) == [1, 0]


def test_oks_exactly_at_the_threshold_matches():
    tk = tp.Tracker()
    tk.step_people(0, [person()])
    o = tp.oks(tk.slots[0][0], tp.poses_of_people([person(2.0)])[0][0], ALL)
    assert 0.0 < o < 1.0
    at = tp.Tracker(oks_threshold=float(o))
    at.step_people(0, [person()])
    assert at.step_people(0, [person(2.0)]) == [0]
    above = tp.Tracker(oks_threshold=float(np.nextafter(o, 2.0)))
    above.step_people(0, [person()])
    assert above.step_people(0, [person(2.0)]) == [1]


def test_age_and_drop_at_max_age():
    tk = tp.Tracker(max_age=2)
    tk.step_people(0, [person()])
    for age in (1, 2):
        assert tk.step_people(0, []) == []
        assert tk.slots[0][0].age == age
    assert tk.step_people(0, [person()]) == [0]  # age 2 is still kept: a track is dropped when its age exceeds max_age
    for _ in range(3):
        tk.step_people(0, [])
    assert tk.slots[0][0] is None
    assert tk.step_people(0, [person()]) == [1]


def test_max_age_zero_keeps_only_tracks_matched_in_the_last_frame():
    tk = tp.Tracker(max_age=0)
    tk.step_people(0, [person()])
    tk.step_people(0, [person(500.0)])
    assert tk.slots[0][0].id == 1 and all(t is None for t in tk.slots[0][1:])


def test_eviction_of_a_full_table_takes_the_largest_age_then_the_smallest_id():
    tk = tp.Tracker(max_age=1000)
    far = [person(1000.0 * k) for k in range(128)]
    assert tk.step_people(0, far) == list(range(128))
    # tracks 0..63 seen again (age 0), 64..127 not (age 1); then 64..95 seen again
    tk.step_people(0, far[:64])
    tk.step_people(0, far[:96])
    ages = {t.id: t.age for t in tk.slots[0]}
    assert ages[0] == 0 and ages[64] == 0 and ages[96] == 2
    new = [person(1000.0 * k, 5000.0) for k in range(3)]
    assert tk.step_people(0, far[:96] + new) == list(range(96)) + [128, 129, 130]
    ids = sorted(t.id for t in tk.slots[0])
    assert 96 not in ids and 97 not in ids and 98 not in ids and 99 in ids and 130 in ids
    assert [t.id for t in tk.slots[0][96:99]] == [128, 129, 130]  # each in the evicted track's slot


def test_new_tracks_take_the_lowest_free_slot():
    tk = tp.Tracker(max_age=0)
    tk.step_people(0, [person(0.0), person(500.0), person(1000.0)])
    tk.step_people(0, [person(0.0), person(1000.0)])  # track 1 dropped: slot 1 free
    assert tk.step_people(0, [person(0.0), person(1000.0), person(2000.0)]) == [0, 2, 3]
    assert tk.slots[0][1].id == 3


def test_unobserved_frames_age_and_give_minus_one():
    tk = tp.Tracker(max_age=1)
    tk.step_people(0, [person()])
    assert tk.step_people(0, [person(), person(100.0)], observed=False) == [-1, -1]
    assert tk.slots[0][0].age == 1 and tk.slots[0][1] is None
    assert tk.step_people(0, [person()]) == [0]
    rec = wire.pack([[person()]], status=[4])[0]
    assert tk.step_record(0, rec) == [-1]
    rec = wire.pack([[person()]])[0]
    assert tk.step_record(0, rec, jpeg_status=11) == [-1]
    assert tk.slots[0][0] is None  # aged past max_age by the two unobserved frames
    assert tk.step_record(0, rec) == [1]


def test_nonfinite_joints_are_skipped_on_both_sides():
    xy = BASE.copy()
    xy[0] = (np.nan, 10.0)
    xy[1] = (np.inf, 8.0)
    tr = tp.Track(0, xy, ALL)
    # T has 15 joints; the person's joints 0 and 1 do not count, nor do its own non-finite ones
    assert tp.oks(tr, BASE, ALL) == 1.0
    other = BASE.copy()
    other[2] = (-np.inf, np.nan)
    assert tp.oks(tr, other, ALL) == 14.0 / 15.0
    assert tp.oks(tr, other, ALL & ~(1 << 3)) == 13.0 / 15.0
    tk = tp.Tracker()
    tk.step(0, xy[None], [ALL])
    assert tk.step(0, BASE[None], [ALL]) == [0]
    assert np.isnan(tk.slots[0][0].xy[0, 0]) is np.False_  # the track took the new pose


def test_single_joint_track_clamps_its_area_to_one():
    tr = tp.Track(0, BASE, 1 << 5)
    assert tp.oks(tr, BASE, ALL) == 1.0
    moved = BASE + np.array([0.01, 0.0])
    dx = moved[5, 0] - BASE[5, 0]
    assert tp.oks(tr, moved, ALL) == np.exp(-((dx * dx + 0.0) / tp.VARS[5] / 1.0 / 2.0))
    assert tp.oks(tp.Track(0, BASE, 0), BASE, ALL) == 0.0  # no joint: OKS 0, never matched


def test_streams_have_independent_id_counters():
    tk = tp.Tracker(streams=3)
    assert tk.step_people(1, [person(), person(300.0)]) == [0, 1]
    assert tk.step_people(0, [person()]) == [0]
    assert tk.step_people(1, [person(900.0)]) == [2]
    assert tk.step_people(2, [person(900.0)]) == [0]
    assert tk.next_id == [1, 3, 1]


def test_a_record_and_its_people_track_alike():
    people = [person(3.0 * k, 7.0 * k, drop=(k, 16 - k)) for k in range(5)]
    a, b = tp.Tracker(), tp.Tracker()
    rec = wire.pack([people])[0]
    for step in range(3):
        moved = [person(3.0 * k + step, 7.0 * k, drop=(k, 16 - k)) for k in range(5)]
        assert a.step_people(0, moved) == b.step_record(0, wire.pack([moved])[0])
    assert b.step_record(0, rec) == list(range(5))
    assert math.isfinite(float(a.last_oks[(0, 0)]))


@pytest.mark.parametrize("thr", [0.0, 0.3, 0.9])
def test_sorted_greedy_result_is_a_matching(thr):
    rng = np.random.default_rng(7)
    tk = tp.Tracker(oks_threshold=thr)
    for _ in range(6):
        people = [person(*rng.normal(0, 20, 2)) for _ in range(int(rng.integers(0, 12)))]
        ids = tk.step_people(0, people)
        assert len(set(ids)) == len(ids) and min(ids, default=0) >= 0
