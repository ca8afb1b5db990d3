"""CPU: the host logic of the capacity-free tier's fallback in ``dropin`` (no device needed)."""
import numpy as np

from improved_body_parts_b200 import dropin, grouping, wire
from improved_body_parts_b200.skeleton import COCO_FROM_PART, NUM_PARTS


def test_capacity_bits_select_the_tier_and_nothing_else():
    G = grouping
    for bit in (G.ST_PEAK_OVERFLOW, G.ST_CAND_OVERFLOW, G.ST_ROW_OVERFLOW):
        assert dropin._over_capacity(bit) and dropin._over_capacity(np.uint32(bit | G.ST_SAMPLE_INDEX))
    for bit in (0, G.ST_SAMPLE_INDEX, G.ST_ASSERT, G.ST_WIRE_OVERFLOW):
        assert not dropin._over_capacity(bit)


def _result(n_persons, rows, seed=0):
    rng = np.random.default_rng(seed)
    K, J = NUM_PARTS, len(COCO_FROM_PART)
    subset = np.full((1, rows, K + 2, 2), -1.0)
    present = rng.random((rows, K)) < 0.6
    subset[0, :, :K, 0] = np.where(present, np.arange(rows * K).reshape(rows, K), -1)
    xy = rng.random((1, rows, J, 2)) * 100
    for j in range(rows):
        for g, part in enumerate(COCO_FROM_PART):
            if not present[j, part]:
                xy[0, j, g] = 0.0
    empty = np.zeros((1, 0))
    return grouping.GroupResult(K=K, L=0, limbs=np.zeros((0, 2), np.int32), peak_count=empty, peak_x=empty, peak_y=empty,
                                peak_score=empty, peak_anchor=empty, conn_count=empty, cand_count=empty, conn_ij=empty,
                                conn_score=empty, conn_norm=empty, n_persons=np.array([n_persons], np.int32),
                                subset=subset, people_xy=xy, people_score=rng.random((1, rows)),
                                status=np.zeros(1, np.uint32)), present


def test_people_of_result_is_what_a_wire_record_gives():
    """predict_many takes a regrouped image's persons from the tier's arrays: same values and types as the persons of a
    wire record, for more persons than a record holds."""
    r, present = _result(200, 210)
    people = dropin._people_of_result(r)
    assert len(people) == 200
    rec = np.zeros((1,), wire.record_dtype(len(COCO_FROM_PART), 200))[0]
    rec["n_persons"] = 200
    for j in range(200):
        rec["rows"][j]["xy"] = r.people_xy[0, j]
        rec["rows"][j]["score"] = r.people_score[0, j]
        rec["rows"][j]["present"] = sum(1 << g for g, part in enumerate(COCO_FROM_PART) if present[j, part])
    expect = wire.people_of(rec)
    assert [[(type(x).__name__, x, type(y).__name__, y) for x, y in p] for p, _ in people] == \
           [[(type(x).__name__, x, type(y).__name__, y) for x, y in p] for p, _ in expect]
    assert [s for _, s in people] == [s for _, s in expect] and all(type(s) is np.float64 for _, s in people)


def test_unbounded_entries_are_declared():
    assert "spg_group_unbounded" in grouping.EXPORTS and "spg_download_unbounded" in grouping.EXPORTS


def test_sizes_record_is_four_words(tmp_path):
    """Grouper.group_unbounded reads spg_unbounded_sizes as four 32-bit words."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    probe, exe = tmp_path / "probe.c", tmp_path / "probe"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "spgroup.h"\nint main(void){printf("%zu %zu %zu %zu %zu",'
                     'sizeof(spg_unbounded_sizes), offsetof(spg_unbounded_sizes, cap_peaks), offsetof(spg_unbounded_sizes, '
                     'cap_rows), offsetof(spg_unbounded_sizes, n_persons), offsetof(spg_unbounded_sizes, status));return 0;}\n')
    subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), str(probe), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).split() == ["16", "0", "4", "8", "12"]
