"""Port of the tracking step (include/spgroup.h "tracking", ``spg_track_frames``) in numpy float64, with the plain sorted
greedy: the behaviour ``dropin.FrameStream(track=...)`` and the device kernel are held to.

A stream keeps at most ``SLOTS`` tracks, each with its id, age and last pose (17 x (x, y) float64 and a presence mask,
as a wire record row stores them).  ``Tracker.step`` takes one frame of a stream, as a wire record (``step_record``) or
as ``process()``-style people (``step_people``), and returns the id of each person."""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np

SLOTS = 128
JOINTS = 17
#: cocoeval.py's kpt_oks_sigmas and the variances its computeOks uses
SIGMAS = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89]) / 10.0
VARS = (SIGMAS * 2) ** 2


class Track:
    __slots__ = ("id", "age", "xy", "present")

    def __init__(self, id_: int, xy: np.ndarray, present: int):
        self.id, self.age, self.xy, self.present = int(id_), 0, np.array(xy, np.float64), int(present)


def _finite(xy: np.ndarray, present: int, g: int) -> bool:
    return bool((present >> g) & 1) and math.isfinite(xy[g, 0]) and math.isfinite(xy[g, 1])


def oks(track: Track, xy: np.ndarray, present: int) -> np.float64:
    """OKS of a person (``xy [17, 2]``, ``present`` mask) against a track's pose as ground truth."""
    T = [g for g in range(JOINTS) if _finite(track.xy, track.present, g)]
    if not T:
        return np.float64(0.0)
    xs, ys = track.xy[T, 0], track.xy[T, 1]
    area = (xs.max() - xs.min()) * (ys.max() - ys.min())
    area = area if area > 1.0 else np.float64(1.0)
    total = np.float64(0.0)
    for g in T:
        if not _finite(xy, present, g):
            continue
        dx, dy = xy[g, 0] - track.xy[g, 0], xy[g, 1] - track.xy[g, 1]
        e = (dx * dx + dy * dy) / VARS[g] / area / np.float64(2.0)
        total = total + np.exp(-e)
    return total / np.float64(len(T))


def poses_of_people(people) -> tuple:
    """``process()``-style people -> ``(xy [P, 17, 2], present [P])``: an integer ``(0, 0)`` is an absent joint, as
    ``wire.pack`` reads it."""
    xy = np.zeros((len(people), JOINTS, 2), np.float64)
    present = []
    for p, (pts, _) in enumerate(people):
        m = 0
        for g, (x, y) in enumerate(pts):
            if isinstance(x, (int, np.integer)) and isinstance(y, (int, np.integer)) and x == 0 and y == 0:
                continue
            xy[p, g] = (x, y)
            m |= 1 << g
        present.append(m)
    return xy, present


class Tracker:
    """Every stream's tracks.  ``slots[s]`` is stream s's table: ``SLOTS`` entries, each a ``Track`` or None."""

    def __init__(self, streams: int = 1, oks_threshold: float = 0.5, max_age: int = 30):
        self.oks_threshold, self.max_age = float(oks_threshold), int(max_age)
        self.slots: List[List[Optional[Track]]] = [[None] * SLOTS for _ in range(int(streams))]
        self.next_id = [0] * int(streams)
        self.last_oks: dict = {}  # (slot, row) -> OKS of the last observed frame

    def step_people(self, stream: int, people, observed: bool = True) -> List[int]:
        xy, present = poses_of_people(people)
        return self.step(stream, xy, present, observed)

    def step_record(self, stream: int, rec, jpeg_status: int = 0) -> List[int]:
        """One wire record (``wire.record_dtype``); a status bit or a JPEG status other than 0 makes it unobserved."""
        n = int(rec["n_persons"])
        rows = rec["rows"][:max(0, min(n, len(rec["rows"])))]
        observed = int(rec["status"]) == 0 and int(jpeg_status) == 0
        return self.step(stream, np.array(rows["xy"], np.float64), [int(m) for m in rows["present"]], observed)

    def step(self, stream: int, xy: np.ndarray, present, observed: bool = True) -> List[int]:
        table = self.slots[stream]
        P = len(present)
        if not observed:
            self._age(table, set())
            return [-1] * P
        self.last_oks = {}
        pairs = []
        for t, tr in enumerate(table):
            if tr is None:
                continue
            for p in range(P):
                o = oks(tr, xy[p], present[p])
                self.last_oks[(t, p)] = o
                if o >= self.oks_threshold:
                    pairs.append((-o, tr.id, p, t))
        pairs.sort()
        ids = [-1] * P
        slot_taken, row_taken = set(), set()
        for _, tid, p, t in pairs:
            if t in slot_taken or p in row_taken:
                continue
            slot_taken.add(t)
            row_taken.add(p)
            table[t].xy, table[t].present, table[t].age = np.array(xy[p], np.float64), int(present[p]), 0
            ids[p] = tid
        self._age(table, slot_taken)
        for p in range(P):
            if p in row_taken:
                continue
            free = [t for t, tr in enumerate(table) if tr is None]
            if free:
                slot = free[0]
            else:  # the largest age, ties to the smallest id
                slot = min(range(SLOTS), key=lambda t: (-table[t].age, table[t].id))
            table[slot] = Track(self.next_id[stream], xy[p], present[p])
            ids[p] = self.next_id[stream]
            self.next_id[stream] += 1
        return ids

    def _age(self, table, matched) -> None:
        for t, tr in enumerate(table):
            if tr is not None and t not in matched:
                tr.age += 1
                if tr.age > self.max_age:
                    table[t] = None
