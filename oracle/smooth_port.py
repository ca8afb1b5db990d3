"""Port of the smoothing step (include/spgroup.h "smoothing", ``spg_smooth_frames``) in numpy float64 scalars: a One-Euro
filter (Casiez, Roussel and Vogel, CHI 2012) per track and joint, the behaviour ``dropin.FrameStream(smooth=...)`` and
the device kernel are held to bit for bit.

A stream keeps ``SLOTS`` filter slots keyed by track id.  ``Smoother.step`` takes one frame of a stream -- its time,
``xy [P, 17, 2]``, presence masks and track ids -- and returns the smoothed ``xy``; ``step_record`` takes a wire record
and its ids.  Every operation is one float64 rounding in the order written, as the kernel does without fused
multiply-add."""
from __future__ import annotations

from typing import List, Optional

import numpy as np

SLOTS = 128
JOINTS = 17
TWO_PI = np.float64(6.283185307179586)
_ONE, _ZERO = np.float64(1.0), np.float64(0.0)


class Slot:
    __slots__ = ("id", "last", "mask", "joint")

    def __init__(self, id_: int, last: int):
        self.id, self.last, self.mask = int(id_), int(last), 0
        self.joint = np.zeros((JOINTS, 5), np.float64)  # per joint xh, yh, dxh, dyh, tj


def used_joints(xy: np.ndarray, present: int) -> List[int]:
    """The joints of a person the filter uses: present in the mask, x and y finite."""
    return [g for g in range(JOINTS) if (present >> g) & 1 and np.isfinite(xy[g, 0]) and np.isfinite(xy[g, 1])]


def scale(xy: np.ndarray, used: List[int]) -> np.float64:
    """The person's size: ((xmax - xmin) + (ymax - ymin)) / 2 over the used joints, at least 1."""
    if not used:
        return _ONE
    xs, ys = xy[used, 0], xy[used, 1]
    sc = ((xs.max() - xs.min()) + (ys.max() - ys.min())) / np.float64(2.0)
    return sc if sc > 1.0 else _ONE


class Smoother:
    """Every stream's filter slots.  ``slots[s]`` is stream s's table: ``SLOTS`` entries, each a ``Slot`` or None;
    ``clock[s]`` its frame count."""

    def __init__(self, streams: int = 1, min_cutoff: float = 1.0, beta: float = 1.0, d_cutoff: float = 1.0):
        self.min_cutoff, self.beta, self.d_cutoff = np.float64(min_cutoff), np.float64(beta), np.float64(d_cutoff)
        self.slots: List[List[Optional[Slot]]] = [[None] * SLOTS for _ in range(int(streams))]
        self.clock = [0] * int(streams)

    def step_record(self, stream: int, rec, ids, t: float) -> np.ndarray:
        """One wire record (``wire.record_dtype``) with its rows' ids; ``[n_persons, 17, 2]`` smoothed."""
        n = max(0, min(int(rec["n_persons"]), len(rec["rows"])))
        rows = rec["rows"][:n]
        return self.step(stream, t, np.array(rows["xy"], np.float64), [int(m) for m in rows["present"]],
                         [int(i) for i in ids[:n]])

    def step(self, stream: int, t: float, xy: np.ndarray, present, ids) -> np.ndarray:
        xy = np.array(xy, np.float64).reshape(len(ids), JOINTS, 2)
        out = xy.copy()
        if stream < 0:
            return out
        t = np.float64(t)
        table = self.slots[stream]
        self.clock[stream] += 1
        clock = self.clock[stream]
        slot_of = [None] * len(ids)
        held = {}  # id -> the slot its first row of the frame found or claimed
        for p, pid in enumerate(ids):  # 2. the live slot holding the id, for the id's first row
            if pid < 0 or pid in held:
                continue
            for k, sl in enumerate(table):
                if sl is not None and sl.id == pid:
                    held[pid] = slot_of[p] = k
                    sl.last = clock
                    break
        for p, pid in enumerate(ids):  # 3. claims in row order
            if pid < 0 or slot_of[p] is not None or pid in held:
                continue
            free = [k for k, sl in enumerate(table) if sl is None]
            if free:
                k = free[0]
            else:
                older = [k for k, sl in enumerate(table) if sl.last < clock]
                if not older:  # more than SLOTS ids in one frame
                    continue
                k = min(older, key=lambda k: (table[k].last, k))
            table[k] = Slot(pid, clock)
            held[pid] = slot_of[p] = k
        with np.errstate(all="ignore"):
            for p, k in enumerate(slot_of):
                if k is None:
                    continue
                sl = table[k]
                used = used_joints(xy[p], present[p])
                sc = scale(xy[p], used)
                for g in used:
                    out[p, g] = self._joint(sl, g, t, xy[p, g, 0], xy[p, g, 1], sc)
        return out

    def _joint(self, sl: Slot, g: int, t, x, y, sc) -> tuple:
        xh, yh, dxh, dyh, tj = sl.joint[g]
        dt = t - tj
        if not ((sl.mask >> g) & 1) or not (dt > 0.0 and np.isfinite(dt)):
            xh, yh, dxh, dyh = x, y, _ZERO, _ZERO
        else:
            vx = (x - xh) / dt / sc
            vy = (y - yh) / dt / sc
            ad = _ONE / (_ONE + _ONE / (TWO_PI * self.d_cutoff * dt))
            dxh = ad * vx + (_ONE - ad) * dxh
            dyh = ad * vy + (_ONE - ad) * dyh
            fc = self.min_cutoff + self.beta * np.sqrt(dxh * dxh + dyh * dyh)
            a = _ONE / (_ONE + _ONE / (TWO_PI * fc * dt))
            xh = a * x + (_ONE - a) * xh
            yh = a * y + (_ONE - a) * yh
        sl.joint[g] = (xh, yh, dxh, dyh, t)
        sl.mask |= 1 << g
        return xh, yh
