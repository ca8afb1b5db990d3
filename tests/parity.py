"""Comparison helpers shared by the parity tests.

The reference's outputs are nested Python structures (evaluate.py:203,276,498):
``all_peaks``  list[K] of list of (x, y, score, id)
``connection_all`` list[L] of ndarray[n,6] | []   rows [idA, idB, score, i, j, norm]
``special_k``  list[int]
``subset``     ndarray[P, K+2, 2] f64
``candidate``  ndarray[N, 4] f64

``diff_structures`` returns human-readable mismatch strings.  Integer content (anchors, ids, counts,
(i, j), membership) must always be identical; floats are compared bit-exactly when ``float_tol == 0``
and within ``float_tol`` (the north-star's 1e-4) otherwise.
"""
from __future__ import annotations

from typing import List

import numpy as np

FLOAT_TOL = 1e-4  # BASELINE.json north_star: "float connection scores within 1e-4"


def _feq(a, b, tol) -> bool:
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    if tol == 0:  # bit-exact values; NaN (maps with non-finite values) compared by position
        return bool(np.array_equal(a, b, equal_nan=True))
    return bool(np.all(np.abs(a - b) <= tol))


def diff_structures(ref, got, float_tol: float = 0.0, max_report: int = 12) -> List[str]:
    r_peaks, r_conn, r_special, r_subset, r_cand = ref
    g_peaks, g_conn, g_special, g_subset, g_cand = got
    out: List[str] = []

    def rep(msg):
        if len(out) < max_report:
            out.append(msg)

    if len(r_peaks) != len(g_peaks):
        rep(f"peaks: {len(r_peaks)} parts vs {len(g_peaks)}")
    for c, (rp, gp) in enumerate(zip(r_peaks, g_peaks)):
        if len(rp) != len(gp):
            rep(f"part {c}: {len(rp)} peaks vs {len(gp)}")
            continue
        for q, (a, b) in enumerate(zip(rp, gp)):
            if int(a[3]) != int(b[3]):
                rep(f"part {c} peak {q}: id {a[3]} vs {b[3]}")
            # integer-ness of border peaks (util.py:201-202) is part of the contract
            a_int = isinstance(a[0], (int, np.integer))
            b_int = isinstance(b[0], (int, np.integer))
            if a_int != b_int:
                rep(f"part {c} peak {q}: integer-coordinate flag {a_int} vs {b_int}")
            if not (_feq(a[0], b[0], float_tol) and _feq(a[1], b[1], float_tol)):
                rep(f"part {c} peak {q}: xy ({a[0]!r},{a[1]!r}) vs ({b[0]!r},{b[1]!r})")
            if not _feq(a[2], b[2], float_tol):
                rep(f"part {c} peak {q}: score {a[2]!r} vs {b[2]!r}")
    if list(r_special) != list(g_special):
        rep(f"special_k {list(r_special)} vs {list(g_special)}")
    for k, (rc, gc) in enumerate(zip(r_conn, g_conn)):
        rc_empty = isinstance(rc, list)
        gc_empty = isinstance(gc, list)
        if rc_empty != gc_empty:
            rep(f"limb {k}: special-ness differs")
            continue
        if rc_empty:
            continue
        if rc.shape != gc.shape:
            rep(f"limb {k}: {rc.shape[0]} connections vs {gc.shape[0]}")
            continue
        if rc.shape[0] == 0:
            continue
        if not np.array_equal(rc[:, [0, 1, 3, 4]], gc[:, [0, 1, 3, 4]]):
            rep(f"limb {k}: accepted (idA,idB,i,j) differ")
        if not _feq(rc[:, 2], gc[:, 2], float_tol):
            rep(f"limb {k}: scores differ, max |d|={np.max(np.abs(rc[:, 2] - gc[:, 2])):.3e}")
        if not _feq(rc[:, 5], gc[:, 5], float_tol):
            rep(f"limb {k}: norms differ, max |d|={np.max(np.abs(rc[:, 5] - gc[:, 5])):.3e}")
    if r_subset.shape != g_subset.shape:
        rep(f"subset shape {r_subset.shape} vs {g_subset.shape}")
    else:
        if not np.array_equal(r_subset[:, :-2, 0], g_subset[:, :-2, 0]):
            rep("subset: person membership (peak ids) differs")
        if not np.array_equal(r_subset[:, -1, 0], g_subset[:, -1, 0]):
            rep("subset: part counts differ")
        if not _feq(r_subset, g_subset, float_tol):
            rep(f"subset: float content differs, max |d|={np.max(np.abs(r_subset - g_subset)):.3e}")
    r_cand = np.asarray(r_cand, np.float64)
    g_cand = np.asarray(g_cand, np.float64)
    if r_cand.shape != g_cand.shape:
        rep(f"candidate shape {r_cand.shape} vs {g_cand.shape}")
    elif not _feq(r_cand, g_cand, float_tol):
        rep("candidate differs")
    return out


def structure_stats(s) -> dict:
    peaks, conn, special, subset, cand = s
    return {"peaks": int(sum(len(p) for p in peaks)),
            "connections": int(sum(0 if isinstance(c, list) else c.shape[0] for c in conn)),
            "special": len(special), "persons": int(subset.shape[0])}
