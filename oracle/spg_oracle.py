"""ctypes front-end of the CPU checker ``libspg_oracle.so`` (see spg_oracle.c).

TEST INFRASTRUCTURE, NOT PRODUCT: only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may import this module.  Nothing under
``improved_body_parts_b200/`` does.

``OracleResult`` holds the flat arrays; ``as_reference_structures`` rebuilds exactly the Python objects
the reference's functions return (``all_peaks``, ``connection_all``, ``special_k``, ``subset``,
``candidate`` -- evaluate.py:203,276,498) so they can be compared with goldens value for value.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
import subprocess
from typing import List, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libspg_oracle.so")

ERR_CAPACITY, ERR_INDEX, ERR_ASSERT, ERR_NONFINITE, ERR_NAN_PRIORITY = -1, -2, -3, -4, -5


class _Params(C.Structure):
    _fields_ = [("thre1", C.c_double), ("thre2", C.c_double), ("connect_ration", C.c_double),
                ("len_rate", C.c_double), ("connection_tole", C.c_double), ("min_mean_score", C.c_double),
                ("mid_num", C.c_int32), ("offset_radius", C.c_int32), ("remove_recon", C.c_int32),
                ("min_parts", C.c_int32), ("crit1_strict", C.c_int32), ("refresh_len_check", C.c_int32)]


def build(force: bool = False) -> str:
    """Compile the checker in place (gcc, seconds).  Building the checker is not using it."""
    src = os.path.join(_HERE, "spg_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-B", "libspg_oracle.so"])
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.spgo_group_batch.restype = C.c_int
        _lib.spgo_find_peaks.restype = C.c_int
        _lib.spgo_find_connections.restype = C.c_int
        _lib.spgo_find_people.restype = C.c_int
        _lib.spgo_max_threads.restype = C.c_int
        _lib.spgo_to_coco.restype = None
    return _lib


def _params_struct(params: dict) -> _Params:
    return _Params(float(params.get("thre1", 0.1)), float(params.get("thre2", 0.1)),
                   float(params.get("connect_ration", 0.8)), float(params.get("len_rate", 16.0)),
                   float(params.get("connection_tole", 0.7)), float(params.get("min_mean_score", 0.45)),
                   int(params.get("mid_num", 20)), int(params.get("offset_radius", 2)),
                   int(params.get("remove_recon", 0)), int(params.get("min_parts", 2)),
                   int(params.get("crit1_strict", 0)), int(params.get("refresh_len_check", 0)))


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


@dataclasses.dataclass
class OracleResult:
    K: int
    L: int
    limbs: np.ndarray            # [L,2] int32
    px: np.ndarray               # [N,capP] f64 refined x (part-major, raster inside a part)
    py: np.ndarray               # [N,capP] f64
    pscore: np.ndarray           # [N,capP] f32
    pxi: np.ndarray              # [N,capP] i32 integer anchors
    pyi: np.ndarray
    pint: np.ndarray             # [N,capP] u8  1 = border peak (integer coords in the reference)
    part_count: np.ndarray       # [N,K] i32
    conn_ij: np.ndarray          # [N,L,capC,2] i32
    conn_score: np.ndarray       # [N,L,capC] f64
    conn_norm: np.ndarray        # [N,L,capC] f64
    conn_count: np.ndarray       # [N,L] i32, -1 = special_k
    cand_count: np.ndarray       # [N,L] i32
    subset: np.ndarray           # [N,capR,K+2,2] f64
    n_persons: np.ndarray        # [N] i32
    status: np.ndarray           # [N] i32

    def n_peaks(self, n: int) -> int:
        return int(self.part_count[n].sum())

    def as_reference_structures(self, n: int):
        """(all_peaks, connection_all, special_k, subset, candidate) of image ``n``."""
        K, L = self.K, self.L
        off = np.concatenate([[0], np.cumsum(self.part_count[n])])
        all_peaks = []
        for c in range(K):
            lst = []
            for g in range(off[c], off[c + 1]):
                if self.pint[n, g]:
                    lst.append((np.int64(self.pxi[n, g]), np.int64(self.pyi[n, g]), self.pscore[n, g], int(g)))
                else:
                    lst.append((np.float64(self.px[n, g]), np.float64(self.py[n, g]), self.pscore[n, g], int(g)))
            all_peaks.append(lst)
        connection_all, special_k = [], []
        for k in range(L):
            m = int(self.conn_count[n, k])
            if m < 0:
                special_k.append(k)
                connection_all.append([])
                continue
            a, b = (int(v) for v in self.limbs[k])
            rows = np.zeros((m, 6))
            ij = self.conn_ij[n, k, :m]
            rows[:, 0] = off[a] + ij[:, 0]
            rows[:, 1] = off[b] + ij[:, 1]
            rows[:, 2] = self.conn_score[n, k, :m]
            rows[:, 3] = ij[:, 0]
            rows[:, 4] = ij[:, 1]
            rows[:, 5] = self.conn_norm[n, k, :m]
            connection_all.append(rows)
        P = int(self.n_persons[n])
        subset = self.subset[n, :P].copy()
        tot = int(off[K])
        candidate = np.stack([self.px[n, :tot], self.py[n, :tot], self.pscore[n, :tot].astype(np.float64),
                              np.arange(tot, dtype=np.float64)], axis=1) if tot else np.zeros((0,))
        return all_peaks, connection_all, special_k, subset, candidate

    def to_coco(self, n: int, coco_from_part: Sequence[int]):
        """evaluate.py:523-543: list of ([17 x (x, y)], score)."""
        P = int(self.n_persons[n])
        cfp = np.asarray(coco_from_part, np.int32)
        kp = np.zeros((P, len(cfp), 2))
        sc = np.zeros((P,))
        sub = np.ascontiguousarray(self.subset[n, :P])
        lib().spgo_to_coco(_p(sub), C.c_int(P), C.c_int(self.K), _p(self.px[n]), _p(self.py[n]), _p(cfp),
                           C.c_int(len(cfp)), _p(kp), _p(sc))
        return kp, sc


def group_batch(heat: np.ndarray, paf: np.ndarray, limbs, image_extent: float, params: dict, *,
                cap_peaks: int = 2048, cap_conn: int = 128, cap_rows: int = 256,
                threads: int = 1) -> OracleResult:
    """Run the whole path on ``heat [N,K,H,W] f32`` and ``paf [N,L,H,W] f32|f64`` (channel-first)."""
    heat = np.ascontiguousarray(heat, np.float32)
    assert paf.dtype in (np.float32, np.float64)
    paf = np.ascontiguousarray(paf)
    N, K, H, W = heat.shape
    L = paf.shape[1]
    assert paf.shape == (N, L, H, W)
    limbs_a = np.ascontiguousarray(np.asarray(limbs, np.int32).reshape(L, 2))
    ps = _params_struct(params)
    r = OracleResult(
        K=K, L=L, limbs=limbs_a,
        px=np.zeros((N, cap_peaks)), py=np.zeros((N, cap_peaks)), pscore=np.zeros((N, cap_peaks), np.float32),
        pxi=np.zeros((N, cap_peaks), np.int32), pyi=np.zeros((N, cap_peaks), np.int32),
        pint=np.zeros((N, cap_peaks), np.uint8), part_count=np.zeros((N, K), np.int32),
        conn_ij=np.zeros((N, L, cap_conn, 2), np.int32), conn_score=np.zeros((N, L, cap_conn)),
        conn_norm=np.zeros((N, L, cap_conn)), conn_count=np.zeros((N, L), np.int32),
        cand_count=np.zeros((N, L), np.int32), subset=np.zeros((N, cap_rows, K + 2, 2)),
        n_persons=np.zeros((N,), np.int32), status=np.zeros((N,), np.int32))
    lib().spgo_group_batch(
        _p(heat), _p(paf), C.c_int(int(paf.dtype == np.float64)), C.c_int(N), C.c_int(K), C.c_int(L), _p(limbs_a),
        C.c_int(H), C.c_int(W), C.c_double(float(image_extent)), C.byref(ps), C.c_int(cap_peaks), C.c_int(cap_conn),
        C.c_int(cap_rows), C.c_int(threads), _p(r.px), _p(r.py), _p(r.pscore), _p(r.pxi), _p(r.pyi), _p(r.pint),
        _p(r.part_count), _p(r.conn_ij), _p(r.conn_score), _p(r.conn_norm), _p(r.conn_count), _p(r.cand_count),
        _p(r.subset), _p(r.n_persons), _p(r.status))
    return r


def max_threads() -> int:
    return int(lib().spgo_max_threads())


COV_NAMES = ("norm0", "special_k", "mid_num1", "candidate", "accept", "assign", "replace", "replace_len_reject",
             "keep_old", "refresh", "assign_len_reject", "merge", "merge_reject", "overlap", "recon_remove",
             "new_person", "pruned", "third_match", "border_peak", "neg_wrap")


def cov_reset() -> None:
    lib().spgo_cov_reset()


def cov_read() -> dict:
    """Counts of the reference branches reached since ``cov_reset`` (names follow evaluate.py's branches)."""
    out = np.zeros(len(COV_NAMES), np.int64)
    n = lib().spgo_cov_read(_p(out), C.c_int(len(COV_NAMES)))
    assert n == len(COV_NAMES)
    return dict(zip(COV_NAMES, (int(v) for v in out)))
