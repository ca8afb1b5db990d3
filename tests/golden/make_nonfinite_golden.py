#!/usr/bin/env python
"""Generate ``tests/golden/nonfinite/``: the reference's grouping on maps holding NaN, +inf, -inf, -0.0 and denormals.

Same procedure as ``make_golden.py``: seeded synthetic maps, the reference's own ``find_peaks -> find_connections ->
find_people`` (evaluate.py, or demo_image.py's inlined copy) lifted verbatim by oracle/ref_loader.py, with one or a few
values written into a map.  Each case records what the reference did:

  ``ok``            its structures, as the other fixtures (golden_io.flatten);
  ``raise``         the exception class and the limb whose find_connections loop raised (a NaN or infinite end point:
                    ``int(round(norm + 1))`` at evaluate.py:226 / demo_image.py:268);
  ``nan_priority``  the first limb whose ``sorted(..., key=priority)`` (evaluate.py:259) saw a NaN key among two or
                    more candidates -- an order the library flags instead of reproducing; nothing else is recorded.

Runs only where a reference checkout is available: ``python tests/golden/make_nonfinite_golden.py``.  The files are
written with fixed zip timestamps, so a rerun rewrites them byte for byte.
"""
from __future__ import annotations

import io
import json
import os
import sys
import traceback
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "nonfinite")
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from golden_io import flatten  # noqa: E402
from improved_body_parts_b200 import skeleton, synth  # noqa: E402

NAN, PINF, NINF = np.float32(np.nan), np.float32(np.inf), np.float32(-np.inf)
VALUES = {"nan": NAN, "pinf": PINF, "ninf": NINF}
H = W = 64  # smooth maps (no background noise) at 64 x 64 keep the files small
LIMB = 0  # the limb the border-score cases paint a line on
SAMPLE_LIMB = 12  # (neck, left shoulder): 23 px between its parts' largest peaks in the base map, so mid_num samples


def _base(**kw):
    return synth.make_image(3, H, W, 3, noise=0.0, **kw)


def _anchor(heat, c, margin):
    """(y, x) of part c's largest value (a peak of a clean map), at least `margin` pixels from the border."""
    m = heat[c].copy()
    m[:margin] = m[-margin:] = 0
    m[:, :margin] = m[:, -margin:] = 0
    return np.unravel_index(int(np.argmax(m)), m.shape)


def _limb_samples(heat, a, b, mid_num=20):
    """The reference's sample pixels (np.linspace + round, evaluate.py:232-235) between the largest peaks of parts a, b,
    from their integer anchors (every sample case keeps those anchors' boxes finite, so they refine as in the clean map
    and stay within a pixel of the line)."""
    (ya, xa), (yb, xb) = _anchor(heat, a, 5), _anchor(heat, b, 5)
    n = min(int(round(np.hypot(xb - xa, yb - ya) + 1)), mid_num)
    return [(int(round(y)), int(round(x))) for x, y in zip(np.linspace(xa, xb, n), np.linspace(ya, yb, n))]


def _paint_line(paf, k, p0, p1, value=0.9, width=1.0):
    """Body-part plane k set to `value` within `width` px of the segment p0 -> p1 ((y, x) each)."""
    yy, xx = np.mgrid[0:H, 0:W]
    (y0, x0), (y1, x1) = p0, p1
    d = np.array([y1 - y0, x1 - x0], np.float64)
    t = np.clip(((yy - y0) * d[0] + (xx - x0) * d[1]) / max(d @ d, 1e-9), 0, 1)
    dist = np.hypot(yy - (y0 + t * d[0]), xx - (x0 + t * d[1]))
    paf[k][dist <= width] = np.float32(value)


def build_cases():
    """name -> (heat, paf, param overrides, variant)."""
    cases = {}
    heat0, paf0 = _base()
    y, x = _anchor(heat0, 0, 5)
    for vn, v in VALUES.items():
        for where, (yy, xx) in (("peak", (y, x)), ("neighbour", (y, x + 1))):
            h = heat0.copy()
            h[0, yy, xx] = v
            cases[f"{vn}_{where}"] = (h, paf0, {}, "evaluate")
        for R in (0, 2, 4):  # only in the radius-2 ring of the peak: inside its box for R >= 2, outside its 3x3 window
            h = heat0.copy()
            h[0, y + 2, x] = v
            cases[f"{vn}_ring2_r{R}"] = (h, paf0, dict(offset_radius=R), "evaluate")
        for row in (0, 1):  # the border band of R = 2: integer anchor, the raw value as score
            h = heat0.copy()
            h[0, row, 50] = v
            cases[f"{vn}_border_row{row}"] = (h, paf0, {}, "evaluate")
    # a NaN network output pixel is a ~16 x 16 NaN block after the x4 bicubic resize (4 taps at 1/4 spacing)
    h = heat0.copy()
    h[2, y - 8:y + 8, x - 8:x + 8] = NAN
    cases["nan_blob16"] = (h, paf0, {}, "evaluate")
    # runs of body-part samples along limb SAMPLE_LIMB between its end parts' largest peaks: the interior samples, or
    # every other one, all NaN / +inf / -inf, or alternating +inf, -inf (their sum is NaN: criterion2 fails)
    sa, sb = skeleton.LIMBS[SAMPLE_LIMB]
    samples = _limb_samples(heat0, sa, sb)
    assert len(samples) == 20, len(samples)
    runs = {"nan": ([NAN], 1), "pinf": ([PINF], 1), "ninf": ([NINF], 1), "pm_inf": ([PINF, NINF], 1),
            "nan_every_other": ([NAN], 2)}
    for vn, (seq, step) in runs.items():
        p = paf0.copy()
        for t, (sy, sx) in enumerate(samples[2:-2:step]):
            p[SAMPLE_LIMB, sy, sx] = seq[t % len(seq)]
        cases[f"samples_{vn}"] = (heat0, p, {}, "evaluate")
    p = paf0.copy()
    sy, sx = samples[len(samples) // 2]
    p[SAMPLE_LIMB, sy, sx] = PINF  # one +inf sample: a candidate with score +inf
    cases["samples_one_pinf"] = (heat0, p, {}, "evaluate")
    a, b = skeleton.LIMBS[LIMB]
    # border peaks with a non-finite score that become candidates: part a blanked, one border peak painted to the
    # B peaks of one person (one candidate) or of two (several)
    for vn, v in (("nan", NAN), ("pinf", PINF), ("ninf", NINF)):
        for persons in (1, 2):
            h, p = synth.make_image(5, H, W, persons, noise=0.0, missing_parts=(a,))
            h[a, 0, 48] = v
            for q in range(persons):
                m = h[b].copy()
                for _ in range(q):
                    yq, xq = np.unravel_index(int(np.argmax(m)), m.shape)
                    m[max(yq - 6, 0):yq + 7, max(xq - 6, 0):xq + 7] = 0
                yb, xb = np.unravel_index(int(np.argmax(m)), m.shape)
                _paint_line(p, LIMB, (0, 48), (yb, xb))
            cases[f"border_{vn}_score_{'one' if persons == 1 else 'several'}"] = (h, p, {}, "evaluate")
    # +inf and -inf border scores at both ends of one pair: priority inf + -inf = NaN (one candidate: reproduced)
    h, p = synth.make_image(5, H, W, 1, noise=0.0, missing_parts=(a, b))
    h[a, 0, 48] = PINF
    h[b, H - 1, 40] = NINF
    _paint_line(p, LIMB, (0, 48), (H - 1, 40))
    cases["border_pinf_ninf_pair"] = (h, p, {}, "evaluate")
    # -0.0 and denormal plateaus (the background is exactly zero), thre1 0.1 / 0 / -0.1
    hz, pz = _base()
    h = hz.copy()
    h[3, 10:16, 10:16] = np.float32(-0.0)
    h[4, 10:16, 10:16] = np.float32(1e-40)                 # positive denormal
    h[5, 20:24, 60:64] = np.float32(-1e-40)                # negative denormal
    h[6, 40:44, 50:54] = np.float32(-0.05)                 # negative plateau: its inner 2 x 2 only reach a negative thre1
    for tn, thr in (("0p1", 0.1), ("0", 0.0), ("m0p1", -0.1)):
        cases[f"zeros_denormals_thre1_{tn}"] = (h, pz, dict(thre1=thr), "evaluate")
    # demo_image.py's inlined copy: its NaN scrub (:179-180) leaves +-inf in the maps
    for vn, v, (yy, xx) in (("pinf_border", PINF, (0, 50)), ("ninf_peak", NINF, (y, x))):
        h = heat0.copy()
        h[0, yy, xx] = v
        cases[f"demo_{vn}"] = (h, paf0, {}, "demo")
    return cases


class _SortSpy:
    """Stands in for builtins.sorted in the reference's globals: records the first limb whose candidate list holds a NaN
    priority among two or more entries (the caller's loop variable `k`)."""

    def __init__(self):
        self.first = None

    def __call__(self, seq, key=None, reverse=False):
        seq = list(seq)
        if self.first is None and len(seq) > 1 and any(np.isnan(float(key(c))) for c in seq):
            self.first = int(sys._getframe(1).f_locals["k"])
        return sorted(seq, key=key, reverse=reverse)


def run_reference(ref, heat, paf, params, demo):
    spy = _SortSpy()
    ns = ref._fn.__globals__ if demo else ref._ns
    ns["sorted"] = spy
    try:
        structs = ref.group(np.ascontiguousarray(heat.transpose(1, 2, 0)), np.ascontiguousarray(paf.transpose(1, 2, 0)),
                            H, params)
    except (ValueError, OverflowError, IndexError) as e:
        tb = traceback.extract_tb(e.__traceback__)
        limb = None
        for fr, _ in traceback.walk_tb(e.__traceback__):
            if fr.f_code.co_name in ("find_connections", "demo_group") and "k" in fr.f_locals:
                limb = int(fr.f_locals["k"])
        first_nan = spy.first
        outcome = dict(outcome="raise", exception=type(e).__name__, limb=limb, line=tb[-1].lineno)
        if first_nan is not None and first_nan < limb:
            outcome = dict(outcome="nan_priority", limb=first_nan)
        return outcome, None
    finally:
        del ns["sorted"]
    if spy.first is not None:
        return dict(outcome="nan_priority", limb=spy.first), None
    return dict(outcome="ok"), structs


def save(path, arrays) -> None:
    """np.savez_compressed with fixed zip timestamps."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main() -> None:
    import torch

    from oracle.ref_loader import DemoReference, Reference

    refs = {"evaluate": Reference(), "demo": DemoReference()}
    assert tuple(refs["evaluate"].limbs) == skeleton.LIMBS, "limb table drifted from the reference"
    os.makedirs(OUT, exist_ok=True)
    manifest = {"generated_by": "tests/golden/make_nonfinite_golden.py", "reference": "hellojialee/Improved-Body-Parts",
                "numpy": np.__version__, "torch": torch.__version__, "cases": {}}
    for name, (heat, paf, over, variant) in build_cases().items():
        params = dict(skeleton.default_params(), **over)
        expect, structs = run_reference(refs[variant], heat, paf, params, variant == "demo")
        if variant == "demo":
            params = dict(params, crit1_strict=1, refresh_len_check=1, min_parts=4)  # as make_golden.py
        arrays = dict(heat=np.ascontiguousarray(heat, np.float32), paf=np.ascontiguousarray(paf, np.float32),
                      image_extent=np.int64(H), params=np.array(json.dumps(params, sort_keys=True)),
                      expect=np.array(json.dumps(dict(expect, variant=variant), sort_keys=True)))
        if structs is not None:
            arrays.update(flatten(structs))
            peaks, conn, _, subset, _ = structs
            expect = dict(expect, peaks=int(sum(len(p) for p in peaks)), persons=int(subset.shape[0]),
                          connections=int(sum(0 if isinstance(c, list) else c.shape[0] for c in conn)))
        path = os.path.join(OUT, name + ".npz")
        save(path, arrays)
        manifest["cases"][name] = dict(expect, variant=variant, bytes=os.path.getsize(path))
        print(f"{name:34s} {manifest['cases'][name]}")
    with open(os.path.join(OUT, "MANIFEST.json"), "w") as fh:
        json.dump(manifest, fh, indent=1, sort_keys=True)
        fh.write("\n")


if __name__ == "__main__":
    main()
