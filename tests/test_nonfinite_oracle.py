"""CPU: grouping on maps holding NaN, +-inf, -0.0 and denormals -- the checker and the port against the reference's own
outcomes (tests/golden/nonfinite, make_nonfinite_golden.py), and the kernels' peak predicate and pass-1 vote modelled
in numpy against torch's ``heat * keep != 0`` (util.py:177-183, evaluate.py:193).

The reference keeps every non-finite pixel (NaN * 0, inf * 0 and -inf * 0 are NaN, never 0), refines it into NaN
coordinates when its box is inside the map, and then raises at evaluate.py:226 for any limb pair with such an end point.
"""
import glob
import json
import os

import numpy as np
import pytest

from golden_io import unflatten
from oracle import grouping_port as gp
from oracle import spg_oracle as so
from parity import diff_structures, structure_stats

HERE = os.path.dirname(os.path.abspath(__file__))
NONFINITE = sorted(glob.glob(os.path.join(HERE, "golden", "nonfinite", "*.npz")))


def load_nonfinite(path):
    """A non-finite golden: inputs, params, the reference's outcome, and its structures when it finished."""
    with np.load(path, allow_pickle=False) as z:
        d = {k: z[k] for k in z.files}
    expect = json.loads(str(d["expect"]))
    return dict(heat=d["heat"], paf=d["paf"], image_extent=int(d["image_extent"]), params=json.loads(str(d["params"])),
                expect=expect, structs=unflatten(d) if expect["outcome"] == "ok" else None,
                name=os.path.basename(path)[:-4])


#: the checker's error code for each outcome the reference can have on these maps
CHECKER_CODE = {"ok": 0, "raise": so.ERR_NONFINITE, "nan_priority": so.ERR_NAN_PRIORITY}


def test_nonfinite_goldens_cover_the_cases():
    names = {os.path.basename(p)[:-4] for p in NONFINITE}
    assert len(names) >= 35
    cases = [load_nonfinite(p) for p in NONFINITE]
    outcomes = {c["expect"]["outcome"] for c in cases}
    assert outcomes == {"ok", "raise", "nan_priority"}
    assert {c["expect"]["variant"] for c in cases} == {"evaluate", "demo"}
    for c in cases:
        assert c["heat"].shape[1] * c["heat"].shape[2] <= 128 * 128
    # the values the goldens put into the maps
    heat = np.concatenate([c["heat"].ravel() for c in cases])
    paf = np.concatenate([c["paf"].ravel() for c in cases])
    for arr in (heat, paf):
        assert np.isnan(arr).any() and np.isposinf(arr).any() and np.isneginf(arr).any()
    assert (np.signbit(heat) & (heat == 0)).any() and ((heat != 0) & (np.abs(heat) < np.finfo(np.float32).tiny)).any()


def test_sample_goldens_hold_runs_on_one_body_part_plane():
    """samples_*: several non-finite values along one limb's line (one for samples_one_pinf); pm_inf holds both signs."""
    runs = [p for p in NONFINITE if os.path.basename(p).startswith("samples_")]
    assert len(runs) >= 6
    for path in runs:
        name = os.path.basename(path)[:-4]
        paf = load_nonfinite(path)["paf"]
        k, y, x = np.nonzero(~np.isfinite(paf))
        assert len(set(k.tolist())) == 1, name
        if name == "samples_one_pinf":
            assert len(k) == 1 and np.isposinf(paf[k, y, x]).all()
            continue
        assert len(k) >= 6, (name, len(k))
        v = paf[k, y, x]
        if name == "samples_pm_inf":
            assert np.isposinf(v).sum() >= 3 and np.isneginf(v).sum() >= 3
        elif "nan" in name:
            assert np.isnan(v).all(), name


def _header_bits(path, pattern):
    import re
    src = open(path).read()
    return {m.group(1): 1 << int(m.group(2)) for m in re.finditer(pattern, src)}


def test_status_bits_agree_across_header_kernels_and_binding():
    """SPG_ST_* in include/spgroup.h, kSt* in csrc/common.cuh and grouping.ST_*: the same value for every bit."""
    from improved_body_parts_b200 import grouping

    root = os.path.dirname(HERE)
    hdr = _header_bits(os.path.join(root, "include", "spgroup.h"), r"SPG_ST_(\w+)\s*=\s*1u\s*<<\s*(\d+)")
    cuh = _header_bits(os.path.join(root, "improved_body_parts_b200", "csrc", "common.cuh"),
                       r"constexpr uint32_t kSt(\w+)\s*=\s*1u\s*<<\s*(\d+)")
    assert set(hdr) == {"PEAK_OVERFLOW", "CAND_OVERFLOW", "ROW_OVERFLOW", "SAMPLE_INDEX", "ASSERT", "WIRE_OVERFLOW",
                        "NONFINITE", "NAN_PRIORITY"}
    for name, bit in hdr.items():
        assert getattr(grouping, "ST_" + name) == bit, name
        camel = "".join(w.capitalize() for w in name.split("_"))
        assert cuh[camel] == bit, name
    # the scorer-internal flag is no published bit
    assert cuh["NanPrioCand"] not in hdr.values()
    assert set(grouping.ST_MEANING) == {grouping.ST_SAMPLE_INDEX, grouping.ST_ASSERT, grouping.ST_NONFINITE,
                                        grouping.ST_NAN_PRIORITY}


def _checker(case):
    return so.group_batch(case["heat"][None], case["paf"][None], gp_limbs(), case["image_extent"], case["params"])


def gp_limbs():
    from improved_body_parts_b200 import skeleton
    return skeleton.LIMBS


@pytest.mark.parametrize("path", NONFINITE, ids=[os.path.basename(p)[:-4] for p in NONFINITE])
def test_checker_matches_the_reference_on_nonfinite_maps(path):
    case = load_nonfinite(path)
    r = _checker(case)
    assert r.status[0] == CHECKER_CODE[case["expect"]["outcome"]], (case["expect"], r.status[0])
    if case["structs"] is not None:
        got = r.as_reference_structures(0)
        diffs = diff_structures(case["structs"], got, float_tol=0.0)
        assert not diffs, "\n".join(diffs)
        assert structure_stats(got) == structure_stats(case["structs"])


@pytest.mark.parametrize("path", NONFINITE, ids=[os.path.basename(p)[:-4] for p in NONFINITE])
def test_port_matches_the_reference_on_nonfinite_maps(path):
    case = load_nonfinite(path)
    e = case["expect"]
    run = lambda: gp.group_image(case["heat"], case["paf"], case["image_extent"], case["params"], gp_limbs())  # noqa: E731
    if e["outcome"] == "raise":
        with pytest.raises((ValueError, OverflowError)) as info:
            run()
        assert type(info.value).__name__ == e["exception"]
    elif e["outcome"] == "nan_priority":
        with pytest.raises(gp.UnorderedPriorities, match=f"limb {e['limb']}:"):
            run()
    else:
        peaks, conns, special, subset, candidate = run()
        diffs = diff_structures(case["structs"], (peaks, conns, special, subset, candidate), float_tol=0.0)
        assert not diffs, "\n".join(diffs)


def test_border_peaks_keep_the_raw_nonfinite_score():
    """A non-finite border pixel is a peak with its integer anchor and its own value as score (util.py:201-202),
    whatever its neighbours -- NaN vetoes only finite neighbours."""
    for name in ("nan_border_row0", "pinf_border_row1", "ninf_border_row0"):
        case = load_nonfinite(os.path.join(HERE, "golden", "nonfinite", name + ".npz"))
        peaks = case["structs"][0][0]
        border = [p for p in peaks if isinstance(p[0], (int, np.integer)) and not np.isfinite(p[2])]
        assert len(border) == 1, name
        v = case["heat"][0, int(border[0][1]), int(border[0][0])]
        assert np.array_equal(np.float32(border[0][2]), v, equal_nan=True)


# ---- the kernels' peak predicate and pass-1 vote, modelled in numpy -------------------------------------------------
F32 = np.float32


def _value_set(thr):
    thr = F32(thr)
    return np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-40, -1e-40, np.nextafter(thr, F32(-np.inf)), thr, 0.5,
                     np.finfo(np.float32).max], np.float32)


def _random_maps(seed, thr, n, H, W):
    rng = np.random.default_rng(seed)
    vals = _value_set(thr)
    # mostly the few finite values, so that peaks and plateaus are common; every value appears in every position class
    p = np.array([3, 3, 3, 6, 6, 4, 4, 10, 10, 10, 6], np.float64)
    return vals[rng.choice(len(vals), size=(n, H, W), p=p / p.sum())]


def _torch_keep(maps, thr):
    """util.keypoint_heatmap_nms + np.nonzero(heat * keep) (evaluate.py:184,193), restated with the same torch ops."""
    import torch
    import torch.nn.functional as F

    heat = torch.from_numpy(maps)[:, None]
    hmax = F.max_pool2d(F.pad(heat, (1, 1, 1, 1), mode="reflect"), (3, 3), stride=1, padding=0)
    keep = (hmax == heat).float() * (heat >= float(thr)).float()
    return (heat * keep)[:, 0].numpy() != 0


def _kernel_predicate(maps, thr):
    """nms_test_group: neighbours clamped to the image (U/C/D rows, columns x-1 .. x+1), then
    !isfinite(v) | (v >= thr & v != 0 & every neighbour <= v)."""
    n, H, W = maps.shape
    thr = F32(thr)
    y = np.arange(H)
    x = np.arange(W)
    ok = np.ones(maps.shape, bool)
    with np.errstate(invalid="ignore"):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                nb = maps[:, np.clip(y + dy, 0, H - 1)][:, :, np.clip(x + dx, 0, W - 1)]
                ok &= nb <= maps
        return ~np.isfinite(maps) | ((maps >= thr) & (maps != 0) & ok)


def _group_vote(maps, thr):
    """nms_group_vote over the float4 groups of each row: fmaxf (drops NaN) >= thr, or the float32 sum of magnitudes
    ((|x| + |y|) + |z|) + |w| is not <= FLT_MAX."""
    n, H, W = maps.shape
    g = maps.reshape(n, H, W // 4, 4)
    with np.errstate(invalid="ignore", over="ignore"):
        mx = np.fmax(np.fmax(g[..., 0], g[..., 1]), np.fmax(g[..., 2], g[..., 3]))
        mag = ((np.abs(g[..., 0]) + np.abs(g[..., 1])) + np.abs(g[..., 2])) + np.abs(g[..., 3])
        return (mx >= F32(thr)) | ~(mag <= np.finfo(np.float32).max), mx >= F32(thr)


@pytest.mark.parametrize("thr", [0.1, 0.0, -0.1])
def test_kernel_peak_predicate_is_torchs_nonzero_heat_times_keep(thr):
    """A million 3x3 windows (10 000 maps of 10 x 10: interior, clipped border and corner windows) over NaN, +-inf, +-0,
    +-denormal, thr - ulp, thr, 0.5 and FLT_MAX."""
    maps = _random_maps(7, thr, 10_000, 10, 10)
    want = _torch_keep(maps, thr)
    got = _kernel_predicate(maps, thr)
    assert np.array_equal(got, want), f"{int((got != want).sum())} pixels differ"
    # every class of pixel is exercised: non-finite peaks, finite peaks, vetoed pixels
    assert (want & ~np.isfinite(maps)).any() and (want & np.isfinite(maps)).any() and (~want).any()
    assert not (want & (maps == 0)).any()  # -0.0 * 1 and 0 * 1 are zeros


@pytest.mark.parametrize("thr", [0.1, 0.0, -0.1])
def test_pass1_vote_covers_every_group_holding_a_peak(thr):
    """nms_queue_groups drops a float4 group unless its vote is set: every group holding a peak must be voted.  The max
    alone (fmaxf drops NaN, -inf never reaches thre1) misses groups whose only peaks are NaN or -inf."""
    maps = _random_maps(8, thr, 20_000, 8, 16)
    peaks = _torch_keep(maps, thr)
    n, H, W = maps.shape
    has_peak = peaks.reshape(n, H, W // 4, 4).any(-1)
    vote, max_only = _group_vote(maps, thr)
    assert not (has_peak & ~vote).any()
    assert (has_peak & ~max_only).any(), "the maps hold no group that the max alone would miss"
    # NaN-only and -inf-only groups, and a group of a NaN next to finite values below thre1
    g = np.array([[[np.nan] * 4, [-np.inf] * 4, [np.nan, F32(thr) - 1, F32(thr) - 1, F32(thr) - 1]]], np.float32)
    v, _ = _group_vote(g.reshape(1, 3, 4), thr)
    assert v.all()
