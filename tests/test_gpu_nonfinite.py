"""GPU: grouping on maps holding NaN, +-inf, -0.0 and denormals.

Every non-finite golden (tests/golden/nonfinite, the reference's own outcomes) through spg_group_batch, the ragged call
and the capacity-free tier: bit-identical structures where the reference finished, SPG_ST_NONFINITE where it raised,
SPG_ST_NAN_PRIORITY where its sort saw a NaN key among others.  Then every peak-finding and pair-scoring schedule, named
by ``stage_kernels()``, against the checker on seeded maps with non-finite values written where the schedules split
their work, and the drop-in functions raising ``GroupingError`` where the reference raised.
"""
import os

import numpy as np
import pytest

from parity import FLOAT_TOL, diff_structures
from test_nonfinite_oracle import NONFINITE, load_nonfinite

pytestmark = pytest.mark.gpu

NAN, PINF, NINF = np.float32(np.nan), np.float32(np.inf), np.float32(-np.inf)


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import grouping, skeleton, synth
    from oracle import spg_oracle as so

    class Env:
        pass

    e = Env()
    e.torch, e.G, e.skeleton, e.synth, e.so, e.dev = torch, grouping, skeleton, synth, so, cuda_device
    e.bit = {"raise": grouping.ST_NONFINITE, "nan_priority": grouping.ST_NAN_PRIORITY}
    e.code_bit = {so.ERR_NONFINITE: grouping.ST_NONFINITE, so.ERR_NAN_PRIORITY: grouping.ST_NAN_PRIORITY,
                  so.ERR_INDEX: grouping.ST_SAMPLE_INDEX, so.ERR_ASSERT: grouping.ST_ASSERT}
    return e


CAPACITY = 0x7


def _assert_same(ref, got, what):
    d = diff_structures(ref, got, float_tol=0.0)
    if d:
        loose = diff_structures(ref, got, float_tol=FLOAT_TOL)
        pytest.fail(f"{what}: not bit-identical ({'within 1e-4' if not loose else 'ALSO outside 1e-4'}):\n" + "\n".join(d))


def _over_capacity(env, case, capP=128):
    """The golden has a part with more peaks than the bounded calls hold (nan_blob16: a 16 x 16 NaN block is 256 peaks)."""
    o = env.so.group_batch(case["heat"][None], case["paf"][None], env.skeleton.LIMBS, case["image_extent"], case["params"])
    return int(o.part_count.max()) > capP


def _check_golden(env, case, status, structs_of, what, bounded=True):
    e = case["expect"]
    status = int(status)
    if bounded and _over_capacity(env, case):  # flagged; the capacity-free tier answers for such an image
        assert status & env.G.ST_PEAK_OVERFLOW, f"{what}: status {status:#x}"
        return
    assert not status & CAPACITY, f"{what}: status {status:#x}"
    if e["outcome"] == "ok":
        assert status == 0, f"{what}: status {status:#x}"
        _assert_same(case["structs"], structs_of(), what)
    else:
        assert status & env.bit[e["outcome"]], f"{what}: {e} but status {status:#x}"


def _dev(env, a):
    return env.torch.from_numpy(np.ascontiguousarray(a)).to(env.dev)


@pytest.mark.parametrize("path", NONFINITE, ids=[os.path.basename(p)[:-4] for p in NONFINITE])
def test_golden_through_group_batch_and_the_tier(env, path):
    case = load_nonfinite(path)
    H, W = case["heat"].shape[1:]
    hd, pd = _dev(env, case["heat"][None]), _dev(env, case["paf"][None])
    g = env.G.Grouper(max_batch=1, max_h=H, max_w=W, max_peaks_per_part=128, max_person_rows=128)
    try:
        g.group_device(hd, pd, case["image_extent"], case["params"])
        r = g.fetch()
        _check_golden(env, case, r.status[0], lambda: r.as_reference_structures(0), "spg_group_batch")
        t = g.group_unbounded(hd[0], pd[0], case["image_extent"], case["params"])
        _check_golden(env, case, t.status[0], lambda: t.as_reference_structures(0), "spg_group_unbounded",
                      bounded=False)
    finally:
        g.close()


def test_goldens_through_one_ragged_call(env):
    cases = [load_nonfinite(p) for p in NONFINITE]
    by_params = {}
    for c in cases:  # one call per parameter set
        by_params.setdefault(repr(sorted(c["params"].items())), []).append(c)
    for group in by_params.values():
        g = env.G.Grouper(max_batch=len(group), max_h=128, max_w=128, max_peaks_per_part=128, max_person_rows=128)
        try:
            maps = [(_dev(env, c["heat"]), _dev(env, c["paf"])) for c in group]
            g.group_ragged(maps, [c["image_extent"] for c in group], group[0]["params"])
            r = g.fetch(len(group))
            assert g.stage_kernels()[0] == "nms_peaks_ragged_kernel", g.stage_kernels()
            assert g.stage_kernels()[1].startswith("limb_score_ragged_kernel"), g.stage_kernels()
            for i, c in enumerate(group):
                _check_golden(env, c, r.status[i], lambda: r.as_reference_structures(i), f"ragged {c['name']}")
        finally:
            g.close()


# ---- the schedule matrix against the checker ------------------------------------------------------------------------
def _peaks_equal(o, r, i, what):
    """Peak lists of image i: counts, anchors, border flags, and x / y / score bit for bit with NaN by position."""
    K = r.peak_count.shape[1]
    off = 0
    for c in range(K):
        n = int(o.part_count[i, c])
        assert int(r.peak_count[i, c]) == n, f"{what}: part {c}: {int(r.peak_count[i, c])} peaks vs {n}"
        sl = slice(off, off + n)
        anc = r.peak_anchor[i, c, :n]
        assert np.array_equal(anc & 0xffff, o.pxi[i, sl]) and np.array_equal((anc >> 16) & 0x7fff, o.pyi[i, sl]), what
        assert np.array_equal(anc >> 31, o.pint[i, sl]), what
        for name, a, b in (("x", r.peak_x[i, c, :n], o.px[i, sl]), ("y", r.peak_y[i, c, :n], o.py[i, sl]),
                           ("score", r.peak_score[i, c, :n], o.pscore[i, sl])):
            assert np.array_equal(a, b, equal_nan=True), f"{what}: part {c} {name}"
        off += n


def _compare(env, o, r, n, what, peaks_only=False):
    for i in range(n):
        _peaks_equal(o, r, i, f"{what} image {i}")
        if peaks_only:
            continue
        st = int(o.status[i])
        if st == 0:
            assert int(r.status[i]) == 0, f"{what} image {i}: status {int(r.status[i]):#x}"
            _assert_same(o.as_reference_structures(i), r.as_reference_structures(i), f"{what} image {i}")
        else:
            assert int(r.status[i]) & env.code_bit[st], f"{what} image {i}: checker {st}, status {int(r.status[i]):#x}"


def _run(env, monkeypatch, heat, paf, extent, params, envvars=(), paf_as_f64=False, **cfg):
    for k, v in envvars:
        monkeypatch.setenv(k, v)
    N, K, H, W = heat.shape
    g = env.G.Grouper(max_batch=N, max_h=H, max_w=W, **cfg)
    try:
        g.group_device(_dev(env, heat), _dev(env, paf), extent, params, paf_as_f64=paf_as_f64)
        return g.fetch(), g.stage_kernels()
    finally:
        g.close()
        for k, _ in envvars:
            monkeypatch.delenv(k)


def _dirty(env, seed, n, H, W, persons=4, interior=True, **kw):
    """Seeded maps with NaN / +inf / -inf written into keypoint planes -- in the border band always, inside the map when
    `interior` (the reference then raises: NaN end points) -- and runs of them along body-part planes."""
    heat, paf = env.synth.make_batch(seed, n, H, W, persons, **kw)
    rng = np.random.default_rng(seed)
    vals = np.array([NAN, PINF, NINF], np.float32)
    for i in range(n):
        for _ in range(6):  # border band of radius 2: integer anchors, raw non-finite scores
            c = int(rng.integers(18))
            y = int(rng.choice([0, 1, H - 2, H - 1])) if rng.random() < 0.5 else int(rng.integers(H))
            x = int(rng.integers(W)) if y in (0, 1, H - 2, H - 1) else int(rng.choice([0, 1, W - 2, W - 1]))
            heat[i, c, y, x] = vals[rng.integers(3)]
        if interior and i % 2:
            c, y, x = int(rng.integers(18)), int(rng.integers(3, H - 3)), int(rng.integers(3, W - 3))
            heat[i, c, y, x] = vals[rng.integers(3)]
        for _ in range(40):
            k, y, x = int(rng.integers(paf.shape[1])), int(rng.integers(H)), int(rng.integers(W))
            paf[i, k, y, x] = vals[rng.integers(3)]
    return heat, paf


def _nms_edges(env, heat, share_groups):
    """Non-finite values in the first and last float4 group of scanner shares / bands of `share_groups` groups, and
    NaN-only / -inf-only groups, in the first part of each image."""
    N, K, H, W = heat.shape
    flat = heat.reshape(N, K, H * W)
    G = H * W // 4
    step = share_groups * max(8, -(-G // (20 * share_groups)))  # some 20 shares: the part stays within the peak capacity
    for i in range(N):
        for s0 in range(0, G, step):
            for g, v in ((s0, NAN), (min(s0 + share_groups, G) - 1, NINF)):
                flat[i, 0, 4 * g + (i % 4)] = v
        g = (G // 2 + 7 * i) % G
        flat[i, 1, 4 * g:4 * g + 4] = NAN
        g = (G // 3 + 5 * i) % G
        flat[i, 2, 4 * g:4 * g + 4] = NINF
    return heat


def test_nms_schedules_on_nonfinite_planes(env, monkeypatch):
    params = env.skeleton.default_params()
    # persistent ring, 128 x 128: scanner shares are 32-group chunks dealt round-robin
    heat, paf = _dirty(env, 9100, 6, 128, 128)
    heat = _nms_edges(env, heat, 32)
    o = env.so.group_batch(heat, paf, env.skeleton.LIMBS, 128, params)
    r, names = _run(env, monkeypatch, heat, paf, 128, params, max_peaks_per_part=128)
    assert names[0] == "nms_peaks_persist_kernel", names
    _compare(env, o, r, 6, "persist", peaks_only=True)
    # one CTA per plane: float4 pass (W % 4 == 0) and the scalar path (W % 4 != 0)
    for H, W in ((128, 128), (57, 61)):
        heat, paf = _dirty(env, 9200 + W, 4, H, W)
        if W % 4 == 0:
            heat = _nms_edges(env, heat, 128 * 32 // 8)  # kNmsThreads / 32 warps, one contiguous slice each
        o = env.so.group_batch(heat, paf, env.skeleton.LIMBS, H, params)
        r, names = _run(env, monkeypatch, heat, paf, H, params, envvars=(("SPG_PERSIST", "0"),), max_peaks_per_part=128)
        assert names[0] == "nms_peaks_kernel", names
        _compare(env, o, r, 4, f"per-plane {H}x{W}", peaks_only=True)
    # banded (planes too large for the ring), as test_planes_too_large_for_the_plane_ring_take_the_banded_nms
    for H, W in ((200, 260), (150, 512), (300, 132)):
        heat, paf = _dirty(env, 9300 + H, 2, H, W, persons=6, scale_range=(1.5, 3.0))
        heat = _nms_edges(env, heat, 32)
        for b in range(2):  # every band's first / last rows (band heights 8 .. 31 rows)
            for y in range(0, H, 8):
                heat[b, 3, y, (5 * y) % W] = NAN
                heat[b, 3, min(y + 7, H - 1), (3 * y + 1) % W] = NINF
        o = env.so.group_batch(heat, paf, env.skeleton.LIMBS, H, params)
        r, names = _run(env, monkeypatch, heat, paf, H, params, max_peaks_per_part=128)
        assert names[0] == "nms_peaks_banded_kernel", names
        _compare(env, o, r, 2, f"banded {H}x{W}", peaks_only=True)


def test_nms_ragged_and_tier_on_nonfinite_planes(env):
    params = env.skeleton.default_params()
    sizes = [(128, 128), (57, 61), (96, 64)]
    imgs = []
    for s, (H, W) in enumerate(sizes):
        heat, paf = _dirty(env, 9400 + s, 1, H, W)
        if W % 4 == 0:
            heat = _nms_edges(env, heat, 32)
        imgs.append((heat, paf))
    g = env.G.Grouper(max_batch=len(sizes), max_h=128, max_w=128, max_peaks_per_part=128, max_person_rows=128)
    try:
        g.group_ragged([(_dev(env, h[0]), _dev(env, p[0])) for h, p in imgs], [h.shape[2] for h, _ in imgs], params)
        r = g.fetch(len(sizes))
        assert g.stage_kernels()[0] == "nms_peaks_ragged_kernel"
        for s, (heat, paf) in enumerate(imgs):
            o = env.so.group_batch(heat, paf, env.skeleton.LIMBS, heat.shape[2], params)
            one = _slice(r, s)
            _compare(env, o, one, 1, f"ragged {sizes[s]}")
            t = g.group_unbounded(_dev(env, heat[0]), _dev(env, paf[0]), heat.shape[2], params)
            _compare(env, o, t, 1, f"tier {sizes[s]}")
    finally:
        g.close()


def _slice(r, i):
    import dataclasses
    fields = {f.name: getattr(r, f.name) for f in dataclasses.fields(r)}
    for k, v in fields.items():
        if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == r.status.shape[0] and k not in ("limbs",):
            fields[k] = v[i:i + 1]
    return type(r)(**fields)


@pytest.mark.parametrize("mode", ["persist_f32", "staged_176", "sampled_512", "f64", "f32_as_f64", "no_screen"])
def test_scoring_schedules_on_nonfinite_maps(env, monkeypatch, mode):
    """Border-band non-finite peaks (raw non-finite scores: +-inf and NaN priorities) and non-finite body-part samples
    through each scoring schedule; every other image also has an interior non-finite pixel (NaN end points)."""
    H, W, n, envvars, f64, as_f64 = 128, 128, 8, (), False, False
    if mode == "staged_176":  # the per-item schedule, whole plane in shared memory
        H = W = 176
        envvars = (("SPG_PERSIST", "0"),)
    elif mode == "sampled_512":
        H = W = 512
        n = 2
    elif mode == "f64":
        f64 = True
    elif mode == "f32_as_f64":
        as_f64 = True
    elif mode == "no_screen":
        envvars = (("SPG_NO_SCREEN", "1"),)
    kw = dict(scale_range=(3.0, 5.0)) if H == 512 else {}
    heat, paf = _dirty(env, 9500 + H + 7 * f64 + 3 * as_f64, n, H, W, persons=8, **kw)
    params = env.skeleton.default_params()
    paf_ref = paf.astype(np.float64) if (f64 or as_f64) else paf
    paf_dev = paf.astype(np.float64) if f64 else paf
    o = env.so.group_batch(heat, paf_ref, env.skeleton.LIMBS, H, params, threads=4)
    assert (o.status == 0).any() and (o.status == env.so.ERR_NONFINITE).any(), o.status
    r, names = _run(env, monkeypatch, heat, paf_dev, H, params, envvars=envvars, paf_as_f64=as_f64,
                    max_peaks_per_part=64, max_person_rows=128)
    want = {"persist_f32": "limb_score_persist_kernel<float>", "staged_176": "limb_score_kernel<float,true>",
            "sampled_512": "limb_score_kernel<float,false>", "f64": "limb_score_kernel<double,",
            "f32_as_f64": "limb_score_persist_kernel<double>", "no_screen": "limb_score_persist_kernel<float>"}[mode]
    assert names[1].startswith(want), names
    _compare(env, o, r, n, mode)


def test_nan_priority_is_flagged_by_every_scorer(env, monkeypatch):
    """border_nan_score_several: a NaN border score on a limb with two candidates -> SPG_ST_NAN_PRIORITY from the
    persistent, the per-item and the tier scorers alike; border_nan_score_one: one candidate, reproduced."""
    for name, bit in (("border_nan_score_several", env.G.ST_NAN_PRIORITY), ("border_nan_score_one", 0)):
        case = load_nonfinite(os.path.join(os.path.dirname(NONFINITE[0]), name + ".npz"))
        for flag in ("1", "0"):
            r, names = _run(env, monkeypatch, case["heat"][None], case["paf"][None], case["image_extent"], case["params"],
                            envvars=(("SPG_PERSIST", flag),))
            assert ("persist" in names[1]) == (flag == "1")
            assert int(r.status[0]) == bit, (name, flag, int(r.status[0]))


def test_dropin_raises_where_the_reference_raised(env):
    from improved_body_parts_b200 import dropin

    for path in NONFINITE:
        case = load_nonfinite(path)
        e = case["expect"]
        dropin.configure(variant=e["variant"])
        try:
            heat = np.ascontiguousarray(case["heat"].transpose(1, 2, 0))
            paf = np.ascontiguousarray(case["paf"].transpose(1, 2, 0))
            ext, params = case["image_extent"], case["params"]
            if e["outcome"] == "ok":
                _assert_same(case["structs"], dropin.group(heat, paf, ext, params), f"group {case['name']}")
                got = dropin.group_many([(heat, paf)] * 2, [ext] * 2, params)
                _assert_same(case["structs"], got[1], f"group_many {case['name']}")
                all_peaks = dropin.find_peaks(heat, params)
                conns, special = dropin.find_connections(all_peaks, paf, ext, params)
                subset, candidate = dropin.find_people(conns, special, all_peaks, params)
                _assert_same(case["structs"], (all_peaks, conns, special, subset, candidate), f"stages {case['name']}")
                continue
            word = "NONFINITE" if e["outcome"] == "raise" else "NAN_PRIORITY"
            with pytest.raises(env.G.GroupingError, match=word):
                dropin.group(heat, paf, ext, params)
            with pytest.raises(env.G.GroupingError, match=word):
                dropin.group_many([(heat, paf)], [ext], params)
            all_peaks = dropin.find_peaks(heat, params)  # peaks never raise in the reference
            with pytest.raises(env.G.GroupingError, match=word):
                dropin.find_connections(all_peaks, paf, ext, params)
        finally:
            dropin.configure(variant="evaluate")
