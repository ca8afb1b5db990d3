"""GPU: the capacity-free grouping tier (``spg_group_unbounded`` / ``Grouper.group_unbounded``) and the drop-in functions
that fall back to it when an image goes past the handle's capacities.

Every result is compared bit for bit: against the reference's own answers (the golden fixtures) and against the CPU
checker run with capacities far above the image's needs."""
import glob
import os
import types

import numpy as np
import pytest

from conftest import ROOT, golden_paths
from golden_io import load_case
from parity import diff_structures

pytestmark = pytest.mark.gpu

CROWD_GOLDENS = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "crowd", "*.npz")))
GOLDENS = golden_paths() + CROWD_GOLDENS
BIG = dict(cap_peaks=1 << 16, cap_conn=8192, cap_rows=8192)  # the checker's capacities: nothing here comes close


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import grouping, skeleton, synth
    from oracle import spg_oracle as so

    return types.SimpleNamespace(torch=torch, G=grouping, skeleton=skeleton, synth=synth, so=so, dev=cuda_device)


def _same(ref, got, what):
    d = diff_structures(ref, got, float_tol=0.0)
    assert not d, f"{what}: not bit-identical:\n" + "\n".join(d)


def _tiny(env, limbs=None, **kw):
    """A handle whose capacities every golden exceeds (as test_capacity_overflows_are_flagged_not_fatal uses)."""
    cfg = dict(max_batch=1, max_h=64, max_w=64, max_peaks_per_part=8, max_person_rows=4, max_cands_per_limb=4)
    cfg.update(kw)
    return env.G.Grouper(limbs if limbs is not None else env.skeleton.LIMBS, **cfg)


def _dev(env, a):
    return env.torch.from_numpy(np.ascontiguousarray(a)).to(env.dev)


@pytest.mark.parametrize("path", GOLDENS, ids=[os.path.relpath(p, os.path.join(ROOT, "tests", "golden"))[:-4]
                                               for p in GOLDENS])
def test_every_golden_through_the_tier(env, path):
    case = load_case(path)
    heat, paf, ext, params = case["heat"], case["paf"], case["image_extent"], case["params"]
    with _tiny(env, case["limbs"]) as g:
        r = g.group_unbounded(_dev(env, heat), _dev(env, paf), ext, params)
    assert r.status[0] == 0, f"status {r.status[0]:#x}"
    got = r.as_reference_structures(0)
    _same(case["structs"], got, "reference")
    o = env.so.group_batch(heat[None], paf[None], case["limbs"], ext, params, **BIG)
    assert o.status[0] == 0
    _same(o.as_reference_structures(0), got, "checker")
    xy, sc = o.to_coco(0, env.skeleton.COCO_FROM_PART)
    P = int(o.n_persons[0])
    assert np.array_equal(r.people_xy[0, :P], xy) and np.array_equal(r.people_score[0, :P], sc)


@pytest.mark.parametrize("path", [p for p in GOLDENS if "f64" not in os.path.basename(p)][:4])
def test_float32_planes_held_as_float64(env, path):
    """SPG_F32_AS_F64: float32 storage, the reference's float64 arithmetic (a single-scale predict() output)."""
    case = load_case(path)
    heat, paf = case["heat"], case["paf"].astype(np.float32)
    with _tiny(env, case["limbs"]) as g:
        r = g.group_unbounded(_dev(env, heat), _dev(env, paf), case["image_extent"], case["params"], paf_as_f64=True)
    o = env.so.group_batch(heat[None], paf[None].astype(np.float64), case["limbs"], case["image_extent"], case["params"],
                           **BIG)
    _same(o.as_reference_structures(0), r.as_reference_structures(0), "checker on the float64 values")


# name -> (seed, H, W, persons, added to the body-part maps, make_image knobs, capacity bits the bounded call sets)
CROWDS = {
    "peaks": (11, 256, 256, 60, 0.0, dict(spikes=3000), 1),     # 242 peaks in a part, 75 rows, 163 candidates
    "rows": (13, 256, 256, 110, 0.0, dict(drop_prob=0.3), 4),  # 84 peaks, 253 rows (dead ones included)
    "cands": (16, 160, 160, 70, 1.0, {}, 2),                    # 70 peaks, 4 900 candidates on a limb
    "all": (20, 256, 256, 240, 1.0, dict(drop_prob=0.6, spikes=3000), 7),
}


def _crowd(env, name):
    seed, H, W, persons, add, kw, _ = CROWDS[name]
    heat, paf = env.synth.make_batch(seed, 1, H, W, persons, **kw)
    return heat[0], (paf[0] + np.float32(add)).astype(np.float32)


@pytest.mark.parametrize("name", list(CROWDS))
def test_crowded_images_flag_the_bounded_call_and_the_tier_equals_the_checker(env, name):
    from improved_body_parts_b200 import dropin
    heat, paf = _crowd(env, name)
    H, W = heat.shape[1:]
    params = env.skeleton.default_params()
    normal = [env.synth.make_image(300 + i, 96 + 8 * i, 120, 6 + i) for i in range(2)]
    maps = [normal[0], (heat, paf), normal[1]]
    g = env.G.Grouper(max_batch=3, max_h=H, max_w=W, max_peaks_per_part=dropin.CAP_PEAKS,
                      max_cands_per_limb=dropin.CAP_CANDS, max_person_rows=dropin.CAP_ROWS)
    try:
        g.group_ragged([(_dev(env, h), _dev(env, p)) for h, p in maps], [h.shape[1] for h, _ in maps], params)
        r = g.fetch(3)
        assert int(r.status[1]) & 7 == CROWDS[name][-1], f"status {int(r.status[1]):#x}"
        for i in (0, 2):  # the other images of the ragged batch
            h, p = maps[i]
            o = env.so.group_batch(h[None], p[None], env.skeleton.LIMBS, h.shape[1], params, **BIG)
            assert r.status[i] == 0
            _same(o.as_reference_structures(0), r.as_reference_structures(i), f"image {i}")
        t = g.group_unbounded(_dev(env, heat), _dev(env, paf), H, params)
        after = g.fetch(3)  # the tier leaves the bounded call's results alone
        for f in ("n_persons", "subset", "people_xy", "status", "peak_x", "conn_ij"):
            assert np.array_equal(getattr(after, f), getattr(r, f)), f
    finally:
        g.close()
    assert t.status[0] == 0
    o = env.so.group_batch(heat[None], paf[None], env.skeleton.LIMBS, H, params, **BIG)
    assert o.status[0] == 0
    _same(o.as_reference_structures(0), t.as_reference_structures(0), "checker")
    xy, sc = o.to_coco(0, env.skeleton.COCO_FROM_PART)
    P = int(o.n_persons[0])
    assert int(t.n_persons[0]) == P
    assert np.array_equal(t.people_xy[0, :P], xy) and np.array_equal(t.people_score[0, :P], sc)


def test_tier_reports_the_sample_index_bit(env):
    heat, paf = _crowd(env, "peaks")
    heat = _with_far_peak(env, heat)
    params = env.skeleton.default_params()
    with _tiny(env, max_h=256, max_w=256) as g:
        r = g.group_unbounded(_dev(env, heat), _dev(env, paf), heat.shape[1], params)
    assert r.status[0] & env.G.ST_SAMPLE_INDEX


def _with_far_peak(env, heat):
    """A peak of the first limb's A part whose refined x lands ~2000 px right of the map: the reference samples outside
    the map there and raises IndexError (evaluate.py:235).  Its 5x5 box sums to ~1e-3 with a large row-weighted sum."""
    heat = heat.copy()
    a = env.skeleton.LIMBS[0][0]
    y, x = heat.shape[1] // 2, heat.shape[2] // 2
    heat[a, y - 2:y + 3, x - 2:x + 3] = 0.0
    heat[a, y, x] = 1.0
    heat[a, y - 2, x - 2:x + 3] = -0.1998
    return heat


# ---- the drop-in functions ----------------------------------------------------------------------------------------
@pytest.fixture()
def dropin(cuda_device):
    from improved_body_parts_b200 import dropin as d
    d.configure(device=0, limbs=d.LIMBS)
    yield d
    d.configure()


def _hwc(a):
    return np.ascontiguousarray(a.transpose(1, 2, 0))


def test_dropin_group_and_chained_stages_take_the_tier(dropin, env):
    assert CROWD_GOLDENS, "tests/golden/crowd/*.npz missing"
    for path in CROWD_GOLDENS:
        case = load_case(path)
        heat, paf, ext, params = _hwc(case["heat"]), _hwc(case["paf"]), case["image_extent"], case["params"]
        _same(case["structs"], dropin.group(heat, paf, ext, params), "group")
        all_peaks = dropin.find_peaks(heat, params)
        conns, special = dropin.find_connections(all_peaks, paf, ext, params)
        subset, candidate = dropin.find_people(conns, special, all_peaks, params)
        _same(case["structs"], (all_peaks, conns, special, subset, candidate), "chained stages")
        # foreign peaks past the capacities still raise, and say why
        copied = [list(p) for p in all_peaks]
        with pytest.raises(env.G.GroupingError, match="capacity"):
            dropin.find_connections(copied, paf, ext, params)


def test_dropin_group_many_mixed_batch(dropin, env):
    crowd = load_case(CROWD_GOLDENS[0])
    small = load_case(golden_paths()[0])
    cases = [small, crowd, small]
    got = dropin.group_many([(_hwc(c["heat"]), _hwc(c["paf"])) for c in cases], [c["image_extent"] for c in cases],
                            crowd["params"])
    for i, c in enumerate(cases):
        _same(c["structs"], got[i], f"image {i}")


def test_dropin_sample_index_still_raises(dropin, env):
    heat, paf = _crowd(env, "peaks")
    heat = _with_far_peak(env, heat)
    params = env.skeleton.default_params()
    with pytest.raises(env.G.GroupingError, match="sample index"):
        dropin.group(_hwc(heat), _hwc(paf), heat.shape[1], params)
    with pytest.raises(env.G.GroupingError, match="sample index"):
        dropin.group_many([(_hwc(heat), _hwc(paf))], [heat.shape[1]], params)


def test_predict_many_with_a_crowded_image(dropin, env, tmp_path):
    """batch > 1: the crowded image's persons come from the tier (more than the wire record holds); the per-image path
    (process(): the three chained stage functions) gives the same file."""
    import cv2
    import torch
    from improved_body_parts_b200 import wire
    from test_gpu_ragged import _stand_in_evaluate, _typed

    shapes = [(120, 160), (512, 512), (160, 120)]
    rng = np.random.default_rng(5)
    coco = types.SimpleNamespace(imgs={}, getImgIds=lambda: sorted(coco.imgs))
    for k, (H, W) in enumerate(shapes):
        iid = 2000 + k
        cv2.imwrite(str(tmp_path / f"{iid:012d}.png"), rng.integers(0, 255, size=(H, W, 3), dtype=np.uint8))
        coco.imgs[iid] = {"file_name": f"{iid:012d}.png"}
    ids = list(coco.imgs)
    params = dict(env.skeleton.default_params(), scale_search=[1.0], rotation_search=[0.0])
    model_params = dict(boxsize=512, stride=4, max_downsample=32, padValue=128)

    def model(x):  # a crowd for the large input, a few persons otherwise
        h, w = int(x.shape[1]) // 4, int(x.shape[2]) // 4
        out = env.synth.make_network_output(h * 1000 + w, h, w, 200 if h >= 128 else 3, noise=0.0)
        return [[torch.from_numpy(out).to(x.device)]]

    results = []
    for batch in (1, 3):
        mod = _stand_in_evaluate(env.skeleton, dropin)
        mod.posenet = model
        dropin.install(mod, device_predict=True, batch=batch)
        results.append(mod.predict_many(coco, str(tmp_path), ids, params, model, model_params, 18, 30))
    per_image, batched = results
    assert len(per_image[2001]) > dropin.CAP_ROWS
    assert list(batched) == list(per_image)
    assert _typed(list(batched.values())) == _typed(list(per_image.values()))
    wire.format_results(per_image, str(tmp_path / "a.json"))
    wire.format_results(batched, str(tmp_path / "b.json"))
    assert (tmp_path / "a.json").read_bytes() == (tmp_path / "b.json").read_bytes()
