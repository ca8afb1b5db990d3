"""GPU: evaluate.py's own geometry (boxsize 640, stride 4, max_downsample 64) on COCO-shaped images, bit for bit against
the CPU chain of ``coco_geometry``: ``postnet_port`` maps, the C checker's structures and ``dropin.keypoints``' people.

At this geometry a 480 x 640 image runs ``postnet_kernel`` with a 0.75 second resize over hundreds of tiles, an image
640 rows high the identity kernel; its 480 x 640 planes take the banded peak finder, widths 427, 375, 359 the per-band
one, the body-part planes the L2-sampling limb scorer; the crowds leave limbs with more than 256 candidates.  Every
device path of a validation run is held to the chain: ``predict`` + ``group``, ``predict_batch`` + ``group_many``,
``predict_many`` on an ``evaluate``-like module and ``FrameStream`` on a replayed frame, for the reference default,
multi-scale, rotation-search and demo settings.  The coverage tests fail if the fixture stops reaching those paths."""
import types

import numpy as np
import pytest

import coco_geometry as cg
from parity import diff_structures

pytestmark = pytest.mark.gpu

_chains = {}


def _chain(cfg, i):
    """The CPU chain of fixture entry i under ``cfg``, computed once per module."""
    if (cfg.name, i) not in _chains:
        _chains[(cfg.name, i)] = cg.cpu_chain(cfg, i)
    return _chains[(cfg.name, i)]


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch

    from improved_body_parts_b200 import dropin, skeleton
    e = types.SimpleNamespace(torch=torch, dropin=dropin, skeleton=skeleton, dev=cuda_device, kernels={}, models={})
    return e


@pytest.fixture(autouse=True)
def _restore_dropin(request):
    """``dropin.configure()`` keeps every setting it is not given: after each test put back all that ``_setup`` and
    ``install`` change (the variant above all), so that later test modules see the defaults."""
    yield
    if "env" in request.fixturenames:
        from improved_body_parts_b200 import dropin, skeleton
        dropin.configure(limbs=skeleton.LIMBS, device=0, variant="evaluate", input_stage="host", decode="host")


def _setup(env, name):
    """``dropin`` configured for ``CONFIGS[name]`` and its stand-in network (built once per configuration)."""
    cfg = cg.CONFIGS[name]
    env.dropin.configure(device=0, limbs=env.skeleton.LIMBS, variant=cfg.variant, input_stage="host", decode="host")
    if name not in env.models:
        env.models[name] = cg.StandIn(env.torch, env.dev, cfg)
    return cfg, env.models[name]


def _same(got, want, what):
    """Bit for bit, a NaN equal to a NaN at the same position (device and host NaN payloads differ)."""
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, got.shape, want.dtype, want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN positions differ"
    bad = got[~nan].view(np.uint8).reshape(-1, got.itemsize) != want[~nan].view(np.uint8).reshape(-1, got.itemsize)
    assert not bad.any(), f"{what}: {int(bad.any(1).sum())} values differ"


def _check_maps(heat, paf, c, what):
    """``DeviceMaps`` (or the ``[1, C, H, W]`` tensors of a frame) against the chain's maps."""
    h = heat.tensor if hasattr(heat, "tensor") else heat
    p = paf.tensor if hasattr(paf, "tensor") else paf
    _same(h[0].permute(1, 2, 0).cpu().numpy(), c.heat, f"{what}: heat")
    _same(p[0].permute(1, 2, 0).double().cpu().numpy(), c.paf, f"{what}: paf")


def _check_structs(got, c, what):
    d = diff_structures(c.structs, got, float_tol=0.0)
    assert not d, f"{what}:\n" + "\n".join(d)


def _typed(v):
    if isinstance(v, (list, tuple)):
        return (type(v).__name__, [_typed(x) for x in v])
    return (type(v).__name__, repr(v))


def _check_people(got, c, what):
    assert _typed(got) == _typed(c.people), f"{what}: people differ"


@pytest.mark.parametrize("name", list(cg.CONFIGS))
def test_predict_then_group_is_the_chain(env, name):
    cfg, model = _setup(env, name)
    d = env.dropin
    params = cfg.params()
    kernels = env.kernels.setdefault(name, set())
    for i in cfg.images:
        spec, c = cg.FIXTURE[i], _chain(cfg, i)
        what = f"{name} image {i} {spec.H}x{spec.W}"
        heat, paf = d.predict(cg.image(i, spec), params, model, cg.MODEL_PARAMS)
        kernels.add(d._grouper().postnet_kernel())
        _check_maps(heat, paf, c, what)
        got = d.group(heat, paf, spec.H, params)
        kernels.update(d._grouper().stage_kernels()[:2])
        _check_structs(got, c, what)
        _check_people(d.keypoints(got[3], got[4]), c, what)


@pytest.mark.parametrize("forward_batch", [1, 4])
@pytest.mark.parametrize("name", list(cg.CONFIGS))
def test_predict_batch_then_group_many_is_the_chain(env, name, forward_batch):
    cfg, model = _setup(env, name)
    d = env.dropin
    params = cfg.params()
    imgs = [cg.image(i, cg.FIXTURE[i]) for i in cfg.images]
    maps = d.predict_batch(imgs, params, model, cg.MODEL_PARAMS, forward_batch=forward_batch)
    for (heat, paf), i in zip(maps, cfg.images):
        _check_maps(heat, paf, _chain(cfg, i), f"{name} image {i}")
    got = d.group_many(maps, [cg.FIXTURE[i].H for i in cfg.images], params)
    env.kernels.setdefault(name + " ragged", set()).update(d._ragged[0].stage_kernels()[:2])
    for g, i in zip(got, cfg.images):
        _check_structs(g, _chain(cfg, i), f"{name} image {i} (forward_batch {forward_batch})")


@pytest.mark.parametrize("name", list(cg.CONFIGS))
def test_predict_many_is_the_chain(env, name, tmp_path):
    import cv2

    from test_gpu_ragged import _stand_in_evaluate
    cfg, model = _setup(env, name)
    coco = types.SimpleNamespace(imgs={}, getImgIds=lambda: sorted(coco.imgs))
    for i in cfg.images:
        iid = 5000 + 3 * i
        assert cv2.imwrite(str(tmp_path / f"{iid:012d}.png"), cg.image(i, cg.FIXTURE[i]))
        coco.imgs[iid] = {"file_name": f"{iid:012d}.png"}
    mod = _stand_in_evaluate(env.skeleton, env.dropin)
    mod.posenet = model
    env.dropin.install(mod, device_predict=True, batch=8)
    got = mod.predict_many(coco, str(tmp_path), list(coco.imgs), cfg.params(), model, dict(cg.MODEL_PARAMS), 18, 30)
    assert list(got) == list(coco.imgs)
    env.kernels.setdefault(name + " predict_many", set()).update(env.dropin._ragged[0].stage_kernels()[:2])
    for (iid, people), i in zip(got.items(), cfg.images):
        _check_people(people, _chain(cfg, i), f"{name} image {i}")


@pytest.mark.parametrize("name", list(cg.CONFIGS))
def test_frame_stream_replay_is_the_chain(env, name):
    """One slot: a frame's first tick captures its graph, the second replays it; both equal the chain."""
    cfg, model = _setup(env, name)
    d = env.dropin
    frames = list(cfg.images[:3]) + list(cfg.images[:3])
    with d.FrameStream(model, cfg.params(), cg.MODEL_PARAMS, slots=1) as fs:
        for k, i in enumerate(frames):
            c = _chain(cfg, i)
            r = fs.result(fs.submit(cg.image(i, cg.FIXTURE[i])), detail=True)
            what = f"{name} image {i} ({'replay' if k >= len(frames) // 2 else 'capture'})"
            _check_maps(r.heat, r.paf, c, what)
            _check_people(r.people, c, what)
        assert fs.captures == len({(cg.FIXTURE[i].H, cg.FIXTURE[i].W) for i in cfg.images[:3]})


def test_the_fixture_reaches_the_kernels(env):
    """Names ``stage_kernels()`` / ``postnet_kernel()`` reported in the tests above: the geometry reaches every path."""
    got = env.kernels.get("default")
    if not got:
        pytest.skip("runs after test_predict_then_group_is_the_chain[default]")
    assert {"postnet_kernel", "postnet_x4_ident_kernel"} <= got, got
    assert {"nms_peaks_banded_kernel", "nms_peaks_kernel"} <= got, got
    assert "limb_score_kernel<float,false,double>" in got, got  # single scale: float32 planes of float64 values, via L2
    assert "limb_score_kernel<double,false>" in env.kernels.get("scales4", set()), env.kernels.get("scales4")
    for key in ("default ragged", "default predict_many"):
        ragged = env.kernels.get(key, set())
        assert "nms_peaks_ragged_kernel" in ragged and any(k.startswith("limb_score_ragged_kernel") for k in ragged), \
            (key, ragged)


def test_the_chain_reaches_the_paths():
    """The CPU chain's own coverage: a limb with more than 256 candidates (the matcher past its parallel rounds), most
    scored pairs with all 20 samples, peaks whose refine box leaves the map, and twins whose limbs tie exactly."""
    cfg = cg.CONFIGS["default"]
    cov = cg.coverage({i: _chain(cfg, i) for i in cfg.images})
    assert cov["max_cands"] > 256, cov
    assert cov["full_samples"] > 0.5, cov
    assert cov["border_images"], cov
    _assert_twins_tie(_chain(cfg, cg.TWINS[0]))


def _assert_twins_tie(c):
    """Each limb of the twins: the two accepted rows have the same score, so their order is the tie-break's."""
    ties = sum(1 for rows in c.structs[1] if len(rows) >= 2 and rows[0, 2] == rows[1, 2])
    assert ties >= 10, ties


@pytest.mark.parametrize("shape", [(480, 640), (427, 640)])
def test_prenet_at_the_validation_geometry_is_the_port(env, shape):
    """``spg_prenet`` and ``spg_prenet_ragged`` against ``prenet_port`` for 480 x 640 -> 640 x 896 and
    427 x 640 -> 640 x 960 inputs, unrotated and rotated."""
    from improved_body_parts_b200 import grouping, synth
    from oracle import prenet_port as pn
    t = env.torch
    H, W = shape
    img = synth.photo(31 + H, H, W)
    m = 640 / H
    angles = [0.0, 15.0]
    want = [pn.prenet_item(img, m, a, 64, 128) for a in angles]
    assert want[0][0].shape[1:3] == cg.geometry(H, W, 1.0)[4:]
    dev = t.from_numpy(img).to(env.dev)
    g = grouping.Grouper(max_batch=1, max_h=64, max_w=64)
    try:
        got = g.prenet(dev, [m], angles, max_downsample=64, pad_value=128)
        ragged = g.prenet_ragged([(dev, m, a) for a in angles], max_downsample=64, pad_value=128)
        for what, items in (("spg_prenet", got), ("spg_prenet_ragged", ragged)):
            for (pair, crop, rev), (ref, ref_crop, _, ref_rev), a in zip(items, want, angles):
                p = pair.cpu().numpy()
                assert np.array_equal(p.view(np.uint32), ref.view(np.uint32)), (what, a, int((p != ref).sum()))
                assert tuple(crop) == tuple(ref_crop) and (rev is None) == (ref_rev is None)
    finally:
        g.close()
