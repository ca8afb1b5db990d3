"""GPU: ``dropin.predict_batch`` with several items per image -- the multi-scale and rotation search: one forward pass
per chunk of ``forward_batch`` items of one input size and one ragged multi-item post-network call -- against
``predict`` per image.  The stand-in network's output for a sample does not depend on the batch it runs in."""
import types

import numpy as np
import pytest

from test_gpu_predict_batch import MODEL_PARAMS, SHAPES, StandIn
from test_gpu_ragged import _stand_in_evaluate, _typed

pytestmark = pytest.mark.gpu

SEARCHES = {"2 scales": ([1.0, 0.5], [0.0]), "5 scales": ([0.5, 1.0, 1.5, 2.0, 2.5], [0.0]),
            "3 angles": ([1.0], [0.0, 30.0, -30.0]), "2 scales x 2 angles": ([1.0, 0.5], [0.0, 30.0])}


@pytest.fixture()
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import dropin, skeleton, synth

    dropin.configure(device=0, limbs=dropin.LIMBS)
    yield types.SimpleNamespace(torch=torch, dropin=dropin, skeleton=skeleton, synth=synth, dev=cuda_device)
    dropin.configure(input_stage="host", variant="evaluate")


def _images(seed=0, shapes=SHAPES):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8) for H, W in shapes]


def _assert_maps_equal(got, want):
    assert len(got) == len(want)
    for i, ((gh, gp), (wh, wp)) in enumerate(zip(got, want)):
        for a, b, name in ((gh, wh, "heat"), (gp, wp, "paf")):
            assert a.as_f64 == b.as_f64 and a.shape == b.shape, f"image {i}: {name}"
            x, y = a.tensor.cpu().numpy(), b.tensor.cpu().numpy()
            assert x.dtype == y.dtype and np.array_equal(x, y, equal_nan=True), f"image {i}: {name}"


def _expected_calls(buckets, forward_batch):
    calls = []
    for (Hp, Wp), members in buckets.items():
        for c0 in range(0, len(members), forward_batch):
            calls.append((2 * min(forward_batch, len(members) - c0), Hp, Wp, 3))
    return calls


@pytest.mark.parametrize("search", list(SEARCHES))
@pytest.mark.parametrize("stage", ["host", "device"])
@pytest.mark.parametrize("forward_batch", [2, 16])
def test_predict_batch_equals_predict(env, search, stage, forward_batch):
    d, t = env.dropin, env.torch
    scales, angles = SEARCHES[search]
    params = dict(env.skeleton.default_params(), scale_search=scales, rotation_search=angles)
    imgs = _images(1, SHAPES[:8])
    model = StandIn(t, env.synth)
    want = [d.predict(img, params, model, MODEL_PARAMS, input_stage=stage) for img in imgs]
    model.calls.clear()
    got = d.predict_batch(imgs, params, model, MODEL_PARAMS, forward_batch=forward_batch, input_stage=stage)
    _assert_maps_equal(got, want)
    # one forward pass per chunk of at most forward_batch items of one input size, in plan_items order
    _, buckets = d.plan_items([im.shape[:2] for im in imgs], params, MODEL_PARAMS)
    assert model.calls == _expected_calls(buckets, forward_batch)
    assert any(len(m) > 2 for m in buckets.values())


def test_demo_variant(env):
    d, t = env.dropin, env.torch
    d.configure(variant="demo")
    params = dict(env.skeleton.default_params(), scale_search=[1.0, 0.5, 1.5], rotation_search=[0.0, 30.0])
    imgs = _images(4, SHAPES[:6])
    model = StandIn(t, env.synth)
    want = [d.predict(img, params, model, MODEL_PARAMS) for img in imgs]
    got = d.predict_batch(imgs, params, model, MODEL_PARAMS, forward_batch=4)
    _assert_maps_equal(got, want)


def test_uint8_cuda_tensors_on_the_device_stage(env):
    d, t = env.dropin, env.torch
    params = dict(env.skeleton.default_params(), scale_search=[1.0, 0.5], rotation_search=[0.0, -30.0])
    imgs = _images(5, SHAPES[:5])
    model = StandIn(t, env.synth)
    want = [d.predict(img, params, model, MODEL_PARAMS, input_stage="device") for img in imgs]
    got = d.predict_batch([t.from_numpy(im).to(env.dev) for im in imgs], params, model, MODEL_PARAMS, forward_batch=3,
                          input_stage="device")
    _assert_maps_equal(got, want)


@pytest.mark.parametrize("search", ["2 scales", "2 scales x 2 angles"])
def test_predict_many_with_forward_batch_equals_the_per_image_path(env, tmp_path, search):
    import cv2
    from improved_body_parts_b200 import wire

    d = env.dropin
    rng = np.random.default_rng(12)
    coco = types.SimpleNamespace(imgs={}, getImgIds=lambda: sorted(coco.imgs))
    for k, (H, W) in enumerate(SHAPES):
        iid = 3000 + 7 * k
        cv2.imwrite(str(tmp_path / f"{iid:012d}.png"), rng.integers(0, 255, size=(H, W, 3), dtype=np.uint8))
        coco.imgs[iid] = {"file_name": f"{iid:012d}.png"}
    ids = list(coco.imgs)[::-1]
    scales, angles = SEARCHES[search]
    params = dict(env.skeleton.default_params(), scale_search=scales, rotation_search=angles)
    model = StandIn(env.torch, env.synth)

    mod = _stand_in_evaluate(env.skeleton, d)
    mod.posenet = model
    d.install(mod, device_predict=True)
    per_image = mod.predict_many(coco, str(tmp_path), ids, params, model, MODEL_PARAMS, 18, 30)
    assert sum(len(v) for v in per_image.values()) > 0
    mod = _stand_in_evaluate(env.skeleton, d)
    mod.posenet = model
    d.install(mod, device_predict=True, batch=6, forward_batch=4)
    model.calls.clear()
    batched = mod.predict_many(coco, str(tmp_path), ids, params, model, MODEL_PARAMS, 18, 30)
    assert max(c[0] for c in model.calls) > 2  # the forward passes were batched
    assert list(batched) == list(per_image)
    assert _typed(list(batched.values())) == _typed(list(per_image.values()))
    wire.format_results(per_image, str(tmp_path / "a.json"))
    wire.format_results(batched, str(tmp_path / "b.json"))
    assert (tmp_path / "a.json").read_bytes() == (tmp_path / "b.json").read_bytes()
