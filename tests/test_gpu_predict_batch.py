"""GPU: ``dropin.predict_batch`` -- predict() for a batch of images, any ``scale_search x rotation_search``: one forward
pass per chunk of ``forward_batch`` items of one input size and one ragged post-network call -- against ``predict`` per
image.

The network is a stand-in whose output for a sample does not depend on the batch it runs in: network-like maps keyed on
the input size, plus a small term taken by indexing and scaling from the sample's own input (elementwise float32 is exact
whatever the batch, and an image read from the wrong slot changes its maps)."""
import types

import numpy as np
import pytest

from test_gpu_ragged import _stand_in_evaluate, _typed

pytestmark = pytest.mark.gpu

MODEL_PARAMS = dict(boxsize=160, stride=4, max_downsample=32, padValue=128)

SEARCHES = {"1 item": ([1.0], [0.0]), "2 scales": ([1.0, 0.5], [0.0]), "5 scales": ([0.5, 1.0, 1.5, 2.0, 2.5], [0.0]),
            "3 angles": ([1.0], [0.0, 30.0, -30.0]), "2 scales x 2 angles": ([1.0, 0.5], [0.0, 30.0])}


class StandIn:
    def __init__(self, torch, synth):
        self.torch, self.synth, self.calls, self._maps = torch, synth, [], {}

    def __call__(self, x):
        t = self.torch
        self.calls.append(tuple(x.shape))
        n, Hp, Wp, _ = x.shape
        h, w = Hp // 4, Wp // 4
        if (h, w) not in self._maps:
            self._maps[(h, w)] = t.from_numpy(self.synth.make_network_output(h * 1000 + w, h, w, 3, noise=0.0)).to(x.device)
        base = self._maps[(h, w)].repeat(n // 2, 1, 1, 1)
        own = x[:, ::4, ::4, :][..., t.arange(50, device=x.device) % 3].permute(0, 3, 1, 2)
        return [[base + own * t.tensor(0.05, dtype=t.float32, device=x.device)]]


@pytest.fixture()
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import dropin, skeleton, synth

    dropin.configure(device=0, limbs=dropin.LIMBS)
    yield types.SimpleNamespace(torch=torch, dropin=dropin, skeleton=skeleton, synth=synth, dev=cuda_device)
    dropin.configure(input_stage="host", variant="evaluate")


# boxsize 160: (120, 160), (60, 80), (90, 120) share a 160 x 224 input; (160, 120), (80, 60) a 160 x 128 one; images 160
# rows high are identity items (crop == image) at scale 1
SHAPES = [(120, 160), (160, 120), (60, 80), (160, 200), (90, 120), (80, 60), (160, 97), (150, 200), (33, 250), (160, 200)]


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
    imgs = _images(1)
    model = StandIn(t, env.synth)
    want = [d.predict(img, params, model, MODEL_PARAMS, input_stage=stage) for img in imgs]
    model.calls.clear()
    got = d.predict_batch(imgs, params, model, MODEL_PARAMS, forward_batch=forward_batch, input_stage=stage)
    _assert_maps_equal(got, want)
    # one forward pass per chunk of at most forward_batch items of one input size, sizes in order of first appearance
    _, buckets = d.plan_items([im.shape[:2] for im in imgs], params, MODEL_PARAMS)
    assert model.calls == _expected_calls(buckets, forward_batch)
    assert any(len(m) > 2 for m in buckets.values()) and len(buckets) >= 3


@pytest.mark.parametrize("params_update,stride", [(dict(scale_search=[1.0, 0.5], rotation_search=[0.0]), 4),
                                                  (dict(scale_search=[1.0], rotation_search=[0.0, 30.0]), 4),
                                                  (dict(scale_search=[1.0], rotation_search=[0.0]), 8),
                                                  (dict(scale_search=[1.0, 0.5], rotation_search=[0.0]), 8)])
def test_predict_batch_equals_predict_at_any_stride(env, params_update, stride):
    """At stride 4 the items are batched; at another stride (no rotation there) every image runs ``predict``, one pair
    per forward pass."""
    d, t = env.dropin, env.torch
    params = dict(env.skeleton.default_params(), **params_update)
    model_params = dict(MODEL_PARAMS, stride=stride)
    imgs = _images(2)[:5]
    model = StandIn(t, env.synth)
    want = [d.predict(img, params, model, model_params) for img in imgs]
    model.calls.clear()
    got = d.predict_batch(imgs, params, model, model_params, forward_batch=8)
    _assert_maps_equal(got, want)
    assert (max(c[0] for c in model.calls) > 2) == (stride == 4)


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


@pytest.mark.parametrize("search,batch,forward_batch", [("1 item", 3, 2), ("1 item", 16, 4), ("2 scales", 6, 4),
                                                        ("2 scales x 2 angles", 6, 4)])
def test_predict_many_with_forward_batch_equals_the_per_image_path(env, tmp_path, search, batch, forward_batch):
    import cv2
    from improved_body_parts_b200 import wire

    d = env.dropin
    rng = np.random.default_rng(11)
    coco = types.SimpleNamespace(imgs={}, getImgIds=lambda: sorted(coco.imgs))
    for k, (H, W) in enumerate(SHAPES):
        iid = 2000 + 7 * k
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
    d.install(mod, device_predict=True, batch=batch, forward_batch=forward_batch)
    model.calls.clear()
    batched = mod.predict_many(coco, str(tmp_path), ids, params, model, MODEL_PARAMS, 18, 30)
    assert max(c[0] for c in model.calls) > 2  # the forward passes were batched
    assert list(batched) == list(per_image)
    assert _typed(list(batched.values())) == _typed(list(per_image.values()))
    wire.format_results(per_image, str(tmp_path / "a.json"))
    wire.format_results(batched, str(tmp_path / "b.json"))
    assert (tmp_path / "a.json").read_bytes() == (tmp_path / "b.json").read_bytes()
