"""GPU: the ragged multi-item post-network stage (``spg_postnet_ragged_items`` / ``Grouper.postnet_ragged_items``).

Images of different sizes, each with the items of one ``product(multiplier, rotate_angle)``, share one call; each image's
maps must equal, bit for bit (NaN-aware), what ``Grouper.postnet(..., rotations=...)`` gives for that image alone."""
import ctypes as C
import itertools
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MD = 16  # max_downsample of the geometry below


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import grouping, synth

    e = types.SimpleNamespace(torch=torch, grouping=grouping, synth=synth, dev=cuda_device)
    e.g = grouping.Grouper(max_batch=128, max_h=1024, max_w=1024)
    e.single = grouping.Grouper(max_batch=1, max_h=1024, max_w=1024)
    yield e
    e.g.close()
    e.single.close()


# (H, W): widths that are not multiples of 4 and sizes that leave partial border tiles; at scale 1 an item's crop is
# the image (identity second resize)
SIZES = [(160, 213), (97, 131), (128, 128), (75, 301), (203, 150), (61, 47), (130, 90), (64, 257), (33, 35), (250, 190)]


def _items(env, H, W, scales, angles, dtype, seed, nan=False, channels=50):
    """predict()'s items of one H x W image: (network output [2, C, h, w], crop, rotate_matrix_reverse or None)."""
    import cv2
    out = []
    for t, (s, angle) in enumerate(itertools.product(scales, angles)):
        H1, W1 = int(np.rint(H * s)), int(np.rint(W * s))
        Hp, Wp = -(-H1 // MD) * MD, -(-W1 // MD) * MD
        net = env.synth.make_network_output(seed + 97 * t, Hp // 4, Wp // 4, 2)
        if channels > net.shape[1]:  # channel offsets: the maps sit inside a wider output
            wide = np.zeros((2, channels) + net.shape[2:], np.float32)
            wide[:, 3:3 + net.shape[1]] = net
            net = wide
        if nan:
            net[np.random.default_rng(seed + t).random(net.shape) < 0.002] = np.nan
        rev = cv2.getRotationMatrix2D((Hp / 2, Wp / 2), -angle, 1) if angle != 0 else None
        out.append((env.torch.from_numpy(net).to(env.dev, dtype), (H1, W1), rev))
    return out


def _images(env, sizes, scales, angles, dtype, nan=False, seed=0, channels=50):
    return [(_items(env, H, W, scales, angles, dtype, seed + 31 * i, nan, channels), (H, W)) for i, (H, W) in enumerate(sizes)]


def _same(a, b, what):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=True), what


def _check_against_single(env, imgs, got, **kw):
    for i, (items, hw) in enumerate(imgs):
        rots = [r for _, _, r in items]
        heat, paf = env.single.postnet([o[None] for o, _, _ in items], [c for _, c, _ in items], hw,
                                       rotations=rots if any(r is not None for r in rots) else None, **kw)
        _same(got[i][0], heat, f"image {i} {hw}: heat")
        _same(got[i][1], paf, f"image {i} {hw}: paf")


CONFIGS = {"2 scales": ([1.0, 0.5], [0.0]), "5 scales": ([0.5, 1.0, 1.5, 2.0, 0.7], [0.0]),
           "scales x angles": ([1.0, 0.5], [0.0, 30.0, -30.0]), "one rotated item": ([1.0], [30.0])}


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("net_dtype", ["float32", "float16"])
def test_ragged_items_equal_per_image_postnet(env, config, net_dtype):
    t = env.torch
    scales, angles = CONFIGS[config]
    imgs = _images(env, SIZES, scales, angles, getattr(t, net_dtype), seed=7)
    got = env.g.postnet_ragged_items(imgs)
    want_kernel = "postnet_rot_ragged_kernel" if any(angles) else "postnet_items_ragged_kernel"
    assert env.g.postnet_kernel() == want_kernel
    assert got[0][1].dtype == (t.float32 if len(scales) * len(angles) == 1 else t.float64)
    _check_against_single(env, imgs, got)


@pytest.mark.parametrize("config", ["2 scales", "5 scales", "scales x angles"])
def test_nan_scrub_and_channel_offsets(env, config):
    t = env.torch
    scales, angles = CONFIGS[config]
    imgs = _images(env, SIZES[:6], scales, angles, t.float32, nan=True, seed=11, channels=56)
    got = env.g.postnet_ragged_items(imgs, paf_chan0=3, heat_chan0=33, nan_scrub=True)
    assert not any(bool(t.isnan(h).any()) or bool(t.isnan(p).any()) for h, p in got)
    _check_against_single(env, imgs, got, paf_chan0=3, heat_chan0=33, nan_scrub=True)
    got = env.g.postnet_ragged_items(imgs, paf_chan0=3, heat_chan0=33)  # without the scrub the NaNs pass through
    assert any(bool(t.isnan(h).any()) for h, _ in got)
    _check_against_single(env, imgs, got, paf_chan0=3, heat_chan0=33)


def test_outs_are_reused(env):
    t = env.torch
    imgs = _images(env, SIZES[:5], [1.0, 0.5, 1.5], [0.0], t.float32, seed=3)
    outs = [(t.full((1, 18) + hw, 7.0, device=env.dev), t.full((1, 30) + hw, 7.0, dtype=t.float64, device=env.dev))
            for _, hw in imgs]
    got = env.g.postnet_ragged_items(imgs, outs=outs)
    assert all(a is o[0] and b is o[1] for (a, b), o in zip(got, outs))
    _check_against_single(env, imgs, got)


def test_more_images_than_one_launch_holds(env):
    t = env.torch
    rng = np.random.default_rng(5)
    sizes = [(int(rng.integers(8, 60)), int(rng.integers(8, 80))) for _ in range(120)]
    imgs = _images(env, sizes, [1.0, 0.6], [0.0], t.float16, seed=900)
    before = env.g.launch_count
    got = env.g.postnet_ragged_items(imgs)
    assert env.g.launch_count - before >= 2
    _check_against_single(env, imgs, got)


def test_one_unrotated_item_is_postnet_ragged(env):
    t = env.torch
    imgs = _images(env, SIZES, [0.8], [0.0], t.float32, seed=21)
    got = env.g.postnet_ragged_items(imgs)
    want = env.g.postnet_ragged([(items[0][0], items[0][1], hw) for items, hw in imgs])
    for i, ((a, b), (c, d)) in enumerate(zip(got, want)):
        _same(a, c, f"image {i}: heat")
        _same(b, d, f"image {i}: paf")


@pytest.mark.parametrize("config", list(CONFIGS))
def test_launch_count_does_not_depend_on_the_number_of_images(env, config):
    t = env.torch
    scales, angles = CONFIGS[config]
    sizes = [SIZES[i % 3] for i in range(40)]  # one image family each
    imgs = _images(env, sizes, scales, angles, t.float32, seed=40)
    counts = []
    for n in (10, 40):
        before = env.g.launch_count
        env.g.postnet_ragged_items(imgs[:n])
        counts.append(env.g.launch_count - before)
    assert counts[0] == counts[1] and counts[0] >= 1


def _raw_call(env, imgs, n_items, rot=True, paf_dtype=None, stride=4, n=None):
    """The C ABI directly: (return code, error message) of one call over imgs' items, with arrays the test may edit."""
    g, grouping, t = env.g, env.grouping, env.torch
    n = len(imgs) if n is None else n
    arr = (grouping._PostnetImage * (len(imgs) * n_items))()
    rots = (grouping._PostnetRotation * (len(imgs) * n_items))()
    keep = []
    for i, (items, (H, W)) in enumerate(imgs):
        heat = t.empty((18, H, W), device=env.dev)
        paf = t.empty((30, H, W), dtype=t.float64, device=env.dev)
        keep += [heat, paf]
        for k, (o, (ch, cw), m) in enumerate(items):
            arr[i * n_items + k] = grouping._PostnetImage(o.data_ptr(), o.stride(0), o.stride(1), o.shape[2], o.shape[3], ch,
                                                          cw, H, W, heat.data_ptr(), paf.data_ptr())
            if m is not None:
                rots[i * n_items + k] = grouping._PostnetRotation(1, 0, (C.c_double * 6)(*np.asarray(m).reshape(6).tolist()))
    fp, fh = g._flip_orders(None, None)
    common = grouping._PostnetCommon(stride, 0, 30, fp.ctypes.data_as(C.POINTER(C.c_int32)),
                                     fh.ctypes.data_as(C.POINTER(C.c_int32)), 0, grouping.F32)

    def call(**edit):
        for fn in edit.values():
            fn(arr, rots, common)
        rc = g._lib.spg_postnet_ragged_items(g._h, C.byref(common), arr, rots if rot else None, n, n_items,
                                             grouping.F64 if paf_dtype is None else paf_dtype, g._stream_ptr(None))
        return rc, g._lib.spg_last_error(g._h).decode()
    return call, keep


def test_bad_input_names_the_image_and_launches_nothing(env):
    t, grouping, g = env.torch, env.grouping, env.g
    imgs = _images(env, SIZES[:4], [1.0, 0.5], [0.0, 30.0], t.float32, seed=1)
    before = g.launch_count
    ok, keep = _raw_call(env, imgs, 4)
    cases = [
        (dict(e=lambda a, r, c: setattr(a[9], "height", a[9].height + 1)), "image 2 item 1"),
        (dict(e=lambda a, r, c: setattr(a[10], "width", a[10].width - 1)), "image 2 item 2"),
        (dict(e=lambda a, r, c: setattr(a[7], "heat_out", a[7].heat_out + 64)), "image 1 item 3"),
        (dict(e=lambda a, r, c: setattr(a[13], "paf_out", a[13].paf_out + 64)), "image 3 item 1"),
        (dict(e=lambda a, r, c: setattr(r[5], "apply", 0)), "image 1 item 1: rotated in some images"),
        (dict(e=lambda a, r, c: setattr(c, "stride", 8)), "stride 4"),
    ]
    for edit, msg in cases:
        call, _ = _raw_call(env, imgs, 4)
        rc, err = call(**edit)
        assert rc == -1 and msg in err, (msg, err)
    call, _ = _raw_call(env, imgs, 4, paf_dtype=grouping.F32)
    rc, err = call()
    assert rc == -1 and "float32" in err
    call, _ = _raw_call(env, imgs, 4)
    rc, err = call(e=lambda a, r, c: [setattr(a[k], "heat_out", a[k].heat_out + 4) for k in range(8, 12)])
    assert rc == -1 and "image 2: heat_out/paf_out must be 16-byte aligned" in err
    call, _ = _raw_call(env, imgs, 4, n=129)
    rc, err = call()
    assert rc == -1 and "max_batch" in err
    # through the binding: a different number of items per image
    with pytest.raises(grouping.GroupingError, match="same number of items"):
        g.postnet_ragged_items([imgs[0], (imgs[1][0][:3], imgs[1][1])])
    assert g.launch_count == before
    rc, err = ok()  # the unedited call is valid and launches
    assert rc == 0 and g.launch_count > before
    t.cuda.synchronize()


def test_empty_call_launches_nothing(env):
    before = env.g.launch_count
    assert env.g.postnet_ragged_items([]) == []
    assert env.g.launch_count == before
