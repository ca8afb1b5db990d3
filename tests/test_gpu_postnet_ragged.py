"""GPU: the ragged post-network stage (``spg_postnet_ragged`` / ``Grouper.postnet_ragged``).

Images of different sizes, identity items (crop == image) and items whose second resize up- or down-samples, share one
call; each image's maps must equal, bit for bit (NaN-aware), what ``Grouper.postnet`` gives for that image alone."""
import ctypes as C
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD  # a NaN payload no kernel writes


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import grouping, synth

    e = types.SimpleNamespace(torch=torch, grouping=grouping, synth=synth, dev=cuda_device)
    e.g = grouping.Grouper(max_batch=160, max_h=1024, max_w=1024)
    e.single = grouping.Grouper(max_batch=1, max_h=1024, max_w=1024)
    yield e
    e.g.close()
    e.single.close()


def _geometry(H, W, scale, md=16):
    """(crop, network output size) of predict()'s one item for an H x W image at `scale`."""
    H1, W1 = int(np.rint(H * scale)), int(np.rint(W * scale))
    return (H1, W1), (-(-H1 // md) * md // 4, -(-W1 // md) * md // 4)


# (H, W, scale): scale 1 gives an identity item; < 1 up-samples in the second resize, > 1 down-samples.  Widths that are
# not multiples of 4 and sizes that leave partial border tiles on purpose.
MIXED = [(160, 213, 1.0), (97, 131, 1.0), (128, 128, 1.0), (75, 301, 0.7), (203, 150, 1.6), (61, 47, 2.3), (130, 90, 0.45),
         (64, 257, 1.0), (33, 35, 1.0), (250, 190, 0.9), (40, 66, 1.3), (2, 9, 3.0)]


def _net(env, seed, h, w, dtype, nan=False):
    out = env.synth.make_network_output(seed, h, w, 2)
    if nan:
        rng = np.random.default_rng(seed)
        out[rng.random(out.shape) < 0.002] = np.nan
    return env.torch.from_numpy(out).to(env.dev, dtype)


def _images(env, spec, dtype, nan=False, seed=0):
    imgs = []
    for i, (H, W, s) in enumerate(spec):
        crop, (h, w) = _geometry(H, W, s)
        imgs.append((_net(env, seed + 31 * i, h, w, dtype, nan), crop, (H, W)))
    return imgs


def _same(a, b, what):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=True), what


def _check_against_single(env, imgs, got, paf_dtype, nan_scrub):
    for i, (net, crop, hw) in enumerate(imgs):
        heat, paf = env.single.postnet([net[None]], [crop], hw, paf_dtype=paf_dtype, nan_scrub=nan_scrub)
        _same(got[i][0], heat, f"image {i} {hw} crop {crop}: heat")
        _same(got[i][1], paf, f"image {i} {hw} crop {crop}: paf")


@pytest.mark.parametrize("net_dtype", ["float32", "float16"])
@pytest.mark.parametrize("paf_dtype", ["float32", "float64"])
@pytest.mark.parametrize("nan_scrub", [False, True])
def test_ragged_equals_per_image_postnet(env, net_dtype, paf_dtype, nan_scrub):
    t = env.torch
    imgs = _images(env, MIXED, getattr(t, net_dtype), nan=nan_scrub, seed=7)
    got = env.g.postnet_ragged(imgs, paf_dtype=getattr(t, paf_dtype), nan_scrub=nan_scrub)
    assert env.g.postnet_kernel() == "postnet_ragged_kernel"
    if nan_scrub:
        assert not any(bool(t.isnan(h).any()) or bool(t.isnan(p).any()) for h, p in got)
    _check_against_single(env, imgs, got, getattr(t, paf_dtype), nan_scrub)


def test_nan_passes_through_without_scrub(env):
    t = env.torch
    imgs = _images(env, MIXED[:4], t.float32, nan=True, seed=11)
    got = env.g.postnet_ragged(imgs)
    assert any(bool(t.isnan(h).any()) for h, _ in got)
    _check_against_single(env, imgs, got, t.float32, False)


def test_pairs_read_in_place_from_a_shared_batch_output(env):
    """k images with one network input size: their pairs are slices of one [2k, 50, h, w] tensor, and that tensor is a
    channel-offset view of a larger one (strides other than the dense ones)."""
    t = env.torch
    spec = [(120, 160, 4 / 3), (60, 80, 8 / 3), (90, 120, 16 / 9), (150, 200, 16 / 15), (160, 213, 1.0)]
    crops = [_geometry(H, W, s)[0] for H, W, s in spec]
    sizes = {_geometry(H, W, s)[1] for H, W, s in spec}
    assert len(sizes) == 1
    h, w = sizes.pop()
    k = len(spec)
    big = t.zeros((2 * k, 53, h, w), dtype=t.float32, device=env.dev)
    for j in range(k):
        big[2 * j:2 * j + 2, 2:52] = _net(env, 400 + j, h, w, t.float32)
    batch = big[:, 2:52]
    imgs = [(batch[2 * j:2 * j + 2], crops[j], spec[j][:2]) for j in range(k)]
    got = env.g.postnet_ragged(imgs)
    _check_against_single(env, [(batch[2 * j:2 * j + 2].contiguous(), crops[j], spec[j][:2]) for j in range(k)], got,
                          t.float32, False)


POST_TABLE_IMAGES = 82  # kPostTableImages in csrc/postnet.cuh: image descriptors per launch


@pytest.mark.parametrize("identity", [True, False])
def test_more_images_than_one_table_holds(env, identity):
    t = env.torch
    rng = np.random.default_rng(5 if identity else 6)
    n = 2 * POST_TABLE_IMAGES + 22
    spec = [(int(rng.integers(8, 70)), int(rng.integers(8, 90)), 1.0 if identity else float(rng.choice([0.6, 1.4])))
            for _ in range(n)]
    imgs = _images(env, spec, t.float16, seed=900)
    with env.grouping.Grouper(max_batch=n, max_h=1024, max_w=1024) as g:
        before = g.launch_count
        got = g.postnet_ragged(imgs)
        assert g.launch_count - before == 3  # two full tables and 22 images
        assert g.postnet_kernel() == ("postnet_x4_ident_ragged_kernel" if identity else "postnet_ragged_kernel")
        _check_against_single(env, imgs, got, t.float32, False)


def test_outputs_stay_inside_their_planes(env):
    """Every image's planes are slices of one sentinel-filled buffer with gaps: the gaps keep the sentinel, the planes
    are written everywhere and equal the per-image maps."""
    t = env.torch
    imgs = _images(env, MIXED, t.float32, seed=3)
    guard, gap = 4096, 772  # plane bases 16-byte aligned, as the call requires
    sizes = []
    for _, _, (H, W) in imgs:
        sizes += [18 * H * W, 30 * H * W]
    buf = t.full((2 * guard + sum(sizes) + (gap + 4) * len(sizes),), SENTINEL, dtype=t.int32, device=env.dev)
    f = buf.view(t.float32)
    outs, spans, pos = [], [], guard
    for _, _, (H, W) in imgs:
        pair = []
        for ch in (18, 30):
            pair.append(f[pos:pos + ch * H * W].view(1, ch, H, W))
            spans.append((pos, pos + ch * H * W))
            pos = -(-(pos + ch * H * W) // 4) * 4 + gap
        outs.append(tuple(pair))
    got = env.g.postnet_ragged(imgs, outs=outs)
    assert all(a is o[0] and b is o[1] for (a, b), o in zip(got, outs))
    b = buf.cpu().numpy()
    mask = np.ones(b.shape, bool)
    for lo, hi in spans:
        mask[lo:hi] = False
        assert not (b[lo:hi] == SENTINEL).any()
    assert (b[mask] == SENTINEL).all()
    _check_against_single(env, imgs, got, t.float32, False)


def test_bad_input_names_the_image_and_launches_nothing(env):
    t, grouping = env.torch, env.grouping
    g = env.g
    imgs = _images(env, MIXED[:4], t.float32, seed=1)
    before = g.launch_count
    net, crop, hw = imgs[1]
    with pytest.raises(grouping.GroupingError, match="image 2"):  # crop larger than the up-sampled output
        g.postnet_ragged(imgs[:2] + [(net, (4 * net.shape[2] + 1, crop[1]), hw)] + imgs[2:])
    with pytest.raises(grouping.GroupingError, match="image 1"):  # a one-row image
        g.postnet_ragged([imgs[0], (net, crop, (1, 40)), imgs[2]])
    with pytest.raises(grouping.GroupingError, match="stride 4"):
        g.postnet_ragged(imgs, stride=8)
    with pytest.raises(grouping.GroupingError, match="image 3"):  # mixed network output dtypes
        g.postnet_ragged(imgs[:3] + [(imgs[3][0].half(), imgs[3][1], imgs[3][2])])
    outs = [(t.empty((1, 18) + tuple(hw), device=env.dev), t.empty((1, 30) + tuple(hw), device=env.dev)) for _, _, hw in imgs]
    H, W = imgs[2][2]
    outs[2] = (t.empty((18 * H * W + 1,), device=env.dev)[1:].view(1, 18, H, W), outs[2][1])  # 4 bytes past an aligned base
    with pytest.raises(grouping.GroupingError, match="image 2: heat_out/paf_out must be 16-byte aligned"):
        g.postnet_ragged(imgs, outs=outs)
    # straight through the C ABI: a NULL heat_out, and n > max_batch
    arr = (grouping._PostnetImage * 161)()
    keep = []
    for i in range(161):
        o, (ch, cw), (H, W) = imgs[i % 4]
        heat = t.empty((18, H, W), device=env.dev)
        paf = t.empty((30, H, W), device=env.dev)
        keep += [heat, paf]
        arr[i] = grouping._PostnetImage(o.data_ptr(), o.stride(0), o.stride(1), o.shape[2], o.shape[3], ch, cw, H, W,
                                        heat.data_ptr(), paf.data_ptr())
    arr[1].heat_out = None
    fp, fh = g._flip_orders(None, None)
    common = grouping._PostnetCommon(4, 0, 30, fp.ctypes.data_as(C.POINTER(C.c_int32)),
                                     fh.ctypes.data_as(C.POINTER(C.c_int32)), 0, grouping.F32)
    rc = g._lib.spg_postnet_ragged(g._h, C.byref(common), arr, 4, grouping.F32, g._stream_ptr(None))
    assert rc == -1 and b"image 1" in g._lib.spg_last_error(g._h)
    arr[1].heat_out = keep[2].data_ptr()
    rc = g._lib.spg_postnet_ragged(g._h, C.byref(common), arr, 161, grouping.F32, g._stream_ptr(None))
    assert rc == -1 and b"max_batch" in g._lib.spg_last_error(g._h)
    common.stride = 2
    rc = g._lib.spg_postnet_ragged(g._h, C.byref(common), arr, 4, grouping.F32, g._stream_ptr(None))
    assert rc == -1 and b"stride 4" in g._lib.spg_last_error(g._h)
    assert g.launch_count == before
    # no images: nothing to launch, and not an error
    assert g.postnet_ragged([]) == [] and g.launch_count == before
