"""GPU: the ragged pre-network stage (spg_prenet_ragged, prenet.cuh) -- members of different source sizes, scales and
angles in one call -- against oracle/prenet_port.py and against spg_prenet of each image alone, and the device input
stage of dropin.predict_batch that runs on it.

The bar is the one of tests/test_gpu_prenet.py: BIT-IDENTICAL pairs."""
import math
import types

import numpy as np
import pytest

from test_gpu_predict_batch import SEARCHES, SHAPES, MODEL_PARAMS, StandIn, _assert_maps_equal
from test_gpu_predict_batch import _images as _batch_images
from test_gpu_prenet import GEOMS, SENTINEL, _images

pytestmark = pytest.mark.gpu

#: members per launch: the descriptors that fit in the kernel-parameter space (PreMember is 136 bytes)
MEMBERS_PER_LAUNCH = 240


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import grouping
    from oracle import prenet_port as pn

    g = grouping.Grouper(max_batch=1, max_h=64, max_w=64)
    yield types.SimpleNamespace(torch=torch, grouping=grouping, pn=pn, dev=cuda_device, g=g)
    g.close()


def _check(env, members, results, md, pv, alone=True):
    """Each member's pair, crop and reverse matrix against the port, and (``alone``) against ``prenet`` of its image
    alone."""
    assert len(results) == len(members)
    for k, ((img, host, scale, angle), (pair, crop, rev)) in enumerate(zip(members, results)):
        ref, ref_crop, _, ref_rev = env.pn.prenet_item(host, env.pn.clamp_scale(scale, host.shape[:2]), angle, md, pv)
        got = pair.cpu().numpy()
        assert got.shape == ref.shape, (k, scale, angle)
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (k, scale, angle, int((got != ref).sum()))
        assert tuple(crop) == tuple(ref_crop)
        assert (rev is None) == (ref_rev is None) and (rev is None or np.array_equal(rev, ref_rev))
        if alone:
            (p1, c1, r1), = env.g.prenet(img, [scale], [angle], max_downsample=md, pad_value=pv)
            assert np.array_equal(p1.cpu().numpy().view(np.uint32), got.view(np.uint32)) and tuple(c1) == tuple(crop)
            assert (r1 is None) == (rev is None) and (rev is None or np.array_equal(r1, rev))


def _launches(env):
    return int(env.g._lib.spg_launch_count(env.g._h))


def test_mixed_sources_in_one_call(env):
    """Every geometry of tests/test_gpu_prenet.py (1x1, 2x3, 40x1400, the copy case H1 == h, W1 * 3 not a multiple of
    8, ...) in one call, rotated and unrotated members shuffled, several members per source."""
    t = env.torch
    members = []
    for gi, ((h, w), scales) in enumerate(GEOMS):
        host = _images(1, h, w, 100 + gi)[0]
        img = t.from_numpy(host).to(env.dev)
        angles = [0, 30, -30, 0.5] if h * w > 6 else [0, 90, 180]
        members += [(img, host, s, a) for s in scales for a in angles]
    order = np.random.default_rng(3).permutation(len(members))
    members = [members[k] for k in order]
    before = _launches(env)
    results = env.g.prenet_ragged([(img, s, a) for img, _, s, a in members], max_downsample=8, pad_value=128)
    assert _launches(env) - before == 3  # one unrotated launch, the rotated members' resize and warp
    assert env.g.prenet_kernel.startswith("prenet_kernel")
    _check(env, members, results, 8, 128)


def test_more_members_than_one_launch_holds(env):
    """Hundreds of small members: unrotated and rotated ones each span several launches, and every pair is exact."""
    t = env.torch
    rng = np.random.default_rng(11)
    sources = []
    for s in range(40):
        host = _images(1, int(rng.integers(2, 24)), int(rng.integers(2, 40)), 200 + s)[0]  # 2 rows: not empty at 0.5
        sources.append((t.from_numpy(host).to(env.dev), host))
    members = []
    for k in range(3 * MEMBERS_PER_LAUNCH + 17):
        img, host = sources[int(rng.integers(len(sources)))]
        members.append((img, host, float(rng.choice([0.5, 1.0, 1.7, 2.3])), float(rng.choice([0, 30, -45]))))
    n_rot = sum(m[3] != 0 for m in members)
    assert n_rot > MEMBERS_PER_LAUNCH and len(members) - n_rot > MEMBERS_PER_LAUNCH
    before = _launches(env)
    results = env.g.prenet_ragged([(img, s, a) for img, _, s, a in members], max_downsample=8, pad_value=33)
    want = math.ceil((len(members) - n_rot) / MEMBERS_PER_LAUNCH) + 2 * math.ceil(n_rot / MEMBERS_PER_LAUNCH)
    assert _launches(env) - before == want
    _check(env, members, results, 8, 33, alone=False)


def test_strided_sources(env):
    """Views inside larger frames (rows further apart than their bytes), next to a contiguous image."""
    t = env.torch
    big = _images(2, 150, 260, 4)
    frames = t.from_numpy(big).to(env.dev)
    views = [(frames[0, 7:7 + 121, 11:11 + 163], big[0, 7:7 + 121, 11:11 + 163]),
             (frames[1, 30:30 + 45, 200:200 + 60], big[1, 30:30 + 45, 200:200 + 60]),
             (frames[1], big[1])]
    assert views[0][0].stride(0) != 163 * 3
    members = [(img, np.ascontiguousarray(host), s, a) for img, host in views for s in (1.37, 0.8) for a in (0, 30)]
    results = env.g.prenet_ragged([(img, s, a) for img, _, s, a in members], max_downsample=64, pad_value=100)
    _check(env, members, results, 64, 100)


def test_outputs_stay_inside_their_slots(env):
    """Every member writes into a slot of one shared buffer: the gaps between the slots and the guard bands keep the
    sentinel, and every pair is written whole."""
    t = env.torch
    members, slots = [], []
    for k, (h, w) in enumerate([(57, 83), (20, 31), (90, 45)]):
        host = _images(1, h, w, 30 + k)[0]
        img = t.from_numpy(host).to(env.dev)
        for s, a in ((1.37, 0), (0.9, 30), (1.0, 0), (1.0, -30)):
            H1, W1 = env.pn.resized_size(h, w, s)
            Hp, Wp = -(-H1 // 16) * 16, -(-W1 // 16) * 16
            members.append((img, host, s, a))
            slots.append((2 * Hp * Wp * 3, (2, Hp, Wp, 3)))
    guard, gap = 4096, 777
    total = 2 * guard + sum(n + gap for n, _ in slots)
    buf = t.full((total,), SENTINEL, dtype=t.int32, device=env.dev).view(t.float32)
    outs, at = [], guard
    for n, shape in slots:
        outs.append(buf[at:at + n].view(shape))
        at += n + gap
    results = env.g.prenet_ragged([(img, s, a) for img, _, s, a in members], max_downsample=16, pad_value=7, out=outs)
    _check(env, members, results, 16, 7, alone=False)
    b = buf.view(t.int32).cpu().numpy()
    assert (b[:guard] == SENTINEL).all() and (b[at:] == SENTINEL).all()
    at = guard
    for n, _ in slots:
        assert not (b[at:at + n] == SENTINEL).any()
        assert (b[at + n:at + n + gap] == SENTINEL).all()
        at += n + gap


def test_invalid_members_are_rejected_before_any_launch(env):
    """Each rule of spg_prenet per member: -1 and "member <index>" in the error, the outputs untouched (nothing was
    launched, not even for the valid members before the bad one), and the handle still works."""
    t, grouping = env.torch, env.grouping
    host = _images(1, 20, 30, 2)[0]
    src = t.from_numpy(host).to(env.dev)
    out = t.full((3, 2, 64, 64, 3), SENTINEL, dtype=t.int32, device=env.dev)
    M = [0.866, 0.5, -3.0, -0.5, 0.866, 12.0]

    def run(bad=None, pad_value=128, md=8, bad_index=2):
        arr = np.zeros(3, grouping.PRENET_MEMBER)
        for k in range(3):
            arr[k] = (src.data_ptr(), src.stride(0), 20, 30, 1.0, k % 2, 0, M, out[k].data_ptr())
        for f, v in (bad or {}).items():
            arr[bad_index][f] = v
        rc = env.g._lib.spg_prenet_ragged(env.g._h, md, pad_value, arr.ctypes.data, 3, None)
        return rc, (env.g._lib.spg_last_error(env.g._h) or b"").decode()

    cases = [(dict(scale=float("nan")), "finite and positive"), (dict(scale=0.0), "finite and positive"),
             (dict(scale=-1.0), "finite and positive"), (dict(scale=float("inf")), "finite and positive"),
             (dict(scale=0.01), "resized image is empty"), (dict(scale=2000.0), "above 32767"),
             (dict(rotate=2), "rotate must be 0 or 1"), (dict(reserved=1), "reserved 0"),
             (dict(matrix=M[:5] + [float("inf")]), "not finite"), (dict(out=0), "out is NULL"),
             (dict(image=0), "image is NULL"), (dict(row_stride=89), "row_stride"), (dict(height=0), "outside [1, 32767]"),
             (dict(width=40000), "outside [1, 32767]")]
    for bad_index in (0, 2):
        for kw, msg in cases:
            rc, err = run(kw, bad_index=bad_index)
            assert rc == -1 and f"member {bad_index}:" in err and msg in err, (kw, rc, err)
    for kw, msg in ((dict(pad_value=256), "pad_value"), (dict(pad_value=-1), "pad_value"), (dict(md=0), "max_downsample")):
        rc, err = run(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)
    t.cuda.synchronize(env.dev)
    assert (out.cpu().numpy() == SENTINEL).all()
    with pytest.raises(grouping.GroupingError, match=r"\(-1\).*member 1: .*empty"):
        env.g.prenet_ragged([(src, 1.0, 0), (src, 0.001, 0)], max_downsample=8, pad_value=128)
    with pytest.raises(grouping.GroupingError, match="member 0"):
        env.g.prenet_ragged([(src.float(), 1.0, 0)], max_downsample=8, pad_value=128)
    rc, err = run()
    assert rc == 0, err
    members = [(src, host, 1.2, 0), (src, host, 1.2, 30)]
    _check(env, members, env.g.prenet_ragged([(src, 1.2, 0), (src, 1.2, 30)], max_downsample=8, pad_value=128), 8, 128)


@pytest.fixture()
def dropin_env(cuda_device):
    import torch
    from improved_body_parts_b200 import dropin, grouping, skeleton, synth

    dropin.configure(device=0, limbs=dropin.LIMBS)
    yield types.SimpleNamespace(torch=torch, dropin=dropin, grouping=grouping, skeleton=skeleton, synth=synth,
                                dev=cuda_device)
    dropin.configure(input_stage="host", variant="evaluate")


@pytest.mark.parametrize("search", ["1 item", "3 angles", "2 scales x 2 angles"])
def test_predict_batch_builds_each_bucket_with_one_ragged_call(dropin_env, monkeypatch, search):
    """Host images and uint8 CUDA tensors in one batch: the maps equal ``predict``'s per image, each input size is
    built with one ``prenet_ragged`` call, and ``prenet`` is not called."""
    e = dropin_env
    d, t, Grouper = e.dropin, e.torch, e.grouping.Grouper
    scales, angles = SEARCHES[search]
    params = dict(e.skeleton.default_params(), scale_search=scales, rotation_search=angles)
    imgs = _batch_images(6, SHAPES[:7])
    batch = [t.from_numpy(im).to(e.dev) if k % 2 else im for k, im in enumerate(imgs)]
    model = StandIn(t, e.synth)
    want = [d.predict(img, params, model, MODEL_PARAMS, input_stage="device") for img in imgs]
    calls = {"prenet": 0, "prenet_ragged": 0}
    for name in calls:
        def counted(self, *a, _f=getattr(Grouper, name), _n=name, **k):
            calls[_n] += 1
            return _f(self, *a, **k)
        monkeypatch.setattr(Grouper, name, counted)
    got = d.predict_batch(batch, params, model, MODEL_PARAMS, forward_batch=4, input_stage="device")
    _assert_maps_equal(got, want)
    _, buckets = d.plan_items([im.shape[:2] for im in imgs], params, MODEL_PARAMS)
    assert calls == {"prenet": 0, "prenet_ragged": len(buckets)}
    assert len(buckets) >= 2
