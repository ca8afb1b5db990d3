"""GPU: the pre-network stage (spg_prenet, prenet.cuh -- evaluate.py:94-121) against its CPU checker oracle/prenet_port.py,
which tests/test_prenet_port.py pins to cv2's generic resize path and to cv2.warpAffine.

The resize is OpenCV's generic integer / float32 algorithm and the warp its fixed-point one, so the bar is BIT-IDENTICAL
pairs."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD  # a NaN no kernel writes


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import grouping, skeleton, synth
    from oracle import postnet_port as pp
    from oracle import postnet_rotation_port as pr
    from oracle import prenet_port as pn
    from oracle import spg_oracle as so

    class Env:
        pass

    e = Env()
    e.torch, e.grouping, e.skeleton, e.synth, e.pp, e.pr, e.pn, e.so, e.dev = torch, grouping, skeleton, synth, pp, pr, pn, so, cuda_device
    return e


def _images(n, h, w, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    img[:, : h // 3] = (np.indices((h // 3, w)).sum(0) % 2 * 255).astype(np.uint8)[None, :, :, None]  # saturating band
    return img


def _check_items(env, imgs, items, scales, angles, md, pv):
    import itertools
    assert len(items) == len(scales) * len(angles)
    for (pair, crop, rev), (scale, angle) in zip(items, itertools.product(scales, angles)):
        got = pair.cpu().numpy()
        for i in range(imgs.shape[0]):
            ref, ref_crop, _, ref_rev = env.pn.prenet_item(imgs[i], scale, angle, md, pv)
            assert got[i].shape == ref.shape, (scale, angle)
            assert np.array_equal(got[i].view(np.uint32), ref.view(np.uint32)), \
                (scale, angle, i, int((got[i] != ref).sum()))
            assert tuple(crop) == tuple(ref_crop)
            assert (rev is None) == (ref_rev is None) and (rev is None or np.array_equal(rev, ref_rev))


GEOMS = [((120, 160), [4 / 3, 1.499]), ((75, 100), [3.41, 0.61]), ((37, 53), [1.0, 0.37]),
         ((1, 1), [3.0]), ((2, 3), [2.5]), ((90, 200), [1.0]), ((40, 1400), [3.0])]


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("geom", GEOMS, ids=[f"{h}x{w}" for (h, w), _ in GEOMS])
def test_kernel_is_the_port_bit_for_bit(env, n, geom):
    (h, w), scales = geom
    t = env.torch
    imgs = _images(n, h, w, 10 * n + h)
    angles = [0, 30, -30, 0.5] if h * w > 6 else [0, 90, 180]
    g = env.grouping.Grouper(max_batch=1, max_h=64, max_w=64)
    try:
        items = g.prenet(t.from_numpy(imgs).to(env.dev), scales, angles, max_downsample=8, pad_value=128)
        assert g.prenet_kernel.startswith("prenet_kernel")
        _check_items(env, imgs, items, scales, angles, 8, 128)
    finally:
        g.close()


def test_unbatched_and_strided_source(env):
    """A [H, W, 3] view inside a larger frame (rows and images further apart than their bytes) and the 3-D form."""
    t = env.torch
    big = _images(2, 150, 260, 4)
    view = t.from_numpy(big).to(env.dev)[:, 7:7 + 121, 11:11 + 163, :]
    assert view.stride(1) != 163 * 3
    imgs = np.ascontiguousarray(big[:, 7:7 + 121, 11:11 + 163, :])
    g = env.grouping.Grouper(max_batch=1, max_h=64, max_w=64)
    try:
        items = g.prenet(view, [1.37, 0.8], [0, 30], max_downsample=64, pad_value=100)
        _check_items(env, imgs, items, [1.37, 0.8], [0, 30], 64, 100)
        one = g.prenet(view[1], [1.37], [0, -30], max_downsample=64, pad_value=100)
        assert one[0][0].dim() == 4
        _check_items(env, imgs[1:], [(p[None], c, r) for p, c, r in one], [1.37], [0, -30], 64, 100)
    finally:
        g.close()


def test_outputs_stay_inside_their_slots(env):
    """Each image's pair in a slot of a larger buffer: the gaps between the slots and the guard bands keep the sentinel."""
    t = env.torch
    imgs = _images(3, 57, 83, 9)
    g = env.grouping.Grouper(max_batch=1, max_h=64, max_w=64)
    try:
        outs, views = [], []
        for scale in (1.37, 0.9):
            H1, W1 = env.pn.resized_size(57, 83, scale)
            Hp, Wp = -(-H1 // 16) * 16, -(-W1 // 16) * 16
            for _ in range(2):  # two angles
                pair, slot, guard = 2 * Hp * Wp * 3, 2 * Hp * Wp * 3 + 1000, 4096
                buf = t.full((2 * guard + 3 * slot,), SENTINEL, dtype=t.int32, device=env.dev).view(t.float32)
                views.append(buf[guard:guard + 3 * slot].view(3, slot)[:, :pair].view(3, 2, Hp, Wp, 3))
                outs.append((buf, pair, slot, guard))
        items = g.prenet(t.from_numpy(imgs).to(env.dev), [1.37, 0.9], [0, 30], max_downsample=16, pad_value=7, out=views)
        _check_items(env, imgs, items, [1.37, 0.9], [0, 30], 16, 7)
        for buf, pair, slot, guard in outs:
            b = buf.view(t.int32).cpu().numpy()
            assert (b[:guard] == SENTINEL).all() and (b[guard + 3 * slot:] == SENTINEL).all()
            for i in range(3):
                assert (b[guard + i * slot + pair:guard + (i + 1) * slot] == SENTINEL).all()
                assert not (b[guard + i * slot:guard + i * slot + pair] == SENTINEL).any()
    finally:
        g.close()


def test_invalid_inputs_are_rejected(env):
    t, grouping = env.torch, env.grouping
    imgs = _images(1, 20, 30, 2)
    src = t.from_numpy(imgs).to(env.dev)
    out = t.empty((1, 2, 64, 64, 3), dtype=t.float32, device=env.dev)
    M = env.pr.rotation_matrices((24, 32), 30)[0].reshape(6).tolist()
    g = grouping.Grouper(max_batch=1, max_h=64, max_w=64)

    def run(scale=1.0, rotate=0, reserved=0, matrix=M, out_ptr=None, pad_value=128, md=8):
        it = (grouping._PrenetItem * 1)(grouping._PrenetItem(scale, rotate, reserved, (C.c_double * 6)(*matrix),
                                                            out.data_ptr() if out_ptr is None else out_ptr, 0))
        rc = g._lib.spg_prenet(g._h, C.c_void_p(src.data_ptr()), C.c_int64(src.stride(0)), C.c_int64(src.stride(1)), 1, 20,
                               30, md, pad_value, it, 1, None)
        return rc, (g._lib.spg_last_error(g._h) or b"").decode()

    try:
        cases = [(dict(scale=float("nan")), "finite and positive"), (dict(scale=0.0), "finite and positive"),
                 (dict(scale=-1.0), "finite and positive"), (dict(scale=float("inf")), "finite and positive"),
                 (dict(scale=0.01), "resized image is empty"), (dict(scale=2000.0), "above 32767"),
                 (dict(pad_value=256), "pad_value"), (dict(pad_value=-1), "pad_value"),
                 (dict(rotate=2), "rotate must be 0 or 1"), (dict(reserved=1), "reserved 0"),
                 (dict(rotate=1, matrix=M[:5] + [float("inf")]), "not finite"), (dict(out_ptr=0), "out is NULL"),
                 (dict(md=0), "max_downsample")]
        for kw, msg in cases:
            rc, err = run(**kw)
            assert rc == -1 and msg in err, (kw, rc, err)
        with pytest.raises(grouping.GroupingError, match=r"\(-1\).*pad_value"):
            g.prenet(src, [1.0], [0], max_downsample=8, pad_value=300)
        with pytest.raises(grouping.GroupingError, match=r"\(-1\).*empty"):
            g.prenet(src, [0.001], [0], max_downsample=8, pad_value=128)
        items = g.prenet(src, [1.2], [0, 30], max_downsample=8, pad_value=128)  # the handle still works
        _check_items(env, imgs, items, [1.2], [0, 30], 8, 128)
    finally:
        g.close()


def test_device_input_predict_with_scale_and_rotation_search(env):
    """dropin.predict(input_stage="device") over 2 scales x 3 angles: the network receives the port's pairs, and the maps
    and the grouping are the checker pipeline's on whatever the network answered per item."""
    from parity import diff_structures
    from test_gpu_postnet import _network_like_output

    from improved_body_parts_b200 import dropin
    t, sk = env.torch, env.skeleton
    rng = np.random.default_rng(5)
    image = rng.integers(0, 255, size=(150, 210, 3), dtype=np.uint8)
    params = dict(sk.default_params(), scale_search=[1.0, 0.75], rotation_search=[0.0, 30.0, -30.0])
    model_params = dict(boxsize=160, stride=4, max_downsample=64, padValue=128)
    for source in ("host", "cuda"):
        seen, answers = [], []

        def model(x):
            seen.append(x.cpu().numpy())
            h, w = x.shape[1] // 4, x.shape[2] // 4
            answers.append(_network_like_output(env, 1000 + len(answers), 1, h, w, 5)[0])
            return [[t.from_numpy(answers[-1]).to(x.device)]]

        dropin.configure(limbs=sk.LIMBS)
        img = image if source == "host" else t.from_numpy(image).to(env.dev)
        heatmap, paf = dropin.predict(img, params, model, model_params, 20, 30, "synthetic", input_stage="device")
        assert len(seen) == 6
        heat_avg, paf_avg = np.zeros((150, 210, 18)), np.zeros((150, 210, 30))
        items = [(x * 160 / 150, a) for x in params["scale_search"] for a in params["rotation_search"]]
        for x, out, (scale, angle) in zip(seen, answers, items):
            pair, crop, pad, M = env.pn.prenet_item(image, scale, angle, 64, 128)
            assert np.array_equal(x.view(np.uint32), pair.view(np.uint32))
            hm, pf = env.pr.post_network_item(out, 4, pair.shape[1:3], pad, image.shape[:2], 30, 48, sk.FLIP_PAF_ORD,
                                              sk.FLIP_HEAT_ORD[:18], rotate_matrix=M)
            heat_avg, paf_avg = env.pp.accumulate(heat_avg, hm, 6), env.pp.accumulate(paf_avg, pf, 6)
        assert np.array_equal(heatmap.numpy(), heat_avg.astype(np.float32).astype(np.float64))
        assert np.array_equal(paf.numpy(), paf_avg)
        all_peaks = dropin.find_peaks(heatmap, params)
        connection_all, special_k = dropin.find_connections(all_peaks, paf, image.shape[0], params)
        subset, candidate = dropin.find_people(connection_all, special_k, all_peaks, params)
        o = env.so.group_batch(np.ascontiguousarray(heat_avg.transpose(2, 0, 1)[None]).astype(np.float32),
                               np.ascontiguousarray(paf_avg.transpose(2, 0, 1)[None]), sk.LIMBS, image.shape[0], params)
        d = diff_structures(o.as_reference_structures(0), (all_peaks, connection_all, special_k, subset, candidate),
                            float_tol=0.0)
        assert not d, "\n".join(d)


def test_configure_and_install_pass_the_input_stage(env):
    import types

    from improved_body_parts_b200 import dropin
    try:
        dropin.configure(input_stage="device")
        assert dropin._input_stage == "device"
        with pytest.raises(ValueError):
            dropin.configure(input_stage="gpu")
        mod = types.SimpleNamespace(limbSeq=env.skeleton.LIMBS)
        dropin.install(mod, device_predict=True)
        assert dropin._input_stage == "host"
        dropin.install(mod, device_predict=True, device_input=True)
        assert dropin._input_stage == "device"
    finally:
        dropin.configure(input_stage="host")
