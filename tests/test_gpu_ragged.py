"""GPU: the ragged grouping call (``spg_group_ragged`` / ``Grouper.group_ragged``) and the batched drop-in functions.

Images of different sizes, extents and channel layouts share one call; every image's results must equal, bit for bit,
what ``spg_group_batch`` returns for that image alone on a handle with the same capacities (the candidate arrays aside:
they are appended atomically and unordered)."""
import ctypes as C
import json
import os
import types

import numpy as np
import pytest

from conftest import golden_paths
from golden_io import load_case
from parity import diff_structures

pytestmark = pytest.mark.gpu

CAPS = dict(max_peaks_per_part=64, max_cands_per_limb=1024, max_person_rows=96)


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import grouping, skeleton, synth, wire

    e = types.SimpleNamespace(torch=torch, grouping=grouping, skeleton=skeleton, synth=synth, wire=wire, dev=cuda_device)
    e.ragged = grouping.Grouper(max_batch=64, max_h=1024, max_w=1024, **CAPS)
    e.single = grouping.Grouper(max_batch=1, max_h=1024, max_w=1024, **CAPS)
    yield e
    e.ragged.close()
    e.single.close()


def _maps(env, heat, paf, paf_dtype, sliced):
    """Device maps of one image: channel slices of a [1, 50, H, W] network-like tensor, or separate tensors."""
    t = env.torch
    K, H, W = heat.shape
    pd = t.float64 if paf_dtype == env.grouping.F64 else t.float32
    if sliced:
        net = t.zeros((1, 50, H, W), dtype=t.float32, device=env.dev)
        net[0, 30:48] = t.from_numpy(heat)
        h = net[:, 30:48]
        if pd == t.float32:
            net[0, :30] = t.from_numpy(paf)
            return h, net[:, :30]
        buf = t.zeros((1, 33, H, W), dtype=pd, device=env.dev)
        buf[0, 1:31] = t.from_numpy(paf.astype(np.float64))
        return h, buf[:, 1:31]
    return t.from_numpy(heat).to(env.dev)[None], t.from_numpy(paf).to(env.dev, pd)[None]


def _same(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=True), what


def _assert_image_equal(r, i, s, what):
    """Image i of a ragged result `r` against image 0 of a single call `s`: every contract array, valid entries only."""
    _same(r.status[i], s.status[0], f"{what}: status")
    _same(r.peak_count[i], s.peak_count[0], f"{what}: peak_count")
    capP = r.peak_x.shape[2]
    for c in range(r.K):
        m = min(int(s.peak_count[0, c]), capP)
        for name in ("peak_x", "peak_y", "peak_score", "peak_anchor"):
            _same(getattr(r, name)[i, c, :m], getattr(s, name)[0, c, :m], f"{what}: {name} part {c}")
    _same(r.cand_count[i], s.cand_count[0], f"{what}: cand_count")
    _same(r.conn_count[i], s.conn_count[0], f"{what}: conn_count")
    for k in range(r.L):
        m = max(int(s.conn_count[0, k]), 0)
        for name in ("conn_ij", "conn_score", "conn_norm"):
            _same(getattr(r, name)[i, k, :m], getattr(s, name)[0, k, :m], f"{what}: {name} limb {k}")
    _same(r.n_persons[i], s.n_persons[0], f"{what}: n_persons")
    P = int(s.n_persons[0])
    for name in ("subset", "people_xy", "people_score"):
        _same(getattr(r, name)[i, :P], getattr(s, name)[0, :P], f"{what}: {name}")


def _record(buf, i, rec_bytes, P, J=17):
    """Header and live rows of record i (the rest of a record is never written)."""
    return bytes(buf[i, :8 + P * (2 * J + 2) * 8])


# ---- the mixed set ------------------------------------------------------------------------------------------------
SHAPES = [(2, 2), (3, 5), (37, 53), (72, 56), (128, 128), (427, 640), (640, 427), (512, 512), (33, 1000), (61, 127),
          (96, 160), (128, 128), (45, 90), (200, 131), (128, 128), (16, 18)]


def _mixed_images(env):
    rng = np.random.default_rng(77)
    imgs = []
    for t in range(40):
        H, W = SHAPES[t % len(SHAPES)]
        if H < 16 or W < 16:
            heat = rng.random((18, H, W), dtype=np.float32)
            paf = rng.random((30, H, W), dtype=np.float32) * np.float32(0.3)
        else:
            persons = int(rng.integers(0, 31)) if H * W >= 128 * 128 else int(rng.integers(0, 6))
            heat, paf = env.synth.make_image(900 + t, H, W, persons)
        imgs.append((heat, paf, float(rng.choice([H, W, 0.5 * H, 1000.0]))))
    # one image with far more peaks than max_peaks_per_part: it overflows, its neighbours must not notice (no body-part
    # signal, so no candidate depends on which peaks the truncated lists kept)
    heat = rng.random((18, 128, 128), dtype=np.float32)
    paf = np.zeros((30, 128, 128), np.float32)
    imgs.insert(17, (heat, paf, 128.0))
    return imgs, 17


@pytest.fixture(scope="module")
def mixed(env):
    return _mixed_images(env)


def _params_variant(env, name):
    d = env.skeleton.default_params()
    if name == "demo":
        return env.skeleton.GroupParams.demo(d)
    if name == "mid65":
        return dict(d, mid_num=65)
    if name.startswith("r"):
        return dict(d, offset_radius=int(name[1:]))
    return d


@pytest.mark.parametrize("pname,dtype_name", [("default", "F32"), ("default", "F64"), ("default", "F32_AS_F64"),
                                              ("demo", "F32_AS_F64"), ("mid65", "F32"), ("r0", "F64"),
                                              ("r1", "F32_AS_F64"), ("r3", "F32"), ("r4", "F32_AS_F64")])
def test_ragged_equals_per_image_calls(env, mixed, pname, dtype_name):
    imgs, overflow = mixed
    t = env.torch
    dtype = getattr(env.grouping, dtype_name)
    params = _params_variant(env, pname)
    as_f64 = dtype == env.grouping.F32_AS_F64
    maps = [_maps(env, h, p, dtype, sliced=(i % 2 == 0)) for i, (h, p, _) in enumerate(imgs)]
    ext = [e for _, _, e in imgs]
    g, s = env.ragged, env.single
    rb = g.wire_record_bytes()
    wire_r = t.zeros((len(maps), rb), dtype=t.uint8, device=env.dev)
    wire_s = t.zeros((1, rb), dtype=t.uint8, device=env.dev)
    g.set_wire_output(wire_r.data_ptr())
    try:
        g.group_ragged(maps, ext, params, paf_as_f64=as_f64)
        r = g.fetch(len(maps))
    finally:
        g.set_wire_output(None)
    assert g.stage_kernels()[0] == "nms_peaks_ragged_kernel" and g.stage_kernels()[1].startswith("limb_score_ragged_kernel")
    rec_r = wire_r.cpu().numpy()
    s.set_wire_output(wire_s.data_ptr())
    try:
        for i, (h, p) in enumerate(maps):
            s.group_device(h, p, ext[i], params, paf_as_f64=as_f64)
            one = s.fetch(1)
            what = f"image {i} {tuple(h.shape[2:])} ({pname}, {dtype_name})"
            if i == overflow:
                assert one.status[0] & env.grouping.ST_PEAK_OVERFLOW
                _same(r.status[i], one.status[0], f"{what}: status")
                continue
            _assert_image_equal(r, i, one, what)
            P = int(one.n_persons[0])
            assert _record(rec_r, i, rb, P) == _record(wire_s.cpu().numpy(), 0, rb, P), f"{what}: wire record"
    finally:
        s.set_wire_output(None)
    assert sum(int(n) for n in r.n_persons) > 0


def test_goldens_in_ragged_calls(env):
    """Golden cases grouped by (limbs, params, paf dtype), each group one ragged call, padded with synthetic images of
    other sizes; every golden image equals its recorded reference structures bit for bit."""
    t = env.torch
    groups = {}
    for path in golden_paths():
        case = load_case(path)
        key = (json.dumps(case["limbs"]), json.dumps(case["params"], sort_keys=True, default=str), str(case["paf"].dtype))
        groups.setdefault(key, []).append((os.path.basename(path), case))
    pads = [env.synth.make_image(31 + j, H, W, 4) for j, (H, W) in enumerate([(61, 83), (150, 97), (48, 200)])]
    for cases in groups.values():
        limbs, params = cases[0][1]["limbs"], cases[0][1]["params"]
        f64 = cases[0][1]["paf"].dtype == np.float64
        maps, ext = [], []
        for _, c in cases:
            maps.append((t.from_numpy(c["heat"]).to(env.dev)[None], t.from_numpy(c["paf"]).to(env.dev)[None]))
            ext.append(float(c["image_extent"]))
        L = len(limbs)
        for heat, paf in pads[:max(0, 3 - len(cases))]:
            pf = np.resize(paf, (L,) + paf.shape[1:]).astype(np.float64 if f64 else np.float32)
            maps.append((t.from_numpy(heat).to(env.dev)[None], t.from_numpy(pf).to(env.dev)[None]))
            ext.append(float(heat.shape[1]))
        with env.grouping.Grouper(limbs, max_batch=len(maps), max_h=256, max_w=256, max_peaks_per_part=128,
                                  max_person_rows=128) as g:
            g.group_ragged(maps, ext, params)
            r = g.fetch(len(maps))
        for i, (name, c) in enumerate(cases):
            assert r.status[i] == 0, f"{name}: status {r.status[i]:#x}"
            d = diff_structures(c["structs"], r.as_reference_structures(i), float_tol=0.0)
            assert not d, f"{name}:\n" + "\n".join(d)


def _small_set(env, n=6, seed=5):
    shapes = [(72, 56), (128, 128), (61, 127), (200, 131), (96, 160), (45, 90), (128, 96), (33, 250)]
    out = []
    for i in range(n):
        H, W = shapes[i % len(shapes)]
        heat, paf = env.synth.make_image(seed + i, H, W, 3 + i % 5)
        out.append((env.torch.from_numpy(heat).to(env.dev)[None], env.torch.from_numpy(paf).to(env.dev)[None], float(H)))
    return out


def test_permuted_batch_gives_permuted_results_and_images_array_is_reusable(env):
    g = env.ragged
    imgs = _small_set(env, 8)
    g.group_ragged([(h, p) for h, p, _ in imgs], [e for _, _, e in imgs])
    base = g.fetch(len(imgs))
    perm = [5, 2, 7, 0, 3, 6, 1, 4]
    g.group_ragged([imgs[j][:2] for j in perm], [imgs[j][2] for j in perm])
    r = g.fetch(len(imgs))
    for i, j in enumerate(perm):
        _assert_image_equal(r, i, types.SimpleNamespace(**{k: getattr(base, k)[j:j + 1] for k in (
            "status", "peak_count", "peak_x", "peak_y", "peak_score", "peak_anchor", "cand_count", "conn_count",
            "conn_ij", "conn_score", "conn_norm", "n_persons", "subset", "people_xy", "people_score")}), f"slot {i}")
    # the descriptors are consumed by the call: overwriting the array right after it changes nothing
    grouping = env.grouping
    arr = (grouping._ImageMaps * len(imgs))()
    for i, (h, p, e) in enumerate(imgs):
        arr[i] = grouping._ImageMaps(h.data_ptr(), p.data_ptr(), h.stride(1), p.stride(1), h.shape[2], h.shape[3], e)
    prm = grouping.params_struct(None)
    rc = g._lib.spg_group_ragged(g._h, arr, len(imgs), grouping.F32, C.byref(prm), g._stream_ptr(None))
    assert rc == 0
    C.memset(arr, 0, C.sizeof(arr))
    g._last_n = len(imgs)
    r = g.fetch(len(imgs))
    for i in range(len(imgs)):
        _assert_image_equal(r, i, types.SimpleNamespace(**{k: getattr(base, k)[i:i + 1] for k in (
            "status", "peak_count", "peak_x", "peak_y", "peak_score", "peak_anchor", "cand_count", "conn_count",
            "conn_ij", "conn_score", "conn_norm", "n_persons", "subset", "people_xy", "people_score")}), f"reuse {i}")


def test_bad_input_names_the_image_and_launches_nothing(env):
    t, grouping = env.torch, env.grouping
    g = env.ragged
    good = _small_set(env, 3)
    maps = [(h, p) for h, p, _ in good]
    ext = [e for _, _, e in good]
    before = g.launch_count
    tall1 = (t.zeros((1, 18, 1, 40), device=env.dev), t.zeros((1, 30, 1, 40), device=env.dev))
    with pytest.raises(grouping.GroupingError, match="image 2"):
        g.group_ragged(maps[:2] + [tall1], ext)
    wide = (t.zeros((1, 18, 8, 1100), device=env.dev), t.zeros((1, 30, 8, 1100), device=env.dev))
    with pytest.raises(grouping.GroupingError, match="image 1"):
        g.group_ragged([maps[0], wide, maps[1]], ext)
    with pytest.raises(grouping.GroupingError, match="max_batch|handle was created"):
        g.group_ragged(maps * 22, ext * 22)
    # a NULL paf and n > max_batch straight through the C ABI
    arr = (grouping._ImageMaps * 65)()
    for i in range(65):
        h, p, e = good[i % 3]
        arr[i] = grouping._ImageMaps(h.data_ptr(), p.data_ptr(), h.stride(1), p.stride(1), h.shape[2], h.shape[3], e)
    arr[1].paf = None
    prm = grouping.params_struct(None)
    rc = g._lib.spg_group_ragged(g._h, arr, 3, grouping.F32, C.byref(prm), g._stream_ptr(None))
    assert rc == -1 and b"image 1" in g._lib.spg_last_error(g._h)
    arr[1].paf = good[1][1].data_ptr()
    rc = g._lib.spg_group_ragged(g._h, arr, 65, grouping.F32, C.byref(prm), g._stream_ptr(None))
    assert rc == -1 and b"max_batch" in g._lib.spg_last_error(g._h)
    assert g.launch_count == before


def test_coco_shaped_batch_matches_the_checker(env):
    from oracle import spg_oracle as so
    shapes = [(480, 640), (640, 480), (427, 640), (612, 612), (375, 500), (360, 640)]
    params = env.skeleton.default_params()
    maps, host, ext = [], [], []
    for i, (H, W) in enumerate(shapes):
        heat, paf = env.synth.make_image(4100 + i, H, W, 1 + (3 * i) % 15)
        host.append((heat, paf))
        maps.append((env.torch.from_numpy(heat).to(env.dev)[None], env.torch.from_numpy(paf).to(env.dev)[None]))
        ext.append(float(H))
    with env.grouping.Grouper(max_batch=len(maps), max_h=640, max_w=640, max_peaks_per_part=128,
                              max_person_rows=128) as g:
        g.group_ragged(maps, ext, params, paf_as_f64=True)
        r = g.fetch(len(maps))
    for i, (heat, paf) in enumerate(host):
        o = so.group_batch(heat[None], paf[None].astype(np.float64), env.skeleton.LIMBS, ext[i], params)
        assert r.status[i] == 0 and o.status[0] == 0
        d = diff_structures(o.as_reference_structures(0), r.as_reference_structures(i), float_tol=0.0)
        assert not d, f"image {i} {shapes[i]}:\n" + "\n".join(d)


def test_wire_records_and_signal(env):
    t = env.torch
    g, s = env.ragged, env.single
    imgs = _small_set(env, 5, seed=60)
    rb = g.wire_record_bytes()
    wire_r = t.zeros((2 + len(imgs), rb), dtype=t.uint8, device=env.dev)
    word = t.zeros((1,), dtype=t.int64, device=env.dev)
    g.set_wire_output(wire_r.data_ptr(), first_record=2)
    g.arm_wire_signal(word.data_ptr(), 77)
    try:
        g.group_ragged([(h, p) for h, p, _ in imgs], [e for _, _, e in imgs])
        r = g.fetch(len(imgs))
    finally:
        g.set_wire_output(None)
    assert int(word.cpu()[0]) == 77
    rec_r = wire_r.cpu().numpy()
    assert not rec_r[:2].any()
    wire_s = t.zeros((1, rb), dtype=t.uint8, device=env.dev)
    s.set_wire_output(wire_s.data_ptr())
    try:
        for i, (h, p, e) in enumerate(imgs):
            s.group_device(h, p, e)
            P = int(s.fetch(1).n_persons[0])
            assert P == int(r.n_persons[i])
            assert _record(rec_r, 2 + i, rb, P) == _record(wire_s.cpu().numpy(), 0, rb, P), f"image {i}"
    finally:
        s.set_wire_output(None)


# ---- the drop-in functions -----------------------------------------------------------------------------------------
@pytest.fixture()
def dropin(cuda_device):
    from improved_body_parts_b200 import dropin as d
    d.configure(device=0, limbs=d.LIMBS)
    yield d
    d.configure()


def test_group_many_equals_group(dropin, env):
    params = env.skeleton.default_params()
    host = [env.synth.make_image(200 + i, H, W, 2 + i) for i, (H, W) in enumerate([(72, 56), (150, 97), (128, 128),
                                                                                    (61, 200)])]
    hwc = [(np.ascontiguousarray(h.transpose(1, 2, 0)), np.ascontiguousarray(p.transpose(1, 2, 0))) for h, p in host]
    ext = [h.shape[0] for h, _ in hwc]
    got = dropin.group_many(hwc, ext, params)
    for i, (h, p) in enumerate(hwc):
        d = diff_structures(dropin.group(h, p, ext[i], params), got[i], float_tol=0.0)
        assert not d, f"image {i}:\n" + "\n".join(d)
    # DeviceMaps (float32 storage of float64 values, what a single-scale predict() returns)
    t = env.torch
    dm = [(dropin.DeviceMaps(t.from_numpy(h).to(env.dev)[None], False),
           dropin.DeviceMaps(t.from_numpy(p).to(env.dev)[None], True)) for h, p in host]
    got = dropin.group_many(dm, ext, params)
    for i, (h, p) in enumerate(dm):
        d = diff_structures(dropin.group(h, p, ext[i], params), got[i], float_tol=0.0)
        assert not d, f"device image {i}:\n" + "\n".join(d)


def _stand_in_evaluate(skeleton, dropin):
    """What predict_many / process() / get_image_name of evaluate.py do (:501-560), calling the module's own names."""
    mod = types.ModuleType("evaluate")
    mod.limbSeq = list(skeleton.LIMBS)

    def _missing(*a, **k):
        raise AssertionError("the original python function was called")

    mod.find_peaks = mod.find_connections = mod.find_people = mod.predict = _missing

    def process(input_image_path, params, model, model_params, heat_layers, paf_layers):
        import cv2
        ori = cv2.imread(input_image_path)
        heatmap, paf = mod.predict(ori, params, model, model_params, heat_layers, paf_layers, input_image_path)
        all_peaks = mod.find_peaks(heatmap, params)
        connection_all, special_k = mod.find_connections(all_peaks, paf, ori.shape[0], params)
        subset, candidate = mod.find_people(connection_all, special_k, all_peaks, params)
        return dropin.keypoints(subset, candidate)

    def get_image_name(coco, image_id):
        return coco.imgs[image_id]["file_name"]

    def predict_many(coco, images_directory, validation_ids, params, model, model_params, heat_layers, paf_layers):
        assert (not set(validation_ids).difference(set(coco.getImgIds())))
        keypoints = {}
        for image_id in validation_ids:
            name = os.path.join(images_directory, mod.get_image_name(coco, image_id))
            keypoints[image_id] = mod.process(name, dict(params), model, dict(model_params), heat_layers + 2, paf_layers)
        return keypoints

    mod.process, mod.get_image_name, mod.predict_many = process, get_image_name, predict_many
    return mod


def _typed(v):
    if isinstance(v, (list, tuple)):
        return (type(v).__name__, [_typed(x) for x in v])
    return (type(v).__name__, repr(v))


@pytest.mark.parametrize("batch", [1, 3, 16])
def test_predict_many_equals_the_per_image_path(dropin, env, tmp_path, batch):
    import cv2
    import torch
    from improved_body_parts_b200 import wire

    shapes = [(120, 160), (160, 120), (107, 160), (153, 153), (94, 125), (125, 94), (90, 160), (160, 128), (106, 160),
              (120, 160)]
    rng = np.random.default_rng(11)
    coco = types.SimpleNamespace(imgs={}, getImgIds=lambda: sorted(coco.imgs))
    for k, (H, W) in enumerate(shapes):
        iid = 1000 + 7 * k
        cv2.imwrite(str(tmp_path / f"{iid:012d}.png"), rng.integers(0, 255, size=(H, W, 3), dtype=np.uint8))
        coco.imgs[iid] = {"file_name": f"{iid:012d}.png"}
    ids = list(coco.imgs)[::-1]
    params = dict(env.skeleton.default_params(), scale_search=[1.0], rotation_search=[0.0])
    model_params = dict(boxsize=160, stride=4, max_downsample=32, padValue=128)

    def model(x):  # deterministic maps with persons, keyed on the input's shape
        h, w = int(x.shape[1]) // 4, int(x.shape[2]) // 4
        out = env.synth.make_network_output(h * 1000 + w, h, w, 3, noise=0.0)
        return [[torch.from_numpy(out).to(x.device)]]

    mod = _stand_in_evaluate(env.skeleton, dropin)
    mod.posenet = model
    dropin.install(mod, device_predict=True)
    per_image = mod.predict_many(coco, str(tmp_path), ids, params, model, model_params, 18, 30)
    assert sum(len(v) for v in per_image.values()) > 0
    if batch > 1:
        mod = _stand_in_evaluate(env.skeleton, dropin)
        mod.posenet = model
        dropin.install(mod, device_predict=True, batch=batch)
        batched = mod.predict_many(coco, str(tmp_path), ids, params, model, model_params, 18, 30)
    else:
        batched = dropin.predict_many(coco, str(tmp_path), ids, params, model, model_params, 18, 30, batch=1)
    assert list(batched) == list(per_image)
    assert _typed(list(batched.values())) == _typed(list(per_image.values()))
    wire.format_results(per_image, str(tmp_path / "a.json"))
    wire.format_results(batched, str(tmp_path / "b.json"))
    assert (tmp_path / "a.json").read_bytes() == (tmp_path / "b.json").read_bytes()
