"""GPU: the device JPEG decoder (spg_jpeg_decode_ragged through dropin.imread_many) against cv2, byte for byte: the
goldens, seeded COCO-sized encodings, ragged batches, the subsequence decode's edge cases, files left to cv2, and
predict_many with decode="device" against host decoding."""
import json
import os
import types

import numpy as np
import pytest

import make_jpeg_golden as mjg
from test_gpu_predict_batch import MODEL_PARAMS, SEARCHES, StandIn
from test_gpu_ragged import _stand_in_evaluate, _typed

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg")
MANIFEST = json.load(open(os.path.join(GOLDEN, "MANIFEST.json")))["cases"]


@pytest.fixture()
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import dropin, grouping, skeleton, synth

    dropin.configure(device=0, limbs=dropin.LIMBS)
    yield types.SimpleNamespace(torch=torch, dropin=dropin, grouping=grouping, skeleton=skeleton, synth=synth,
                                dev=cuda_device)
    dropin.configure(decode="host", input_stage="host", variant="evaluate")


def _write(tmp_path, name, data):
    p = str(tmp_path / name)
    with open(p, "wb") as f:
        f.write(data)
    return p


def _assert_cv2(paths, images):
    for p, img in zip(paths, images):
        assert img is not None and img.is_cuda, p
        got = img.cpu().numpy()
        assert got.dtype == np.uint8 and np.array_equal(got, cv2.imread(p)), p


def _device_status(env, data):
    """The decoder's own status for one file the parser accepts (no host fallback)."""
    t = env.torch
    rec = env.grouping.jpeg_parse(data)
    assert int(rec["status"]) == 0
    buf = t.from_numpy(np.frombuffer(data, np.uint8).copy()).to(env.dev)
    out = t.empty((int(rec["height"]), int(rec["width"]), 3), dtype=t.uint8, device=env.dev)
    st = t.full((1,), -1, dtype=t.int32, device=env.dev)
    arr = np.zeros(1, env.grouping.JPEG_RECORD)
    arr[0] = rec
    arr[0]["data"], arr[0]["out"], arr[0]["decode_status"] = buf.data_ptr(), out.data_ptr(), st.data_ptr()
    env.dropin._grouper().jpeg_decode(arr)
    return int(st.cpu()[0]), out


def test_goldens(env):
    """Every golden comes back as cv2 decodes it; the ones the device path takes are decoded there."""
    decoded = dict(np.load(os.path.join(GOLDEN, "decoded.npz")))
    names = sorted(MANIFEST)
    paths = [os.path.join(GOLDEN, n + ".jpg") for n in names]
    images, host = env.dropin.imread_many(paths)
    assert host == sum(MANIFEST[n]["status"] != "ok" for n in names)
    for n, p, img in zip(names, paths, images):
        want = decoded[n] if n in decoded else cv2.imread(p)  # cv2.imread keeps what it decoded of a truncated file
        if want is None:
            assert img is None, n
        else:
            assert np.array_equal(img.cpu().numpy(), want), n
    for n in names:
        with open(os.path.join(GOLDEN, n + ".jpg"), "rb") as f:
            data = f.read()
        status = MANIFEST[n]["status"]
        if status in ("ok", "corrupt", "range"):
            st, out = _device_status(env, data)
            assert st == {"ok": 0, "corrupt": 11, "range": 12}[status], n
            if status == "ok":
                assert np.array_equal(out.cpu().numpy(), decoded[n]), n


@pytest.mark.parametrize("shape", [(480, 640), (427, 640)])
@pytest.mark.parametrize("restart", [0, 5])
def test_coco_sized(env, tmp_path, shape, restart):
    paths = []
    for k, s in enumerate(("444", "422", "420", "440")):
        data = mjg.encode(mjg.content(200 + k + restart, *shape), s, 95, restart=restart)
        paths.append(_write(tmp_path, f"{s}.jpg", data))
    paths.append(_write(tmp_path, "grey.jpg", mjg.encode(mjg.content(210, *shape, grey=True), quality=90, restart=restart)))
    images, host = env.dropin.imread_many(paths)
    assert host == 0
    _assert_cv2(paths, images)


def test_ragged_batch_equals_one_file_per_call(env, tmp_path):
    rng = np.random.default_rng(3)
    paths = []
    for k in range(24):
        h, w = int(rng.integers(1, 300)), int(rng.integers(1, 300))
        s = ["444", "422", "420", "440"][k % 4]
        data = mjg.encode(mjg.content(300 + k, h, w, grey=k % 7 == 6), s, int(rng.integers(20, 100)),
                          restart=int(rng.integers(0, 3)) * int(rng.integers(1, 9)), optimize=bool(k % 3 == 0))
        if k % 5 == 0:
            data = mjg.insert_segment(data, 0xE1, mjg.exif(1 + k % 8, "MM" if k % 2 else "II"))
        paths.append(_write(tmp_path, f"{k}.jpg", data))
    together, host = env.dropin.imread_many(paths)
    assert host == 0
    _assert_cv2(paths, together)
    for p, img in zip(paths, together):
        alone, _ = env.dropin.imread_many([p])
        assert env.torch.equal(alone[0], img), p


def test_many_subsequences(env, tmp_path):
    """A 2000 x 3000 4:2:0 file: thousands of subsequences over many CTAs."""
    p = _write(tmp_path, "big.jpg", mjg.encode(mjg.content(400, 2000, 3000), "420", 95))
    images, host = env.dropin.imread_many([p])
    assert host == 0
    _assert_cv2([p], images)


def test_segment_shorter_than_one_subsequence(env, tmp_path):
    data = mjg.encode(np.full((8, 8, 3), 128, np.uint8), "420", 50)
    rec = env.grouping.jpeg_parse(data)
    assert int(rec["scan_length"]) * 8 < 1024
    p = _write(tmp_path, "tiny.jpg", data)
    images, host = env.dropin.imread_many([p])
    assert host == 0
    _assert_cv2([p], images)


def _packed_ff_offsets(data, rec):
    """Raw offsets of the stuffed pairs and the offsets their 0xFF data bytes get in the unstuffed stream."""
    seg = np.frombuffer(data, np.uint8)[int(rec["scan_offset"]):int(rec["scan_offset"]) + int(rec["scan_length"])]
    raw = np.nonzero((seg[:-1] == 0xFF) & (seg[1:] == 0x00))[0]
    return raw, raw - np.arange(len(raw))


def test_stuffed_pairs_on_chunk_and_subsequence_boundaries(env, tmp_path):
    """Files where a 0xFF 0x00 pair straddles an unstuffing chunk (4096 bytes), and where the unstuffed 0xFF byte is the
    last byte before a subsequence boundary (every 128 bytes) or the first after it."""
    found = {"chunk": None, "sub_end": None, "sub_start": None}
    for seed in range(200):
        data = mjg.encode(mjg.content(500 + seed, 480, 640), "420", 97)
        rec = env.grouping.jpeg_parse(data)
        raw, packed = _packed_ff_offsets(data, rec)
        if found["chunk"] is None and (raw % 4096 == 4095).any():
            found["chunk"] = data
        if found["sub_end"] is None and (packed % 128 == 127).any():
            found["sub_end"] = data
        if found["sub_start"] is None and (packed % 128 == 0).any():
            found["sub_start"] = data
        if all(v is not None for v in found.values()):
            break
    assert all(v is not None for v in found.values()), [k for k, v in found.items() if v is None]
    paths = [_write(tmp_path, f"{k}.jpg", v) for k, v in found.items()]
    images, host = env.dropin.imread_many(paths)
    assert host == 0
    _assert_cv2(paths, images)


def test_long_codes(env, tmp_path):
    """Optimised tables at quality 100 on a noisy image: AC codes longer than the 9-bit lookup."""
    img = np.random.default_rng(7).integers(0, 256, (480, 640, 3)).astype(np.uint8)
    data = mjg.encode(img, "444", 100, optimize=True)
    rec = env.grouping.jpeg_parse(data)
    assert (rec["ac"][0]["maxcode"][10:17] >= 0).any()
    p = _write(tmp_path, "long.jpg", data)
    images, host = env.dropin.imread_many([p])
    assert host == 0
    _assert_cv2([p], images)


def test_files_left_to_cv2(env, tmp_path):
    whole = mjg.encode(mjg.content(600, 64, 96), "420", 80)
    files = {"progressive.jpg": mjg.encode(mjg.content(601, 64, 96), "420", 80, progressive=True),
             "truncated.jpg": whole[:len(whole) // 2], "garbage.jpg": mjg.garbage_scan(whole, 5),
             "short.jpg": whole[:len(whole) // 2].rstrip(b"\xff") + b"\xff\xd9", "ok.jpg": whole}
    paths = [_write(tmp_path, k, v) for k, v in files.items()]
    png = str(tmp_path / "image.png")
    cv2.imwrite(png, mjg.content(602, 30, 40))
    paths.append(png)
    images, host = env.dropin.imread_many(paths)
    assert host == 5
    for p, img in zip(paths, images):
        want = cv2.imread(p)
        if want is None:
            assert img is None, p
        else:
            assert np.array_equal(img.cpu().numpy(), want), p
    assert _device_status(env, files["short.jpg"])[0] == 11


def test_decode_rejects_bad_records(env):
    g = env.dropin._grouper()
    arr = np.zeros(1, env.grouping.JPEG_RECORD)
    arr[0] = env.grouping.jpeg_parse(mjg.encode(mjg.content(700, 16, 16), "420", 80))
    with pytest.raises(env.grouping.GroupingError, match="NULL"):
        g.jpeg_decode(arr)
    arr[0]["status"] = 3
    with pytest.raises(env.grouping.GroupingError, match="status"):
        g.jpeg_decode(arr)


@pytest.mark.parametrize("forward_batch", [1, 2])
def test_predict_many_with_device_decode(env, tmp_path, forward_batch):
    """predict_many with decode="device" returns what it returns with cv2.imread, both with the device input stage, on a
    directory of seeded JPEGs that includes a progressive file."""
    from improved_body_parts_b200 import wire

    d = env.dropin
    coco = types.SimpleNamespace(imgs={}, getImgIds=lambda: sorted(coco.imgs))
    shapes = [(120, 160), (160, 120), (60, 80), (160, 200), (90, 120), (80, 60), (160, 97), (33, 250), (150, 200)]
    for k, (H, W) in enumerate(shapes):
        iid = 3000 + 7 * k
        data = mjg.encode(mjg.content(800 + k, H, W), ["444", "422", "420", "440"][k % 4], 90, restart=k % 3,
                          progressive=k == 4)
        _write(tmp_path, f"{iid:012d}.jpg", data)
        coco.imgs[iid] = {"file_name": f"{iid:012d}.jpg"}
    ids = list(coco.imgs)
    params = dict(env.skeleton.default_params(), scale_search=SEARCHES["1 item"][0], rotation_search=[0.0])
    model = StandIn(env.torch, env.synth)
    results = []
    for decode in (False, True):
        mod = _stand_in_evaluate(env.skeleton, d)
        mod.posenet = model
        d.install(mod, device_predict=True, device_input=True, batch=4, forward_batch=forward_batch, device_decode=decode)
        results.append(mod.predict_many(coco, str(tmp_path), ids, params, model, MODEL_PARAMS, 18, 30))
    host, device = results
    assert sum(len(v) for v in host.values()) > 0
    assert list(device) == list(host)
    assert _typed(list(device.values())) == _typed(list(host.values()))
    wire.format_results(host, str(tmp_path / "a.json"))
    wire.format_results(device, str(tmp_path / "b.json"))
    assert (tmp_path / "a.json").read_bytes() == (tmp_path / "b.json").read_bytes()
