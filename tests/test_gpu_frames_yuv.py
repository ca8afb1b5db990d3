"""GPU: ``dropin.FrameStream`` on ``dropin.YUVFrame`` frames -- NV12, I420 and YUYV planes, on the host or on the device,
converted by ``spg_yuv_to_bgr`` inside the tick's graph -- against ``dropin.predict`` + ``dropin.group`` of
``cv2.cvtColor``'s image of the frame (frames_reference.py): people by value and type, wire records, maps and the
``detail`` image equal.  With one and two scales and a rotation search, with both input stages, for a pitched CUDA NV12
surface, in ``submit_many`` ticks that mix YUV, BGR and JPEG frames, and for frames of one format whose content changes
from tick to tick while each slot keeps the one graph it captured."""
import types

import numpy as np
import pytest

import make_jpeg_golden as mjg
from frames_reference import MODEL_PARAMS, StandIn, _live, _reference, _typed
from oracle import yuv_port as yp

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

SEARCHES = {"1 item": ([1.0], [0.0]), "2 scales": ([1.0, 0.5], [0.0]), "3 angles": ([1.0], [0.0, 30.0, -30.0])}


@pytest.fixture()
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import dropin, skeleton, synth, wire

    dropin.configure(device=0, limbs=dropin.LIMBS)
    yield types.SimpleNamespace(torch=torch, dropin=dropin, skeleton=skeleton, synth=synth, wire=wire, dev=cuda_device)
    dropin.configure(input_stage="host", variant="evaluate")


def _params(env, search="1 item"):
    scales, angles = SEARCHES[search]
    return dict(env.skeleton.default_params(), scale_search=scales, rotation_search=angles)


def _planes(fmt, H, W, seed):
    """A photo-like frame's planes in ``fmt``: cv2's YUV of a seeded image, chroma taken at even rows and columns."""
    img = mjg.content(seed, H + H % 2, W)
    yuv = cv2.cvtColor(img, cv2.COLOR_BGR2YUV)[:H]
    Y, U, V = yuv[..., 0].copy(), yuv[..., 1], yuv[..., 2]
    if fmt == "yuyv":
        p = np.empty((H, 2 * W), np.uint8)
        p[:, 0::4], p[:, 1::4], p[:, 2::4], p[:, 3::4] = Y[:, 0::2], U[:, 0::2], Y[:, 1::2], V[:, 0::2]
        return (p,)
    u, v = U[0::2, 0::2].copy(), V[0::2, 0::2].copy()
    if fmt == "nv12":
        uv = np.empty((H // 2, W), np.uint8)
        uv[:, 0::2], uv[:, 1::2] = u, v
        return Y, uv
    return Y, u, v


def _frame(env, fmt, H, W, seed, cuda=False):
    """``(YUVFrame, cv2's BGR image of it)``."""
    planes = _planes(fmt, H, W, seed)
    image = cv2.cvtColor(yp.cv2_layout(fmt, planes), yp.cv2_code(fmt))
    if cuda:
        planes = [env.torch.from_numpy(p).to(env.dev) for p in planes]
    return env.dropin.YUVFrame(fmt, planes), image


def _assert_same(env, got, want, what):
    assert _typed(got.people) == _typed(want.people), f"{what}: people"
    status = int(env.wire.as_records(want.record, 17, env.dropin.CAP_ROWS)[0]["status"])
    if status & env.dropin.CAPACITY_BITS:  # past the capacities the bounded record is unspecified but for its status
        assert int(env.wire.as_records(got.record, 17, env.dropin.CAP_ROWS)[0]["status"]) == status, f"{what}: status"
    else:
        assert _live(env, got.record) == _live(env, want.record), f"{what}: wire record"
    for a, b, name in ((got.heat, want.heat, "heat"), (got.paf, want.paf, "paf")):
        x, y = a.tensor.cpu().numpy(), b.tensor.cpu().numpy()
        assert a.as_f64 == b.as_f64 and x.dtype == y.dtype and np.array_equal(x, y, equal_nan=True), f"{what}: {name}"
    if want.image is not None:
        assert got.image is not None and got.image.dtype == np.uint8 and np.array_equal(got.image, want.image), \
            f"{what}: image"


def _want(env, image, params, model, input_stage="device", converted=True):
    """The reference's FrameResult: predict + group of ``image`` (cv2's image of a YUV frame, whose ``detail`` image it
    is when ``converted``)."""
    heat, paf, people, record = _reference(env, image, params, model, input_stage=input_stage)
    return env.dropin.FrameResult(people, record, heat, paf, image if converted else None)


@pytest.mark.parametrize("search", list(SEARCHES))
@pytest.mark.parametrize("cuda", [False, True], ids=["host", "cuda"])
@pytest.mark.parametrize("fmt", yp.FORMATS)
def test_submit_equals_predict_on_cv2s_image(env, fmt, cuda, search):
    params = _params(env, search)
    model = StandIn(env.torch, env.synth)
    shapes = [(120, 160), (120, 160), (90, 120), (120, 160)] if fmt != "yuyv" else [(121, 160), (121, 160), (90, 120)]
    persons = 0
    with env.dropin.FrameStream(model, params, MODEL_PARAMS, slots=2) as fs:
        for n, (H, W) in enumerate(shapes):
            frame, image = _frame(env, fmt, H, W, 100 + n, cuda)
            got = fs.result(fs.submit(frame), detail=True)
            _assert_same(env, got, _want(env, image, params, model), f"frame {n}")
            persons += len(got.people)
        assert fs.host_decodes == 0
    assert persons > 0


@pytest.mark.parametrize("search", ["1 item", "3 angles"])
@pytest.mark.parametrize("fmt", yp.FORMATS)
def test_host_input_stage(env, fmt, search):
    params = _params(env, search)
    model = StandIn(env.torch, env.synth)
    with env.dropin.FrameStream(model, params, MODEL_PARAMS, slots=2, input_stage="host") as fs:
        for n in range(3):
            frame, image = _frame(env, fmt, 120, 160, 200 + n)
            got = fs.result(fs.submit(frame), detail=True)
            _assert_same(env, got, _want(env, image, params, model, input_stage="host"), f"frame {n}")
        with pytest.raises(ValueError, match="host frames"):
            fs.submit(_frame(env, fmt, 120, 160, 0, cuda=True)[0])


def test_pitched_cuda_nv12_surface(env):
    """The Y and UV views of one pitched device surface, as a hardware decoder hands out a frame."""
    torch = env.torch
    params = _params(env, "2 scales")
    model = StandIn(env.torch, env.synth)
    H, W, pitch = 120, 160, 256
    surface = torch.zeros((H + H // 2, pitch), dtype=torch.uint8, device=env.dev)
    with env.dropin.FrameStream(model, params, MODEL_PARAMS, slots=2) as fs:
        for n in range(4):
            y, uv = _planes("nv12", H, W, 300 + n)
            surface[:H, :W] = torch.from_numpy(y).to(env.dev)
            surface[H:, :W] = torch.from_numpy(uv).to(env.dev)
            surface[:, W:] = 255 - n  # the pitch's padding is never read
            frame = env.dropin.YUVFrame("nv12", (surface[:H, :W], surface[H:, :W]))
            image = cv2.cvtColor(yp.cv2_layout("nv12", (y, uv)), cv2.COLOR_YUV2BGR_NV12)
            got = fs.result(fs.submit(frame), detail=True)
            _assert_same(env, got, _want(env, image, params, model), f"frame {n}")
        assert fs.captures == 2


@pytest.mark.parametrize("search", ["1 item", "3 angles"])
def test_ticks_mix_yuv_bgr_and_jpeg(env, search):
    params = _params(env, search)
    model = StandIn(env.torch, env.synth)

    def tick(seed):
        frames, wants = [], []
        specs = [("nv12", False, 120, 160), ("i420", True, 90, 120), ("yuyv", False, 121, 160), ("bgr", True, 120, 160),
                 ("jpeg", False, 90, 120), ("nv12", True, 120, 160), ("yuyv", True, 90, 120), ("bgr", False, 160, 120),
                 ("i420", False, 160, 120)]
        for j, (kind, cuda, H, W) in enumerate(specs):
            if kind == "bgr":
                img = mjg.content(seed * 100 + j, H, W)
                frames.append(env.torch.from_numpy(img).to(env.dev) if cuda else img)
                wants.append((img, False))
            elif kind == "jpeg":
                data = mjg.encode(mjg.content(seed * 100 + j, H, W), "420", quality=90)
                frames.append(data)
                wants.append((cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR), True))
            else:
                frame, image = _frame(env, kind, H, W, seed * 100 + j, cuda)
                frames.append(frame)
                wants.append((image, True))
        return frames, wants

    persons = 0
    with env.dropin.FrameStream(model, params, MODEL_PARAMS, slots=2) as fs:
        for n in range(3):
            frames, wants = tick(400 + n)
            tickets = fs.submit_many(frames)
            for j, (t, (image, converted)) in enumerate(zip(tickets, wants)):
                got = fs.result(t, detail=True)
                _assert_same(env, got, _want(env, image, params, model, converted=converted), f"tick {n} frame {j}")
                persons += len(got.people)
        assert fs.captures == 2  # one per slot for the one tick key
        assert fs.host_decodes == 0
    assert persons > 0


@pytest.mark.parametrize("cuda", [False, True], ids=["host", "cuda"])
@pytest.mark.parametrize("fmt", yp.FORMATS)
def test_frames_of_one_format_replay_one_graph_per_slot(env, fmt, cuda):
    params = _params(env)
    model = StandIn(env.torch, env.synth)
    images = set()
    with env.dropin.FrameStream(model, params, MODEL_PARAMS, slots=2) as fs:
        for n in range(12):
            frame, image = _frame(env, fmt, 120, 160, 500 + n, cuda)
            got = fs.result(fs.submit(frame), detail=True)
            _assert_same(env, got, _want(env, image, params, model), f"frame {n}")
            images.add(image.tobytes())
        assert fs.captures == 2  # exactly one graph per slot and key
    assert len(images) == 12  # the frames differ in content
