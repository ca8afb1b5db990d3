"""GPU: ``spg_yuv_to_bgr`` (``Grouper.yuv_to_bgr``) against ``cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420 / _YUYV)``:
byte-identical on every (Y, U, V) triple, on seeded COCO-sized and tiny frames, and on pitched planes and outputs; one
call over mixed members equals one call per member; a bad member is refused by name before anything runs; and the call
recorded into a CUDA graph converts whatever the planes hold when the graph replays."""
import numpy as np
import pytest

from oracle import yuv_port as yp

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

COCO = [(480, 640), (428, 640), (640, 480), (612, 612), (334, 500)]


@pytest.fixture()
def g(cuda_device):
    from improved_body_parts_b200.grouping import Grouper

    with Grouper(max_batch=1, device=0) as h:
        yield h


def _cv2(fmt, planes):
    return cv2.cvtColor(yp.cv2_layout(fmt, planes), yp.cv2_code(fmt))


def _device_planes(torch, planes, pad=0):
    """The planes on the device, each row ``pad`` bytes wider than its data when pad > 0 (a pitched surface)."""
    out = []
    for p in planes:
        buf = torch.zeros((p.shape[0], p.shape[1] + pad), dtype=torch.uint8, device="cuda:0")
        buf[:, :p.shape[1]] = torch.from_numpy(p).to("cuda:0")
        out.append(buf[:, :p.shape[1]])
    return out


def _member(fmt, dplanes, out):
    """A YUV_MEMBER for device planes (2-D uint8 tensors, stride (pitch, 1)) and a [H, W, 3] output view."""
    from improved_body_parts_b200 import grouping

    m = np.zeros(1, grouping.YUV_MEMBER)
    m["format"] = {"nv12": grouping.YUV_NV12, "i420": grouping.YUV_I420, "yuyv": grouping.YUV_YUYV}[fmt]
    m["height"], m["width"] = out.shape[0], out.shape[1]
    for k, p in enumerate(dplanes):
        m["planes"][0, k], m["pitches"][0, k] = p.data_ptr(), p.stride(0)
    m["out"], m["out_pitch"] = out.data_ptr(), out.stride(0)
    return m


def _convert(g, torch, fmt, planes, pad=0):
    H, W = planes[0].shape[0], planes[0].shape[1] // (2 if fmt == "yuyv" else 1)
    dplanes = _device_planes(torch, planes, pad)
    buf = torch.full((H, W * 3 + pad), 7, dtype=torch.uint8, device="cuda:0")
    out = buf[:, :3 * W].view(H, W, 3)
    g.yuv_to_bgr(_member(fmt, dplanes, out))
    torch.cuda.synchronize()
    if pad:  # nothing past a row's pixels is written
        assert bool((buf[:, 3 * W:] == 7).all())
    return out.cpu().numpy()


@pytest.mark.parametrize("fmt", yp.FORMATS)
def test_every_triple_equals_cv2(g, fmt):
    import torch
    planes = yp.every_triple(fmt)
    assert np.array_equal(_convert(g, torch, fmt, planes), _cv2(fmt, planes))
    assert g.launch_count >= 1


@pytest.mark.parametrize("fmt", yp.FORMATS)
@pytest.mark.parametrize("H,W", COCO + [(2, 2), (2, 6), (6, 14), (10, 642)])
def test_seeded_frames_equal_cv2(g, fmt, H, W):
    import torch
    planes = yp.random_planes(np.random.default_rng(H * 7919 + W), fmt, H, W)
    assert np.array_equal(_convert(g, torch, fmt, planes), _cv2(fmt, planes))


@pytest.mark.parametrize("fmt", yp.FORMATS)
@pytest.mark.parametrize("pad", [1, 64, 3])
def test_pitched_planes_and_output(g, fmt, pad):
    import torch
    planes = yp.random_planes(np.random.default_rng(pad), fmt, 90, 126)
    assert np.array_equal(_convert(g, torch, fmt, planes, pad), _cv2(fmt, planes))


def test_pitched_host_upload(g):
    """Host planes uploaded row for row into a pitched device surface, as a video reader's pinned upload lays them."""
    import torch
    H, W, pitch = 120, 160, 256
    y, uv = yp.random_planes(np.random.default_rng(3), "nv12", H, W)
    host = torch.zeros((H + H // 2, pitch), dtype=torch.uint8).pin_memory()
    host[:H, :W] = torch.from_numpy(y)
    host[H:, :W] = torch.from_numpy(uv)
    surface = host.to("cuda:0", non_blocking=True)
    out = torch.empty((H, W, 3), dtype=torch.uint8, device="cuda:0")
    g.yuv_to_bgr(_member("nv12", [surface[:H, :W], surface[H:, :W]], out))
    assert np.array_equal(out.cpu().numpy(), _cv2("nv12", (y, uv)))


def test_mixed_members_equal_one_call_each(g):
    import torch
    rng = np.random.default_rng(5)
    specs = [("nv12", 480, 640), ("yuyv", 427, 640), ("i420", 6, 2), ("nv12", 2, 2), ("i420", 612, 612),
             ("yuyv", 1, 2), ("nv12", 334, 500)] * 3
    frames = [(fmt, yp.random_planes(rng, fmt, H, W), H, W) for fmt, H, W in specs]
    dplanes = [_device_planes(torch, planes, pad=j % 3) for j, (_, planes, _, _) in enumerate(frames)]
    one = [torch.zeros((H, W, 3), dtype=torch.uint8, device="cuda:0") for _, _, H, W in frames]
    each = [torch.zeros((H, W, 3), dtype=torch.uint8, device="cuda:0") for _, _, H, W in frames]
    members = np.concatenate([_member(fmt, d, o) for (fmt, _, _, _), d, o in zip(frames, dplanes, one)])
    launches = g.launch_count
    g.yuv_to_bgr(members)
    assert g.launch_count == launches + 1  # one launch for every member
    for (fmt, _, _, _), d, o in zip(frames, dplanes, each):
        g.yuv_to_bgr(_member(fmt, d, o))
    for j, ((fmt, planes, _, _), a, b) in enumerate(zip(frames, one, each)):
        assert np.array_equal(a.cpu().numpy(), b.cpu().numpy()), j
        assert np.array_equal(a.cpu().numpy(), _cv2(fmt, planes)), j


def test_bad_members_are_refused_by_name(g):
    import torch
    from improved_body_parts_b200 import grouping
    planes = _device_planes(torch, yp.random_planes(np.random.default_rng(0), "nv12", 4, 6))
    out = torch.full((4, 6, 3), 9, dtype=torch.uint8, device="cuda:0")
    good = _member("nv12", planes, out)

    def bad(**fields):
        m = good.copy()
        for k, v in fields.items():
            if k.startswith("plane") or k.startswith("pitch"):
                name, i = k.rstrip("0123456789"), int(k[-1])
                m[name + "s" if name == "plane" else "pitches"][0, i] = v
            else:
                m[k] = v
        return m

    cases = {"format": bad(format=0), "format 4": bad(format=4), "reserved": bad(reserved=1), "outside": bad(height=0),
             "even": bad(height=3), "even width": bad(width=5), "plane 1 is NULL": bad(plane1=0),
             "plane 0's pitch": bad(pitch0=5), "plane 1's pitch": bad(pitch1=4), "out is NULL": bad(out=0),
             "out_pitch": bad(out_pitch=17)}
    for what, m in cases.items():
        with pytest.raises(grouping.GroupingError, match=r"SPG_E_INVALID|member 1") as e:
            g.yuv_to_bgr(np.concatenate([good, m]))
        assert "member 1" in str(e.value), (what, str(e.value))
        assert what.split()[0] in str(e.value), (what, str(e.value))
    i420 = _member("i420", _device_planes(torch, yp.random_planes(np.random.default_rng(0), "i420", 4, 6)), out)
    i420["planes"][0, 2] = 0
    with pytest.raises(grouping.GroupingError, match="member 0: plane 2 is NULL"):
        g.yuv_to_bgr(i420)
    yuyv = _member("yuyv", _device_planes(torch, yp.random_planes(np.random.default_rng(0), "yuyv", 3, 6)), out[:3])
    g.yuv_to_bgr(yuyv)  # an odd height is fine for 4:2:2
    torch.cuda.synchronize()
    assert bool((out[3] == 9).all())  # nothing of a refused call ran: the last row is still the fill
    g.yuv_to_bgr(np.zeros(0, grouping.YUV_MEMBER))  # no member: nothing to do


@pytest.mark.parametrize("fmt", yp.FORMATS)
def test_recorded_call_converts_the_new_contents(g, fmt):
    import torch
    rng = np.random.default_rng(17)
    H, W = 120, 160
    first = yp.random_planes(rng, fmt, H, W)
    dplanes = _device_planes(torch, first, pad=32)
    out = torch.empty((H, W, 3), dtype=torch.uint8, device="cuda:0")
    member = _member(fmt, dplanes, out)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        g.yuv_to_bgr(member)
    for n in range(3):
        planes = first if n == 0 else yp.random_planes(rng, fmt, H, W)
        for d, p in zip(dplanes, planes):
            d.copy_(torch.from_numpy(p))
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), _cv2(fmt, planes)), n
