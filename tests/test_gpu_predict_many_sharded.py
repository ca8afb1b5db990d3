"""GPU: ``predict_many`` sharded over 2 ranks (spawned processes, the launcher's ``validate``) against one process.

13 images: 12 synthetic COCO-shaped uint8 PNGs of 3 aspect ratios and one square image whose network output carries the
crowded golden of ``tests/golden/crowd/``, so that the capacity-free tier runs on rank 1.  The network is the stand-in
of test_gpu_predict_batch.py (its output for a sample does not depend on the batch), so every ``forward_batch`` gives
one process's maps.  Rank 0's dict and its ``format_results`` file must be byte-identical to a single process's, at
``batch=4``, ``forward_batch`` 1 and 4, ``[1] x [0]`` and ``[0.5, 1] x [0, 30]``.  The two ranks run on two GPUs, and
also on one GPU that both share (where a box has only one)."""
import datetime
import glob
import os

import numpy as np
import pytest

from golden_io import load_case
from test_gpu_predict_batch import StandIn
from test_predict_many_sharded import TIMEOUT, _free_port, _launcher, _stand_in

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL_PARAMS = dict(boxsize=320, stride=4, max_downsample=64, padValue=128)
SHAPES = [(480, 640), (640, 480), (427, 640)] * 4
CROWD_SHAPE, CROWD_AT = (320, 320), 9  # images 7..12 are rank 1's block of 13
CONFIGS = [(1, [1.0], [0.0]), (4, [1.0], [0.0]), (1, [0.5, 1.0], [0.0, 30.0]), (4, [0.5, 1.0], [0.0, 30.0])]


class Network(StandIn):
    """``StandIn``, except that a square input answers with the crowded golden's maps in its top-left corner."""

    def __call__(self, x):
        from improved_body_parts_b200.skeleton import FLIP_HEAT_ORD, FLIP_PAF_ORD, NUM_PARTS
        h, w = int(x.shape[1]) // 4, int(x.shape[2]) // 4
        if h == w and (h, w) not in self._maps:
            case = load_case(sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "crowd", "*.npz")))[0])
            out = np.zeros((2, 50, h, w), np.float32)
            k = min(h, case["heat"].shape[1])
            out[0, :30, :k, :k], out[0, 30:48, :k, :k] = case["paf"][:, :k, :k], case["heat"][:, :k, :k]
            out[1, :30] = out[0, :30][np.argsort(FLIP_PAF_ORD)][..., ::-1]
            out[1, 30:48] = out[0, 30:48][np.argsort(FLIP_HEAT_ORD[:NUM_PARTS])][..., ::-1]
            self._maps[(h, w)] = self.torch.from_numpy(out).to(x.device)
        return super().__call__(x)


def _images(directory):
    import cv2
    rng = np.random.default_rng(2031)
    shapes = list(SHAPES)
    shapes.insert(CROWD_AT, CROWD_SHAPE)
    ids, names = [], {}
    for k, (H, W) in enumerate(shapes):
        iid = 5000 + 13 * k
        ids.append(iid)
        names[iid] = f"{iid:012d}.png"
        cv2.imwrite(os.path.join(directory, names[iid]), rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8))
    return ids, names


def _evaluate(directory, ids, names):
    """Every config's ``validate`` on this process: (results, tier calls per config)."""
    import torch

    from improved_body_parts_b200 import dropin, skeleton, synth
    tier = []
    unbounded = dropin._unbounded

    def counted(*a, **k):
        tier[-1] += 1
        return unbounded(*a, **k)

    dropin._unbounded = counted
    try:
        out = []
        for fb, scales, angles in CONFIGS:
            tier.append(0)
            params = dict(skeleton.default_params(), scale_search=scales, rotation_search=angles)
            mod = _stand_in(dropin, directory, ids, names, params, MODEL_PARAMS, Network(torch, synth))
            dropin.install(mod, device_predict=True, batch=4, forward_batch=fb)
            out.append(_launcher().validate(mod, dump_name="x"))
        return out, tier
    finally:
        dropin._unbounded = unbounded


def _rank(rank, world, port, devices, directory, ids, names, q):
    import torch
    import torch.distributed as dist

    from improved_body_parts_b200 import dropin
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(devices[rank])
    dist.init_process_group("cuda:nccl,cpu:gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=TIMEOUT))
    try:
        dropin.configure(device=devices[rank], limbs=dropin.LIMBS)
        q.put((rank,) + _evaluate(directory, ids, names))
    finally:
        dist.destroy_process_group()


def _typed(v):
    if isinstance(v, (list, tuple)):
        return (type(v).__name__, [_typed(x) for x in v])
    return (type(v).__name__, repr(v))


@pytest.mark.parametrize("devices", [(0, 1), (0, 0)], ids=["two GPUs", "one shared GPU"])
def test_two_ranks_write_the_single_process_file(cuda_device, tmp_path, devices):
    import torch
    import torch.multiprocessing as mp

    from improved_body_parts_b200 import dropin, wire
    if max(devices) >= torch.cuda.device_count():
        pytest.skip(f"needs {max(devices) + 1} CUDA devices")
    ids, names = _images(str(tmp_path))
    dropin.configure(device=0, limbs=dropin.LIMBS)
    try:
        want, want_tier = _evaluate(str(tmp_path), ids, names)
    finally:
        dropin.configure(input_stage="host", variant="evaluate")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank, args=(r, 2, port, devices, str(tmp_path), ids, names, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        got = {r: (res, tier) for r, res, tier in (q.get(timeout=4 * TIMEOUT) for _ in procs)}
        for p in procs:
            p.join(timeout=TIMEOUT)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    assert all(v is None for v in got[1][0])
    assert all(t > 0 for t in want_tier) and all(t > 0 for t in got[1][1]) and got[0][1] == [0] * len(CONFIGS), \
        "the crowded image is regrouped on the tier, on rank 1"
    for k, (one, sharded) in enumerate(zip(want, got[0][0])):
        assert sum(len(v) for v in one.values()) > 0
        assert list(sharded) == list(one) == ids, CONFIGS[k]
        assert _typed(list(sharded.values())) == _typed(list(one.values())), CONFIGS[k]
        wire.format_results(one, str(tmp_path / "one.json"))
        wire.format_results(sharded, str(tmp_path / "sharded.json"))
        assert (tmp_path / "one.json").read_bytes() == (tmp_path / "sharded.json").read_bytes(), CONFIGS[k]
