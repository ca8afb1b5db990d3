"""CPU, 2 and 3 gloo ranks as spawned processes: ``predict_many`` sharded over ranks through the launcher's ``validate``
(rank 0 runs a stand-in ``evaluate.validation()``, the other ranks ``dropin.serve_predict_many``).

``predict``, ``predict_batch`` and ``_people_of_batch`` are replaced in every process by functions that give
deterministic people from the bytes of each image, so the test checks the sharding itself: blocks, batching inside a
block, the gather, the order of the dict, the types of its values, the failure path -- and that rank 0's dict and its
``format_results`` file equal a single process's."""
import datetime
import importlib.util
import os
import socket
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMEOUT = 120  # seconds for a whole run; a hung collective fails the test instead of blocking the suite

PARAMS = dict(scale_search=[1.0], rotation_search=[0.0])
MODEL_PARAMS = dict(boxsize=64, stride=4, max_downsample=32, padValue=128)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _write_images(directory, n):
    """``n`` tiny PNGs of different sizes; ids in a shuffled order, as validation ids need not be sorted."""
    import cv2
    rng = np.random.default_rng(n)
    ids = [int(v) for v in rng.permutation(np.arange(100, 100 + 7 * n, 7))]
    names = {}
    for k, iid in enumerate(ids):
        names[iid] = f"{iid:012d}.png"
        cv2.imwrite(os.path.join(directory, names[iid]), rng.integers(0, 256, size=(9 + k % 4, 11 + k % 3, 3), dtype=np.uint8))
    return ids, names


def _digest(image):
    return int(image.astype(np.int64).sum()) * 31 + image.shape[0] * 7 + image.shape[1]


def _fake_predict(image, params, model, model_params, heat_layers=None, paf_layers=None, input_image_path=None):
    return ("maps", _digest(image))


def _fake_predict_batch(images, params, model, model_params, *, forward_batch):
    return [("maps", _digest(im)) for im in images]


def _fake_people_of_batch(maps, extents, params):
    """Per image: 0-3 persons, ``np.float64`` coordinates and scores, integer ``(0, 0)`` for a missing joint."""
    out = []
    for (_, s), extent in zip(maps, extents):
        people = []
        for p in range(s % 4):
            pts = [(0, 0) if (g + p + s) % 5 == 0 else (np.float64(s % 97 + g / 8), np.float64(extent + p / 3))
                   for g in range(17)]
            people.append((pts, np.float64(1 - 1 / (s % 11 + p + 2))))
        out.append(people)
    return out


def _fakes(dropin):
    dropin.predict, dropin.predict_batch, dropin._people_of_batch = _fake_predict, _fake_predict_batch, _fake_people_of_batch


def _stand_in(dropin, directory, ids, names, params=PARAMS, model_params=MODEL_PARAMS, posenet="network"):
    """An ``evaluate`` module as far as ``validation()`` -> ``predict_many`` goes (evaluate.py:546-560, :587-613)."""
    coco = types.SimpleNamespace(imgs={i: {"file_name": n} for i, n in names.items()}, getImgIds=lambda: list(names))
    mod = types.ModuleType("evaluate")
    mod.limbSeq = list(dropin.LIMBS)
    mod.posenet = posenet
    mod.get_image_name = lambda c, image_id: c.imgs[image_id]["file_name"]

    def validation(model, dump_name=None):
        return mod.predict_many(coco, directory, ids, params, model, model_params, 18, 30)

    mod.validation = validation
    return mod


def _launcher():
    spec = importlib.util.spec_from_file_location("run_evaluate_b200", os.path.join(ROOT, "tools", "run_evaluate_b200.py"))
    L = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(L)
    return L


def _rank(rank, world, port, directory, ids, names, batch, forward_batch, q):
    import torch.distributed as dist

    from improved_body_parts_b200 import dropin
    from improved_body_parts_b200.grouping import GroupingError

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=TIMEOUT))
    try:
        _fakes(dropin)
        mod = _stand_in(dropin, directory, ids, names)
        dropin.install(mod, device_predict=True, batch=batch, forward_batch=forward_batch)
        try:
            got = _launcher().validate(mod, dump_name="x")
        except GroupingError as e:
            q.put((rank, "GroupingError", str(e)))
        else:
            q.put((rank, "ok", got))
    finally:
        dist.destroy_process_group()


def _run(world, directory, ids, names, batch, forward_batch):
    """Every rank's ``(status, value)``, in rank order; no process outlives the call."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank, args=(r, world, port, directory, ids, names, batch, forward_batch, q))
             for r in range(world)]
    for p in procs:
        p.start()
    try:
        out = dict((r, (s, v)) for r, s, v in (q.get(timeout=TIMEOUT) for _ in procs))
        for p in procs:
            p.join(timeout=TIMEOUT)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    return [out[r] for r in range(world)]


def _single(monkeypatch, directory, ids, names, batch, forward_batch):
    from improved_body_parts_b200 import dropin
    for name, fn in (("predict", _fake_predict), ("predict_batch", _fake_predict_batch),
                     ("_people_of_batch", _fake_people_of_batch)):
        monkeypatch.setattr(dropin, name, fn)
    mod = _stand_in(dropin, directory, ids, names)
    try:
        dropin.install(mod, device_predict=True, batch=batch, forward_batch=forward_batch)
        return _launcher().validate(mod, dump_name="x")
    finally:
        dropin.configure(limbs=dropin.LIMBS, input_stage="host")


# (world, images, batch, forward_batch): uneven blocks (5 over 3 is 2, 2, 1), a rank with an empty block (2 over 3),
# batch larger than every block, and blocks of several grouping batches
CASES = [(2, 6, 2, 1), (3, 5, 2, 2), (3, 2, 4, 2), (2, 5, 16, 1), (3, 11, 2, 1)]


@pytest.mark.parametrize("world,n,batch,forward_batch", CASES)
def test_rank0_returns_what_one_process_returns(tmp_path, monkeypatch, world, n, batch, forward_batch):
    from improved_body_parts_b200 import wire

    ids, names = _write_images(str(tmp_path), n)
    want = _single(monkeypatch, str(tmp_path), ids, names, batch, forward_batch)
    assert list(want) == ids and sum(len(v) for v in want.values()) > 0
    results = _run(world, str(tmp_path), ids, names, batch, forward_batch)
    assert [s for s, _ in results] == ["ok"] * world
    assert all(v is None for _, v in results[1:])
    got = results[0][1]
    assert list(got) == list(want)
    assert [repr(v) for v in got.values()] == [repr(v) for v in want.values()]
    wire.format_results(want, str(tmp_path / "one.json"))
    wire.format_results(got, str(tmp_path / "sharded.json"))
    assert (tmp_path / "one.json").read_bytes() == (tmp_path / "sharded.json").read_bytes()


@pytest.mark.parametrize("failing_rank", [2, 0])
def test_a_failing_block_raises_on_rank0_and_every_rank_ends(tmp_path, failing_rank):
    """A block that raises (here ``cv2.imread`` of a missing file) sends its text in place of its dict: rank 0 raises
    GroupingError naming the rank and the image, and every process returns."""
    from improved_body_parts_b200.sharding import shard_range

    ids, names = _write_images(str(tmp_path), 7)
    lo, hi = shard_range(len(ids), failing_rank, 3)
    bad = ids[lo + 1]
    os.remove(tmp_path / names[bad])
    results = _run(3, str(tmp_path), ids, names, 2, 1)
    status, msg = results[0]
    assert status == "GroupingError"
    assert f"rank {failing_rank}, image {bad}:" in msg and "AttributeError" in msg, msg
    assert [s for s, _ in results[1:]] == ["ok", "ok"] and all(v is None for _, v in results[1:])


@pytest.mark.parametrize("args,env,msg", [
    (["--gpus", "2"], {}, "--gpus needs --batch > 1"),
    (["--gpus", "2", "--batch", "1"], {"WORLD_SIZE": "2", "LOCAL_RANK": "0"}, "--gpus needs --batch > 1"),
    (["--gpus", "2", "--batch", "8"], {}, "runs under torchrun --nproc-per-node 2"),
    (["--gpus", "4", "--batch", "8"], {"WORLD_SIZE": "2", "LOCAL_RANK": "0"}, "runs under torchrun --nproc-per-node 4"),
    (["--gpus", "2", "--batch", "8", "--device", "1"], {"WORLD_SIZE": "2", "LOCAL_RANK": "0"}, "drop --device"),
])
def test_launcher_gpus_argument_errors(tmp_path, monkeypatch, args, env, msg):
    from test_predict_batch_host import _launcher as launch
    for k in ("WORLD_SIZE", "LOCAL_RANK", "RANK"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    r = launch(args, tmp_path)
    assert r.returncode == 2 and msg in r.stderr, (args, r.stderr[-2000:])


def test_prepare_checks_gpus(tmp_path, monkeypatch):
    for k in ("WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    L = _launcher()
    with pytest.raises(ValueError, match="batch > 1"):
        L.prepare(str(tmp_path), gpus=2)
    with pytest.raises(ValueError, match="torchrun"):
        L.prepare(str(tmp_path), gpus=2, batch=4)
