#!/usr/bin/env python
"""Run the reference's ``evaluate.py`` UNCHANGED with its grouping stage on the H100 path.

    python tools/run_evaluate_b200.py --reference /path/to/Improved-Body-Parts [--config utils/config] [--check] [--batch N]
                                      [--forward-batch M] [--device-decode]
    torchrun --nproc-per-node G tools/run_evaluate_b200.py --reference ... --batch N [--forward-batch M] --gpus G

What it does (SURVEY.md §8b, INTEGRATION.md §1) -- the reference checkout is never modified:

1. stubs the modules ``evaluate.py`` imports but this host lacks (``pycocotools``, ``matplotlib``, ``configobj``,
   ``apex``) -- only the missing ones, and only as empty shells;
2. imports ``evaluate`` with a clean ``sys.argv`` (its module body runs argparse, ``evaluate.py:48``,
   and ``GetConfig``, ``:52``) and restores ``CUDA_VISIBLE_DEVICES``, which the module pins to "0" (``:28``) -- one
   process per GPU needs its own device;
3. ``dropin.install(evaluate)``: rebinds ``evaluate.find_peaks / find_connections / find_people`` (looked up by name
   at the call sites ``:509-511``) and takes ``limbSeq`` from the module (``:54``); with ``--batch N`` (N > 1) it also
   replaces ``predict`` by the device one and ``predict_many`` (``:550-560``) by ``dropin.predict_many``, which groups
   N images per call; ``--forward-batch M`` (M > 1, with N > 1) also runs the network on up to M images of the same
   input size at once (``dropin.predict_batch``; with several scales or a rotation search in ``utils/config``, up to M
   items: the images' scaled and rotated copies); ``--device-decode`` (with N > 1) also decodes each group of N JPEG
   files on the GPU (``dropin.imread_many``) in place of ``cv2.imread`` (``:502``), and builds the network input on the
   GPU as well (``device_input=True``), which the decoded images feed;
4. fills the globals ``evaluate.__main__`` would set (``:643-646``): ``params, model_params`` from the reference's own
   ``utils/config`` through ``skeleton.read_reference_ini`` (``utils/config_reader.py:7`` hard-codes the author's path),
   ``show_eval_speed``;
5. optionally replaces ``format_results`` (``:563-582``) by ``wire.format_results`` (same file contents);
6. with ``--device-cocoeval`` (``prepare(..., device_cocoeval=True)``) binds ``evaluate.COCOeval`` to
   ``cocoeval.COCOeval``, which scores the results on the GPU (``:617-620``), and ``evaluate.COCO`` to
   ``cocoeval.COCO`` where pycocotools is missing, so that ``validation()`` produces its metric without pycocotools.

``prepare()`` returns the module; building ``evaluate.posenet`` (``:626-641``: checkpoint + apex amp) and calling
``evaluate.validation(...)`` is then exactly what ``evaluate.__main__`` does.  With ``--check`` the launcher runs one
synthetic image through ``evaluate``'s own call sequence (``:509-511``) on the GPU and prints what it found.

With ``--gpus G`` (``prepare(..., gpus=G)``), every one of the G processes torchrun starts joins the process group, is
pinned to its ``LOCAL_RANK`` device and installs the ``predict_many`` that shards the images over the ranks.  Each rank
then builds ``evaluate.posenet`` on its device and calls ``validate(evaluate, ...)``: rank 0 runs
``evaluate.validation()`` unchanged, the other ranks serve their blocks of its ``predict_many``.  ``--check`` runs on
every rank, on that rank's device.
"""
from __future__ import annotations

import argparse
import importlib
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_OPTIONAL = ("pycocotools", "pycocotools.coco", "pycocotools.cocoeval", "matplotlib", "matplotlib.pyplot", "configobj",
             "apex")


def _stub_missing() -> list:
    stubbed = []
    for name in _OPTIONAL:
        if name in sys.modules:
            continue
        try:
            importlib.import_module(name)
        except Exception:
            mod = types.ModuleType(name)
            mod.__spg_stub__ = True
            sys.modules[name] = mod
            parent, _, child = name.rpartition(".")
            if parent:
                setattr(sys.modules[parent], child, mod)
            stubbed.append(name)
    for name, attr in (("pycocotools.coco", "COCO"), ("pycocotools.cocoeval", "COCOeval"), ("configobj", "ConfigObj")):
        m = sys.modules.get(name)
        if m is not None and getattr(m, "__spg_stub__", False) and not hasattr(m, attr):
            setattr(m, attr, dict if attr == "ConfigObj" else object)
    return stubbed


def gpus_error(gpus: int, batch: int):
    """Why ``--gpus gpus`` cannot run here, or None: it needs ``batch > 1`` (the sharded path is the batched
    ``predict_many``) and a ``torchrun --nproc-per-node gpus`` environment."""
    if batch < 2:
        return "--gpus needs --batch > 1"
    if "LOCAL_RANK" not in os.environ or os.environ.get("WORLD_SIZE") != str(gpus):
        return f"--gpus {gpus} runs under torchrun --nproc-per-node {gpus} (WORLD_SIZE={os.environ.get('WORLD_SIZE')})"
    return None


def init_ranks() -> int:
    """One process per GPU under torchrun: pin this process to ``LOCAL_RANK`` and join the process group (NCCL for CUDA
    tensors, gloo for the CPU objects ``predict_many`` broadcasts and gathers); returns the local rank."""
    import torch
    import torch.distributed as dist
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    if not dist.is_initialized():
        dist.init_process_group(backend="cuda:nccl,cpu:gloo")
    return local


def prepare(reference_root: str, config_path: str = None, device: int = None, install: bool = True,
            replace_format_results: bool = False, batch: int = 1, forward_batch: int = 1, gpus: int = None,
            device_cocoeval: bool = False, device_decode: bool = False):
    """Import the reference's ``evaluate`` module (unchanged) and put the H100 grouping path behind its call sites.

    ``gpus=G`` (under ``torchrun --nproc-per-node G``, with ``batch > 1``) joins the process group, pins this rank to
    its ``LOCAL_RANK`` device and installs the ``predict_many`` that shards the images over the G ranks; run
    ``validate`` on every rank.  ``device_cocoeval=True`` puts the GPU keypoint evaluation behind ``evaluate.COCOeval``
    (and the minimal loader behind ``evaluate.COCO`` when pycocotools was stubbed).  ``device_decode=True`` (with
    ``batch > 1``) decodes ``predict_many``'s JPEG files on the GPU, with the device input stage."""
    if device_decode and batch < 2:
        raise ValueError("device_decode needs batch > 1: only the batched predict_many reads the image files")
    if gpus is not None:
        err = gpus_error(int(gpus), int(batch))
        if err:
            raise ValueError(err)
        if device is not None:
            raise ValueError("gpus= takes each rank's device from LOCAL_RANK: pass no device")
        device = init_ranks()
    reference_root = os.path.abspath(reference_root)
    if not os.path.isfile(os.path.join(reference_root, "evaluate.py")):
        raise FileNotFoundError(f"no evaluate.py under {reference_root}")
    for p in (ROOT, reference_root):
        if p not in sys.path:
            sys.path.insert(0, p)
    stubbed = _stub_missing()
    visible = os.environ.get("CUDA_VISIBLE_DEVICES")
    argv, sys.argv = sys.argv, [os.path.join(reference_root, "evaluate.py")]
    cwd = os.getcwd()
    try:
        os.chdir(reference_root)  # the module appends ".." to sys.path and uses relative data paths
        evaluate = importlib.import_module("evaluate")
    finally:
        os.chdir(cwd)
        sys.argv = argv
        if visible is None:
            os.environ.pop("CUDA_VISIBLE_DEVICES", None)  # evaluate.py:28 pinned it to "0"
        else:
            os.environ["CUDA_VISIBLE_DEVICES"] = visible
    from improved_body_parts_b200 import dropin, skeleton, wire

    if install:
        if device is not None:
            dropin.configure(device=device)
        if batch > 1:  # the batched grouping takes the maps the device predict() leaves on the GPU
            extra = dict(forward_batch=forward_batch) if forward_batch > 1 else {}
            if device_decode:
                extra.update(device_input=True, device_decode=True)
            dropin.install(evaluate, device_predict=True, batch=batch, **extra)
        else:
            dropin.install(evaluate)
    evaluate.params, evaluate.model_params = skeleton.read_reference_ini(
        config_path or os.path.join(reference_root, "utils", "config"))
    evaluate.show_eval_speed = False
    if replace_format_results:
        evaluate.format_results = wire.format_results
    if device_cocoeval:
        from improved_body_parts_b200 import cocoeval
        evaluate.COCOeval = cocoeval.COCOeval
        if "pycocotools.coco" in stubbed:
            evaluate.COCO = cocoeval.COCO
    evaluate.__spg_stubbed__ = stubbed
    return evaluate


def validate(evaluate, **kwargs):
    """``evaluate.validation(evaluate.posenet, **kwargs)`` on rank 0, which returns its result; on every other rank,
    ``dropin.serve_predict_many(evaluate.posenet)``, which runs that rank's share of ``predict_many`` and returns None.
    Each rank builds ``evaluate.posenet`` on its own device first, as ``evaluate.__main__`` does (``:626-641``).  In a
    single process this is ``evaluate.validation(...)``."""
    from improved_body_parts_b200 import dropin, sharding
    if sharding._world()[0] != 0:
        dropin.serve_predict_many(evaluate.posenet)
        return None
    try:
        return evaluate.validation(evaluate.posenet, **kwargs)
    finally:
        dropin.end_serving()  # the other ranks return, also when validation raised


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reference", default=os.environ.get("SPG_REFERENCE_ROOT"), required="SPG_REFERENCE_ROOT" not in os.environ,
                    help="a checkout of the reference (default: $SPG_REFERENCE_ROOT)")
    ap.add_argument("--config", default=None, help="the reference's utils/config INI (default: <reference>/utils/config)")
    ap.add_argument("--device", type=int, default=None)
    ap.add_argument("--check", action="store_true", help="group one synthetic image through evaluate's call sites on the GPU")
    ap.add_argument("--batch", type=int, default=1,
                    help="images per grouping call in predict_many (> 1 implies the device predict; default 1)")
    ap.add_argument("--forward-batch", type=int, default=1,
                    help="images per network forward pass in predict_many (> 1 needs --batch > 1; default 1)")
    ap.add_argument("--device-cocoeval", action="store_true",
                    help="score validation() with the GPU COCOeval (and the minimal COCO loader without pycocotools)")
    ap.add_argument("--device-decode", action="store_true",
                    help="decode predict_many's JPEG files on the GPU, with the device input stage (needs --batch > 1)")
    ap.add_argument("--gpus", type=int, default=None,
                    help="under torchrun --nproc-per-node G: shard predict_many's images over the G GPUs (needs --batch > 1)")
    a = ap.parse_args()
    if a.batch < 1:
        ap.error("--batch must be >= 1")
    if a.forward_batch < 1:
        ap.error("--forward-batch must be >= 1")
    if a.forward_batch > 1 and a.batch < 2:
        ap.error("--forward-batch > 1 needs --batch > 1")
    if a.device_decode and a.batch < 2:
        ap.error("--device-decode needs --batch > 1")
    if a.gpus is not None:
        if a.gpus < 1:
            ap.error("--gpus must be >= 1")
        if a.device is not None:
            ap.error("--gpus takes each rank's device from LOCAL_RANK: drop --device")
        err = gpus_error(a.gpus, a.batch)
        if err:
            ap.error(err)
    ev = prepare(a.reference, a.config, a.device, batch=a.batch, forward_batch=a.forward_batch, gpus=a.gpus,
                 device_cocoeval=a.device_cocoeval, device_decode=a.device_decode)
    rank = f"rank {os.environ['RANK']}: " if a.gpus is not None else ""
    print(f"{rank}evaluate imported from {ev.__file__}; stubbed: {ev.__spg_stubbed__}; limbs: {len(ev.limbSeq)}; "
          f"find_peaks -> {ev.find_peaks.__module__}.{ev.find_peaks.__name__}")
    if a.check:
        import numpy as np
        from improved_body_parts_b200 import synth
        heat, paf = synth.make_image(7, 128, 128, 6)
        hw, pw = np.ascontiguousarray(heat.transpose(1, 2, 0)), np.ascontiguousarray(paf.transpose(1, 2, 0))
        peaks = ev.find_peaks(hw, ev.params)                                   # evaluate.py:509
        conns, special = ev.find_connections(peaks, pw, hw.shape[0], ev.params)  # :510
        subset, candidate = ev.find_people(conns, special, peaks, ev.params)    # :511
        print(f"{rank}check: {sum(len(p) for p in peaks)} peaks, {sum(len(c) for c in conns if len(c))} connections, "
              f"{len(subset)} persons")
    if a.gpus is not None:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
