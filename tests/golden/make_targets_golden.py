"""Regenerate tests/golden/targets/ or tests/golden/targets_space/: the reference data server's own classes
(AugmentSelection, Transformer, Heatmapper of py_cocodata_server/), run unmodified on seeded synthetic samples.  Needs the
reference checkout and cv2; matplotlib is stubbed.
Usage: python tests/golden/make_targets_golden.py [reference_root] [targets | targets_space]

targets/ is the reference's CanonicalConfig at sizes 256 and 512 (stride 4).  targets_space/ varies what that config
admits (space_cases): the stride (1, 2, 3, 5, 6, 8), sizes that are not powers of two, sigma, paf_sigma, both Gaussian
thresholds (keypoint_gaussian_thre sets gaussian_size), a non-integer paf_thre and the limb table; each case also records
that configuration (stride, gaussian_size, sigma, paf_sigma, keypoint_gaussian_thre, limb_gaussian_thre, paf_thre,
limbs).

Each case records the source's size and mask kinds (source() rebuilds it), objpos / scale_provided / joints, the augmentation, the matrix M
(AugmentSelection.affine), the moved joints, the warped image (as its uint8 codes: the reference's float32 image is
exactly np.float32(code) / 255., checked here), both float32 masks and the labels.  augment_draws.npz holds seeded
AugmentSelection.random draws.
"""
from __future__ import annotations

import importlib.util
import json
import os
import random
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def load_reference(root):
    sys.modules.setdefault("matplotlib", types.ModuleType("matplotlib"))
    plt = types.ModuleType("matplotlib.pyplot")
    sys.modules["matplotlib.pyplot"] = plt
    sys.modules["matplotlib"].pyplot = plt
    mods = {}
    for name, rel in (("ref_config", "config/config.py"), ("ref_transformer", "py_cocodata_server/py_data_transformer.py"),
                      ("ref_heatmapper", "py_cocodata_server/py_data_heatmapper.py")):
        spec = importlib.util.spec_from_file_location(name, os.path.join(root, rel))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        mods[name] = m
    return mods["ref_config"], mods["ref_transformer"], mods["ref_heatmapper"]


def sized_config(cfg_mod, size):
    class Sized(cfg_mod.CanonicalConfig):
        def __init__(self):
            super().__init__()
            self.width = self.height = size
            self.mask_shape = (self.height // self.stride, self.width // self.stride)
            self.parts_shape = (self.height // self.stride, self.width // self.stride, self.num_layers)
            self.offset_shape = (self.height // self.stride, self.width // self.stride, self.offset_layers)
    return Sized()


def space_config(cfg_mod, size, stride, tp=None, limbs=None):
    """A CanonicalConfig at ``size`` x ``size`` and ``stride`` with the transform parameters ``tp`` set and, when given,
    the limb table ``limbs``: every shape and layer index the reference derives follows."""
    class Space(cfg_mod.CanonicalConfig):
        def __init__(self):
            super().__init__()
            self.width = self.height = size
            self.stride = stride
            if limbs is not None:
                self.limbs_conn = [tuple(l) for l in limbs]
                self.paf_layers = len(self.limbs_conn)
                self.num_layers = self.paf_layers + self.heat_layers + 2
                self.heat_start = self.paf_layers
                self.bkg_start = self.paf_layers + self.heat_layers
                self.offset_start = self.num_layers
            self.mask_shape = (self.height // self.stride, self.width // self.stride)
            self.parts_shape = (self.height // self.stride, self.width // self.stride, self.num_layers)
            self.offset_shape = (self.height // self.stride, self.width // self.stride, self.offset_layers)
            self.transform_params = cfg_mod.TransformationParams(stride)
            for k, v in (tp or {}).items():
                setattr(self.transform_params, k, v)
    return Space()


def source(h, w, miss="random", all_="random"):
    """The deterministic synthetic source of a case (tests rebuild it from h, w and the mask kinds)."""
    y, x = np.mgrid[0:h, 0:w]
    img = np.stack([(x * 3 + y) % 256, (x + y * 2) % 256, (x * y // 7) % 256], -1)
    img = ((img + ((x * x + 5 * y * y) // 97 % 13)[..., None]) % 256).astype(np.uint8)  # compresses; no rng noise
    masks = []
    for kind in (miss, all_):
        if kind == "random":
            m = np.where(((x // 37 + y // 29) % 3 == 0), 0, 255).astype(np.uint8)
            m[(x * 13 + y * 7) % 101 == 0] = 127
        else:
            m = np.full((h, w), kind, np.uint8)
        masks.append(m)
    return img, masks[0], masks[1]


def persons(rng, P, h, w, far=False, coincident=False):
    j = np.zeros((P, 18, 3))
    for p in range(P):
        c = rng.uniform([0, 0], [w, h])
        j[p, :, 0:2] = c + rng.normal(0, max(h, w) / 10, (18, 2))
        j[p, :, 2] = rng.choice([0, 1, 2, 3], 18, p=[0.3, 0.5, 0.15, 0.05])
    if far and P:
        j[0, 0, 0:2] = (-3e6, 5e5)
        j[0, 4, 0:2] = (w * 40.0, -h * 25.0)
        j[min(1, P - 1), 7, 0:2] = (-1.0, -1.0)
        j[:, :, 2][:, [0, 4]] = 1
    if coincident and P:
        j[0, 1, :] = (w / 2, h / 2, 1)
        j[0, 0, :] = (w / 2, h / 2, 1)  # limb 0 (neck, nose): dnorm == 0
    return j


def cases():
    yield dict(name="p0_unrandom", size=256, hw=(300, 400), P=0, aug=("un",))
    yield dict(name="p1_rot_scale", size=256, hw=(480, 640), P=1, aug=(False, 25.0, (10, -7), 1.2))
    yield dict(name="p5_flip", size=256, hw=(640, 427), P=5, aug=(True, -13.0, (-30, 12), 0.8))
    yield dict(name="p15_random", size=256, hw=(480, 640), P=15, aug=("rand", 11))
    yield dict(name="p100_crowd", size=256, hw=(480, 640), P=100, aug=("rand", 12))
    yield dict(name="p5_far_coincident", size=256, hw=(480, 640), P=5, far=True, coincident=True,
               aug=(False, 5.0, (0, 0), 1.0))
    yield dict(name="src_1x1", size=256, hw=(1, 1), P=1, aug=(True, 33.0, (3, 4), 1.1), scale=0.05)
    yield dict(name="masks_255_0", size=256, hw=(427, 640), P=5, miss=255, all_=0, aug=("rand", 13))
    yield dict(name="masks_0_255", size=256, hw=(427, 640), P=5, miss=0, all_=255, aug=(True, -40.0, (50, -50), 0.7))
    yield dict(name="d512_p5", size=512, hw=(480, 640), P=5, aug=("rand", 14))
    yield dict(name="d512_p15_flip", size=512, hw=(640, 427), P=15, aug=(True, 17.0, (-20, 25), 1.25))


# a short table: one limb twice and one from a part to itself (skipped as dnorm == 0, as any coincident ends)
SHORT_LIMBS = ((1, 0), (2, 3), (1, 0), (5, 5), (8, 9))


def space_cases():
    from improved_body_parts_b200 import skeleton
    odd = dict(sigma=5.5, paf_sigma=3.25, keypoint_gaussian_thre=0.05, limb_gaussian_thre=0.03, paf_thre=2.5)
    yield dict(name="s1_64_limbs24", size=64, stride=1, hw=(120, 90), P=4, limbs=skeleton.LIMBS_24,
               tp=dict(sigma=2.5, paf_sigma=2.0, paf_thre=0.75), aug=(False, 10.0, (3, -2), 1.1))
    yield dict(name="s1_48_flip", size=48, stride=1, hw=(100, 75), P=6, tp=dict(sigma=3.0, paf_sigma=1.5),
               aug=(True, -20.0, (0, 4), 1.3))
    yield dict(name="s2_128_p15", size=128, stride=2, hw=(480, 640), P=15, aug=("rand", 21))
    yield dict(name="s2_96_odd_params", size=96, stride=2, hw=(427, 640), P=8, tp=odd, aug=(True, 31.0, (-9, 7), 0.9))
    yield dict(name="s3_255_flip", size=255, stride=3, hw=(640, 427), P=10, aug=(True, -13.0, (12, -30), 1.05))
    yield dict(name="s3_96_far_coincident", size=96, stride=3, hw=(300, 400), P=5, far=True, coincident=True,
               tp=dict(sigma=4.0, keypoint_gaussian_thre=0.2), aug=(False, 5.0, (0, 0), 1.0))
    yield dict(name="s5_160_limbs24", size=160, stride=5, hw=(480, 640), P=12, limbs=skeleton.LIMBS_24,
               aug=("rand", 22))
    yield dict(name="s6_96_short_limbs", size=96, stride=6, hw=(375, 500), P=9, limbs=SHORT_LIMBS, coincident=True,
               tp=odd, aug=(False, -35.0, (20, 10), 1.2))
    yield dict(name="s8_368_p10", size=368, stride=8, hw=(480, 640), P=10, aug=("rand", 23))
    yield dict(name="s8_256_masks_0_255", size=256, stride=8, hw=(427, 640), P=5, miss=0, all_=255,
               tp=dict(sigma=12.0, paf_sigma=9.0, limb_gaussian_thre=0.001, paf_thre=5.5), aug=(True, 40.0, (50, -50), 0.7))


def main(root, kind="targets"):
    cfg_mod, tr, hm = load_reference(root)
    space = kind == "targets_space"
    out = os.path.join(HERE, kind)
    os.makedirs(out, exist_ok=True)
    rng = np.random.default_rng(20261019 if space else 20261016)
    manifest = {}
    for c in (space_cases() if space else cases()):
        if space:
            config = space_config(cfg_mod, c["size"], c["stride"], c.get("tp"), c.get("limbs"))
        else:
            config = sized_config(cfg_mod, c["size"])
        h, w = c["hw"]
        img, mm, ma = source(h, w, c.get("miss", "random"), c.get("all_", "random"))
        joints = persons(rng, c["P"], h, w, c.get("far", False), c.get("coincident", False))
        meta = {"objpos": [[float(rng.uniform(0, w)), float(rng.uniform(0, h))]],
                "scale_provided": [c.get("scale", float(rng.uniform(0.3, 1.2)))], "joints": joints.copy()}
        a = c["aug"]
        if a[0] == "un":
            aug = tr.AugmentSelection.unrandom()
        elif a[0] == "rand":
            random.seed(a[1])
            while True:
                aug = tr.AugmentSelection.random(config.transform_params)
                if not aug.tint:
                    break
        else:
            aug = tr.AugmentSelection(a[0], False, a[1], a[2], a[3])
        M, _ = aug.affine(meta["objpos"][0], meta["scale_provided"][0], config)
        src_joints = meta["joints"].copy()
        ti, tm, ta, meta = tr.Transformer(config).transform(img, mm, ma, meta, aug)
        labels = hm.Heatmapper(config).create_heatmaps(meta["joints"].astype(np.float32), ta)
        codes = np.rint(ti * 255).astype(np.uint8)
        assert np.array_equal(codes.astype(np.float32) / 255., ti)
        extra = {}
        if space:
            p = config.transform_params
            extra = dict(stride=config.stride, gaussian_size=hm.Heatmapper(config).gaussian_size, sigma=np.float64(p.sigma),
                         paf_sigma=np.float64(p.paf_sigma), keypoint_gaussian_thre=np.float64(p.keypoint_gaussian_thre),
                         limb_gaussian_thre=np.float64(p.limb_gaussian_thre),
                         paf_thre=np.float64(p.paf_thre), limbs=np.array(config.limbs_conn, np.int32))
        np.savez_compressed(os.path.join(out, c["name"] + ".npz"), size=c["size"], source_hw=np.array([h, w]),
                            mask_kinds=np.array([str(c.get("miss", "random")), str(c.get("all_", "random"))]), objpos=np.array(meta["objpos"][0]),
                            scale_provided=np.float64(meta["scale_provided"][0]), joints_src=src_joints,
                            aug_flip=aug.flip, aug_degree=aug.degree, aug_crop=np.array(aug.crop), aug_scale=aug.scale,
                            M=M, joints=meta["joints"], image_codes=codes, mask_miss=tm, mask_all=ta, labels=labels, **extra)
        manifest[c["name"]] = {"size": c["size"], "source": [h, w], "persons": c["P"]}
        if space:
            manifest[c["name"]].update(stride=c["stride"], gaussian_size=int(extra["gaussian_size"]),
                                       limbs=len(config.limbs_conn))
    if space:
        with open(os.path.join(out, "MANIFEST.json"), "w") as f:
            json.dump({"generator": "tests/golden/make_targets_golden.py targets_space",
                       "reference": "py_cocodata_server (unmodified)", "numpy": np.__version__, "cases": manifest}, f,
                      indent=1, sort_keys=True)
        return
    draws = []
    random.seed(2024)
    config = cfg_mod.CanonicalConfig()
    for _ in range(64):
        a = tr.AugmentSelection.random(config.transform_params)
        draws.append([a.flip, a.tint, a.degree, a.crop[0], a.crop[1], a.scale])
    np.savez_compressed(os.path.join(out, "augment_draws.npz"), seed=2024, draws=np.array(draws, np.float64))
    with open(os.path.join(out, "MANIFEST.json"), "w") as f:
        json.dump({"generator": "tests/golden/make_targets_golden.py", "reference": "py_cocodata_server (unmodified)",
                   "numpy": np.__version__, "cases": manifest}, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))  # improved_body_parts_b200.skeleton's limb tables
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference", sys.argv[2] if len(sys.argv) > 2 else "targets")
