"""Regenerate tests/golden/tint/: the reference data server's own colour distortion (``Transformer.distort_color``) and,
for whole samples, ``AugmentSelection.random`` + ``Transformer.transform`` + ``Heatmapper.create_heatmaps``
(py_cocodata_server/), run unmodified with seeded ``np.random`` and ``random``.  Needs the reference checkout and cv2;
the reference is loaded as make_targets_golden.py loads it.
Usage: python tests/golden/make_tint_golden.py REFERENCE_ROOT

- ``color_*.npz``: one ``distort_color`` call on make_targets_golden.source(h, w) (a strided view of a wider source when
  ``pad_cols`` > 0): the numpy seed, the three draws it made, the row block of the cv2 that made it and the output.
  Widths cover every class of cv2's HSV->BGR tail: width % 32 = 0 (640), 11 (427), 20 (500), 1 (1, 33), 31 (31, 63).
- ``gen_*.npz``: a sequential gen()-style loop over a few samples (both generators seeded once): per sample the
  selection, the draws (zeros when untinted), M, the moved joints, the warped image's uint8 codes, both masks and the
  labels.
"""
from __future__ import annotations

import json
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "tint")
sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

import make_targets_golden as mtg  # noqa: E402

COLOR_CASES = [  # name, (h, w), pad columns, np.random seed
    ("color_640", (24, 640), 0, 1),
    ("color_427", (31, 427), 0, 2),
    ("color_500", (20, 500), 0, 3),
    ("color_1x1", (1, 1), 0, 4),
    ("color_33", (17, 33), 0, 5),
    ("color_31", (9, 31), 0, 6),
    ("color_63", (12, 63), 0, 7),
    ("color_427_strided", (29, 427), 13, 8),
    ("color_64x50", (50, 64), 0, 9),
]
GEN_CASES = [  # name, output size, per sample (h, w) and persons; seed searched from `seed` for >= 2 tinted samples
    ("gen_256", 256, [((480, 640), 5), ((427, 640), 3), ((375, 500), 8), ((640, 427), 2)], 100),
    ("gen_512", 512, [((500, 375), 4), ((480, 640), 6), ((333, 250), 1)], 200),
]


def probe_row_block(cv2) -> int:
    """The row block of this cv2 (improved_body_parts_b200.targets.cv2_row_block, restated without the package)."""
    for w in range(1, 4097):
        out = cv2.cvtColor(np.full((2, w, 3), (0, 1, 1), np.uint8), cv2.COLOR_HSV2BGR)[:, :, 0]
        if not (out == 1).any():
            return w
    raise RuntimeError("no vector block")


def draws_of(seed: int):
    rs = np.random.RandomState(seed)
    return [int(rs.randint(21)), int(rs.randint(81)), int(rs.randint(61))]


def main(root):
    import cv2
    cfg_mod, tr, hm = mtg.load_reference(root)
    os.makedirs(OUT, exist_ok=True)
    block = probe_row_block(cv2)
    meta_common = {"cv2": cv2.__version__, "cv2_cpu_features": cv2.getCPUFeaturesLine(), "row_block": block}
    manifest = {}
    for name, (h, w), pad, seed in COLOR_CASES:
        big, _, _ = mtg.source(h, w + pad)
        img = big[:, pad // 2:pad // 2 + w]
        assert pad == 0 or not img.flags["C_CONTIGUOUS"]
        np.random.seed(seed)
        out = tr.Transformer.distort_color(img)
        d = draws_of(seed)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), source_hw=np.array([h, w]), pad_cols=pad, seed=seed,
                            draws=np.array(d), row_block=block, cv2_version=cv2.__version__, out=out)
        manifest[name] = {"source": [h, w], "pad_cols": pad, "seed": seed, "draws": d, "row_block": block}
    for name, size, specs, seed in GEN_CASES:
        config = mtg.sized_config(cfg_mod, size)
        while True:  # the first seed whose loop tints at least two samples and leaves one untinted
            random.seed(seed)
            tints = [tr.AugmentSelection.random(config.transform_params).tint for _ in specs]
            if sum(tints) >= 2 and not all(tints):
                break
            seed += 1
        rng = np.random.default_rng(seed)
        srcs, metas = [], []
        for (h, w), P in specs:
            srcs.append(mtg.source(h, w))
            joints = mtg.persons(rng, P, h, w)
            metas.append({"objpos": [[float(rng.uniform(0, w)), float(rng.uniform(0, h))]],
                          "scale_provided": [float(rng.uniform(0.3, 1.2))], "joints": joints})
        random.seed(seed)
        np.random.seed(seed)
        rec = {k: [] for k in ("aug", "draws", "M", "joints", "image_codes", "mask_miss", "mask_all", "labels")}
        for (img, mm, ma), meta in zip(srcs, metas):  # gen(): transform (which draws its own selection) + heatmaps
            st = np.random.get_state()
            r_state = random.getstate()
            aug = tr.AugmentSelection.random(config.transform_params)
            random.setstate(r_state)
            d = [int(np.random.randint(21)), int(np.random.randint(81)), int(np.random.randint(61))] if aug.tint \
                else [0, 0, 0]
            np.random.set_state(st)
            M, _ = aug.affine(meta["objpos"][0], meta["scale_provided"][0], config)
            m2 = {k: (v.copy() if k == "joints" else v) for k, v in meta.items()}
            ti, tm, ta, m2 = tr.Transformer(config).transform(img, mm, ma, m2)
            labels = hm.Heatmapper(config).create_heatmaps(m2["joints"].astype(np.float32), ta)
            codes = np.rint(ti * 255).astype(np.uint8)
            assert np.array_equal(codes.astype(np.float32) / 255., ti)
            rec["aug"].append([aug.flip, aug.tint, aug.degree, aug.crop[0], aug.crop[1], aug.scale])
            for k, v in (("draws", d), ("M", M), ("joints", m2["joints"]), ("image_codes", codes), ("mask_miss", tm),
                         ("mask_all", ta), ("labels", labels)):
                rec[k].append(v)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), size=size, seed=seed, row_block=block,
                            cv2_version=cv2.__version__, source_hw=np.array([s[0] for s in specs]),
                            objpos=np.array([m["objpos"][0] for m in metas]),
                            scale_provided=np.array([m["scale_provided"][0] for m in metas]),
                            **{f"joints_src_{i}": m["joints"] for i, m in enumerate(metas)},
                            **{f"joints_{i}": j for i, j in enumerate(rec["joints"])},
                            aug=np.array(rec["aug"], np.float64), draws=np.array(rec["draws"]), M=np.array(rec["M"]),
                            image_codes=np.array(rec["image_codes"]), mask_miss=np.array(rec["mask_miss"]),
                            mask_all=np.array(rec["mask_all"]), labels=np.array(rec["labels"]))
        manifest[name] = {"size": size, "seed": seed, "sources": [list(s[0]) for s in specs],
                          "persons": [s[1] for s in specs], "draws": rec["draws"], "tint": [a[1] for a in rec["aug"]],
                          "row_block": block}
    with open(os.path.join(OUT, "MANIFEST.json"), "w") as f:
        json.dump({"generator": "tests/golden/make_tint_golden.py", "reference": "py_cocodata_server (unmodified)",
                   "numpy": np.__version__, **meta_common, "cases": manifest}, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
