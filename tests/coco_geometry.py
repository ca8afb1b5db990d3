"""evaluate.py's validation geometry on COCO-shaped images, and the CPU chain the device paths are held to there.

``validation()`` runs ``predict`` with ``boxsize = 640``, ``stride = 4``, ``max_downsample = 64`` (utils/config) on images of
about 480 x 640.  Every image becomes a 640-row crop: a 480 x 640 image a 640 x 853 crop padded to 640 x 896, whose
160 x 224 network output is resized x4 and then by 0.75 back to the image; an image 640 rows high keeps its size, so its
second resize is the identity.  This module holds

* ``FIXTURE``: seeded images of COCO shapes, two of them crowded, one with a pair of identical persons (``twins``);
* ``geometry``: each item's sizes restated from evaluate.py:87-100 (not taken from ``dropin.plan_items``);
* the network's answers: per item, maps from ``synth.render`` of skeletons placed in the item's crop, persons 15-80 %
  of the image height, some straddling the border; ``StandIn`` returns them on the device, keyed by input shape and
  by a marker the image carries in its blue channel, so that the batched paths can mix images in one forward pass and
  a CUDA graph can replay the lookup;
* ``cpu_chain``: ``postnet_port`` / ``postnet_rotation_port`` per item and ``accumulate`` (the maps ``predict()``
  returns), then the C checker's structures and ``dropin.keypoints``' people;
* ``coverage``: what the chain says about the paths the maps reach (candidates per limb, samples per pair, peaks at
  the border).

Nothing under ``improved_body_parts_b200/`` imports this file."""
import dataclasses
import itertools

import numpy as np

MODEL_PARAMS = dict(boxsize=640, stride=4, max_downsample=64, padValue=128)
SHAPES = [(480, 640), (640, 480), (427, 640), (640, 427), (612, 612), (375, 500), (500, 375), (333, 500), (640, 359)]

#: the blue channel of image i is 130 + 5 i: the lookup key of the stand-in network (robust to a 1-LSB resize difference
#: and to the warp of a rotated item; the padding, 128, stays below it)
MARKER0, MARKER_STEP = 130, 5


@dataclasses.dataclass(frozen=True)
class Spec:
    H: int
    W: int
    persons: int
    seed: int
    twins: bool = False  # two identical persons a whole number of network pixels apart (identity second resize only)


def _fixture():
    out = []
    for i in range(22):
        H, W = SHAPES[i % len(SHAPES)]
        out.append(Spec(H, W, 1 + (3 * i) % 8, 7000 + 13 * i))
    out.insert(5, Spec(480, 640, 20, 7400))   # crowded
    out.insert(14, Spec(427, 640, 21, 7500))  # crowded
    out[3] = Spec(640, 427, 3, 7600, twins=True)
    return out


FIXTURE = _fixture()
CROWDED = [i for i, s in enumerate(FIXTURE) if s.persons >= 20]
TWINS = [i for i, s in enumerate(FIXTURE) if s.twins]


def geometry(H, W, s, model_params=MODEL_PARAMS):
    """evaluate.py:87-100 for one scale of ``scale_search``: ``(multiplier, scale, H1, W1, Hp, Wp)`` -- the multiplier
    ``s * boxsize / H``, the scale after the 2600 / 3800 clamp, the size of ``cv2.resize(image, (0, 0), fx=scale,
    fy=scale)`` (``cvRound``: to nearest, ties to even) and ``padRightDownCorner`` of it up to multiples of
    ``max_downsample``."""
    m = s * model_params["boxsize"] / H
    scale = m
    if scale * H > 2600 or scale * W > 3800:
        scale = min(2600 / H, 3800 / W)
    H1, W1 = int(np.rint(H * scale)), int(np.rint(W * scale))
    md = model_params["max_downsample"]
    Hp = H1 if H1 % md == 0 else H1 + md - H1 % md
    Wp = W1 if W1 % md == 0 else W1 + md - W1 % md
    return m, scale, H1, W1, Hp, Wp


def image(i, spec):
    """The uint8 BGR image of fixture entry i: blue is the marker, green and red a photo-like texture."""
    from improved_body_parts_b200 import synth
    img = synth.photo(spec.seed, spec.H, spec.W)
    img[:, :, 0] = MARKER0 + MARKER_STEP * i
    return img


def _skeletons(spec, base_hw):
    """Joints ``[P, 18, 2]`` in network pixels of the scale-1 crop (``base_hw``): persons 15-80 % of the image height
    (the template is 35.5 units tall, the crop 160 network rows), centres anywhere in the crop, so some bodies straddle
    the border."""
    from improved_body_parts_b200 import synth
    rng = np.random.default_rng(spec.seed)
    bh, bw = base_hw
    if spec.twins:  # one person and its copy 40 network pixels to the right, both inside the crop; coordinates in 1/8 px
        j = synth.sample_skeletons(rng, 1, bh, bw, scale_range=(1.4, 1.4), jitter=0.4)
        j[0, :, 0] += 30.0 - j[0, :, 0].mean()
        j[0, :, 1] += 0.5 * bh - j[0, :, 1].mean()
        j = np.round(j * 8) / 8
        return np.concatenate([j, j + np.array([40.0, 0.0])])
    P = spec.persons
    if P >= 20:  # a crowd: a row of persons 44 % of the image high, shoulder to shoulder
        scale = rng.uniform(1.9, 2.1, size=(P, 1, 1))
        body = synth._TEMPLATE[None] * scale + rng.normal(0.0, 0.6, size=(P, 18, 2))
        body[..., 0] += 0.5 * bw + 8.0 * (np.arange(P)[:, None] - (P - 1) / 2) + rng.normal(0.0, 1.0, size=(P, 1))
        body[..., 1] += 0.5 * bh + rng.normal(0.0, 3.0, size=(P, 1))
        return body
    scale = rng.uniform(0.7, 3.5, size=(P, 1, 1))
    body = synth._TEMPLATE[None] * scale + rng.normal(0.0, 0.6, size=(P, 18, 2))
    body[..., 0] += rng.uniform(0.0, bw - 1.0, size=(P, 1))
    body[..., 1] += rng.uniform(0.0, bh - 1.0, size=(P, 1))
    return body


def network_output(spec, s, h, w):
    """What the network answers for (image, mirror) of the item at scale ``s`` of ``scale_search``: ``[2, 50, h, w]``
    float32 in the network's channel layout; the persons are those of the scale-1 crop, drawn ``s`` times larger."""
    from improved_body_parts_b200 import skeleton, synth
    _, _, H1, W1, _, _ = geometry(spec.H, spec.W, 1.0)
    joints = _skeletons(spec, (H1 / 4, W1 / 4)) * s
    rng = np.random.default_rng(spec.seed + 1)
    noise = 0.0 if spec.twins else synth.NOISE_MAX  # the twins' maps are exact translates of each other
    visible = np.ones(joints.shape[:2], bool)
    heat, paf = synth.render(joints, visible, h, w, rng, noise=noise, sigma_scale=s)
    if spec.persons >= 20:  # a crowd's limb maps blur into one wide band, as a network's do: many candidates per limb
        paf = synth.render(joints, visible, h, w, rng, noise=noise, sigma_scale=3 * s)[1]
    out = np.zeros((2, 50, h, w), np.float32)
    out[0, :30], out[0, 30:48] = paf, heat
    out[1, :30] = paf[np.argsort(skeleton.FLIP_PAF_ORD)][..., ::-1]
    out[1, 30:48] = heat[np.argsort(skeleton.FLIP_HEAT_ORD[:18])][..., ::-1]
    if not spec.twins:
        out[1] += (rng.random((50, h, w), dtype=np.float32) - 0.5) * np.float32(0.004)
    return out


@dataclasses.dataclass(frozen=True)
class Config:
    name: str
    scale_search: tuple
    rotation_search: tuple = (0.0,)
    variant: str = "evaluate"
    images: tuple = tuple(range(len(FIXTURE)))  # fixture entries the configuration runs on
    nan_items: bool = False  # a few NaN values in every network output (the demo variant scrubs them)

    def params(self):
        from improved_body_parts_b200 import skeleton
        return dict(skeleton.default_params(), scale_search=list(self.scale_search),
                    rotation_search=list(self.rotation_search))

    def group_params(self):
        """The grouping parameters ``dropin`` runs with (the demo variant's three deviations included), as a dict."""
        from improved_body_parts_b200 import skeleton
        p = self.params()
        return dataclasses.asdict(skeleton.GroupParams.demo(p) if self.variant == "demo" else
                                  skeleton.GroupParams.from_dict(p))


#: the reference default; four scales (float64 planes, fused items); five scales (past one launch's items, sums continued
#: through memory); a rotation search; the demo variant.  The CPU chain at 640 x 896 and beyond costs seconds per item,
#: so the configurations past the default run on a few images: one non-identity and one identity second resize each.
CONFIGS = {
    "default": Config("default", (1.0,)),
    "scales4": Config("scales4", (0.5, 1.0, 1.5, 2.0), images=(0, 3)),
    "scales5": Config("scales5", (0.5, 1.0, 1.5, 2.0, 0.75), images=(1,)),
    "rotation": Config("rotation", (1.0,), (0.0, 15.0, -15.0), images=(0, 3)),
    "demo": Config("demo", (1.0,), variant="demo", images=(0, 2, 3, 5), nan_items=True),
}


def items(cfg, i):
    """Per item of ``product(multiplier, rotation_search)`` (evaluate.py:90) of fixture entry i:
    ``(s, angle, geometry, network output)``; the rotated items of a scale share its network output."""
    spec = FIXTURE[i]
    outs = {}
    res = []
    for s, angle in itertools.product(cfg.scale_search, cfg.rotation_search):
        geo = geometry(spec.H, spec.W, s)
        if s not in outs:
            o = network_output(spec, s, geo[4] // 4, geo[5] // 4)
            if cfg.nan_items:
                rng = np.random.default_rng(spec.seed + 5)
                o[rng.random(o.shape) < 2e-4] = np.nan
            outs[s] = o
        res.append((s, angle, geo, outs[s]))
    return res


class StandIn:
    """The network: ``model(x)[-1][0]`` is, per sample pair of ``x [2k, Hp, Wp, 3]``, the output ``items`` gives for the
    image whose marker the pair's first sample carries.  Pure device operations (a max, a table lookup, a gather), so
    a CUDA graph can hold it; the tables are built up front."""

    def __init__(self, torch, dev, cfg):
        self.torch = torch
        self.tables = {}
        for i in cfg.images:
            for _, _, geo, out in items(cfg, i):
                rows = self.tables.setdefault((geo[4], geo[5]), {})
                rows[i] = out
        for key, rows in self.tables.items():
            lut = torch.zeros(256, dtype=torch.long)
            order = sorted(rows)
            for r, i in enumerate(order):
                lut[i] = r
            self.tables[key] = (lut.to(dev), torch.from_numpy(np.stack([rows[i] for i in order])).to(dev))

    def __call__(self, x):
        t = self.torch
        n, Hp, Wp, _ = x.shape
        lut, outs = self.tables[(int(Hp), int(Wp))]
        code = t.round((x[0::2, :, :, 0].amax(dim=(1, 2)) * 255 - MARKER0) / MARKER_STEP).long().clamp(0, 255)
        return [[outs[lut[code]].reshape(n, 50, Hp // 4, Wp // 4)]]


@dataclasses.dataclass
class Chain:
    heat: np.ndarray     # [H, W, 18] float32, what find_peaks reads (evaluate.py:173)
    paf: np.ndarray      # [H, W, 30] float64
    oracle: object       # spg_oracle.OracleResult of the image
    structs: tuple       # (all_peaks, connection_all, special_k, subset, candidate)
    people: list         # dropin.keypoints(subset, candidate)


def cpu_maps(cfg, i):
    """evaluate.py:126-161 on the stand-in's outputs: every item through the ports, float64 sums in item order (the demo
    variant's NaN scrub after every item, demo_image.py:179-180)."""
    from improved_body_parts_b200 import skeleton
    from oracle import postnet_port as pp
    from oracle import postnet_rotation_port as pr
    spec = FIXTURE[i]
    its = items(cfg, i)
    heat_avg, paf_avg = np.zeros((spec.H, spec.W, 18)), np.zeros((spec.H, spec.W, 30))
    for s, angle, (_, _, H1, W1, Hp, Wp), out in its:
        M = pr.rotation_matrices((Hp, Wp), angle)[1] if angle != 0 else None
        hm, pf = pr.post_network_item(out, 4, (Hp, Wp), [0, 0, Hp - H1, Wp - W1], (spec.H, spec.W), 30, 48,
                                      skeleton.FLIP_PAF_ORD, skeleton.FLIP_HEAT_ORD[:18], rotate_matrix=M)
        heat_avg = pp.accumulate(heat_avg, hm, len(its))
        paf_avg = pp.accumulate(paf_avg, pf, len(its))
        if cfg.variant == "demo":
            heat_avg[np.isnan(heat_avg)] = 0.0
            paf_avg[np.isnan(paf_avg)] = 0.0
    return heat_avg.astype(np.float32), paf_avg


def cpu_chain(cfg, i):
    from improved_body_parts_b200 import dropin, skeleton
    from oracle import spg_oracle as so
    heat, paf = cpu_maps(cfg, i)
    o = so.group_batch(np.ascontiguousarray(heat.transpose(2, 0, 1))[None], np.ascontiguousarray(paf.transpose(2, 0, 1))[None],
                       skeleton.LIMBS, FIXTURE[i].H, cfg.group_params())
    assert o.status[0] == 0, f"image {i}: checker status {o.status[0]}"
    structs = o.as_reference_structures(0)
    return Chain(heat, paf, o, structs, dropin.keypoints(structs[3], structs[4]))


def coverage(chains, mid_num=20, radius=2):
    """What the chain's results reach: the largest number of candidates of one limb, the share of scored pairs (two peaks
    of a limb's parts at distinct positions) that take all ``mid_num`` samples (``round(norm + 1) >= mid_num``,
    evaluate.py:226), and the images with a peak whose refine box (``radius``) leaves the map."""
    from improved_body_parts_b200 import skeleton
    max_cands, full, scored, border = 0, 0, 0, []
    for i, c in chains.items():
        max_cands = max(max_cands, int(c.oracle.cand_count[0].max()))
        peaks = c.structs[0]
        for a, b in skeleton.LIMBS:
            if not peaks[a] or not peaks[b]:
                continue
            pa = np.array([(float(p[0]), float(p[1])) for p in peaks[a]])
            pb = np.array([(float(p[0]), float(p[1])) for p in peaks[b]])
            norm = np.hypot(pb[None, :, 0] - pa[:, None, 0], pb[None, :, 1] - pa[:, None, 1])
            scored += int((norm > 0).sum())
            full += int((np.rint(norm + 1) >= mid_num).sum())
        H, W = c.heat.shape[:2]
        n = c.oracle.n_peaks(0)
        x, y = c.oracle.pxi[0, :n], c.oracle.pyi[0, :n]
        if ((x < radius) | (y < radius) | (x > W - 1 - radius) | (y > H - 1 - radius)).any():
            border.append(i)
    return dict(max_cands=max_cands, full_samples=full / max(scored, 1), border_images=border)
