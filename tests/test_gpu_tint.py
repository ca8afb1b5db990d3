"""GPU: the colour distortion kernel (spg_targets_tint) against the numpy port bit for bit and against the reference's
goldens, and make_batch / Transformer with tint=True."""
import copy
import os
import random

import numpy as np
import pytest

import tint_port as tt
from improved_body_parts_b200 import grouping, targets

pytestmark = pytest.mark.gpu
COLOR = tt.golden_paths("color")
GEN = tt.golden_paths("gen")


def _ulp(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _tint(cuda_device, views, draws, row_block=32):
    """Tint uint8 [h, w, 3] CUDA views (rows may be strided) in place, one call."""
    g = targets._Device.grouper(targets.TargetConfig(), 0)
    recs = targets.tint_records([(v.data_ptr(), v.stride(0), v.shape[0], v.shape[1]) for v in views], draws, row_block)
    g.targets_tint(recs)
    assert (g._lib.spg_stage_kernel(g._h, 6) or b"").decode() == "targets_tint_kernel"


@pytest.mark.parametrize("draws,block", [((10, 20, 20), 32), ((10, 20, 20), 1 << 30), ((0, 0, 0), 32),
                                         ((20, 80, 60), 32), ((3, 71, 9), 32), ((17, 5, 44), 1 << 30)])
def test_every_triple_equals_the_port(cuda_device, draws, block):
    """All 2^24 BGR triples in rows 4096 wide: block 32 leaves no tail, block 2^30 makes every pixel tail."""
    import torch
    t = tt.all_triples().reshape(4096, 4096, 3)
    d = torch.from_numpy(t).to(cuda_device)
    _tint(cuda_device, [d], [draws], block)
    assert np.array_equal(d.cpu().numpy(), tt.distort_color(t, draws, block))


def test_a_ragged_batch_of_every_tail_length_and_alignment(cuda_device):
    """Widths 1..64 and 427 (every width % 32), heights 1..5, rows contiguous or strided at offsets of 0..17 bytes into
    a wider buffer, with their own draws: one call."""
    import torch
    rng = np.random.default_rng(7)
    srcs, views, draws = [], [], []
    for k, w in enumerate(list(range(1, 65)) + [427, 640]):
        h, pad = 1 + k % 5, (0 if k % 3 == 0 else 1 + k % 17)
        buf = torch.from_numpy(rng.integers(0, 256, (h, 3 * w + pad + 17), dtype=np.uint8)).to(cuda_device)
        off = k % 18 if pad else 0
        views.append(torch.as_strided(buf[:, off:off + 3 * w], (h, w, 3), (buf.stride(0), 3, 1)))
        srcs.append(views[-1].cpu().numpy())
        draws.append((int(rng.integers(0, 21)), int(rng.integers(0, 81)), int(rng.integers(0, 61))))
    _tint(cuda_device, views, draws)
    for k, (v, s, d) in enumerate(zip(views, srcs, draws)):
        assert np.array_equal(v.cpu().numpy(), tt.distort_color(s, d, 32)), k


def test_bytes_outside_the_rows_are_untouched(cuda_device):
    import torch
    buf = torch.from_numpy(np.arange(7 * 200, dtype=np.int64).astype(np.uint8).reshape(7, 200)).to(cuda_device)
    ref = buf.cpu().numpy()
    v = torch.as_strided(buf[:, 5:5 + 3 * 61], (7, 61, 3), (200, 3, 1))
    _tint(cuda_device, [v], [(20, 80, 60)])
    got = buf.cpu().numpy()
    assert np.array_equal(got[:, :5], ref[:, :5]) and np.array_equal(got[:, 5 + 183:], ref[:, 5 + 183:])
    assert np.array_equal(got[:, 5:188].reshape(7, 61, 3), tt.distort_color(ref[:, 5:188].reshape(7, 61, 3), (20, 80, 60)))


@pytest.mark.parametrize("path", COLOR, ids=lambda p: os.path.basename(p)[:-4])
def test_kernel_equals_the_reference_golden(cuda_device, path):
    """The source as the reference saw it (a strided view of a wider source where the case has one) tinted in place."""
    import torch
    z = np.load(path)
    h, w = (int(v) for v in z["source_hw"])
    pad = int(z["pad_cols"])
    from make_targets_golden import source
    big = torch.from_numpy(source(h, w + pad)[0]).to(cuda_device)
    v = big[:, pad // 2:pad // 2 + w]
    assert v.is_contiguous() == (pad == 0)
    _tint(cuda_device, [v], [tuple(int(x) for x in z["draws"])], int(z["row_block"]))
    assert np.array_equal(v.cpu().numpy(), z["out"])


def test_distort_color_static_draws_like_the_reference(cuda_device):
    z = np.load(COLOR[0])
    np.random.seed(int(z["seed"]))
    out = targets.Transformer.distort_color(tt.color_source(z), row_block=int(z["row_block"]), device=0)
    assert np.array_equal(out, z["out"])


def test_malformed_records_raise_and_launch_nothing(cuda_device):
    import torch
    img = torch.zeros((4, 5, 3), dtype=torch.uint8, device=cuda_device)
    g = targets._Device.grouper(targets.TargetConfig(), 0)
    good = (img.data_ptr(), 15, 4, 5)
    bad = [([good, (0, 15, 4, 5)], [(0, 0, 0)] * 2, 32, "NULL"),
           ([good, (img.data_ptr(), 14, 4, 5)], [(0, 0, 0)] * 2, 32, "row_stride"),
           ([good, good], [(0, 0, 0), (21, 0, 0)], 32, "draws"),
           ([good, good], [(0, 0, 0), (0, 81, 0)], 32, "draws"),
           ([good, good], [(0, 0, 0), (0, 0, -1)], 32, "draws"),
           ([good, good], [(0, 0, 0)] * 2, 0, "row_block"),
           ([good, (img.data_ptr(), 15, 0, 5)], [(0, 0, 0)] * 2, 32, "outside")]
    launches = g.launch_count
    for imgs, draws, block, match in bad:
        with pytest.raises(grouping.GroupingError, match=match):
            g.targets_tint(targets.tint_records(imgs, draws, block))
    assert g.launch_count == launches
    assert int(img.sum()) == 0  # sample 0 was valid and was not tinted either


def _gen_samples(z):
    from make_targets_golden import source
    samples = []
    for i, (h, w) in enumerate(z["source_hw"]):
        img, mm, ma = source(int(h), int(w))
        samples.append((img, mm, ma, {"objpos": [list(z["objpos"][i])], "scale_provided": [float(z["scale_provided"][i])],
                                      "joints": z[f"joints_src_{i}"].copy()}))
    return samples


@pytest.mark.parametrize("path", GEN, ids=lambda p: os.path.basename(p)[:-4])
def test_make_batch_with_seeded_generators_equals_the_reference_gen_loop(cuda_device, path):
    z = np.load(path)
    cfg = targets.TargetConfig(int(z["size"]), int(z["size"]))
    cfg.tint_row_block = int(z["row_block"])
    samples = _gen_samples(z)
    random.seed(int(z["seed"]))
    np.random.seed(int(z["seed"]))
    images, miss, labels = (t.cpu().numpy() for t in targets.make_batch(samples, [None] * len(samples), cfg, tint=True))
    for i in range(len(samples)):
        assert np.array_equal(images[i], z["image_codes"][i].astype(np.float32) / 255.), i
        assert np.array_equal(miss[i, 0], z["mask_miss"][i]), i
        ref = z["labels"][i]
        assert np.array_equal(labels[i, 48], ref[48]) and _ulp(labels[i, :30], ref[:30]).max() <= 1, i
        for c in list(range(30, 48)) + [49]:
            assert np.array_equal(labels[i, c] == 0, ref[c] == 0) and _ulp(labels[i, c], ref[c]).max() <= 5, (i, c)


def test_make_batch_equals_transform_and_leaves_untinted_samples_alone(cuda_device):
    """A mixed batch: equal to Transformer(tint=True).transform + create_heatmaps per sample under the same seed, and
    its untinted samples byte-identical to make_batch(tint=False) on the same selections."""
    rng = np.random.default_rng(4)
    cfg = targets.TargetConfig(256, 256)
    samples, augs = [], []
    for i, (h, w) in enumerate([(480, 640), (427, 640), (1, 1), (333, 250), (375, 500), (64, 50)]):
        j = np.zeros((3, 18, 3))
        j[:, :, 0:2] = rng.uniform([0, 0], [w, h], (3, 18, 2))
        j[:, :, 2] = rng.choice([0, 1, 2], (3, 18))
        samples.append((rng.integers(0, 256, (h, w, 3), dtype=np.uint8), np.full((h, w), 255, np.uint8),
                        np.where(rng.random((h, w)) < 0.3, 255, 0).astype(np.uint8),
                        {"objpos": [[w / 2, h / 2]], "scale_provided": [0.6], "joints": j}))
        augs.append(targets.AugmentSelection(bool(i % 2), i % 3 != 1, float(rng.uniform(-40, 40)), (3, -4), 1.1))
    np.random.seed(9)
    out = [t.cpu().numpy() for t in targets.make_batch(samples, augs, cfg, tint=True)]
    np.random.seed(9)
    tr, hm = targets.Transformer(cfg, tint=True), targets.Heatmapper(cfg)
    for i, (s, aug) in enumerate(zip(samples, augs)):
        ti, tm, ta, m2 = tr.transform(s[0], s[1], s[2], copy.deepcopy(s[3]), aug)
        lab = hm.create_heatmaps(m2["joints"].astype(np.float32), ta)
        assert np.array_equal(out[0][i], ti) and np.array_equal(out[1][i, 0], tm) and np.array_equal(out[2][i], lab), i
    plain = [i for i, a in enumerate(augs) if not a.tint]
    ref = [t.cpu().numpy() for t in targets.make_batch([samples[i] for i in plain], [augs[i] for i in plain], cfg)]
    for k, i in enumerate(plain):
        assert all(np.array_equal(o[i], r[k]) for o, r in zip(out, ref)), i
    tinted = [i for i, a in enumerate(augs) if a.tint]
    assert tinted and not np.array_equal(out[0][tinted[0]], targets.make_batch(
        [samples[tinted[0]]], [targets.AugmentSelection(augs[tinted[0]].flip, False, augs[tinted[0]].degree, (3, -4), 1.1)],
        cfg)[0][0].cpu().numpy())
