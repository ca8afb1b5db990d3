"""GPU: the training-sample kernels (spg_targets_warp / spg_targets_maps) against the numpy port, bit for bit, and the
public interface of improved_body_parts_b200/targets.py."""
import os
import random

import numpy as np
import pytest

import targets_port as tp
from improved_body_parts_b200 import grouping, skeleton, targets

pytestmark = pytest.mark.gpu
CASES = tp.golden_paths()
SPACE = tp.golden_paths("targets_space")


def _ulp(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _kernels(cuda_device, z):
    """image, mask_miss, mask_all, labels of a golden case from the kernels, with the case's M, joints, stride,
    parameters and limb table."""
    import torch
    cfg = tp.target_config(z)
    params = targets.target_params(cfg)
    n, m = z["size"], z["size"] // cfg.stride
    src = [torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device) for a in (z["img"], z["mask_miss_src"], z["mask_all_src"])]
    out = [torch.empty(s, dtype=torch.float32, device=cuda_device)
           for s in ((n, n, 3), (m, m), (m, m), (cfg.num_layers, m, m))]
    h, w = z["img"].shape[:2]
    ws = np.zeros(1, grouping.TARGET_SAMPLE)
    ws[0] = (src[0].data_ptr(), src[1].data_ptr(), src[2].data_ptr(), 3 * w, w, h, w, z["M"].reshape(6), out[0].data_ptr(),
             out[1].data_ptr(), out[2].data_ptr())
    j = torch.from_numpy(np.ascontiguousarray(z["joints"], np.float32)).to(cuda_device)
    wj = np.zeros(1, grouping.TARGET_JOINTS)
    wj[0] = (j.data_ptr(), z["joints"].shape[0], 0, out[2].data_ptr(), out[3].data_ptr())
    g = targets._Device.grouper(cfg, 0)
    g.targets_warp(params, ws)
    g.targets_maps(params, wj)
    assert (g._lib.spg_stage_kernel(g._h, 6) or b"").decode() == "targets_maps_kernel"
    return [t.cpu().numpy() for t in out]


def _hold_the_golden_contract(z, im, mm, ma, lab):
    """The reference's own output: image, masks and channel L+K exact, body parts within 1 ULP, keypoints and channel
    L+K+1 within 5 ULP with the same zeros."""
    L, ref = len(tp.case_params(z)["limbs"]), z["labels"]
    assert lab.shape == ref.shape
    assert np.array_equal(im, z["image"]) and np.array_equal(mm, z["mask_miss"]) and np.array_equal(ma, z["mask_all"])
    assert np.array_equal(lab[L + 18], ref[L + 18])
    assert _ulp(lab[:L], ref[:L]).max(initial=0) <= 1
    for c in list(range(L, L + 18)) + [L + 19]:
        assert np.array_equal(lab[c] == 0, ref[c] == 0) and _ulp(lab[c], ref[c]).max() <= 5, c


@pytest.mark.parametrize("path", CASES + SPACE, ids=lambda p: os.path.basename(p)[:-4])
def test_kernels_equal_the_port_and_hold_the_golden_contract(cuda_device, path):
    z = tp.load_case(path)
    im, mm, ma, lab = _kernels(cuda_device, z)
    pim, pmm, pma, plab = tp.port_case(z, "rounded")
    assert np.array_equal(im, pim) and np.array_equal(mm, pmm) and np.array_equal(ma, pma)
    for c in range(len(plab)):
        assert np.array_equal(lab[c].view(np.int32), plab[c].view(np.int32)), f"channel {c}"
    _hold_the_golden_contract(z, im, mm, ma, lab)


@pytest.mark.parametrize("path", [p for p in SPACE if os.path.basename(p).startswith(("s2_", "s8_"))],
                         ids=lambda p: os.path.basename(p)[:-4])
def test_make_batch_holds_the_golden_contract_at_strides_2_and_8(cuda_device, path):
    """make_batch from the golden's source, meta and augmentation with a config of its stride and parameters."""
    z = tp.load_case(path)
    cfg = tp.target_config(z)
    aug = targets.AugmentSelection(bool(z["aug_flip"]), False, float(z["aug_degree"]), tuple(int(v) for v in z["aug_crop"]),
                                   float(z["aug_scale"]))
    meta = {"objpos": [list(z["objpos"])], "scale_provided": [float(z["scale_provided"])], "joints": z["joints_src"]}
    images, miss, labels = targets.make_batch([(z["img"], z["mask_miss_src"], z["mask_all_src"], meta)], [aug], cfg)
    im, mm, lab = images[0].cpu().numpy(), miss[0, 0].cpu().numpy(), labels[0].cpu().numpy()
    L = len(cfg.limbs_conn)
    _hold_the_golden_contract(z, im, mm, z["mask_all"], lab)
    assert np.array_equal(lab[L + 18], tp.erode3(z["mask_all"]))


def _ragged_batch(seed, n=64, size=256):
    rng = np.random.default_rng(seed)
    random.seed(seed)
    cfg = targets.TargetConfig(size, size)
    sizes = [(480, 640), (640, 427), (375, 500), (1, 1), (333, 250), (612, 612)]
    samples, augs = [], []
    for i in range(n):
        h, w = sizes[i % len(sizes)]
        P = 100 if i == 7 else int(rng.integers(0, 31))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        mm = np.where(rng.random((h, w)) < 0.1, 0, 255).astype(np.uint8)
        ma = np.where(rng.random((h, w)) < 0.3, 255, 0).astype(np.uint8)
        j = np.zeros((P, 18, 3))
        j[:, :, 0:2] = rng.uniform([-50, -50], [w + 50, h + 50], (P, 18, 2))
        j[:, :, 2] = rng.choice([0, 1, 2], (P, 18), p=[0.3, 0.5, 0.2])
        meta = {"objpos": [[float(rng.uniform(0, w)), float(rng.uniform(0, h))]],
                "scale_provided": [float(rng.uniform(0.2, 1.2))], "joints": j}
        aug = targets.AugmentSelection.random(cfg.transform_params)
        aug.tint = False
        samples.append((img, mm, ma, meta))
        augs.append(aug)
    return cfg, samples, augs


def test_make_batch_equals_the_port_on_a_ragged_batch(cuda_device):
    cfg, samples, augs = _ragged_batch(11)
    images, miss, labels = targets.make_batch(samples, augs, cfg)
    images, miss, labels = images.cpu().numpy(), miss.cpu().numpy(), labels.cpu().numpy()
    for i, ((img, mm, ma, meta), aug) in enumerate(zip(samples, augs)):
        M, _ = aug.affine(meta["objpos"][0], meta["scale_provided"][0], cfg)
        joints = targets.transform_joints(meta["joints"], M, aug.flip, cfg).astype(np.float32)
        pim, pmm, pma = tp.warp_sample(img, mm, ma, M, (cfg.width, cfg.height), cfg.stride)
        plab = tp.label_maps(joints, pma, skeleton.LIMBS, 4, 9, 7, 0.015, 4, 14, exp="rounded")
        assert np.array_equal(images[i], pim) and np.array_equal(miss[i, 0], pmm), i
        assert np.array_equal(labels[i].view(np.int32), plab.view(np.int32)), i


def test_make_batch_equals_transform_and_create_heatmaps_and_is_composition_free(cuda_device):
    import copy
    cfg, samples, augs = _ragged_batch(12, n=9)
    images, miss, labels = (t.cpu().numpy() for t in targets.make_batch(samples, augs, cfg))
    tr, hm = targets.Transformer(cfg), targets.Heatmapper(cfg)
    for i, ((img, mm, ma, meta), aug) in enumerate(zip(samples, augs)):
        ti, tm, ta, m2 = tr.transform(img, mm, ma, copy.deepcopy(meta), aug)
        lab = hm.create_heatmaps(m2["joints"].astype(np.float32), ta)
        assert np.array_equal(images[i], ti) and np.array_equal(miss[i, 0], tm) and np.array_equal(labels[i], lab), i
        alone = [t.cpu().numpy() for t in targets.make_batch([samples[i]], [aug], cfg)]
        assert np.array_equal(alone[0][0], images[i]) and np.array_equal(alone[1][0], miss[i])
        assert np.array_equal(alone[2][0], labels[i])


# a standing skeleton in image pixels relative to (centre x, top), parts in skeleton.PART_NAMES order
_TEMPLATE = np.array([(0, 0), (0, 48), (-32, 48), (-44, 104), (-48, 160), (32, 48), (44, 104), (48, 160), (-20, 168),
                      (-24, 248), (-24, 328), (20, 168), (24, 248), (24, 328), (-8, -8), (8, -8), (-18, 0), (18, 0)],
                     np.float64)


def test_round_trip_skeletons_to_labels_to_grouping(cuda_device):
    import torch
    cfg = targets.TargetConfig()
    hm = targets.Heatmapper(cfg)
    rng = np.random.default_rng(3)
    labels, expected = [], []
    for n in range(2):
        xs = np.array([100.0, 256.0, 412.0]) + rng.uniform(-6, 6, 3)
        j = np.zeros((3, 18, 3), np.float32)
        for p, x in enumerate(xs):
            j[p, :, 0:2] = _TEMPLATE + (x, 70.0 + rng.uniform(-8, 8)) + rng.uniform(-2, 2, (18, 2))
            j[p, :, 2] = 1
        labels.append(hm.create_heatmaps(j, np.zeros((128, 128), np.float32)))
        expected.append((j[:, :, 0:2] - cfg.stride / 2 + 0.5) / cfg.stride)
    lab = torch.from_numpy(np.stack(labels)).to(cuda_device)
    with grouping.Grouper(max_batch=2, device=0) as g:
        g.group_device(lab[:, 30:48], lab[:, 0:30], 128.0)
        r = g.fetch()
    for n in range(2):
        assert int(r.n_persons[n]) == 3, r.n_persons
        found = r.people_xy[n, :3]  # [3, 17, 2] COCO order
        for p in range(3):
            want = expected[n][p][list(skeleton.COCO_FROM_PART)]
            best = min(range(3), key=lambda q: np.abs(found[q] - want).max())
            assert np.abs(found[best] - want).max() <= 1.0, (n, p, found[best], want)


# members per launch of the training-sample kernels: kTgtWarpMax, kTgtMapsMax, kTgtTintMax in csrc/targets.cuh
WARP_TABLE, MAPS_TABLE, TINT_TABLE = 247, 784, 682


def test_more_samples_than_one_table_holds(cuda_device):
    """800 tiny samples through targets_tint, targets_warp and targets_maps, one call each: every kernel's launches split
    at its table's capacity, and every sample equals a call of its own."""
    import torch
    n, h, w, P = 800, 6, 7, 2
    cfg = targets.TargetConfig(8, 8)
    params = targets.target_params(cfg)
    g = targets._Device.grouper(cfg, 0)
    rng = np.random.default_rng(23)
    src = torch.from_numpy(rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)).to(cuda_device)
    masks = torch.from_numpy(rng.integers(0, 256, (2, n, h, w), dtype=np.uint8)).to(cuda_device)
    joints = np.zeros((n, P, 18, 3), np.float32)
    joints[..., 0:2] = rng.uniform(-2, 10, (n, P, 18, 2))
    joints[..., 2] = rng.choice([0, 1, 2], (n, P, 18))
    joints = torch.from_numpy(joints).to(cuda_device)
    n_persons = rng.integers(0, P + 1, n)
    mats = np.zeros((n, 2, 3))
    for i in range(n):
        a, s = rng.uniform(-np.pi, np.pi), rng.uniform(0.7, 1.4)
        mats[i] = [[s * np.cos(a), -s * np.sin(a), rng.uniform(-2, 6)], [s * np.sin(a), s * np.cos(a), rng.uniform(-2, 6)]]
    draws = [(int(rng.integers(0, 21)), int(rng.integers(0, 81)), int(rng.integers(0, 61))) for _ in range(n)]

    def outputs():
        return (torch.full((n, 8, 8, 3), -1.0, device=cuda_device), torch.full((2, n, 2, 2), -1.0, device=cuda_device),
                torch.full((n, 50, 2, 2), -1.0, device=cuda_device))

    def run(idx, img, out):
        g.targets_tint(targets.tint_records([(img[i].data_ptr(), 3 * w, h, w) for i in idx], [draws[i] for i in idx]))
        ws = np.zeros(len(idx), grouping.TARGET_SAMPLE)
        wj = np.zeros(len(idx), grouping.TARGET_JOINTS)
        for k, i in enumerate(idx):
            ws[k] = (img[i].data_ptr(), masks[0, i].data_ptr(), masks[1, i].data_ptr(), 3 * w, w, h, w, mats[i].reshape(6),
                     out[0][i].data_ptr(), out[1][0, i].data_ptr(), out[1][1, i].data_ptr())
            wj[k] = (joints[i].data_ptr(), n_persons[i], 0, out[1][1, i].data_ptr(), out[2][i].data_ptr())
        g.targets_warp(params, ws)
        g.targets_maps(params, wj)

    batch_src, alone_src = src.clone(), src.clone()
    batch, alone = outputs(), outputs()
    before = g.launch_count
    run(range(n), batch_src, batch)
    ranges = [-(-n // c) for c in (TINT_TABLE, WARP_TABLE, MAPS_TABLE)]
    assert ranges == [2, 4, 2] and g.launch_count - before == sum(ranges)
    for i in range(n):
        run([i], alone_src, alone)
    assert torch.equal(batch_src, alone_src) and not torch.equal(batch_src, src)
    for b, a in zip(batch, alone):
        assert (b >= 0).all() and torch.equal(b.view(torch.int32), a.view(torch.int32))
