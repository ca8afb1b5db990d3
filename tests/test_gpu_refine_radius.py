"""GPU: the persistent peak finder at every refinement radius, against the CPU checker with zero tolerance.

nms_peaks_persist_kernel is compiled once per offset_radius (0 .. kMaxRefineRadius), so each radius is a kernel of its
own.  Each runs on a seeded 30-person batch whose planes outnumber the CTAs more than six times over (every plane slot
and peak list of the rings is reused), once with a peak capacity that some plane fills exactly and once with one that
many planes exceed.  Planes within the capacity must equal the checker's peaks bit for bit; a plane over it must keep
the checker's count, raise ST_PEAK_OVERFLOW and keep only peaks the checker has, bit for bit, in raster order.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_IMAGES = 64  # 64 x 18 planes over at most 132 CTAs: > 6 planes per CTA


@pytest.fixture(scope="module")
def batch():
    from improved_body_parts_b200 import synth

    return synth.make_batch(90210, N_IMAGES, 128, 128, 30, spikes=20)


def _checker_peaks(o, n, K):
    """Per part of image n: the checker's peaks as (anchor, x, y, score) tuples in raster order."""
    off = np.concatenate([[0], np.cumsum(o.part_count[n])])
    out = []
    for c in range(K):
        g = np.arange(off[c], off[c + 1])
        anchor = (o.pyi[n, g].astype(np.uint32) << 16) | o.pxi[n, g].astype(np.uint32) | (o.pint[n, g].astype(np.uint32) << 31)
        out.append((anchor, o.px[n, g], o.py[n, g], o.pscore[n, g]))
    return out


@pytest.mark.parametrize("radius", [0, 1, 2, 3, 4])
def test_persistent_peak_finder_at_every_radius(cuda_device, batch, radius):
    import torch
    from improved_body_parts_b200 import grouping as G, skeleton
    from oracle import spg_oracle as so

    heat, paf = batch
    params = dict(skeleton.default_params(), offset_radius=radius)
    o = so.group_batch(heat, paf, skeleton.LIMBS, 128, params, threads=4)
    K = heat.shape[1]
    counts = o.part_count[:, :K]
    ref = [_checker_peaks(o, n, K) for n in range(N_IMAGES)]
    reached = int(counts.max())
    exceeded = int(np.percentile(counts, 25))
    assert reached <= 128 and (counts > exceeded).sum() > 100, "the batch no longer spans the capacities"
    for capP in (reached, exceeded):
        g = G.Grouper(max_batch=N_IMAGES, max_peaks_per_part=capP, max_person_rows=128)
        try:
            g.nms_peaks(torch.from_numpy(heat).to(cuda_device), params)
            assert g.stage_kernels()[0] == "nms_peaks_persist_kernel", g.stage_kernels()
            r = g.fetch()
        finally:
            g.close()
        assert np.array_equal(r.peak_count, counts), f"radius {radius}, capP {capP}: peak counts differ"
        assert np.array_equal((r.status & G.ST_PEAK_OVERFLOW) != 0, (counts > capP).any(axis=1)), f"radius {radius}, capP {capP}"
        for n in range(N_IMAGES):
            for c in range(K):
                a_ref, x_ref, y_ref, s_ref = ref[n][c]
                m = min(int(counts[n, c]), capP)
                a, x, y, s = (r.peak_anchor[n, c, :m], r.peak_x[n, c, :m], r.peak_y[n, c, :m], r.peak_score[n, c, :m])
                where = f"radius {radius}, capP {capP}, image {n}, part {c}"
                if counts[n, c] <= capP:
                    sel = np.arange(m)
                else:  # the kept peaks are some of the checker's, in raster order
                    assert np.all(np.diff(a & 0x7fffffff) > 0), where
                    sel = np.searchsorted(a_ref & 0x7fffffff, a & 0x7fffffff)
                    assert np.all(sel < len(a_ref)), where
                assert np.array_equal(a, a_ref[sel]), where
                assert np.array_equal(x.view(np.uint64), x_ref[sel].view(np.uint64)), where
                assert np.array_equal(y.view(np.uint64), y_ref[sel].view(np.uint64)), where
                assert np.array_equal(s.view(np.uint32), s_ref[sel].view(np.uint32)), where
