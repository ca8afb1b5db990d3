"""GPU: every limb_score schedule publishes the survivor count of every (image, limb), special_k limbs included.

A limb one of whose parts has no peaks (special_k, evaluate.py:272-274) has no candidates and no survivors.  Its
survivor count must read 0 whatever the handle's memory held before, on the persistent kernel (at most 64 peaks per
part) and on the per-item kernel alike."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cap,schedule", [(64, "persist"), (128, "limb_score_kernel")])
def test_special_limbs_publish_zero_survivors(cuda_device, cap, schedule):
    import torch
    from improved_body_parts_b200 import skeleton, synth
    from improved_body_parts_b200.grouping import Grouper

    heat, paf = synth.make_batch(31, 3, 128, 128, 8)
    heat[0, 1] = 0.0  # image 0: part 1 has no peaks, so every limb of part 1 is special
    heat[2, 5] = 0.0
    g = Grouper(max_batch=3, max_h=128, max_w=128, max_peaks_per_part=cap)
    try:
        views = g.device_tensors()
        views["surv_count"].fill_(-7)  # what the memory held before: must not show through
        views["cand_count"].fill_(-7)
        torch.cuda.synchronize()
        g.group_device(torch.from_numpy(heat).to(cuda_device), torch.from_numpy(paf).to(cuda_device), 128,
                       skeleton.default_params())
        torch.cuda.synchronize()
        surv = views["surv_count"][:3].cpu().numpy()
        cand = views["cand_count"][:3].cpu().numpy()
        kernel = g.stage_kernels()[1]
    finally:
        g.close()
    assert schedule in kernel
    special = cand == -1
    limbs = np.asarray(skeleton.LIMBS)
    assert special[0][(limbs == 1).any(1)].all() and special[2][(limbs == 5).any(1)].all()
    assert (surv[special] == 0).all(), f"{kernel}: special limbs publish stale survivor counts {surv[special]}"
    assert (surv >= 0).all() and (cand >= -1).all() and (surv[~special] > 0).any()
