"""The training loss's case table: seeded (stack count, weights, channel layout, target shape, batch divisor) cases that
together cover what ``improved_body_parts_b200.loss`` admits, each well under 2 GB of device memory with the port's
autograd beside it.  ``tests/test_gpu_loss_space.py`` runs them; ``tests/test_loss_host.py`` checks the coverage."""
from __future__ import annotations

from typing import List, NamedTuple, Tuple

SW = [0.1, 0.2, 0.4, 1.6, 6.4]


class LossCase(NamedTuple):
    name: str
    focal: bool
    nstack_weight: List[float]
    scale_weight: List[float]
    B: int
    C: int                    # label channels (MultiTaskLossParallel: offset_start)
    H: int
    W: int
    heat: Tuple[int, int]     # focal: (heat_start, bkg_start)
    batch_size: int           # focal: the divisor, opt.batch_size
    grad_output: float
    seed: int
    extra: int = 0            # l2: prediction channels past offset_start

    @property
    def nstack(self) -> int:
        return len(self.nstack_weight)

    @property
    def pred_channels(self) -> int:
        return self.C + self.extra


CASES = [
    # 16 x 16: the coarsest scale is 1 x 1; an empty keypoint range at 0; the divisor below B
    LossCase("ns1_c2_16x16", True, [2.5], SW, 3, 2, 16, 16, (0, 0), 2, 3.0, 1),
    # one band of 16 rows; the keypoint range starts at 0; the divisor above B
    LossCase("ns2_c3_16x256", True, [0.1, 2.5], SW, 2, 3, 16, 256, (0, 1), 5, 65536.0, 2),
    # one column of 16: every scale past 0 takes scalar accesses; a stack weight of 0; the range ends at C
    LossCase("ns3_c12_256x16", True, [0.0, 1.0, 0.3], SW, 2, 12, 256, 16, (2, 12), 2, 1.0, 3),
    # an odd C whose range covers C - 2; W = 80 switches between vector and scalar access
    LossCase("ns4_c57_48x80", True, [1.0, 0.3, 0.1, 2.5], SW, 2, 57, 48, 80, (1, 56), 2, 3.0, 4),
    # more than 20 (scale, stack) slots; a scale weight of 0; B = 1
    LossCase("ns5_c50_112x208", True, [1.0, 2.5, 0.1, 0.3, 1.0], [0.1, 0.2, 0.0, 1.6, 6.4], 1, 50, 112, 208, (30, 48), 1,
             0.5, 5),
    # L2 at B = 16, predictions 3 channels past offset_start
    LossCase("ns6_l2_c3_128x128_b16", False, [1.0, 0.1, 0.3, 2.5, 0.0, 1.0], SW, 16, 3, 128, 128, (0, 0), 16, 3.0, 6, 3),
    # the last CTA's loop over 35 slots passes 32; an empty range past 0
    LossCase("ns7_c2_256x384_b2", True, [0.3, 1.0, 2.5, 0.1, 1.0, 0.0, 1.0], SW, 2, 2, 256, 384, (1, 1), 2, 1.0, 7),
    # 40 slots at B = 1 and 512 x 512; an empty range at C (bkg_start == C)
    LossCase("ns8_c3_512x512_b1", True, [1.0, 0.1, 0.3, 2.5, 1.0, 1.0, 0.0, 1.0], SW, 1, 3, 512, 512, (3, 3), 1, 3.0, 8),
    # L2 with 8 stacks and 50 channels plus 3
    LossCase("ns8_l2_c50_64x96", False, [2.5, 1.0, 0.3, 0.1, 1.0, 1.0, 0.0, 1.0], SW, 2, 50, 64, 96, (0, 0), 2, 65536.0, 9,
             3),
]


def device_bytes(c: LossCase) -> int:
    """An upper bound on the device memory a case takes with the port beside it: the targets, the predictions with
    their gradients twice over, and the port's ~12 tensors of [nstack, B, C, h, w] float32 per scale."""
    px = sum((c.H >> j) * (c.W >> j) for j in range(5))
    pred = c.B * c.pred_channels * px * 4 * c.nstack
    return c.B * (c.C + 1) * c.H * c.W * 4 + 4 * pred + 12 * pred
