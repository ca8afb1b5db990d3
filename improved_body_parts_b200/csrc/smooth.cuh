// smooth.cuh -- tracked people's keypoints smoothed across a stream's frames (include/spgroup.h "smoothing"): a
// One-Euro filter per track and joint, its state in a table of slots keyed by track id, one CTA per stream of a call.
// The frame table travels as a __grid_constant__ parameter with one CTA per frame, as track.cuh's does; the CTA of a
// stream's first frame in the call runs that stream's frames in order and the others return.
#pragma once

#include "../../include/spgroup.h"
#include "common.cuh"

namespace spg {

constexpr int kSmoothThreads = 512;
constexpr int kSmoothJoints = 17;
constexpr int kSmoothSlots = SPG_TRACK_SLOTS;
// per person row, in dynamic shared memory: its scale (double), its slot (int) and its used joints (unsigned)
constexpr size_t kSmoothRowBytes = sizeof(double) + sizeof(int) + sizeof(unsigned);

// One frame of a call.
struct SmoothFrame {
    const unsigned char *record;
    const int *stream;
    const long long *ids;
    const double *time;
    double *xy;
    int first_cta;  // the frame's CTA (fill_table)
};
constexpr int kSmoothTableMax = (int)((kParamBytes - 64) / sizeof(SmoothFrame));
struct SmoothRagged {
    int n;
    SmoothFrame img[kSmoothTableMax];
};

static_assert(sizeof(SmoothRagged) + 64 <= kParamBytes, "a launch's parameters fit the kernel-parameter limit");
static_assert(sizeof(spg_smooth_slot) == 24 + kSmoothJoints * 5 * 8 &&
              sizeof(spg_smooth_table) == 16 + kSmoothSlots * sizeof(spg_smooth_slot), "spg_smooth_table layout");
static_assert(sizeof(spg_smooth_frame) == 40, "spg_smooth_frame layout");

}  // namespace spg
