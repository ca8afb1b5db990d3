// yuv.cuh -- cv2.cvtColor's YUV -> BGR conversions on the device (include/spgroup.h "YUV frames"): NV12, I420 and YUYV
// with OpenCV's integer BT.601 limited-range formula, bit for bit.  One ragged launch per call: the member table travels
// as a __grid_constant__ parameter and a CTA finds its frame by binary search over first_cta (ragged_member).  A thread
// converts one 2x2 block of a 4:2:0 frame, or one 2x1 pair of a 4:2:2 frame, which share one U and one V.
#pragma once

#include "../../include/spgroup.h"
#include "common.cuh"

namespace spg {

constexpr int kYuvThreads = 256;

// One frame of a call.
struct YuvMember {
    const unsigned char *plane[3];  // NV12: Y, UV; I420: Y, U, V; YUYV: the packed plane
    long long pitch[3];
    unsigned char *out;             // [h][w][3] BGR
    long long out_pitch;
    int format;                     // SPG_YUV_*
    int h, w;
    int units;                      // blocks (4:2:0) or pairs (4:2:2) per block row: w / 2
    int first_cta;
};
constexpr int kYuvTableMax = (int)((kParamBytes - 16) / sizeof(YuvMember));
struct YuvRagged {
    int n;
    YuvMember img[kYuvTableMax];  // first_cta increasing
};
static_assert(sizeof(YuvRagged) <= kParamBytes, "a launch's parameters fit the kernel-parameter limit");

}  // namespace spg
