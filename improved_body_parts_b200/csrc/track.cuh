// track.cuh -- people tracked across a stream's frames (include/spgroup.h "tracking"): the OKS of every live track with
// every person of a frame, greedy matching, and the table's update, one CTA per stream of a call.  The frame table
// travels as a __grid_constant__ parameter with one CTA per frame; the CTA of a stream's first frame in the call runs
// that stream's frames in order and the others return, so which frames share a stream is read on the device and a
// recorded launch serves any assignment of frames to streams.
#pragma once

#include "../../include/spgroup.h"
#include "common.cuh"

namespace spg {

constexpr int kTrackThreads = 512;
constexpr int kTrackJoints = 17;
constexpr int kTrackSlots = SPG_TRACK_SLOTS;
// the OKS matrix of one frame, [slot][person row], in dynamic shared memory
constexpr size_t kTrackSmem = (size_t)kTrackSlots * kTrackSlots * sizeof(double);

// One frame of a call.
struct TrackFrame {
    const unsigned char *record;
    const int *stream;
    const int *jpeg_status;  // may be null
    long long *ids;
    double *oks;             // may be null
    int first_cta;           // the frame's CTA (fill_table)
};
constexpr int kTrackTableMax = (int)((kParamBytes - 64) / sizeof(TrackFrame));
struct TrackRagged {
    int n;
    TrackFrame img[kTrackTableMax];
};

static_assert(sizeof(TrackRagged) + 64 <= kParamBytes, "a launch's parameters fit the kernel-parameter limit");
static_assert(sizeof(spg_track) == 296 && sizeof(spg_track_table) == 16 + kTrackSlots * 296, "spg_track_table layout");

}  // namespace spg
