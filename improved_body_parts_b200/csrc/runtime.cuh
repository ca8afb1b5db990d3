// runtime.cuh -- the host runtime that every stage's translation unit shares: the handle, its scratch and its error
// text, the one launch path, and the checks and ragged-launch dealing of more than one stage.  spgroup.cu defines the
// functions declared here; what only one stage uses lives in that stage's unit.  Internal: no kernels, and nothing here
// is part of the C ABI (include/spgroup.h).
#pragma once

#include "../../include/spgroup.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include "common.cuh"

namespace spg {

// the stage numbers of spg_stage_kernel (include/spgroup.h)
enum : int { kStageNms, kStageScore, kStageMatch, kStageAssemble, kStagePostnet, kStagePrenet, kStageTargets, kStageLoss, kStageCoco, kStageJpeg, kStageYuv, kStageTrack, kStageSmooth, kStageCount };

// device scratch that grows on demand (grow) and lives until spg_destroy
struct Scratch {
    void *p = nullptr;
    size_t bytes = 0;
};

}  // namespace spg

struct spg_handle {
    spg_config cfg{};
    int device = 0;
    int sm_count = 0;
    size_t smem_optin = 0;
    std::vector<std::pair<const void *, size_t>> smem_rooms;  // smem_room's cache: kernel -> dynamic shared memory it may take
    spg::Workspace ws{};
    std::vector<void *> allocs;
    spg::Scratch in_heat, in_paf;  // staging for spg_group_host
    unsigned int *done_counter = nullptr;          // "last CTA done" counter of the in-kernel wire signal
    unsigned int *score_queue = nullptr;           // 2 x 2 words: item queues of limb_score_persist_kernel (launch_score)
    unsigned long long *armed_flag = nullptr;      // spg_arm_wire_signal: consumed by the next assemble launch
    unsigned long long armed_value = 0;
    spg::Scratch heat_acc;  // postnet: float64 accumulator of the keypoint maps over the scale loop
    spg::Scratch pre_grid;  // prenet: the padded uint8 images of a launch's rotated members
    spg::Scratch coco_sort, coco_acc;  // spg_coco_evaluate: sort keys and CUB scratch; spg_coco_accumulate: the curves
    spg::Scratch jpeg;  // spg_jpeg_decode_ragged: records, unstuffed streams, subsequence states, coefficients, planes
    // the capacity-free tier (spg_group_unbounded): fixed-size words, tables sized by the peak counts, the candidate list
    // with the sort's scratch, the person table and outputs; `ub_ws` describes the last call's results
    spg::Scratch ub_small, ub_peaks, ub_cands, ub_people;
    spg::Workspace ub_ws{};
    bool ub_valid = false;
    cudaStream_t streams[2] = {nullptr, nullptr};
    int64_t launches = 0;
    const char *stage_kernel[spg::kStageCount] = {"", "", "", "", "", "", "", "", "", "", "", "", ""};
    // tuning / A-B switches, read from the environment ONCE in spg_create (never per launch); none changes a result
    int persist = 1;      // persistent warp-specialised nms_peaks / limb_score when they apply (SPG_PERSIST=0 turns them off)
    int screen = 1;       // limb_score phase A on (SPG_NO_SCREEN=1 turns it off: every pair is evaluated exactly)
    int exact_warps = 14; // scorer warps of the persistent limb_score (SPG_EXACT_WARPS; DESIGN.md §8 has the sweep)
    int ma_warps = spg::kMAMatchWarps;  // matcher warps of the fused kernel (SPG_MA_WARPS, tuning)
    int fuse_ma = 1;      // whole-path calls run the fused match+assemble kernel (SPG_FUSE_MA=0: the two kernels back to back)
    int cand_dtype = SPG_F32;  // dtype of the planes the current candidates were scored on
    int stage = 0;  // 0 none, 1 peaks, 2 candidates, 3 connections, 4 people
    bool frames_reserved = false;  // spg_reserve_frame was called: captured calls reset the scorer's queue
    std::string err;
};

namespace spg {

// the call's error: h->err, or spg_create's (h == nullptr); returns `code`
int fail(spg_handle *h, int code, const char *fmt, ...);

#define SPG_CUDA(h, call)                                                                              \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) return fail((h), SPG_E_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_)); \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
    }
    ~DeviceGuard() {
        int cur = -1;
        cudaGetDevice(&cur);
        if (prev >= 0 && cur != prev) cudaSetDevice(prev);
    }
};

int grow(spg_handle *h, Scratch &s, size_t bytes);

// whether `st` is capturing a CUDA graph
int stream_capturing(spg_handle *h, cudaStream_t st, bool *capturing);

// grow() for a call on `st`: while `st` captures, an allocation would invalidate the capture, so a buffer below `bytes`
// is SPG_E_CAPTURE instead (`what` names the buffer); the caller has enqueued nothing yet
int grow_on(spg_handle *h, Scratch &s, size_t bytes, cudaStream_t st, const char *what);

// Every kernel launch on a handle goes through here: it raises the kernel's dynamic shared memory limit to `smem`,
// launches, records `name` as the kernel of `stage` (spg_stage_kernel), counts the launch (spg_launch_count) and turns
// a launch error into the call's error.
template <typename... P, typename... A>
int launch(spg_handle *h, int stage, const char *name, void (*kern)(P...), dim3 grid, int block, size_t smem, cudaStream_t st,
           const A &...args) {
    if (smem > 0) SPG_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, block, smem, st>>>(args...);
    h->stage_kernel[stage] = name;
    h->launches++;
    SPG_CUDA(h, cudaGetLastError());
    return SPG_OK;
}

// The dynamic shared memory a launch of `kern` may ask for: the opt-in limit less the kernel's static __shared__ arrays,
// because a block needs dynamic + static <= opt-in (cudaFuncSetAttribute refuses a larger dynamic size).  Every plan that
// sizes dynamic shared memory by the shape or the capacities compares against this, not against smem_optin.  Queried
// once per kernel and handle; if the query fails, the opt-in limit is returned and the launch reports the CUDA error.
template <typename... P>
size_t smem_room(spg_handle *h, void (*kern)(P...)) {
    const void *key = reinterpret_cast<const void *>(kern);
    for (const auto &r : h->smem_rooms)
        if (r.first == key) return r.second;
    cudaFuncAttributes fa{};
    if (cudaFuncGetAttributes(&fa, kern) != cudaSuccess) return h->smem_optin;
    const size_t room = fa.sharedSizeBytes < h->smem_optin ? h->smem_optin - fa.sharedSizeBytes : 0;
    h->smem_rooms.emplace_back(key, room);
    return room;
}

// Every ragged launch's table boundaries: given each member's CTA count, consecutive ranges of at most `capacity`
// members (the kernel's table) and at most 2^31 - 1 CTAs (grid.x), and each member's first CTA inside its range.  Fails
// only when one member alone has more CTAs than grid.x holds; it is named as `what` and ids[i] (nullptr: its position).
struct RaggedRange {
    size_t begin, end;  // members [begin, end)
    unsigned ctas;      // grid.x
};
int deal_ragged(spg_handle *h, const std::vector<long long> &ctas, size_t capacity, const char *what, const int *ids,
                std::vector<RaggedRange> &ranges, std::vector<int> &first_cta);

// range g of the members into the table r, each at its first CTA
template <class Table, class M>
void fill_table(Table &r, const std::vector<M> &ms, const std::vector<int> &first_cta, const RaggedRange &g) {
    r.n = (int)(g.end - g.begin);
    for (int k = 0; k < r.n; k++) {
        r.img[k] = ms[g.begin + k];
        r.img[k].first_cta = first_cta[g.begin + k];
    }
}

// Lays arrays out in one Scratch, each 256-byte aligned: a pass with base == nullptr measures, a pass with the grown
// buffer hands out the pointers.
struct Carver {
    unsigned char *base = nullptr;
    size_t bytes = 0;
    template <typename T>
    T *take(size_t count) {
        const size_t o = (bytes + 255) & ~(size_t)255;
        bytes = o + std::max<size_t>(count, 1) * sizeof(T);
        return base ? reinterpret_cast<T *>(base + o) : nullptr;
    }
};

// `what` given: a call on `st`, which grows nothing while `st` captures (grow_on)
template <typename F>
int carve(spg_handle *h, Scratch &s, F &&layout, cudaStream_t st = nullptr, const char *what = nullptr) {
    Carver m;
    layout(m);
    int rc;
    if ((rc = what ? grow_on(h, s, m.bytes, st, what) : grow(h, s, m.bytes))) return rc;
    Carver c;
    c.base = static_cast<unsigned char *>(s.p);
    layout(c);
    return SPG_OK;
}

int check_batch(spg_handle *h, int n);
int check_dims(spg_handle *h, int n, int H, int W);

// warpAffine's inversion of its matrix (imgproc/src/imgwarp.cpp), in its operation order (the host code is built
// without FMA contraction): the kernels then repeat its fixed-point coordinates bit for bit
void invert_affine(const double *M, double *m);

// spg_create's check of the capacities against the sampled limb-scoring kernels, which every limb-scoring plan falls
// back to (group.cu)
int check_score_room(spg_handle *h);

}  // namespace spg
