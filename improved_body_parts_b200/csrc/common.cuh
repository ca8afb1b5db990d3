// common.cuh -- shared definitions for the sm_90a grouping kernels.
//
// Arithmetic contract: every floating-point operation that feeds a discrete decision of the reference
// (rounding of sample coordinates, threshold tests, sort keys) is reproduced in the reference's precision
// and operation order.  The translation unit is built with -fmad=false and uses the explicit *_rn
// intrinsics where an accidental contraction would change a rounding, so results are bit-identical to
// numpy/Python on the host (see DESIGN.md "numerics").
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

namespace spg {

// Clock trace of the first CTAs of a launch (development builds only: `make trace` -> libspgroup_trace.so, which is
// never loaded by the package).  SPG_TR(slot, dep) stores clock64() once `dep` (any 32-bit value) is available;
// SPG_TR_FIRST / SPG_TR_LAST keep the earliest / latest such stamp of several warps (the buffer starts zeroed);
// SPG_TR_ADD sums a value over several warps.
#ifdef SPG_TRACE
constexpr int kTraceCtas = 64, kTraceSlots = 1024;
__device__ unsigned long long g_spg_trace[kTraceCtas * kTraceSlots];
__device__ __forceinline__ void trace_put(int slot, int dep, int mode) {  // mode 0: store, 1: value, 2: first, 3: last, 4: add
    if (blockIdx.x < kTraceCtas && (threadIdx.x & 31) == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%clock64;" : "=l"(t) : "r"(dep) : "memory");
        unsigned long long *w = &g_spg_trace[blockIdx.x * kTraceSlots + slot];
        if (mode == 2) atomicCAS(w, 0ull, t);
        else if (mode == 3) atomicMax(w, t);
        else if (mode == 4) atomicAdd(w, (unsigned long long)(unsigned)dep);
        else *w = mode == 1 ? (unsigned long long)(unsigned)dep : t;
    }
}
#define SPG_TR(slot, dep) ::spg::trace_put((slot), (int)(dep), 0)
#define SPG_TRV(slot, v) ::spg::trace_put((slot), (int)(v), 1)
#define SPG_TR_FIRST(slot, dep) ::spg::trace_put((slot), (int)(dep), 2)
#define SPG_TR_LAST(slot, dep) ::spg::trace_put((slot), (int)(dep), 3)
#define SPG_TR_ADD(slot, v) ::spg::trace_put((slot), (int)(v), 4)
// Start and exit time of every CTA (up to kTraceSpanCtas) of a launch, in %globaltimer nanoseconds: unlike clock64 one
// clock for all SMs, so CTAs on different SMs can be compared.  SPG_TR_CTA_START: thread 0 at entry; SPG_TR_CTA_EXIT:
// every warp at its end, the latest stays.
constexpr int kTraceSpanCtas = 1024;
__device__ unsigned long long g_spg_cta_span[kTraceSpanCtas * 2];
__device__ __forceinline__ void trace_cta(int exit) {
    if (blockIdx.x < kTraceSpanCtas && (threadIdx.x & 31) == 0 && (exit || threadIdx.x == 0)) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t) :: "memory");
        if (exit) atomicMax(&g_spg_cta_span[2 * blockIdx.x + 1], t);
        else g_spg_cta_span[2 * blockIdx.x] = t;
    }
}
#define SPG_TR_CTA_START() ::spg::trace_cta(0)
#define SPG_TR_CTA_EXIT() ::spg::trace_cta(1)
#else
#define SPG_TR(slot, dep) do {} while (0)
#define SPG_TRV(slot, v) do {} while (0)
#define SPG_TR_FIRST(slot, dep) do {} while (0)
#define SPG_TR_LAST(slot, dep) do {} while (0)
#define SPG_TR_ADD(slot, v) do {} while (0)
#define SPG_TR_CTA_START() do {} while (0)
#define SPG_TR_CTA_EXIT() do {} while (0)
#endif

constexpr int kMaxParts = 32;        // K
constexpr int kMaxLimbs = 64;        // L
constexpr int kMaxCapPeaks = 128;    // peaks per (image, part); two 64-bit "used" masks in limb_match
constexpr int kMaxCapRows = 128;     // subset rows per image; four 32-bit alive masks in assemble
constexpr int kMaxRefineRadius = 4;  // (2r+1)^2 <= 81 <= numpy's 128-element pairwise block
constexpr int kMaxOutJoints = 32;
constexpr int kMAMatchWarps = 7;   // matcher warps of match_assemble_kernel by default; the launch may use 1..15 (blockDim.x = 32 * (1 + matchers))

// status bits, identical to SPG_ST_* in include/spgroup.h
constexpr uint32_t kStPeakOverflow = 1u << 0;
constexpr uint32_t kStCandOverflow = 1u << 1;
constexpr uint32_t kStRowOverflow = 1u << 2;
constexpr uint32_t kStSampleIndex = 1u << 3;
constexpr uint32_t kStAssert = 1u << 4;
constexpr uint32_t kStWireOverflow = 1u << 5;
constexpr uint32_t kStNonfinite = 1u << 6;
constexpr uint32_t kStNanPriority = 1u << 7;
// Scorer-internal, never published: a candidate of the limb has a NaN priority.  publish_limb turns it into
// kStNanPriority when the limb has another candidate to be sorted against.
constexpr uint32_t kStNanPrioCand = 1u << 31;

struct Params {
    double thre1, thre2, connect_ration, len_rate, connection_tole, min_mean_score;
    int32_t mid_num, offset_radius, remove_recon, min_parts;
    int32_t crit1_strict, refresh_len_check;  // demo_image.py's two deviations from evaluate.py (0 = evaluate.py)
};

// Device workspace of one handle (all arrays [max_batch][...]).
struct Workspace {
    int K, L, J, capP, capC, capR, max_batch;
    int16_t limbs[kMaxLimbs * 2];       // [L][2]; lives in the kernel parameter (constant) bank
    int16_t out_from_part[kMaxOutJoints];  // [J]
    // peaks
    double *peak_x, *peak_y;       // [N][K][capP]
    float *peak_score;
    uint32_t *peak_anchor;
    int32_t *peak_count;           // [N][K]
    // candidates (unordered; the matcher orders them by (priority desc, i*nB+j asc))
    double *cand_prio, *cand_score;  // [N][L][capC]
    uint32_t *cand_ij;
    unsigned long long *cand_key;    // f32 planes only: (order-preserving bits of the f32 priority << 32) | ~((i << 16) | j)
    int32_t *cand_count;             // [N][L]  -1 = special_k
    int32_t *surv_count;             // [N][L]  pairs that survived limb_score's screen (diagnostic)
    // connections, acceptance order
    uint32_t *conn_ij;             // [N][L][capP]
    double *conn_score, *conn_norm;
    int32_t *conn_count;           // [N][L]
    // persons
    double *subset;                // [N][capR][K+2][2]
    int32_t *n_persons;            // [N]
    double *people_xy;             // [N][capR][J][2]
    double *people_score;          // [N][capR]
    uint32_t *status;              // [N]
    // wire records (include/spgroup.h "wire records"); wire == nullptr: off.  May point into a peer GPU's memory.
    unsigned char *wire;
    long long wire_first;          // record index of image 0 of a call
    int wire_rows;                 // person rows per record
};

// ---------------------------------------------------------------------------------------------
// mbarrier + 1-D bulk-copy (TMA engine, SASS UBLKCP) helpers.  A plane row band / a whole plane is
// one contiguous span of global memory, so the descriptor-less 1-D form is the natural fit.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        " .reg .pred p;\n"
        " mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        " selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// Same, for waits that can be long (role hand-offs in persistent kernels): pass a suspend-time hint so the warp is
// parked by the hardware instead of polling, and does not take issue slots from the warps it is waiting for.
__device__ __forceinline__ void mbar_wait_sleep(uint64_t *bar, uint32_t parity, uint32_t hint_ns = 20000u) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile(
            "{\n"
            " .reg .pred p;\n"
            " mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
            " selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity), "r"(hint_ns)
            : "memory");
    }
}

// ---------------------------------------------------------------------------------------------
// Ragged launches: one launch covers many members (images, items or samples) whose descriptors travel in a table passed
// as a __grid_constant__ kernel parameter, so a call returns with nothing of the caller's left to copy.  grid.x walks the
// members' CTAs back to back; member k starts at img[k].first_cta (increasing).  A table fits the kernel-parameter limit
// (CUDA 12.1 and later) together with the launch's other arguments.
// ---------------------------------------------------------------------------------------------
constexpr int kParamBytes = 32764;

// the member whose CTAs hold CTA `cta`: the last one whose first CTA is <= cta
template <class R>
__device__ __forceinline__ const auto &ragged_member(const R &r, int cta) {
    int lo = 0, hi = r.n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (r.img[mid].first_cta <= cta) lo = mid;
        else hi = mid - 1;
    }
    return r.img[lo];
}

// numpy's pairwise summation order for 8 <= n <= 128 (and the plain loop for n < 8): what both
// `score_box.sum()` (f32) and `(score_box * grid).sum()` (f64) use in utils/util.py:206-211.
template <typename T>
__device__ __forceinline__ T pairwise_sum(const T *a, int n) {
    if (n < 8) {
        T res = (T)0;
        for (int i = 0; i < n; i++) res = res + a[i];
        return res;
    }
    T r[8];
#pragma unroll
    for (int k = 0; k < 8; k++) r[k] = a[k];
    int i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int k = 0; k < 8; k++) r[k] = r[k] + a[i + k];
    }
    T res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; i++) res = res + a[i];
    return res;
}

}  // namespace spg
