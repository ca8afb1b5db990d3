// nms_peaks_persist.cuh -- K1, persistent warp-specialised form (planes that fit a 3-deep ring, W % 4 == 0).
//
// Same results as nms_peaks_kernel (nms_peaks.cuh); different schedule.  4608 short-lived CTAs per launch spend
// most of their life in launch / first-copy latency and in a one-warp refinement tail that keeps their shared
// memory pinned.  Here one CTA per SM stays resident and walks over its (image, part) planes:
//
//   loader    (warp 0)       waits for a free plane slot (ring of 3) and issues the plane's bulk copy (TMA, SASS
//                            UBLKCP) onto the slot's `full` mbarrier.
//   scanners  (warps 1-28)   per plane: pass 1 queues the float4 groups of their share that reach thre1, pass 2 runs
//                            the 8-neighbour test on the queue and appends peaks to the plane's list (ring of 6).
//   finishers (warps 29-31)  take planes round-robin (finisher f: the planes of slot f): rank the list by raster index
//                            (= np.nonzero order), refine each peak from the plane still in its slot, write the outputs,
//                            then release the plane slot and recycle the list.
#pragma once

#include "nms_peaks.cuh"

namespace spg {

constexpr int kNmsPSlots = 3;  // plane ring; the role constants are in nms_peaks.cuh

// Clock trace (`make trace`, tools/trace_nms_peaks.py): 16 words per plane for a CTA's first 64 planes.
// Loader: 0 before its wait on `free`, 1 copy issued.  Scanners: 2 first past `full`, 5 last out of pass 1 (= before the
// wait on `lfree`), 4 last past `lfree`, 6 first / 7 last done with the plane, 8 last to arrive on `ready`, 11 queued
// groups (sum).
// Finishers: 9 start, 10 end (= the slot released), 12 peaks (value), 13 before the wait on `ready`.
constexpr int kNmsTrWords = 16, kNmsTrPlanes = 64;
#define SPG_NMS_TR(kind, j, f, dep) do { if ((j) < kNmsTrPlanes) kind(kNmsTrWords * (j) + (f), dep); } while (0)

inline size_t nms_persist_smem_bytes(int H, int W, int capP) {
    const size_t plane = (((size_t)H * W * sizeof(float)) + 127) & ~(size_t)127;
    const size_t queues = (size_t)kNmsPScanners * 32 * kNmsPMaxIter * sizeof(uint16_t);
    return kNmsPSlots * plane + kNmsPLists * (size_t)capP * sizeof(uint32_t) + queues + 64;
}

// R = a.radius, the refinement radius: one instantiation per radius (launch_nms dispatches).
template <int R>
__global__ void __launch_bounds__(kNmsPThreads, 1) nms_peaks_persist_kernel(NmsArgs a, int n_items) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t bar_full[kNmsPSlots], bar_free[kNmsPSlots], bar_ready[kNmsPLists], bar_lfree[kNmsPLists];
    __shared__ int s_cnt[kNmsPLists];

    const Workspace &ws = a.ws;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int H = a.H, W = a.W, K = ws.K, capP = ws.capP;
    const size_t plane_bytes = (size_t)H * W * sizeof(float);
    const size_t plane_stride = (plane_bytes + 127) & ~(size_t)127;
    uint32_t *s_lists = reinterpret_cast<uint32_t *>(smem_raw + kNmsPSlots * plane_stride);  // [lists][capP]
    uint16_t *s_queues = reinterpret_cast<uint16_t *>(s_lists + kNmsPLists * (size_t)capP);
    const int W4 = W >> 2, groups = H * W4;
    // g / W4 without a division: groups < 2^16 here (launch condition), so umulhi(g, ceil(2^32 / W4)) is exact
    const uint32_t w4_magic = W4 > 1 ? 0xffffffffu / (uint32_t)W4 + 1u : 0u;

    if (tid == 0) {
        for (int s = 0; s < kNmsPSlots; s++) {
            mbar_init(&bar_full[s], 1);
            mbar_init(&bar_free[s], 1);  // the finisher of the slot's plane
        }
        for (int l = 0; l < kNmsPLists; l++) {
            mbar_init(&bar_ready[l], kNmsPScanners);
            mbar_init(&bar_lfree[l], 1);
            s_cnt[l] = 0;
        }
        fence_mbar_init();
    }
    __syncthreads();

    const int G = gridDim.x;
    const int nj = ((int)blockIdx.x < n_items) ? (n_items - 1 - (int)blockIdx.x) / G + 1 : 0;

    if (warp == 0) {
        // =========================== loader ===========================
        if (lane == 0) {
            for (int j = 0; j < nj; j++) {
                const int s = j % kNmsPSlots;
                SPG_NMS_TR(SPG_TR, j, 0, j);
                if (j >= kNmsPSlots) mbar_wait_sleep(&bar_free[s], ((j / kNmsPSlots) - 1) & 1);
                const int item = (int)blockIdx.x + j * G;
                const int n_local = item / K, c = item - n_local * K;
                const unsigned char *src =
                    reinterpret_cast<const unsigned char *>(a.heat + (int64_t)n_local * a.img_stride + (int64_t)c * a.chan_stride);
                unsigned char *dst = smem_raw + s * plane_stride;
                mbar_expect_tx(&bar_full[s], (uint32_t)plane_bytes);
                for (size_t off = 0; off < plane_bytes; off += 32768) {
                    const uint32_t bytes = (uint32_t)min((size_t)32768, plane_bytes - off);
                    bulk_g2s(dst + off, src + off, bytes, &bar_full[s]);
                }
                SPG_NMS_TR(SPG_TR, j, 1, j);
            }
        }
    } else if (warp <= kNmsPScanners) {
        // =========================== scanners ===========================
        // The plane's float4 groups are dealt to the scanners 32 at a time (warp w: groups w * 32 .. w * 32 + 31, then
        // 28 * 32 further on, ...; <= kNmsPMaxIter rounds, launch condition), so that the groups that reach thre1 -- a
        // person's blob covers a few rows -- and with them pass 2's work spread over all scanners.  With one contiguous
        // slice per warp, the few warps whose slices held the blobs did most of pass 2 while the slot stayed held.
        const int w = warp - 1;
        uint16_t *wq = s_queues + (size_t)w * (32 * kNmsPMaxIter);
        const float thr = a.thr;
        for (int j = 0; j < nj; j++) {
            const int s = j % kNmsPSlots, l = j % kNmsPLists;
            mbar_wait_sleep(&bar_full[s], (j / kNmsPSlots) & 1);
            SPG_NMS_TR(SPG_TR_FIRST, j, 2, j);
            const float *buf = reinterpret_cast<const float *>(smem_raw + s * plane_stride);
            uint32_t *list = s_lists + (size_t)l * capP;
            // pass 1: queue the float4 groups of this warp's share that reach thre1
            const int nq = nms_queue_groups<kNmsPMaxIter>(buf, w * 32, kNmsPScanners * 32, groups, thr, lane, wq);
            SPG_NMS_TR(SPG_TR_LAST, j, 5, nq);
            SPG_NMS_TR(SPG_TR_ADD, j, 11, nq);
            // the list of plane j - kNmsPLists must be finished before pass 2 appends to this one (pass 1 does not need it)
            if (j >= kNmsPLists) mbar_wait_sleep(&bar_lfree[l], ((j / kNmsPLists) - 1) & 1);
            SPG_NMS_TR(SPG_TR_LAST, j, 4, j);
            // pass 2: the 8-neighbour test of the queued groups
            for (int q = lane; q < nq; q += 32) {
                const int g = wq[q];
                const int y = W4 > 1 ? (int)__umulhi((uint32_t)g, w4_magic) : g, xq = g - y * W4;
                nms_test_group(buf, y, 4 * xq, H, W, thr, &s_cnt[l], list, capP);
            }
            __syncwarp();
            if (lane == 0) {
                SPG_NMS_TR(SPG_TR_FIRST, j, 6, j);
                SPG_NMS_TR(SPG_TR_LAST, j, 7, j);
                mbar_arrive(&bar_ready[l]);  // this warp's peaks are in the list; the finisher frees the slot
                SPG_NMS_TR(SPG_TR_LAST, j, 8, j);
            }
        }
    } else {
        // =========================== finishers ===========================
        const int f = warp - 1 - kNmsPScanners;
        for (int j = f; j < nj; j += kNmsPFinishers) {
            const int l = j % kNmsPLists;
            SPG_NMS_TR(SPG_TR, j, 13, j);
            mbar_wait_sleep(&bar_ready[l], (j / kNmsPLists) & 1);
            SPG_NMS_TR(SPG_TR, j, 9, j);
            SPG_NMS_TR(SPG_TRV, j, 12, s_cnt[l]);
            const int s = j % kNmsPSlots;
            // refine from the plane still staged in slot s, not from L2: with every SM streaming, an L2 read took most
            // of a finisher's ~14 000 cycles per plane, and the last plane's finisher is the kernel's tail
            nms_finish_plane<R>(a, s_lists + (size_t)l * capP, s_cnt[l], (int)blockIdx.x + j * G, lane, w4_magic,
                                reinterpret_cast<const float *>(smem_raw + s * plane_stride));
            __syncwarp();
            SPG_NMS_TR(SPG_TR, j, 10, j);
            if (lane == 0) {
                mbar_arrive(&bar_free[s]);  // the plane is not needed any more
                s_cnt[l] = 0;
                mbar_arrive(&bar_lfree[l]);  // list + counter may be reused (plane j + kNmsPLists)
            }
        }
    }
}

}  // namespace spg
