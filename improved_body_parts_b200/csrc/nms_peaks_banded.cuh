// nms_peaks_banded.cuh -- K1, persistent warp-specialised form for planes of ANY size (W % 4 == 0), band by band.
//
// Same results as nms_peaks_kernel (nms_peaks.cuh); different schedule.  4608 short-lived CTAs per launch spend
// most of their life in launch / first-copy latency and in a one-warp refinement tail that keeps their shared
// memory pinned.  Here one CTA per SM stays resident and walks over its (image, part) planes, BAND by band:
//
//   loader    (warp 0)       waits for a free band slot and issues the band's bulk copy (TMA, SASS UBLKCP) -- the band's
//                            rows plus one halo row above and below -- onto the slot's `full` mbarrier.
//   scanners  (warps 1-28)   four teams of seven; per band: pass 1 queues the float4 groups that reach thre1, pass 2 runs the
//                            8-neighbour test on the queue and appends peaks to the PLANE's list (ring of 6); then the team
//                            releases the band slot.
//   finishers (warps 29-31)  take planes round-robin: rank the list by raster index (= np.nonzero order), refine each
//                            peak from L2 (the plane was just streamed), write the outputs, recycle the list.
//
// The whole-plane form (nms_peaks_persist.cuh: ring of 3 planes, 28 scanner slices) is the faster one when three planes fit
// in shared memory (e.g. 128 x 128 planes); this kernel takes the planes that do not fit (e.g. 512 x 512 planes, where it
// is faster than the one-CTA-per-plane kernel) with bands of ~16 KB
// (+ one halo row above and below) through a ring of 8 or 12 slots, so that ~150 KB per SM stay in flight whatever the
// plane size.
#pragma once

#include "nms_peaks_persist.cuh"

namespace spg {

// the role constants (kNmsP*) are in nms_peaks.cuh; a band is <= (warps per team) * 32 * kNmsPMaxIter float4 groups
constexpr int kNmsBMaxSlots = 16;
constexpr int kNmsBTeams = 4;            // banded form: scanner teams of 7 warps, team g scans the bands t = g, g + 4, ... of the CTA's sequence
constexpr int kNmsBBandGroups = 1024;    // banded form: target band size in float4 groups (16 KB)

struct NmsBanding {
    int band_rows, n_bands, slots, teams;
    size_t band_stride, smem;  // bytes
};
// Band geometry for an H x W plane within `smem_limit` bytes of shared memory; slots == 0: does not fit.
inline NmsBanding nms_banding(int H, int W, int capP, size_t smem_limit) {
    NmsBanding g{};
    const int W4 = W / 4;
    const size_t fixed = kNmsPLists * (size_t)capP * sizeof(uint32_t) + (size_t)kNmsPScanners * 32 * kNmsPMaxIter * sizeof(uint16_t) + 64;  // lists + per-warp queues
    if (smem_limit <= fixed) return g;
    g.teams = kNmsBTeams;
    const int team_warps = kNmsPScanners / kNmsBTeams;
    g.band_rows = std::max(1, std::min(H, kNmsBBandGroups / std::max(W4, 1)));
    if ((size_t)g.band_rows * W4 > (size_t)team_warps * 32 * kNmsPMaxIter) return g;  // a single row wider than a team's reach
    g.n_bands = (H + g.band_rows - 1) / g.band_rows;
    g.band_stride = (((size_t)std::min(g.band_rows + 2, H) * W * sizeof(float)) + 127) & ~(size_t)127;
    // a multiple of the team count: band t and band t - slots (same slot) then belong to the same team, which consumes its
    // bands in order -- a team never waits on a slot whose previous band it has not seen land (mbarrier parity waits alias
    // beyond one phase)
    g.slots = (int)std::min<size_t>(kNmsBMaxSlots, (smem_limit - fixed) / g.band_stride) / kNmsBTeams * kNmsBTeams;
    g.smem = (size_t)g.slots * g.band_stride + fixed;
    return g;
}

__global__ void __launch_bounds__(kNmsPThreads, 1) nms_peaks_banded_kernel(NmsArgs a, int n_items, int n_slots, int n_bands) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t bar_full[kNmsBMaxSlots], bar_free[kNmsBMaxSlots], bar_ready[kNmsPLists], bar_lfree[kNmsPLists];
    __shared__ int s_cnt[kNmsPLists];

    const Workspace &ws = a.ws;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int H = a.H, W = a.W, K = ws.K, capP = ws.capP;
    const int BR = a.band_rows, S = n_slots, NB = n_bands;
    constexpr int T = kNmsBTeams, TW = kNmsPScanners / kNmsBTeams;  // teams, warps per team
    const size_t band_stride = (((size_t)min(BR + 2, H) * W * sizeof(float)) + 127) & ~(size_t)127;
    uint32_t *s_lists = reinterpret_cast<uint32_t *>(smem_raw + (size_t)S * band_stride);  // [lists][capP]
    uint16_t *s_queues = reinterpret_cast<uint16_t *>(s_lists + kNmsPLists * (size_t)capP);
    const int W4 = W >> 2;
    // g / W4 without a division: g < 2^16 here (a band's group count), so umulhi(g, ceil(2^32 / W4)) is exact
    const uint32_t w4_magic = W4 > 1 ? 0xffffffffu / (uint32_t)W4 + 1u : 0u;

    if (tid == 0) {
        for (int s = 0; s < S; s++) {
            mbar_init(&bar_full[s], 1);
            mbar_init(&bar_free[s], TW);
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
            int s = 0, round = 0;  // slot of band t = j * NB + b, and t / S
            for (int j = 0; j < nj; j++) {
                const int item = (int)blockIdx.x + j * G;
                const int n_local = item / K, c = item - n_local * K;
                const float *plane = a.heat + (int64_t)n_local * a.img_stride + (int64_t)c * a.chan_stride;
                for (int b = 0; b < NB; b++) {
                    if (round > 0) mbar_wait_sleep(&bar_free[s], (round - 1) & 1);
                    const int r0 = b * BR, lo = max(r0 - 1, 0), hi = min(r0 + BR + 1, H);
                    const uint32_t bytes = (uint32_t)((size_t)(hi - lo) * W * sizeof(float));
                    mbar_expect_tx(&bar_full[s], bytes);
                    bulk_g2s(smem_raw + (size_t)s * band_stride, plane + (size_t)lo * W, bytes, &bar_full[s]);
                    if (++s == S) { s = 0; round++; }
                }
            }
        }
    } else if (warp <= kNmsPScanners) {
        // =========================== scanners ===========================
        // Four teams of seven warps; team g takes the bands t = g, g + 4, ... of the CTA's band sequence, so a warp pays the per-band costs (two
        // barrier operations, the queue set-up) once per ~147 float4 groups, as it did with whole planes, while the ring
        // turns over in 17 KB steps.
        const int w = warp - 1, team = w / TW, tw = w - team * TW;
        uint16_t *wq = s_queues + (size_t)w * (32 * kNmsPMaxIter);
        const float thr = a.thr;
        for (int j = 0; j < nj; j++) {
            const int l = j % kNmsPLists;
            uint32_t *list = s_lists + (size_t)l * capP;
            if (j >= kNmsPLists) mbar_wait_sleep(&bar_lfree[l], ((j / kNmsPLists) - 1) & 1);
            for (int b = (team - (j * NB) % T + T) % T; b < NB; b += T) {
                const int t = j * NB + b, round = t / S, s = t - round * S;  // band t (t mod T == team) sits in slot t mod S
                mbar_wait_sleep(&bar_full[s], round & 1);
                const int r0 = b * BR, r1 = min(r0 + BR, H), lo = max(r0 - 1, 0);
                const int groups = (r1 - r0) * W4;
                // `band` points at the (virtual) start of global row 0, so rows are addressed by their global index
                const float *band = reinterpret_cast<const float *>(smem_raw + (size_t)s * band_stride) - (size_t)lo * W;
                // pass 1: queue the float4 groups of this warp's share that reach thre1 (groups are dealt to the team's
                // warps 32 at a time)
                const int nq = nms_queue_groups<kNmsPMaxIter>(band + (size_t)r0 * W, tw * 32, TW * 32, groups, thr, lane, wq);
                // pass 2: the 8-neighbour test of the queued groups
                for (int q = lane; q < nq; q += 32) {
                    const int g = wq[q];
                    const int yl = W4 > 1 ? (int)__umulhi((uint32_t)g, w4_magic) : g, xq = g - yl * W4;
                    const int y = r0 + yl, x0 = 4 * xq;
                    nms_test_group(band, y, x0, H, W, thr, &s_cnt[l], list, capP);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&bar_free[s]);  // the band is not needed any more
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_ready[l]);      // this warp's peaks of the plane are in the list
        }
    } else {
        // =========================== finishers ===========================
        const int f = warp - 1 - kNmsPScanners;
        for (int j = f; j < nj; j += kNmsPFinishers) {
            const int l = j % kNmsPLists;
            mbar_wait_sleep(&bar_ready[l], (j / kNmsPLists) & 1);
            nms_finish_plane(a, s_lists + (size_t)l * capP, s_cnt[l], (int)blockIdx.x + j * G, lane, 0u);
            __syncwarp();
            if (lane == 0) {
                s_cnt[l] = 0;
                mbar_arrive(&bar_lfree[l]);  // list + counter may be reused (plane j + kNmsPLists)
            }
        }
    }
}

}  // namespace spg
