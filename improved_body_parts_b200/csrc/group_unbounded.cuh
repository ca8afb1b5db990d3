// group_unbounded.cuh -- the capacity-free grouping tier: peaks -> connections -> people of ONE image with every list
// sized from the image itself instead of the handle's capacities.
//
// The bounded kernels keep their fixed limits (128 peaks per part, 128 person rows, max_cands_per_limb candidates): the
// matcher's "used" flags are two 64-bit masks and the person table lives in shared memory.  An image past one of them gets
// a status bit.  This tier regroups such an image with the reference's answer (evaluate.py:169-498, :523-543), whatever
// its size, from the same device functions the bounded schedules share:
//
//   1. ub_peaks_kernel<false>   one CTA per part counts its peaks (nms_is_peak); the host sizes the peak tables from the
//      counts.  ub_peaks_kernel<true> then writes them in raster order (np.nonzero, evaluate.py:193) through an ordered
//      block scan, each finished by nms_finish_peak (border test + refine_centroid).
//   2. ub_score_kernel<false>   one thread per (limb, A peak) scores the row i of the limb's pairs with score_pair_exact
//      and counts the candidates (evaluate.py:211-255); the host turns the counts into offsets.  ub_score_kernel<true>
//      scores them again and writes each candidate at its generation-order position (i-major), so no list is truncated.
//   3. A stable segmented radix sort (CUB) orders each limb's candidates by priority, descending: equal keys keep their
//      generation order, which is Python's stable sorted(..., reverse=True) (:259).  ub_match_kernel, one thread per limb,
//      runs the greedy acceptance (:263-270) with byte flags sized to the peak counts.
//   4. ub_assemble_kernel, one CTA: thread 0 runs find_people's limb loop (:279-488) connection by connection on a person
//      table in global memory, with the transitions of assemble.cuh (apply_zero_or_one, apply_two_rows); rows are born in
//      acceptance order, so a row's birth stamp is its index.  Then the whole CTA runs emit_people: the prune (:491-496),
//      `subset`, the COCO-ordered joints and the person scores (:523-543).
//
// Limits of the tier (the host checks them before the first write and fails the call instead):
//   - peaks per part <= 65535: candidate and connection (i, j) are packed in 16 bits each (cand_ij, conn_ij);
//   - person rows <= 32767: the owner map of the person table holds row numbers in 16 bits; the table has one row per
//     accepted connection, which bounds the rows assembly can create;
//   - candidates per image < 2^31 (the sort's item count).
#pragma once

#include <cub/cub.cuh>

#include "assemble.cuh"
#include "limb_score.cuh"
#include "nms_peaks.cuh"

namespace spg {

constexpr int kUbPeakThreads = 1024;
constexpr int kUbScoreThreads = 128;
constexpr int kUbAssembleThreads = 1024;
constexpr int kUbMaxPeaks = 65535;
constexpr int kUbMaxRows = 32767;

// Arrays of the tier.  `ws` carries the skeleton (K, L, J, limbs, out_from_part) and the result arrays, laid out as the
// bounded ones with the tier's sizes: capP = the largest part's peak count, capR = the person table's rows, one image.
struct UbArgs {
    Workspace ws;
    const float *heat;
    const void *paf;
    int64_t heat_chan_stride, paf_chan_stride;  // elements
    int H, W;
    int32_t *row_count;                 // [L][capP] candidates of pair row (limb, i)
    const int64_t *row_off;             // [L][capP] first candidate of pair row (limb, i) in the image's list
    const int64_t *seg_off;             // [L + 1] first candidate of each limb
    unsigned long long *cand_key_out;   // sorted keys (unused after the sort)
    const uint32_t *sorted;             // [n_cand] candidate index in priority order
    uint32_t *cand_idx;                 // [n_cand] identity (the sort's values)
    unsigned char *used;                // [L][2][capP] greedy-matching flags, zeroed by the host
    PersonTable table;                  // rows / slots / owner in global memory
};

// NMS of part blockIdx.x over the whole plane in raster order: tile by tile, an exclusive block scan of the peak flags
// gives each peak its np.nonzero rank.  WRITE = false only counts (ws.peak_count[c]); WRITE = true finishes every peak at
// [c][rank] of the tier's tables.
template <bool WRITE>
__global__ void __launch_bounds__(kUbPeakThreads) ub_peaks_kernel(UbArgs u, NmsArgs a) {
    using Scan = cub::BlockScan<int, kUbPeakThreads>;
    __shared__ typename Scan::TempStorage scan_tmp;
    const int c = blockIdx.x, tid = threadIdx.x;
    const int H = u.H, W = u.W;
    const float *plane = u.heat + (int64_t)c * u.heat_chan_stride;
    const int64_t npix = (int64_t)H * W;
    int base = 0;
    for (int64_t p0 = 0; p0 < npix; p0 += kUbPeakThreads) {
        const int64_t p = p0 + tid;
        int y = 0, x = 0, pk = 0;
        if (p < npix) {
            y = (int)(p / W);
            x = (int)(p - (int64_t)y * W);
            pk = nms_is_peak(plane, 0, H, W, y, x, plane[p], a.thr) ? 1 : 0;
        }
        int pos, total;
        Scan(scan_tmp).ExclusiveSum(pk, pos, total);
        if (WRITE && pk) nms_finish_peak(a, plane, H, W, (size_t)c * u.ws.capP + base + pos, y, x);
        base += total;
        __syncthreads();  // scan_tmp is reused by the next tile
    }
    if (!WRITE && tid == 0) u.ws.peak_count[c] = base;
}

// Order-preserving 64-bit key of a float64 priority (-0.0 folded into +0.0: Python's sort sees them equal).
__device__ __forceinline__ unsigned long long ub_prio_key(double prio) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(__dadd_rn(prio, 0.0));
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

// Pair row (limb blockIdx.x, A peak i) of the limb's nA x nB pairs: every pair scored in generation order (:218-255).
// WRITE = false: u.row_count[limb][i] = its candidates; WRITE = true: the candidates from u.row_off[limb][i] on.
template <typename T, typename TA, bool WRITE>
__global__ void __launch_bounds__(kUbScoreThreads) ub_score_kernel(UbArgs u, ScoreArgs sa) {
    __shared__ double s_rcp[kScreenMaxMid + 1];
    for (int m = threadIdx.x; m <= kScreenMaxMid; m += blockDim.x) s_rcp[m] = m > 0 ? __ddiv_rn(1.0, (double)m) : 0.0;
    __syncthreads();
    const Workspace &ws = u.ws;
    const int k = blockIdx.x, i = blockIdx.y * kUbScoreThreads + threadIdx.x;
    const int pa = ws.limbs[2 * k], pb = ws.limbs[2 * k + 1];
    const int nA = ws.peak_count[pa], nB = ws.peak_count[pb];
    if (i >= nA || nB == 0) return;
    const int capP = ws.capP, H = u.H, W = u.W;
    const T *plane = reinterpret_cast<const T *>(u.paf) + (int64_t)k * u.paf_chan_stride;
    const PairGeom g{ws.peak_x + (size_t)pa * capP, ws.peak_y + (size_t)pa * capP, ws.peak_x + (size_t)pb * capP,
                     ws.peak_y + (size_t)pb * capP, ws.peak_score + (size_t)pa * capP, ws.peak_score + (size_t)pb * capP, s_rcp};
    const bool ain = inside_map(g.ax[i], g.ay[i], H, W);
    const TA thre2 = (TA)sa.thre2;
    const size_t slot = (size_t)k * capP + i;
    const int64_t out = WRITE ? u.row_off[slot] : 0;
    int nc = 0;
    uint32_t flags = 0;
    for (int j = 0; j < nB; j++) {
        double score, prio;
        const bool ok = score_pair_exact<T, 1, TA>(plane, H, W, sa, g, i, j, ain && inside_map(g.bx[j], g.by[j], H, W), thre2,
                                                   score, prio, flags);
        if (ok) {
            if (WRITE) {
                const int64_t o = out + nc;
                ws.cand_prio[o] = prio;
                ws.cand_score[o] = score;
                ws.cand_ij[o] = ((uint32_t)i << 16) | (uint32_t)j;
                ws.cand_key[o] = ub_prio_key(prio);
                u.cand_idx[o] = (uint32_t)o;
            }
            nc++;
        }
    }
    if (!WRITE) u.row_count[slot] = nc;
    // a NaN priority is judged per limb, by ub_match_kernel, once the limb's candidate count is known
    flags &= ~kStNanPrioCand;
    if (flags) atomicOr(ws.status, flags);
}

// Greedy acceptance of limb k's candidates in priority order (:263-270), one thread per limb.
__global__ void ub_match_kernel(UbArgs u) {
    const Workspace &ws = u.ws;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= ws.L) return;
    const int capP = ws.capP;
    const int pa = ws.limbs[2 * k], pb = ws.limbs[2 * k + 1];
    const int nA = ws.peak_count[pa], nB = ws.peak_count[pb];
    const int64_t c0 = u.seg_off[k], c1 = u.seg_off[k + 1];
    ws.cand_count[k] = (int)(c1 - c0);
    if (nA == 0 || nB == 0) {  // special_k (:272-274)
        ws.conn_count[k] = -1;
        return;
    }
    // a NaN priority among two or more candidates: the reference's sort order (:259) is not reproduced
    if (c1 - c0 > 1) {
        bool nan_prio = false;
        for (int64_t c = c0; c < c1; c++) nan_prio |= isnan(ws.cand_prio[c]);
        if (nan_prio) atomicOr(ws.status, kStNanPriority);
    }
    unsigned char *usedA = u.used + (size_t)k * 2 * capP, *usedB = usedA + capP;
    const int lim = min(nA, nB);
    const size_t cb = (size_t)k * capP;
    int m = 0;
    for (int64_t c = c0; c < c1 && m < lim; c++) {
        const uint32_t idx = u.sorted[c];
        const uint32_t ij = ws.cand_ij[idx];
        const int i = (int)(ij >> 16), j = (int)(ij & 0xffff);
        if (usedA[i] || usedB[j]) continue;
        usedA[i] = 1;
        usedB[j] = 1;
        const double vx = __dsub_rn(ws.peak_x[(size_t)pb * capP + j], ws.peak_x[(size_t)pa * capP + i]);
        const double vy = __dsub_rn(ws.peak_y[(size_t)pb * capP + j], ws.peak_y[(size_t)pa * capP + i]);
        ws.conn_ij[cb + m] = ij;
        ws.conn_score[cb + m] = ws.cand_score[idx];
        ws.conn_norm[cb + m] = __dsqrt_rn(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)));
        m++;
    }
    ws.conn_count[k] = m;
}

// find_people + the process() tail for the image, one CTA.  The person table `u.table` has capR = ws.capR rows.
__global__ void __launch_bounds__(kUbAssembleThreads) ub_assemble_kernel(UbArgs u, AssembleArgs a) {
    __shared__ int s_out;
    const Workspace &ws = a.ws;
    const PersonTable &t = u.table;
    const int tid = threadIdx.x, K = ws.K, L = ws.L, capP = ws.capP, capR = ws.capR;
    if (tid == 0) {
        int off = 0;
        for (int c = 0; c < K; c++) {
            t.off[c] = off;
            off += ws.peak_count[c];
        }
        t.off[K] = off;
    }
    for (int i = tid; i < K * capP; i += kUbAssembleThreads) {
        t.owner[i] = -1;
        t.ps[i] = ws.peak_score[i];
    }
    __syncthreads();
    int nrows = 0;
    if (tid == 0) {
        for (int k = 0; k < L; k++) {
            const int cc = ws.conn_count[k];
            if (cc < 0) continue;  // special_k (:290)
            ConnCtx c;
            c.A = ws.limbs[2 * k];
            c.B = ws.limbs[2 * k + 1];
            const int offA = t.off[c.A];
            c.offB = t.off[c.B];
            c.slotA = t.slot + (size_t)c.A * capR;
            c.slotB = t.slot + (size_t)c.B * capR;
            c.ownB_base = t.owner + (size_t)c.B * capP;
            c.psB_base = t.ps + (size_t)c.B * capP;
            for (int r = 0; r < cc; r++) {
                const uint32_t ij = ws.conn_ij[(size_t)k * capP + r];
                c.s = ws.conn_score[(size_t)k * capP + r];
                c.len = ws.conn_norm[(size_t)k * capP + r];
                c.ia = (int)(ij >> 16);
                c.jb = (int)(ij & 0xffff);
                c.idA = offA + c.ia;
                c.idB = c.offB + c.jb;
                c.psA = (double)t.ps[(size_t)c.A * capP + c.ia];
                c.psB = (double)c.psB_base[c.jb];
                c.ownA = t.owner + (size_t)c.A * capP + c.ia;
                c.ownB = c.ownB_base + c.jb;
                const int ra = *c.ownA, rb = *c.ownB;
                if (ra >= 0 && rb >= 0 && ra != rb) {
                    apply_two_rows(t, a, c.A, c.B, ra, rb, c.s, c.len);
                } else {
                    apply_zero_or_one(t, a, c, ra, rb, nrows, nrows);  // a new row is born at index nrows
                    if (ra < 0 && rb < 0) nrows++;
                }
            }
        }
        s_out = nrows;
    }
    __syncthreads();
    AsmResult res;
    res.nrows = s_out;
    res.flags = 0;
    __syncthreads();
    emit_people(a, t, nullptr, 0, &s_out, 0, 0, res, tid, kUbAssembleThreads);
}

}  // namespace spg
