// cocoeval.cuh -- pycocotools' COCOeval for iouType='keypoints' (the metric evaluate.py:617-621 reports) on the device:
// computeOks, evaluateImg and accumulate over every (category, image) unit at once.
//
// Inputs are the packed arrays of spg_coco_data (include/spgroup.h); cocoeval.cu sorts the detections with CUB's stable
// radix sort on coco_score_key, which orders like numpy's mergesort of -score (NaN last, -0.0 == 0.0, ties in input
// order).  Then:
//   coco_oks_kernel:        one thread per OKS matrix entry (ragged over units).  The 17 terms are summed in numpy's
//                           pairwise order (sequential below 8 terms; 8 strided accumulators combined as
//                           ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the tail, up to 128 terms) and divided by their
//                           count.  exp is CUDA's double exp (within 1 ULP); every other operation is numpy's, in
//                           numpy's order (-fmad=false: no contraction).
//   coco_match_kernel:      one warp per (unit, area range, threshold): evaluateImg's greedy matcher.  Ground truths
//                           are visited in its order (not ignored first, each group in annotation order) 32 at a time;
//                           a ballot finds the last NaN OKS (which resets the running threshold), a shuffle max and a
//                           ballot find the last ground truth at the maximum -- the sequential scan's `iou < thr`
//                           rule, its crowd skip and its break at the first ignored ground truth after a match.
//   coco_accumulate_kernel: one CTA per (category, area range, maxDet, threshold): block scans of the tp / fp counts
//                           over the category's score-sorted detections, the precision envelope as a reverse max scan,
//                           and a lower-bound search of each recall threshold.  Integer scans and one thread per value
//                           of each float64 operation: nothing depends on the launch or the SM count.
#pragma once

#include <cub/cub.cuh>

#include "../../include/spgroup.h"
#include "common.cuh"

namespace spg {

constexpr int kCocoThreads = 256;
constexpr int kCocoWarps = kCocoThreads / 32;
constexpr int kCocoMaxKpt = 128;  // numpy's pairwise sum has one block of 8 accumulators up to 128 terms

// Ascending order of this key is numpy's order of -score: NaN last, -0.0 folded into 0.0, +-inf ordinary values.
__device__ __forceinline__ unsigned long long coco_score_key(double score) {
    double x = -score;
    if (x != x) return ~0ull;
    if (x == 0.0) x = 0.0;
    const unsigned long long b = (unsigned long long)__double_as_longlong(x);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

// the unit of entry `i` of a ragged array with `n + 1` starts: the last unit whose start is <= i
__device__ __forceinline__ int coco_unit_of(const int32_t *start, int n, int i) {
    int lo = 0, hi = n;  // start[lo] <= i < start[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (start[mid] <= i) lo = mid;
        else hi = mid;
    }
    return lo;
}

// the sort keys of every detection: its score's, and its position as the value
__global__ void coco_keys_kernel(spg_coco_data d, unsigned long long *key, int32_t *val) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d.n_dt; i += gridDim.x * blockDim.x) {
        key[i] = coco_score_key(d.dt_score[i]);
        val[i] = i;
    }
}

// the unit and the category of each detection in score order: the keys of the two stable sorts that follow
__global__ void coco_group_keys_kernel(spg_coco_data d, const int32_t *by_score, uint32_t *unit_key, uint32_t *cat_key) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < d.n_dt; j += gridDim.x * blockDim.x) {
        const int u = d.dt_unit[by_score[j]];
        unit_key[j] = (uint32_t)u;
        cat_key[j] = (uint32_t)(u / d.n_images);
    }
}

__global__ void coco_rank_kernel(spg_coco_data d, spg_coco_eval e) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < d.n_dt; j += gridDim.x * blockDim.x) {
        const int i = e.dt_order[j];
        e.dt_rank[i] = j - d.dt_start[d.dt_unit[i]];
    }
}

// np.max((0, v)) of one coordinate: NaN propagates
__device__ __forceinline__ double coco_pos(double v) { return v != v ? v : (v > 0.0 ? v : 0.0); }

__global__ void coco_oks_kernel(spg_coco_params p, spg_coco_data d, spg_coco_eval e) {
    const int n_units = d.n_images * d.n_cats;
    const int K = p.n_kpt;
    const double eps = 2.220446049250313e-16;  // np.spacing(1)
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d.n_ious; i += gridDim.x * blockDim.x) {
        const int u = coco_unit_of(d.iou_start, n_units, i);
        const int G = d.gt_start[u + 1] - d.gt_start[u];
        const int local = i - d.iou_start[u];
        const int row = local / G, col = local - row * G;
        const int gi = d.gt_start[u] + col;
        const int di = e.dt_order[d.dt_start[u] + row];
        const double *g = d.gt_kpts + (size_t)gi * K * 3;
        const double *t = d.dt_kpts + (size_t)di * K * 3;
        int k1 = 0;
        for (int k = 0; k < K; k++) k1 += g[3 * k + 2] > 0.0;
        const double *bb = d.gt_bbox + (size_t)gi * 4;
        const double x0 = bb[0] - bb[2], x1 = bb[0] + bb[2] * 2.0;
        const double y0 = bb[1] - bb[3], y1 = bb[1] + bb[3] * 2.0;
        const double area = d.gt_area[gi] + eps;
        const int n = k1 > 0 ? k1 : K;
        const int full = n - n % 8;
        double r[8], res = 0.0;
        bool combined = false;
        int c = 0;
        for (int k = 0; k < K; k++) {
            if (k1 > 0 && !(g[3 * k + 2] > 0.0)) continue;
            double dx, dy;
            if (k1 > 0) {
                dx = t[3 * k] - g[3 * k];
                dy = t[3 * k + 1] - g[3 * k + 1];
            } else {
                dx = coco_pos(x0 - t[3 * k]) + coco_pos(t[3 * k] - x1);
                dy = coco_pos(y0 - t[3 * k + 1]) + coco_pos(t[3 * k + 1] - y1);
            }
            const double ek = (dx * dx + dy * dy) / p.kpt_vars[k] / area / 2.0;
            const double v = exp(-ek);
            if (n < 8) {
                res += v;
            } else if (c < 8) {
                r[c] = v;
            } else if (c < full) {
                r[c & 7] += v;
            } else {
                if (!combined) res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
                combined = true;
                res += v;
            }
            c++;
        }
        if (n >= 8 && !combined) res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
        e.ious[i] = res / (double)n;
    }
}

// evaluateImg(image, category, areaRng[a], maxDets[-1]) for every unit, area range and threshold: one warp each
__global__ void __launch_bounds__(kCocoThreads) coco_match_kernel(spg_coco_params p, spg_coco_data d, spg_coco_eval e) {
    const int lane = threadIdx.x & 31;
    const long long w = (long long)blockIdx.x * kCocoWarps + (threadIdx.x >> 5);
    const int T = p.n_iou, A = p.n_area;
    if (w >= (long long)d.n_images * d.n_cats * A * T) return;
    const int t = (int)(w % T), a = (int)((w / T) % A), u = (int)(w / ((long long)T * A));
    const unsigned lt = (1u << lane) - 1u;
    const int g0 = d.gt_start[u], G = d.gt_start[u + 1] - g0;
    const int k0 = d.kept_start[u], D = d.kept_start[u + 1] - k0;
    const double lo = p.area_rng[2 * a], hi = p.area_rng[2 * a + 1];
    const double cap = 1 - 1e-10, thr = cap < p.iou_thrs[t] ? cap : p.iou_thrs[t];  // Python's min([t, 1 - 1e-10])
    int64_t *gtm = e.gt_matches + ((size_t)a * T + t) * d.n_gt + g0;
    int64_t *dtm = e.dt_matches + ((size_t)a * T + t) * d.n_kept + k0;
    uint8_t *dig = e.dt_ignore + ((size_t)a * T + t) * d.n_kept + k0;
    auto ignored = [&](int g) {
        const double ar = d.gt_area[g0 + g];
        return (d.gt_flags[g0 + g] & SPG_COCO_IGNORE) || ar < lo || ar > hi;
    };
    // evaluateImg's order of the ground truths: the stable sort by _ignore
    int n_keep = 0;
    for (int c = 0; c < G; c += 32) n_keep += __popc(__ballot_sync(~0u, c + lane < G && !ignored(c + lane)));
    for (int c = 0, keep_seen = 0, ign_seen = 0; c < G; c += 32) {
        const int g = c + lane;
        const bool valid = g < G, ig = valid && ignored(g);
        const unsigned bk = __ballot_sync(~0u, valid && !ig), bi = __ballot_sync(~0u, ig);
        const int pos = ig ? n_keep + ign_seen + __popc(bi & lt) : keep_seen + __popc(bk & lt);
        if (valid) {
            gtm[pos] = 0;
            if (t == 0) {
                e.gt_order[(size_t)a * d.n_gt + g0 + pos] = g0 + g;
                e.gt_ignore[(size_t)a * d.n_gt + g0 + pos] = ig;
            }
        }
        keep_seen += __popc(bk);
        ign_seen += __popc(bi);
    }
    __syncwarp();
    const double *ious = e.ious + d.iou_start[u];
    for (int r = 0; r < D; r++) {
        const int di = e.dt_order[d.dt_start[u] + r];
        const double *row = ious + (size_t)r * G;
        double s = thr;   // the running `iou`
        int m = -1, mg = -1, mph = 0;  // the match: its position in the order, its index in the unit, ignored or not
        // phase 0 scans the ground truths that are not ignored; phase 1 the ignored ones, reached only without a match
        // (the scan breaks at the first ignored ground truth once a match that is not ignored exists)
        for (int ph = 0; ph < 2 && m < 0; ph++) {
            for (int c = 0, seen = 0; c < G; c += 32) {
                const int g = c + lane;
                const bool member = g < G && (int)ignored(g) == ph;
                const unsigned bm = __ballot_sync(~0u, member);
                const int pos = (ph ? n_keep : 0) + seen + __popc(bm & lt);
                seen += __popc(bm);
                const bool elig = member && !(gtm[pos] > 0 && !(d.gt_flags[g0 + g] & SPG_COCO_CROWD));
                const double v = elig ? row[g] : 0.0;
                // a NaN OKS is taken (`NaN < iou` is false) and makes the next eligible one taken whatever its value
                const unsigned bn = __ballot_sync(~0u, elig && v != v);
                unsigned region = ~0u;
                if (bn) {
                    const int q = 31 - __clz(bn);
                    s = __longlong_as_double(0x7ff8000000000000LL);
                    m = __shfl_sync(~0u, pos, q);
                    mg = c + q;
                    mph = ph;
                    region = q == 31 ? 0u : (~0u << (q + 1));
                }
                const bool cand = elig && ((region >> lane) & 1u) && !(v < s);
                if (__ballot_sync(~0u, cand)) {
                    double mx = cand ? v : -INFINITY;
                    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(~0u, mx, o));
                    const int q = 31 - __clz(__ballot_sync(~0u, cand && v == mx));  // ties: the last
                    s = mx;
                    m = __shfl_sync(~0u, pos, q);
                    mg = c + q;
                    mph = ph;
                }
            }
        }
        if (lane == 0) {
            int64_t id = 0;
            if (m >= 0) {
                id = d.gt_id[g0 + mg];
                gtm[m] = d.dt_id[di];
            }
            const double ad = d.dt_area[di];
            dtm[r] = id;
            dig[r] = (m >= 0 && mph) || (id == 0 && (ad < lo || ad > hi));
        }
        __syncwarp();
    }
}

struct CocoCounts {
    int n, tp, fp;
};
struct CocoCountsSum {
    __device__ __forceinline__ CocoCounts operator()(const CocoCounts &a, const CocoCounts &b) const {
        return {a.n + b.n, a.tp + b.tp, a.fp + b.fp};
    }
};
struct CocoMin {
    __device__ __forceinline__ int operator()(int a, int b) const { return a < b ? a : b; }
};
struct CocoMax {
    __device__ __forceinline__ double operator()(double a, double b) const { return a < b ? b : a; }
};

// accumulate() of one (category k, area range a, maxDet m, threshold t): precision[t, :, k, a, m], scores[t, :, k, a, m]
// and recall[t, k, a, m].  Scratch: the category's detections at most once each, as the cumulative true positives
// `tp`, their detection `src` and the precision `pr` (then its envelope) at each kept position.
__global__ void __launch_bounds__(kCocoThreads) coco_accumulate_kernel(spg_coco_params p, spg_coco_data d, spg_coco_eval e,
                                                                       double *precision, double *recall, double *scores,
                                                                       int32_t *tp, int32_t *src, double *pr) {
    using Scan3 = cub::BlockScan<CocoCounts, kCocoThreads>;
    using ScanD = cub::BlockScan<double, kCocoThreads>;
    using RedI = cub::BlockReduce<int, kCocoThreads>;
    __shared__ union {
        typename Scan3::TempStorage s3;
        typename ScanD::TempStorage sd;
        typename RedI::TempStorage ri;
    } tmp;
    __shared__ int s_int;
    const int T = p.n_iou, R = p.n_rec, A = p.n_area, M = p.n_max_dets, K = d.n_cats, I = d.n_images;
    int b = blockIdx.x;
    const int t = b % T; b /= T;
    const int m = b % M; b /= M;
    const int a = b % A;
    const int k = b / A;
    const int tid = threadIdx.x;
    const double lo = p.area_rng[2 * a], hi = p.area_rng[2 * a + 1];
    const int c0 = d.dt_start[k * I], c1 = d.dt_start[(k + 1) * I];  // the category's detections in cat_order
    // this CTA's scratch: its (area, maxDet, threshold) plane of n_dt entries, at the category's own range [c0, c1) of it,
    // so that the CTAs of different categories never share a slot
    const size_t at = (((size_t)a * M + m) * T + t) * d.n_dt + c0;
    tp += at;
    src += at;
    pr += at;
    const size_t out_r = ((size_t)k * A + a) * M + m;  // (k, a, m) of [.., K, A, M]
    const size_t step_r = (size_t)K * A * M;

    // npig: the category's ground truths that are not ignored in this area range
    int own = 0;
    for (int g = d.gt_start[k * I] + tid; g < d.gt_start[(k + 1) * I]; g += kCocoThreads) {
        const double ar = d.gt_area[g];
        own += !((d.gt_flags[g] & SPG_COCO_IGNORE) || ar < lo || ar > hi);
    }
    const int npig_b = RedI(tmp.ri).Sum(own);
    if (tid == 0) s_int = npig_b;
    __syncthreads();
    const int npig = s_int;
    if (npig == 0) {  // `continue`: the slots keep their -1
        for (int r = tid; r < R; r += kCocoThreads) {
            precision[((size_t)t * R + r) * step_r + out_r] = -1.0;
            scores[((size_t)t * R + r) * step_r + out_r] = -1.0;
        }
        if (tid == 0) recall[(size_t)t * step_r + out_r] = -1.0;
        return;
    }
    const double eps = 2.220446049250313e-16;
    const int lim = p.max_dets[m];
    // 1. the kept detections in score order: cumulative tp and fp, and the precision at each
    CocoCounts carry{0, 0, 0};
    for (int base = c0; base < c1; base += kCocoThreads) {
        const int j = base + tid;
        CocoCounts x{0, 0, 0};
        int i = -1;
        if (j < c1) {
            i = e.cat_order[j];
            const int rank = e.dt_rank[i], u = d.dt_unit[i];
            // rank < the unit's kept count too: a max_dets table that is not ascending cannot index past the unit
            if (rank < lim && rank < d.kept_start[u + 1] - d.kept_start[u]) {
                const size_t q = ((size_t)a * T + t) * d.n_kept + d.kept_start[u] + rank;
                const bool matched = e.dt_matches[q] != 0, ign = e.dt_ignore[q] != 0;
                x = {1, matched && !ign, !matched && !ign};
            }
        }
        CocoCounts y, agg;
        Scan3(tmp.s3).InclusiveScan(x, y, CocoCountsSum(), agg);
        if (x.n) {
            const int pos = carry.n + y.n - 1;
            const int ctp = carry.tp + y.tp, cfp = carry.fp + y.fp;
            tp[pos] = ctp;
            src[pos] = i;
            pr[pos] = (double)ctp / (((double)cfp + (double)ctp) + eps);
        }
        carry = CocoCountsSum()(carry, agg);
        __syncthreads();
    }
    const int nd = carry.n;
    // 2. the envelope: each precision becomes the maximum of itself and every later one
    double right = -INFINITY;
    for (int base = nd - 1; base >= 0; base -= kCocoThreads) {
        const int pos = base - tid;
        const double x = pos >= 0 ? pr[pos] : -INFINITY;
        double y, agg;
        ScanD(tmp.sd).InclusiveScan(x, y, CocoMax(), agg);
        if (pos >= 0) pr[pos] = CocoMax()(y, right);
        right = CocoMax()(right, agg);
        __syncthreads();
    }
    // 3. recall, then each recall threshold's first position with rc >= it (numpy's searchsorted, side='left'); from the
    // first threshold whose position is nd on, the slots stay 0 (pycocotools' try/except ends its loop there)
    if (tid == 0) recall[(size_t)t * step_r + out_r] = nd ? (double)tp[nd - 1] / (double)npig : 0.0;
    auto lower_bound = [&](double x) {
        int l = 0, h = nd;
        while (l < h) {
            const int mid = (l + h) >> 1;
            const double rc = (double)tp[mid] / (double)npig;
            if (rc < x || (x != x && rc == rc)) l = mid + 1;  // numpy's less-than: NaN after everything
            else h = mid;
        }
        return l;
    };
    int first_out = R;
    for (int r = tid; r < R; r += kCocoThreads)
        if (lower_bound(p.rec_thrs[r]) >= nd) {
            first_out = r;
            break;
        }
    const int stop = RedI(tmp.ri).Reduce(first_out, CocoMin());
    if (tid == 0) s_int = stop;
    __syncthreads();
    for (int r = tid; r < R; r += kCocoThreads) {
        double q = 0.0, ss = 0.0;
        if (r < s_int) {
            const int pos = lower_bound(p.rec_thrs[r]);
            q = pr[pos];
            ss = d.dt_score[src[pos]];
        }
        precision[((size_t)t * R + r) * step_r + out_r] = q;
        scores[((size_t)t * R + r) * step_r + out_r] = ss;
    }
}

}  // namespace spg
