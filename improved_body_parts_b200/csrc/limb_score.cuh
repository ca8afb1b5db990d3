// limb_score.cuh -- K2a: line-integral scoring of every candidate keypoint pair of every limb.
//
// Replaces the scoring half of find_connections (/root/reference/evaluate.py:211-255).
//
// One CTA per (image, limb).  The limb's body-part plane (H*W elements, one contiguous span) is staged
// into shared memory by the bulk-copy engine (TMA, SASS UBLKCP) in a few large chunks on one mbarrier,
// while the threads stage the two end-point peak lists; HBM is read exactly once per plane element and
// all nearest-neighbour gathers hit shared memory.  Planes that do not fit in shared memory (e.g.
// 512x512) are sampled through L2 instead (STAGE = false).
//
// Two phases keep the kernel on the HBM roofline instead of the issue roofline (nA*nB pairs per limb,
// ~3 % of which are real limbs):
//   A. SCREEN, one thread per pair, cheap f32 arithmetic.  A pair can only become a candidate if at
//      least ceil(connect_ration*m) of its m samples exceed thre2 (:246), i.e. it tolerates at most
//      maxfail = m - ceil(.) failing samples.  The screen looks at <= 10 interior samples (positions in
//      1/64-px fixed point from one FFMA) and counts a failure only when it is CERTAIN: the position is
//      at least 1.5/64 px away from a rounding boundary (so it rounds to the same pixel as the reference's
//      f64 position) and the map value there is <= thre2.  More than maxfail certain failures => the reference rejects the pair => drop it.
//      Anything uncertain (near-boundary sample, sample count m near a rounding boundary, an end point that
//      is not inside the map [0, W-1] x [0, H-1], coincident end points) survives.  The screen can only drop pairs the reference
//      drops; it never decides an accept.
//   B. EXACT, one thread per surviving pair: the reference's arithmetic operation for operation --
//      f64 np.linspace positions, half-to-even rounding, SEQUENTIAL sum of the samples in the plane's
//      precision (Python sum() over np.float32, :241; a shuffle-tree reduction would round differently and
//      can flip threshold / ordering decisions), f32/f64 score and priority exactly as numpy promotes them.
// Survivors are handed from A to B through a bitmask + prefix sums in shared memory (balanced, ordered,
// no atomics); candidates are appended with a warp-aggregated shared-memory atomic and written unordered --
// the matcher orders them by (priority desc, i*nB+j asc), the reference's stable-sort order (:259).
#pragma once

#include "common.cuh"

namespace spg {

struct ScoreArgs {
    const void *paf;
    int64_t img_stride, chan_stride;  // elements
    int H, W, image_base, mid_num, screen;
    int crit1_strict;                                // demo_image.py:288 compares with `>` where evaluate.py:246 uses `>=`
    int exact_warps;                                 // persistent kernel: scorer warps (the rest screen)
    double image_extent, thre2, connect_ration;
    Workspace ws;
};

constexpr int kScoreThreads = 512;
constexpr uint32_t kBulkChunkBytes = 32768;
constexpr int kScreenMaxMid = 63;       // per-m tables (maxfail, sample positions, reciprocals)
#ifndef SPG_SCREEN_SAMPLES
#define SPG_SCREEN_SAMPLES 10
#endif
constexpr int kScreenSamples = SPG_SCREEN_SAMPLES;  // interior samples looked at per pair (build-time: `make variants` for the tuning sweep)
constexpr int kScreenMaxDim = 2048;     // f32 error of a 1/64-px position stays << 1 unit up to this map size
// The persistent screen's rows open with this many samples spread evenly over the interior, then take the others in
// order (build_screen_row).  Same samples, same failures counted: only the order in which a warp's lanes look at them
// changes.  The order itself was measured not to change the speed; the register allocation ptxas makes of the
// persistent kernel with this builder does (DESIGN.md §3, K2a).
constexpr int kScreenSpreadFirst = kScreenSamples < 6 ? kScreenSamples : 6;

// per-m constants of the screen (m = number of samples the reference would take for the pair)
struct alignas(8) ScreenTab {
    float inv;            // 1 / (m - 1)
    signed char maxfail;  // failures the connect_ration criterion tolerates
    unsigned char qn;     // interior samples the screen looks at
    unsigned char pad[2];
};

// The per-m tables of both kernels, in this order: rcp[m] = RN(1/m) (phase B), ScreenTab tab[m], ts[m][kScreenSamples]
// (sample positions of the screen); m = 0 .. kScreenMaxMid.
__host__ __device__ constexpr size_t screen_tables_bytes() {
    return (((size_t)(kScreenMaxMid + 1) * (sizeof(double) + sizeof(ScreenTab) + kScreenSamples * sizeof(float))) + 15) & ~(size_t)15;
}

// Builds row m of the per-m tables.  spread: the persistent kernel's sample order (kScreenSpreadFirst), else ascending.
__device__ __forceinline__ void build_screen_row(const ScoreArgs &a, int m, double *rcp, ScreenTab *tab, float *ts, bool spread) {
    // fewest samples that must exceed thre2: smallest integer >= connect_ration*m in f64, as :246 compares
    const double need = __dmul_rn(a.connect_ration, (double)m);
    int need_i = (int)need;
    if ((double)need_i < need || (a.crit1_strict && (double)need_i == need)) need_i++;  // strict: smallest integer > need
    rcp[m] = m > 0 ? __ddiv_rn(1.0, (double)m) : 0.0;
    // up to kScreenSamples samples spread over the interior [lo, hi] (the ends sit on the peaks and rarely fail); sample r
    // of the qn sits at lo + r * (hi - lo) / (qn - 1).  Entries past qn repeat sample qn - 1 (tail clamped: every entry
    // is a valid sample index).
    const int lo = m / 8, hi = m - 1 - lo;
    const int qn = max(0, min(kScreenSamples, hi - lo + 1));
    auto put = [&](int q, int r) { ts[m * kScreenSamples + q] = (float)(qn > 1 ? lo + (r * (hi - lo)) / (qn - 1) : lo); };
    if (!spread) {
        for (int q = 0; q < kScreenSamples; q++) put(q, min(q, max(qn - 1, 0)));
    } else {
        // first s1 samples at ranks ~ q * (qn - 1) / (s1 - 1): the step is >= 1, so they are distinct and the last is
        // qn - 1; then the ranks not taken yet, ascending; then the tail
        const int s1 = min(kScreenSpreadFirst, qn);
        const float step = s1 > 1 ? (float)(qn - 1) / (float)(s1 - 1) : 0.0f;
        uint32_t taken = 0;  // bit r: sample r is in the first s1
        for (int q = 0; q < s1; q++) {
            const int r = min((int)__fadd_rn(__fmul_rn((float)q, step), 0.5f), qn - 1);
            taken |= 1u << r;
            put(q, r);
        }
        for (int q = s1, r = 0; q < kScreenSamples; q++) {
            if (q < qn) {
                while (taken >> r & 1u) r++;
                put(q, r++);
            } else {
                put(q, max(qn - 1, 0));
            }
        }
    }
    ScreenTab t;
    t.inv = m > 1 ? 1.0f / (float)(m - 1) : 0.0f;
    t.maxfail = (signed char)max(min(m - need_i, 127), -1);
    t.qn = (unsigned char)qn;
    t.pad[0] = t.pad[1] = 0;
    tab[m] = t;
}

inline size_t score_smem_bytes(size_t plane_bytes, int capP) {
    const size_t plane = (plane_bytes + 127) & ~(size_t)127;
    const size_t peaks = (size_t)capP * (4 * sizeof(double) + 6 * sizeof(float) + 2);
    const size_t words = ((size_t)capP * capP + 31) / 32;
    return plane + ((peaks + 15) & ~(size_t)15) + screen_tables_bytes() + words * (sizeof(uint32_t) + sizeof(uint16_t)) + 16;
}

// inside the map [0, W-1] x [0, H-1]
__device__ __forceinline__ bool inside_map(double x, double y, int H, int W) {
    return x >= 0.0 && x <= (double)(W - 1) && y >= 0.0 && y <= (double)(H - 1);
}

struct PairGeom {  // one limb's end-point lists in shared memory
    const double *ax, *ay, *bx, *by;
    const float *as, *bs;
    const double *rcp;  // rcp[d] = RN(1/d), d = 1 .. mid_num-1
};

// Phase B: the reference's evaluation of one pair (evaluate.py:224-255).  Returns true if it is a candidate.  `flags`
// collects what the reference would raise for -- kStNonfinite (a non-finite pair length: round() at :226 raises),
// kStSampleIndex (a sample outside the map: :235 raises) -- and kStNanPrioCand for a candidate with a NaN priority.
// kExactBatch: samples of the exact evaluation whose index computations and loads are in flight together (register budget)
// T: the type the plane is STORED in; TA: the type the reference's arithmetic runs in (TA = double with T = float is
// SPG_F32_AS_F64: float64 maps whose values are exact float32 numbers, the single-scale output of predict()).
template <typename T, int kExactBatch = 1, typename TA = T>
__device__ __forceinline__ bool score_pair_exact(const T *__restrict__ plane, int H, int W, const ScoreArgs &a,
                                                 const PairGeom &g, int i, int j, bool interior, TA thre2,
                                                 double &score, double &prio, uint32_t &flags) {
    const double ax = g.ax[i], ay = g.ay[i], bx = g.bx[j], by = g.by[j];
    const double vx = __dsub_rn(bx, ax), vy = __dsub_rn(by, ay);                            // :224
    const double n2 = __dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy));
    // a NaN or infinite end point (or a length past DBL_MAX): int(round(norm + 1)) at :226 raises before the norm == 0
    // test.  Returning here also keeps a NaN position away from every index computation below.
    if (!isfinite(n2)) {
        flags |= kStNonfinite;
        return false;
    }
    if (n2 == 0.0) return false;                             // norm == 0 (:228-230); sqrt(x) == 0 iff x == 0
    // norm = sqrt(n2) (:225) is only materialised when a decision needs it:
    //  - m = min(round(norm + 1), mid_num) (:226): n2 >= mid_num^2 implies norm >= mid_num, hence m = mid_num;
    //  - the distance prior (:241) is negative iff norm > 0.5*extent (correctly rounded division is monotone
    //    and 1 - 2^-53 is representable), which cannot happen while n2 <= (0.5*extent)^2 * (1 - 1e-9).
    const double half = __dmul_rn(0.5, a.image_extent);
    const double Md = (double)a.mid_num;
    double norm = 0.0;
    int m = a.mid_num;
    const bool need_norm = n2 < __dmul_rn(Md, Md) || n2 > __dmul_rn(__dmul_rn(half, half), 1.0 - 1e-9);
    if (need_norm) {
        norm = __dsqrt_rn(n2);
        m = min(__double2int_rn(__dadd_rn(norm, 1.0)), a.mid_num);                           // round() half-even
    }
    // np.linspace(A, B, m): step = delta/(m-1); y_t = t*step + start (two roundings); y_{m-1} = stop.
    // delta/(m-1) by Markstein's correction: with y = RN(1/d), q0 = RN(delta*y), r = RN(delta - q0*d) (exact, FMA),
    // RN(q0 + r*y) is the correctly rounded quotient (tests/test_numerics.py checks it against exact rationals).
    double stepx = 0.0, stepy = 0.0;
    if (m > 1) {
        const double dd = (double)(m - 1);
        if (m - 1 <= kScreenMaxMid) {
            const double y = g.rcp[m - 1];
            const double qx = __dmul_rn(vx, y), qy = __dmul_rn(vy, y);
            stepx = __fma_rn(__fma_rn(-qx, dd, vx), y, qx);
            stepy = __fma_rn(__fma_rn(-qy, dd, vy), y, qy);
        } else {  // mid_num beyond the reciprocal table (the reference accepts any mid_num): the plain correctly rounded division
            stepx = __ddiv_rn(vx, dd);
            stepy = __ddiv_rn(vy, dd);
        }
    }
    TA sum = (TA)0;
    int above = 0;
    if (interior) {
        // both end points lie inside the map ([0, W-1] x [0, H-1]) and the samples stay between them (to within an
        // f64 rounding error): no index can leave the map, no negative index can wrap
        const int last = m - 1;
        double td = 0.0;
        if constexpr (kExactBatch <= 1) {
            // plane in shared memory, tight register budget: the plain loop
#pragma unroll 4
            for (int t = 0; t < last; t++) {
                // :235 nearest neighbour, half-to-even: x + 1.5 * 2^52 leaves round(x) in the low word for |x| < 2^31
                // (a DADD instead of F2I.F64 on the quarter-rate conversion pipe)
                const int xi = __double2loint(__dadd_rn(__dadd_rn(__dmul_rn(td, stepx), ax), 6755399441055744.0));
                const int yi = __double2loint(__dadd_rn(__dadd_rn(__dmul_rn(td, stepy), ay), 6755399441055744.0));
                const TA v = (TA)plane[yi * W + xi];
                sum = sum + v;  // sequential, in sample order, in the plane's precision (:241)
                above += v > thre2;
                td = __dadd_rn(td, 1.0);
            }
        } else {
            // The m-1 samples before the end point, kExactBatch at a time: all index computations and loads of a batch
            // are independent and in flight together (the plane is read through L2); samples past m-1 read a valid
            // address (sample 0) and are not accumulated, so no sample sees a different operation sequence.
            for (int t0 = 0; t0 < last; t0 += kExactBatch) {
                T vv[kExactBatch > 0 ? kExactBatch : 1];
#pragma unroll
                for (int u = 0; u < kExactBatch; u++) {
                    const double tdu = t0 + u < last ? __dadd_rn(td, (double)u) : 0.0;
                    const int xi = __double2loint(__dadd_rn(__dadd_rn(__dmul_rn(tdu, stepx), ax), 6755399441055744.0));
                    const int yi = __double2loint(__dadd_rn(__dadd_rn(__dmul_rn(tdu, stepy), ay), 6755399441055744.0));
                    vv[u] = plane[yi * W + xi];
                }
#pragma unroll
                for (int u = 0; u < kExactBatch; u++) {
                    if (t0 + u < last) {
                        sum = sum + (TA)vv[u];  // sequential, in sample order, in the plane's precision (:241)
                        above += (TA)vv[u] > thre2;
                    }
                }
                td = __dadd_rn(td, (double)kExactBatch);
            }
        }
        const TA v = (TA)(m > 1 ? plane[__double2int_rn(by) * W + __double2int_rn(bx)]
                               : plane[__double2int_rn(ay) * W + __double2int_rn(ax)]);
        sum = sum + v;
        above += v > thre2;
    } else {
        for (int t = 0; t < m; t++) {
            double sx, sy;
            if (t == m - 1 && m > 1) {
                sx = bx;
                sy = by;
            } else {
                sx = __dadd_rn(__dmul_rn((double)t, stepx), ax);
                sy = __dadd_rn(__dmul_rn((double)t, stepy), ay);
            }
            int yi = __double2int_rn(sy), xi = __double2int_rn(sx);
            if (yi < 0) yi += H;  // numpy index semantics: negatives wrap once
            if (xi < 0) xi += W;
            if (yi < 0 || yi >= H || xi < 0 || xi >= W) {  // the reference would raise IndexError
                flags |= kStSampleIndex;
                return false;
            }
            const TA v = (TA)plane[(size_t)yi * W + xi];
            sum = sum + v;
            above += v > thre2;
        }
    }
    // :241 -- `image_width` is the image HEIGHT at the call site (:510)
    double prior = 0.0;  // only its value when negative matters: min(prior, 0)
    if (need_norm && norm > half) prior = __dsub_rn(__ddiv_rn(half, norm), 1.0);
    if (sizeof(TA) == 4) {
        float s = __fdiv_rn((float)sum, (float)m);
        s = __fadd_rn(s, prior < 0.0 ? __double2float_rn(prior) : 0.0f);  // f32 + weak Python float
        const float pr = __fadd_rn(__fadd_rn(__fmul_rn(0.5f, s), __fmul_rn(0.25f, g.as[i])), __fmul_rn(0.25f, g.bs[j]));
        score = (double)s;
        prio = (double)pr;
    } else {
        score = __dadd_rn(__ddiv_rn((double)sum, (double)m), prior < 0.0 ? prior : 0.0);
        prio = __dadd_rn(__dadd_rn(__dmul_rn(0.5, score), (double)__fmul_rn(0.25f, g.as[i])),
                         (double)__fmul_rn(0.25f, g.bs[j]));
    }
    const double need = __dmul_rn(a.connect_ration, (double)m);
    const bool crit1 = a.crit1_strict ? (double)above > need : (double)above >= need;       // :246 (demo_image.py:288: `>`)
    const bool crit2 = score > 0.0;                                                         // :251
    if (crit1 && crit2 && isnan(prio)) flags |= kStNanPrioCand;
    return crit1 && crit2;
}

// Candidate `pos` of limb slot `out_base`: pair (i, j) with its score and priority, plus the one-word sort key when the
// priority is an f32 value (TA = float): 32 order-preserving bits + the tie-break fit one word.
template <typename TA>
__device__ __forceinline__ void store_candidate(const Workspace &ws, size_t out_base, int pos, int i, int j, double score, double prio) {
    const uint32_t ij = ((uint32_t)i << 16) | (uint32_t)j;
    ws.cand_prio[out_base + pos] = prio;
    ws.cand_score[out_base + pos] = score;
    ws.cand_ij[out_base + pos] = ij;
    if (sizeof(TA) == 4) {
        const uint32_t b = __float_as_uint((float)prio);
        const uint32_t ord = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
        ws.cand_key[out_base + pos] = ((unsigned long long)ord << 32) | (unsigned long long)(~ij);
    }
}

// Publishes limb `slot` of image n: candidate count (-1 = special_k), survivors of the screen, status bits (`flags` as
// score_pair_exact collects them: a NaN priority matters only when the limb has another candidate to sort it against).
__device__ __forceinline__ void publish_limb(const Workspace &ws, int n, size_t slot, int ncand, int nsurv, uint32_t flags) {
    ws.cand_count[slot] = min(ncand, ws.capC);
    if (ws.surv_count) ws.surv_count[slot] = nsurv;
    if ((flags & kStNanPrioCand) && ncand > 1) flags |= kStNanPriority;
    flags &= ~kStNanPrioCand;
    if (ncand > ws.capC) flags |= kStCandOverflow;
    if (flags) atomicOr(&ws.status[n], flags);
}

// largest float32 <= t: for float32-stored values v, (double)v > t  <=>  v > screen_threshold(t) -- lets the float32
// screen apply the float64 comparison of SPG_F32_AS_F64 exactly
__host__ __device__ inline float f32_not_above(double t) {
    float f = (float)t;
    if ((double)f > t) f = nextafterf(f, -INFINITY);
    return f;
}

// The per-limb schedule: the CTA scores limb k of image n_local of `a` (plane a.paf + n_local * img_stride +
// k * chan_stride, geometry a.H x a.W, a.image_extent) and writes to slot a.image_base + n_local.  `ws` is a.ws, passed
// apart so that a kernel's per-CTA copy of the arguments never has its limb table indexed (that would put it in local memory).
template <typename T, bool STAGE, typename TA>
__device__ __forceinline__ void limb_score_plane(const ScoreArgs &a, const Workspace &ws, int n_local, int k) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t bar;
    __shared__ int s_count;
    __shared__ uint32_t s_flags;
    __shared__ int s_total_surv;
    __shared__ uint32_t s_magic;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = a.image_base + n_local;
    const int H = a.H, W = a.W, capP = ws.capP;
    // Start the plane copy before anything that depends on a global load: it is the longest latency of the CTA.
    const T *gplane = reinterpret_cast<const T *>(a.paf) + (int64_t)n_local * a.img_stride + (int64_t)k * a.chan_stride;
    const size_t plane_bytes = (size_t)H * W * sizeof(T);
    if (tid == 0) {
        s_count = 0;
        s_flags = 0;
        if (STAGE) {
            mbar_init(&bar, 1);
            fence_mbar_init();
            mbar_expect_tx(&bar, (uint32_t)plane_bytes);
            for (size_t off = 0; off < plane_bytes; off += kBulkChunkBytes) {
                const uint32_t bytes = (uint32_t)min((size_t)kBulkChunkBytes, plane_bytes - off);
                bulk_g2s(smem_raw + off, reinterpret_cast<const unsigned char *>(gplane) + off, bytes, &bar);
            }
        }
    }
    const int pa = ws.limbs[2 * k], pb = ws.limbs[2 * k + 1];
    const int nA = min(ws.peak_count[(size_t)n * ws.K + pa], capP);
    const int nB = min(ws.peak_count[(size_t)n * ws.K + pb], capP);
    const size_t slot = (size_t)n * ws.L + k;
    if (nA == 0 || nB == 0) {  // special_k (evaluate.py:272-274)
        if (tid == 0) {
            publish_limb(ws, n, slot, -1, 0, 0);  // no candidates, no survivors (the slot is never left as it was)
            if (STAGE) mbar_wait(&bar, 0);  // the copy must land before the CTA (and its shared memory) goes away
        }
        return;
    }

    unsigned char *after = smem_raw + (STAGE ? ((plane_bytes + 127) & ~(size_t)127) : 0);
    double *s_ax = reinterpret_cast<double *>(after);
    double *s_ay = s_ax + capP;
    double *s_bx = s_ay + capP;
    double *s_by = s_bx + capP;
    float *s_as = reinterpret_cast<float *>(s_by + capP);
    float *s_bs = s_as + capP;
    float *s_fax = s_bs + capP;
    float *s_fay = s_fax + capP;
    float *s_fbx = s_fay + capP;
    float *s_fby = s_fbx + capP;
    unsigned char *s_ain = reinterpret_cast<unsigned char *>(s_fby + capP);  // end point inside the map
    unsigned char *s_bin = s_ain + capP;
    const size_t peaks_bytes = ((size_t)capP * (4 * sizeof(double) + 6 * sizeof(float) + 2) + 15) & ~(size_t)15;
    double *s_rcp = reinterpret_cast<double *>(after + peaks_bytes);  // per-m tables (build_screen_row)
    ScreenTab *s_tab = reinterpret_cast<ScreenTab *>(s_rcp + (kScreenMaxMid + 1));
    float *s_ts = reinterpret_cast<float *>(s_tab + (kScreenMaxMid + 1));
    uint32_t *s_mask = reinterpret_cast<uint32_t *>(after + peaks_bytes + screen_tables_bytes());  // survivor bitmask, bit p = i*nB + j
    const int npairs = nA * nB;
    const int nwords = (npairs + 31) >> 5;
    uint16_t *s_prefix = reinterpret_cast<uint16_t *>(s_mask + (((size_t)capP * capP + 31) >> 5));

    // end-point lists (refined float coordinates + peak scores), overlapped with the plane copy
    const size_t baseA = ((size_t)n * ws.K + pa) * capP, baseB = ((size_t)n * ws.K + pb) * capP;
    // warp-specialised prologue: warp 0 stages the A list, warp 1 the B list, warps 2-3 build the per-m tables;
    // the other warps go straight to the barrier (the prologue is pure issue overhead for them)
    const bool screen = a.screen && a.mid_num <= kScreenMaxMid && H <= kScreenMaxDim && W <= kScreenMaxDim;
    if (warp == 0) {
        for (int i = lane; i < nA; i += 32) {
            const double x = ws.peak_x[baseA + i], y = ws.peak_y[baseA + i];
            s_ax[i] = x; s_ay[i] = y;
            s_fax[i] = (float)(x * 64.0); s_fay[i] = (float)(y * 64.0);  // 1/64-px units for the screen
            s_as[i] = ws.peak_score[baseA + i];
            s_ain[i] = inside_map(x, y, H, W);
        }
    } else if (warp == 1) {
        for (int j = lane; j < nB; j += 32) {
            const double x = ws.peak_x[baseB + j], y = ws.peak_y[baseB + j];
            s_bx[j] = x; s_by[j] = y;
            s_fbx[j] = (float)(x * 64.0); s_fby[j] = (float)(y * 64.0);
            s_bs[j] = ws.peak_score[baseB + j];
            s_bin[j] = inside_map(x, y, H, W);
        }
    } else if (warp < 4) {
        const int m = tid - 64;
        if (m <= a.mid_num && m <= kScreenMaxMid) build_screen_row(a, m, s_rcp, s_tab, s_ts, false);
        if (tid == 64 + 63) s_magic = nB > 1 ? 0xffffffffu / (uint32_t)nB + 1u : 0u;  // ceil(2^32 / nB)
    }
    __syncthreads();
    if (STAGE) mbar_wait(&bar, 0);
    const T *plane = STAGE ? reinterpret_cast<const T *>(smem_raw) : gplane;
    // f32 plane: `> thre2` is an f32 compare against (float)thre2; f64 arithmetic on f32 storage: the equivalent f32 threshold
    const T thre2 = (sizeof(T) == 4 && sizeof(TA) == 8) ? (T)f32_not_above(a.thre2) : (T)a.thre2;
    const TA thre2_exact = (TA)a.thre2;

    // ---------------- phase A: conservative screen ----------------
    const uint32_t magic = s_magic;  // p / nB == umulhi(p, magic) for p < 2^14
    for (int base = 0; base < npairs; base += kScoreThreads) {
        const int p = base + tid;
        bool keep = false;
        if (p < npairs) {
            keep = true;
            if (screen) {
                const int i = nB > 1 ? (int)__umulhi((uint32_t)p, magic) : p;
                const int j = p - i * nB;
                if (s_ain[i] && s_bin[j]) {
                    const float ax64 = s_fax[i], ay64 = s_fay[i];
                    const float dx64 = s_fbx[j] - ax64, dy64 = s_fby[j] - ay64;
                    const float n2 = (dx64 * dx64 + dy64 * dy64) * (1.0f / 4096.0f);  // px^2
                    if (n2 > 1e-6f) {
                        const float q = n2 * rsqrtf(n2) + 1.0f;  // approximate norm + 1: m is only trusted 0.01 away from a tie
                        // branch-free: lanes with long and short pairs must reach the sample loop together
                        const float r = rintf(q);
                        const bool longp = q >= (float)a.mid_num + 0.51f;
                        int m = longp ? a.mid_num : min((int)r, a.mid_num);
                        if (!longp && !(fabsf(q - r) < 0.49f)) m = -1;  // m within 0.01 of a rounding tie -> survive
                        asm volatile("" : "+r"(m));  // keep ONE copy of the sample loop (no specialisation on m == mid_num)
                        if (m >= 1) {
                            const ScreenTab tb = s_tab[m];
                            const int maxfail = tb.maxfail;
                            const int qn = tb.qn;
                            const float inv = tb.inv;
                            const float sx64 = dx64 * inv, sy64 = dy64 * inv;
                            const float *ts = s_ts + m * kScreenSamples;
                            int fails = 0;
                            for (int q2 = 0; q2 < qn; q2++) {
                                const float tf = ts[q2];
                                // position in 1/64 px, off from the reference's f64 position by < 0.51 units
                                const int xs = __float2int_rn(__fmaf_rn(tf, sx64, ax64));
                                const int ys = __float2int_rn(__fmaf_rn(tf, sy64, ay64));
                                // rounding boundaries sit at 32 (mod 64); within {31,32,33} the pixel is uncertain
                                const unsigned cx = (unsigned)(xs + 33) & 63u, cy = (unsigned)(ys + 33) & 63u;
                                const T v = plane[((ys + 32) >> 6) * W + ((xs + 32) >> 6)];
                                fails += (min(cx, cy) > 2u) && !(v > thre2);
                            }
                            keep = fails <= maxfail;
                        }
                    }
                }
            }
        }
        const uint32_t bits = __ballot_sync(0xffffffffu, keep);
        if (lane == 0 && (base >> 5) + warp < nwords) s_mask[(base >> 5) + warp] = bits;  // word = p / 32
    }
    __syncthreads();
    // exclusive prefix of popcounts over the mask words (one warp)
    if (warp == 0) {
        int running = 0;
        for (int w0 = 0; w0 < nwords; w0 += 32) {
            const int w = w0 + lane;
            const int c = w < nwords ? __popc(s_mask[w]) : 0;
            int incl = c;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int o = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += o;
            }
            if (w < nwords) s_prefix[w] = (uint16_t)(running + incl - c);
            running += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) s_total_surv = running;
    }
    __syncthreads();

    // ---------------- phase B: exact evaluation of the survivors ----------------
    const int total_surv = s_total_surv;
    PairGeom g{s_ax, s_ay, s_bx, s_by, s_as, s_bs, s_rcp};
    const size_t out_base = slot * ws.capC;
    for (int sidx = tid; sidx < total_surv; sidx += kScoreThreads) {
        // largest word w with prefix[w] <= sidx, then the (sidx - prefix[w])-th set bit of it
        int lo = 0, hi = nwords - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if ((int)s_prefix[mid] <= sidx) lo = mid; else hi = mid - 1;
        }
        const int bit = __fns(s_mask[lo], 0, sidx - (int)s_prefix[lo] + 1);
        const int p = (lo << 5) + bit;
        const int i = nB > 1 ? (int)__umulhi((uint32_t)p, magic) : p;
        const int j = p - i * nB;
        double score, prio;
        uint32_t flags = 0;
        const bool ok = score_pair_exact<T, 1, TA>(plane, H, W, a, g, i, j, s_ain[i] && s_bin[j], thre2_exact, score, prio, flags);
        if (flags) atomicOr(&s_flags, flags);
        if (ok) {
            const int pos = atomicAdd(&s_count, 1);  // warp-aggregated by ptxas (REDUX + one ATOMS)
            if (pos < ws.capC) store_candidate<TA>(ws, out_base, pos, i, j, score, prio);
        }
    }
    __syncthreads();
    if (tid == 0) publish_limb(ws, n, slot, s_count, total_surv, s_flags);
}

template <typename T, bool STAGE, typename TA = T>
__global__ void __launch_bounds__(kScoreThreads, 3) limb_score_kernel(ScoreArgs a) {
    limb_score_plane<T, STAGE, TA>(a, a.ws, blockIdx.x / a.ws.L, blockIdx.x % a.ws.L);
}

// ---- ragged batches: images of different sizes in one launch (the counterpart of nms_peaks_ragged_kernel) ----
struct ScoreImage {
    const void *paf;
    int64_t chan_stride;  // elements
    double image_extent;
    int H, W, slot;
};
constexpr int kScoreRaggedMaxImages = 128;  // ScoreArgs + 128 x 40 B of kernel parameter
struct ScoreRagged {
    ScoreImage img[kScoreRaggedMaxImages];
};

// Block b: limb b % L of image r.img[b / L] (largest plane first), scored with that image's geometry and extent.
template <typename T, bool STAGE, typename TA = T>
__global__ void __launch_bounds__(kScoreThreads, 3) limb_score_ragged_kernel(ScoreArgs a, const __grid_constant__ ScoreRagged r) {
    const ScoreImage &im = r.img[blockIdx.x / a.ws.L];
    ScoreArgs b = a;  // score_pair_exact reads the extent from the arguments
    b.paf = im.paf;
    b.img_stride = 0;
    b.chan_stride = im.chan_stride;
    b.H = im.H;
    b.W = im.W;
    b.image_extent = im.image_extent;
    b.image_base = im.slot;
    limb_score_plane<T, STAGE, TA>(b, a.ws, 0, blockIdx.x % a.ws.L);
}

}  // namespace spg
