// limb_score_persist.cuh -- K2a, persistent warp-specialised form (f32 planes that fit a 3-deep ring).
//
// Same arithmetic and outputs as limb_score_kernel (limb_score.cuh: conservative f32 screen, then the
// reference's exact evaluation of the survivors, evaluate.py:211-255); different schedule.  The one-CTA-per-
// (image, limb) kernel pays a prologue per item and serialises load -> screen -> exact inside a CTA.  Here one
// CTA per SM stays resident and walks over the items it draws from a device-side queue (item = image * L + limb) with
// three roles and two rings:
//
//   loader    (warp 0)     issues the plane's bulk copy (TMA, SASS UBLKCP) into one of 3 plane slots as soon as the
//                          screeners have left the slot's previous item, and publishes the item's two end-point
//                          lists -- fetched into registers one item earlier, so no global latency sits on the
//                          critical path -- into one of kMetaSlots meta slots; it closes items (counters, status)
//                          when their meta slot comes back.
//   screeners (most warps) the f32 screen of every pair of the item, one chunk of 32 pairs per warp and pass;
//                          survivors are appended, warp-aggregated, to the meta slot's list.  When a screener
//                          leaves an item it releases the PLANE slot: the exact phase does not hold it.
//   scorers   (few warps)  exact evaluation of the survivors in chunks of 32 from a shared counter.  They read the
//                          plane's values back through L2 (where the copy just came from) instead of shared
//                          memory, so the 3 plane slots turn over at the screeners' pace while up to kMetaSlots
//                          items wait for, or are in, their exact phase.
//
// Why this shape (measured with a clock trace of the previous form, all workers screening then scoring with the
// plane held until the exact phase was over): a warp runs this code at a small fraction of the issue rate, a 32-pair
// exact pass is long on one warp, and the ring is only 3 planes deep, so the slot cycle
// (copy + screen + exact + hand-offs) -- not HBM, not issue slots -- set the pace.
//
// All hand-offs are mbarriers (no __syncthreads after start-up); the per-m tables are built once per CTA.
#pragma once

#include "limb_score.cuh"

namespace spg {

constexpr int kPersistThreads = 1024;
constexpr int kPersistSlots = 3;   // plane ring
constexpr int kMetaSlots = 5;      // end-point lists + survivor list + counters ring
constexpr int kWorkerWarps = kPersistThreads / 32 - 1;  // 31
constexpr int kPersistMaxCapP = 64;
constexpr int kScreenTailBypass = 4;
constexpr int kPersistListCap = 1024;  // survivors queued per item; the (rare) excess is evaluated inline by the screener

// Clock trace (`make trace`, tools/trace_limb_score.py): 16 words per item for a CTA's first 64 items.
// Loader: 0 iteration start, 1 copy issued, 2/3 waits for / got the meta slot of item j - kMetaSlots, 4 lists published,
// 8 item closed, 9 survivors (value), 10 candidates (value).  Screeners: 5 first past `full`, 6 first / 7 last to leave.
// Scorers: 11 last to leave.
constexpr int kTrItemWords = 16, kTrItems = 64;
#define SPG_TR_ITEM(kind, j, f, dep) do { if ((j) < kTrItems) kind(kTrItemWords * (j) + (f), dep); } while (0)

struct PersistHdr {
    int nA, nB, npairs, n, k, special;
    uint32_t magic;
    int pad;
};

// One item's two end-point lists in shared memory.  Fixed capacity so that every field offset is an immediate in
// the worker code (a run-time capacity costs an IMAD per access).  `fa`/`fb` are the end points in 1/64 px for the
// screen; a point that is not inside the map is stored as (-1, 0), which makes the pair skip the screen.
struct alignas(16) PeakSlot {
    double ax[kPersistMaxCapP], ay[kPersistMaxCapP], bx[kPersistMaxCapP], by[kPersistMaxCapP];
    float as[kPersistMaxCapP], bs[kPersistMaxCapP];
    float2 fa[kPersistMaxCapP], fb[kPersistMaxCapP];
    unsigned char ain[kPersistMaxCapP], bin[kPersistMaxCapP];
};

struct alignas(16) MetaSlot {
    PeakSlot peaks;
    uint16_t list[kPersistListCap];
    PersistHdr hdr;
    int nsurv, ncand, bnext;  // survivors appended, candidates written, next exact chunk
    uint32_t flags;
};

constexpr size_t kPersistPlaneOffset = (screen_tables_bytes() + kMetaSlots * sizeof(MetaSlot) + 127) & ~(size_t)127;
inline size_t persist_smem_bytes(size_t plane_bytes, int /*capP*/) {
    const size_t plane = (plane_bytes + 127) & ~(size_t)127;
    return kPersistPlaneOffset + kPersistSlots * plane + 128;
}

constexpr uint32_t kScreenBias = 0x4B400000u >> 6;

struct ScreenCtx {
    const PeakSlot *ps;
    uint32_t base;  // shared-memory address of the plane, minus the rounding bias (see screen_pair)
    const ScreenTab *tab;
    const float *ts;  // [kScreenMaxMid + 1][kScreenSamples]
    int W, mid_num, nB;
    uint32_t magic;
    float thre2;
};

// The conservative f32 screen of one pair (limb_score.cuh explains why it may only report certain failures).
// Branch-free: a lane that takes no part (valid = false), a pair with an end point outside the map (x = -1), a
// coincident pair or one whose sample count is within 0.01 of a rounding tie gets m = 0, whose table row has no
// samples.  Every lane executes every sample up to the warp's maximum (rows are padded with a valid sample index),
// so the samples are independent straight-line code.
__device__ __forceinline__ void screen_pair(const ScreenCtx &c, int pc, bool valid, int &fails, int &qn, int &maxfail) {
    const int i = c.nB > 1 ? (int)__umulhi((uint32_t)pc, c.magic) : pc;
    const int jj = pc - i * c.nB;
    const float2 fa = c.ps->fa[i], fb = c.ps->fb[jj];
    const float dx64 = fb.x - fa.x, dy64 = fb.y - fa.y;
    const float n2 = (dx64 * dx64 + dy64 * dy64) * (1.0f / 4096.0f);  // px^2
    float rs;  // one MUFU.RSQ, no denormal fix-up: n2 below 1e-6 is not screened anyway
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(rs) : "f"(n2));
    const float qf = n2 * rs + 1.0f;  // approximate norm + 1 (NaN for n2 = 0: falls out below)
    const float r = rintf(qf);
    const bool longp = qf >= (float)c.mid_num + 0.51f;
    int m = longp ? c.mid_num : min((int)r, c.mid_num);
    if (!longp && !(fabsf(qf - r) < 0.49f)) m = 0;  // m within 0.01 of a rounding tie -> survive
    // coincident pairs and pairs with an end point outside the map are left to the exact path
    if (!(n2 > 1e-6f) || !valid || fminf(fa.x, fb.x) < 0.0f) m = 0;
    m = max(m, 0);
    const ScreenTab tb = c.tab[m];  // m = 0: no samples
    qn = tb.qn;
    maxfail = tb.maxfail;
    const float sx64 = dx64 * tb.inv, sy64 = dy64 * tb.inv;
    // +33 folded into the start point: with u = pos + 33 (1/64 px), the pixel is u >> 6 for every sample that is not
    // within {31,32,33} (mod 64) of a rounding boundary, i.e. u & 63 > 2
    const float ax64o = fa.x + 33.0f, ay64o = fa.y + 33.0f;
    const float *ts = c.ts + m * kScreenSamples;
    const int qmax = __reduce_max_sync(0xffffffffu, qn);
    // Round-to-nearest-even through the 1.5 * 2^23 trick (positions are in [0, 2^22)): the low bits of the float
    // pos + 1.5 * 2^23 are the rounded position u (an FADD instead of F2I, which runs on the quarter-rate conversion
    // pipe).  The bias is never subtracted: its low 6 bits are zero, so bits & 63 == u & 63, and bits >> 6 ==
    // (u >> 6) + kScreenBias; the kScreenBias * (W + 1) elements that adds to the index are taken off the plane's address once
    // (kScreenBias; the offset comes from shared memory so that it stays ONE register operand instead of being
    // re-split into immediates at every sample)
    const uint32_t base = c.base;
    // Every lane runs the warp's maximum number of samples; a lane with fewer samples of its own re-reads padded
    // entries of its row (its last sample, or sample 0 of the empty row), which can only repeat a failure it has
    // already counted -- so instead of masking those samples out one by one, the lane's tolerance is raised by their
    // number: more than maxfail + padded counted failures still means more than maxfail real ones.
    fails = 0;
    auto sample = [&](int q2) {
        const float tf = ts[q2];
        const uint32_t xb = __float_as_uint(__fadd_rn(__fmaf_rn(tf, sx64, ax64o), 12582912.0f));
        const uint32_t yb = __float_as_uint(__fadd_rn(__fmaf_rn(tf, sy64, ay64o), 12582912.0f));
        float v;
        asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(base + 4u * ((yb >> 6) * (uint32_t)c.W + (xb >> 6))));
        fails += (int)(min(xb & 63u, yb & 63u) > 2u) & (int)!(v > c.thre2);
    };
    if (qmax == kScreenSamples) {  // the common case (a warp with at least one pair of >= mid_num samples): no trip checks
#pragma unroll
        for (int q2 = 0; q2 < kScreenSamples; q2++) sample(q2);
    } else {
#pragma unroll
        for (int q2 = 0; q2 < kScreenSamples; q2++) {
            if (q2 >= qmax) break;
            sample(q2);
        }
    }
    maxfail += qmax - qn;
}

// TA = float: f32 planes, f32 arithmetic; double: f32 planes evaluated in float64 (SPG_F32_AS_F64).
// Items are dealt from a device-side queue: queue[0] is the next ticket (ticket = item = image * L + limb), queue[1]
// counts the CTAs that have drawn a ticket >= n_items; the last of them resets both to 0 for the next launch.  Both
// words are 0 when the kernel starts.
template <typename TA>
__global__ void __launch_bounds__(kPersistThreads, 1) limb_score_persist_kernel(ScoreArgs a, int n_items, unsigned int *queue) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    // full: plane copy landed + lists published; screened: every screener has left the item -- its survivor list is
    // complete (scorers) and its plane slot can be refilled (loader); mfree: every scorer has left the meta slot
    __shared__ uint64_t bar_full[kPersistSlots], bar_screened[kMetaSlots], bar_mfree[kMetaSlots];
    __shared__ uint32_t s_bias_bytes;  // 4 * kScreenBias * (W + 1)
    SPG_TR_CTA_START();

    using T = float;
    const Workspace &ws = a.ws;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int H = a.H, W = a.W, capP = ws.capP, L = ws.L;
    const size_t plane_bytes = (size_t)H * W * sizeof(T);
    const size_t plane_stride = (plane_bytes + 127) & ~(size_t)127;
    // layout: per-m tables, meta ring, then the plane ring -- everything but the planes at compile-time offsets
    double *s_rcp = reinterpret_cast<double *>(smem_raw);
    ScreenTab *s_tab = reinterpret_cast<ScreenTab *>(s_rcp + (kScreenMaxMid + 1));
    float *s_ts = reinterpret_cast<float *>(s_tab + (kScreenMaxMid + 1));
    MetaSlot *s_meta = reinterpret_cast<MetaSlot *>(smem_raw + screen_tables_bytes());
    unsigned char *s_planes = smem_raw + kPersistPlaneOffset;
    const int nE = min(max(a.exact_warps, 1), kWorkerWarps - 1), nS = kWorkerWarps - nE;  // scorer / screener warps

    // ---- one-time set-up
    if (tid == 0) {
        for (int s = 0; s < kPersistSlots; s++) {
            mbar_init(&bar_full[s], 2);  // plane copy (expect_tx) + end-point lists
        }
        for (int e = 0; e < kMetaSlots; e++) {
            mbar_init(&bar_screened[e], nS);
            mbar_init(&bar_mfree[e], nE);
            s_meta[e].nsurv = 0; s_meta[e].ncand = 0; s_meta[e].bnext = 0; s_meta[e].flags = 0;
        }
        s_bias_bytes = 4u * kScreenBias * (uint32_t)(W + 1);
        fence_mbar_init();
    }
    if (tid >= 32 && tid < 32 + kScreenMaxMid + 1) build_screen_row(a, tid - 32, s_rcp, s_tab, s_ts, true);
    __syncthreads();

    const bool screen = a.screen && a.mid_num <= kScreenMaxMid && H <= kScreenMaxDim && W <= kScreenMaxDim;
    const T thre2 = sizeof(TA) == 8 ? f32_not_above(a.thre2) : (T)a.thre2;  // the screen's float32 threshold
    const TA thre2_exact = (TA)a.thre2;
    auto plane_of = [&](int n_local, int k) {
        return reinterpret_cast<const T *>(a.paf) + (int64_t)n_local * a.img_stride + (int64_t)k * a.chan_stride;
    };

    if (warp == 0) {
        // =========================== loader ===========================
        constexpr int kMaxE = kPersistMaxCapP / 32;  // list entries per lane
        double r_xa[kMaxE], r_ya[kMaxE], r_xb[kMaxE], r_yb[kMaxE];
        float r_sa[kMaxE], r_sb[kMaxE];
        int r_cntA = 0, r_cntB = 0, r_item = 0;
        // Draws the CTA's next item from the queue and loads its end-point lists into registers.  Items go to whichever
        // CTA asks first, so every SM stays busy until the queue is empty: with a fixed stride of G = 132 CTAs over
        // item = image * 30 + limb, CTA c would only ever score the limbs k = c (mod 6), and limbs differ a lot in how
        // many pairs survive the screen.  A ticket >= n_items ends the CTA's items (its lists load item n_items - 1,
        // unused).
        auto fetch = [&]() {
            int t = 0;
            if (lane == 0) t = (int)atomicAdd(queue, 1u);
            r_item = __shfl_sync(0xffffffffu, t, 0);
            const int item = min(r_item, n_items - 1);
            const int n_local = item / L, k = item - n_local * L;
            const int n = a.image_base + n_local;
            const int pa = ws.limbs[2 * k], pb = ws.limbs[2 * k + 1];
            r_cntA = ws.peak_count[(size_t)n * ws.K + pa];
            r_cntB = ws.peak_count[(size_t)n * ws.K + pb];
            const size_t baseA = ((size_t)n * ws.K + pa) * capP, baseB = ((size_t)n * ws.K + pb) * capP;
#pragma unroll
            for (int u = 0; u < kMaxE; u++) {
                const int e = lane + 32 * u;
                if (e < capP) {  // whole capacity: independent of the counters
                    r_xa[u] = ws.peak_x[baseA + e]; r_ya[u] = ws.peak_y[baseA + e];
                    r_xb[u] = ws.peak_x[baseB + e]; r_yb[u] = ws.peak_y[baseB + e];
                    r_sa[u] = ws.peak_score[baseA + e]; r_sb[u] = ws.peak_score[baseB + e];
                }
            }
        };
        // every scorer has left the meta slot of item jp: publish counters + status, recycle the slot's counters
        auto close_item = [&](int jp) {
            if (lane == 0) {
                MetaSlot &ms = s_meta[jp % kMetaSlots];
                SPG_TR_ITEM(SPG_TR, jp, 8, ms.nsurv);
                SPG_TR_ITEM(SPG_TRV, jp, 9, ms.nsurv);
                SPG_TR_ITEM(SPG_TRV, jp, 10, ms.ncand);
                publish_limb(ws, ms.hdr.n, (size_t)ms.hdr.n * L + ms.hdr.k, ms.hdr.special ? -1 : ms.ncand, ms.nsurv, ms.flags);
                ms.nsurv = 0; ms.ncand = 0; ms.bnext = 0; ms.flags = 0;
            }
            __syncwarp();
        };
        // Item j of the CTA goes through plane slot j % kPersistSlots and meta slot j % kMetaSlots.  Once the queue is
        // empty, one more "item" is published: a header with npairs = -1 and no plane, which tells the screeners (and
        // through them the scorers) that there are no more items.
        fetch();
        int j = 0;
        for (;; j++) {
            const int s = j % kPersistSlots, e = j % kMetaSlots;
            SPG_TR_ITEM(SPG_TR, j, 0, j);
            if (j >= kPersistSlots) {  // the plane slot's previous item has been screened
                const int jp = j - kPersistSlots;
                mbar_wait_sleep(&bar_screened[jp % kMetaSlots], (jp / kMetaSlots) & 1);
            }
            const bool live = r_item < n_items;
            const int n_local = r_item / L, k = r_item - n_local * L;
            const int n = a.image_base + n_local;
            if (lane == 0) {  // plane first (arrival 1 of 2 on `full`, carries the byte count)
                const unsigned char *gplane = reinterpret_cast<const unsigned char *>(plane_of(n_local, k));
                unsigned char *dst = s_planes + s * plane_stride;
                const size_t bytes_in = live ? plane_bytes : 0;
                mbar_expect_tx(&bar_full[s], (uint32_t)bytes_in);
                for (size_t off = 0; off < bytes_in; off += kBulkChunkBytes) {
                    const uint32_t bytes = (uint32_t)min((size_t)kBulkChunkBytes, plane_bytes - off);
                    bulk_g2s(dst + off, gplane + off, bytes, &bar_full[s]);
                }
            }
            SPG_TR_ITEM(SPG_TR, j, 1, j);
            if (j >= kMetaSlots) {
                SPG_TR_ITEM(SPG_TR, j, 2, j);
                mbar_wait_sleep(&bar_mfree[e], ((j / kMetaSlots) - 1) & 1);
                SPG_TR_ITEM(SPG_TR, j, 3, j);
                close_item(j - kMetaSlots);
            }
            MetaSlot &ms = s_meta[e];
            PeakSlot &ps = ms.peaks;
#pragma unroll
            for (int u = 0; u < kMaxE; u++) {
                const int q = lane + 32 * u;
                if (q < capP) {
                    const double xa = r_xa[u], ya = r_ya[u], xb = r_xb[u], yb = r_yb[u];
                    ps.ax[q] = xa; ps.ay[q] = ya; ps.bx[q] = xb; ps.by[q] = yb;
                    ps.as[q] = r_sa[u]; ps.bs[q] = r_sb[u];
                    const bool ain = inside_map(xa, ya, H, W), bin = inside_map(xb, yb, H, W);
                    ps.fa[q] = ain ? make_float2((float)(xa * 64.0), (float)(ya * 64.0)) : make_float2(-1.0f, 0.0f);
                    ps.fb[q] = bin ? make_float2((float)(xb * 64.0), (float)(yb * 64.0)) : make_float2(-1.0f, 0.0f);
                    ps.ain[q] = ain;
                    ps.bin[q] = bin;
                }
            }
            const int nA = min(r_cntA, capP), nB = min(r_cntB, capP);
            const bool special = nA == 0 || nB == 0;
            if (lane == 0) {
                PersistHdr h;
                h.nA = nA; h.nB = nB; h.npairs = !live ? -1 : special ? 0 : nA * nB; h.n = n; h.k = k; h.special = special;
                h.magic = nB > 1 ? 0xffffffffu / (uint32_t)nB + 1u : 0u;
                h.pad = 0;
                ms.hdr = h;
            }
            __syncwarp();
            SPG_TR_ITEM(SPG_TR, j, 4, j);
            if (lane == 0) mbar_arrive(&bar_full[s]);  // arrival 2 of 2: lists + header are in place
            if (!live) break;
            fetch();  // in flight while the next iteration waits for its slots
        }
        for (int jp = max(0, j - kMetaSlots + 1); jp < j; jp++) {  // the items still in the meta ring (j: the end header)
            mbar_wait_sleep(&bar_mfree[jp % kMetaSlots], (jp / kMetaSlots) & 1);
            close_item(jp);
        }
        if (lane == 0) {  // this CTA has drawn its last ticket
            __threadfence();
            if (atomicAdd(queue + 1, 1u) == gridDim.x - 1) {  // so has every other: reset the queue for the next launch
                __threadfence();
                *(volatile unsigned int *)queue = 0u;
                *(volatile unsigned int *)(queue + 1) = 0u;
            }
        }
    } else {
        // exact evaluation of one pair + candidate append.  `plane` is the shared-memory copy for a screener whose
        // survivor does not fit the list, the global plane (read through L2) for the scorers.
        auto exact_one = [&](MetaSlot &ms, const T *plane, int p) {
            const PersistHdr &h = ms.hdr;
            const PeakSlot &ps = ms.peaks;
            const int nB = h.nB;
            const int i = nB > 1 ? (int)__umulhi((uint32_t)p, h.magic) : p;
            const int jj = p - i * nB;
            PairGeom g{ps.ax, ps.ay, ps.bx, ps.by, ps.as, ps.bs, s_rcp};
            double score, prio;
            uint32_t flags = 0;
            const bool ok = score_pair_exact<T, 10, TA>(plane, H, W, a, g, i, jj, ps.ain[i] && ps.bin[jj], thre2_exact, score, prio, flags);
            if (flags) atomicOr(&ms.flags, flags);
            if (ok) {
                const size_t out_base = ((size_t)h.n * L + h.k) * ws.capC;
                const int pos = atomicAdd(&ms.ncand, 1);
                if (pos < ws.capC) store_candidate<TA>(ws, out_base, pos, i, jj, score, prio);
            }
        };

        if (warp <= nS) {
            // =========================== screeners ===========================
            // Item j is cut into chunks of 32 pairs; screener w takes chunks (w + j) mod nS, + nS, ...: the rotation
            // moves the odd second chunk of an item (pairs beyond 32 * nS) to a different warp every item.  Screeners
            // never wait for each other: their only wait is `full`.
            int c0 = warp - 1;
            for (int j = 0;; j++) {
                const int s = j % kPersistSlots, e = j % kMetaSlots;
                // `full` also means the meta slot's list and counters are recycled (the loader closed item j - kMetaSlots)
                mbar_wait_sleep(&bar_full[s], (j / kPersistSlots) & 1);
                SPG_TR_ITEM(SPG_TR_FIRST, j, 5, j);
                MetaSlot &ms = s_meta[e];
                const int npairs = ms.hdr.npairs;
                if (c0 * 32 < npairs) {  // warps without pairs skip the item
                    const T *plane = reinterpret_cast<const T *>(s_planes + s * plane_stride);
                    const ScreenCtx sc{&ms.peaks, smem_u32(plane) - *(volatile uint32_t *)&s_bias_bytes, s_tab, s_ts, W, a.mid_num,
                                       ms.hdr.nB, ms.hdr.magic, thre2};
                    for (int c = c0; c * 32 < npairs; c += nS) {
                        const int p = c * 32 + lane;
                        bool keep = p < npairs;
                        // a last chunk of only a few pairs (31 x 31 peaks leave 1) is not worth a pass: they go straight to
                        // the exact phase, where they ride along in a chunk that exists anyway
                        if (screen && npairs - c * 32 > kScreenTailBypass) {
                            int fails, qn, maxfail;
                            screen_pair(sc, min(p, npairs - 1), keep, fails, qn, maxfail);
                            if (qn > 0) keep = fails <= maxfail;
                        }
                        const uint32_t km = __ballot_sync(0xffffffffu, keep);
                        if (km) {
                            int at = 0;
                            if (lane == 0) at = atomicAdd(&ms.nsurv, __popc(km));
                            at = __shfl_sync(0xffffffffu, at, 0);
                            if (keep) {
                                const int at_me = at + __popc(km & ((1u << lane) - 1u));
                                if (at_me < kPersistListCap) ms.list[at_me] = (uint16_t)p;
                                else exact_one(ms, plane, p);  // list full: evaluate right here, from the staged plane
                            }
                        }
                    }
                }
                __syncwarp();
                SPG_TR_ITEM(SPG_TR_FIRST, j, 6, j);
                SPG_TR_ITEM(SPG_TR_LAST, j, 7, j);
                if (lane == 0) mbar_arrive(&bar_screened[e]);  // release: this warp's survivors are in the list, the plane is no longer read
                if (npairs < 0) break;  // the end header (passed on to the scorers by the arrival above)
                if (++c0 == nS) c0 = 0;
            }
        } else {
            // =========================== scorers ===========================
            for (int j = 0;; j++) {
                const int e = j % kMetaSlots;
                mbar_wait_sleep(&bar_screened[e], (j / kMetaSlots) & 1);  // every screener has left item j: the list is complete
                MetaSlot &ms = s_meta[e];
                if (ms.hdr.npairs < 0) break;  // the end header
                const int ns = min(ms.nsurv, kPersistListCap);
                if (ns > 0) {
                    const T *gplane = plane_of(ms.hdr.n - a.image_base, ms.hdr.k);  // the plane's slot may already hold another item
                    for (;;) {
                        if (*(volatile int *)&ms.bnext * 32 >= ns) break;  // all chunks taken: no need to draw a number
                        int c = 0;
                        if (lane == 0) c = atomicAdd(&ms.bnext, 1);
                        c = __shfl_sync(0xffffffffu, c, 0);
                        if (c * 32 >= ns) break;
                        const int t = c * 32 + lane;
                        if (t < ns) exact_one(ms, gplane, ms.list[t]);
                        __syncwarp();
                    }
                }
                __syncwarp();
                SPG_TR_ITEM(SPG_TR_LAST, j, 11, j);
                if (lane == 0) mbar_arrive(&bar_mfree[e]);  // release: this warp's candidates and counters are visible to the loader
            }
        }
    }
    SPG_TR_CTA_EXIT();
}

}  // namespace spg
