// nms_peaks.cuh -- K1: 3x3 heat-map NMS + ordered peak extraction + centroid refinement.
//
// Replaces find_peaks (/root/reference/evaluate.py:169-203), i.e. util.keypoint_heatmap_nms
// (utils/util.py:177-183) followed by np.nonzero (:193) and util.refine_centroid (:186-211) per peak.
//
// One CTA per (image, part) plane.  The plane is streamed through shared memory in row bands of full
// rows (one contiguous span each) with the 1-D bulk-copy engine, double buffered on two mbarriers, so
// HBM is read exactly once per pixel and the 3x3 window reads hit shared memory.  Detection scans
// float4 groups and rejects a group with one compare when none of its 4 values reaches thre1 (the
// common case).  Peaks are appended unordered and then rank-sorted by raster index, which restores
// np.nonzero's order exactly (peak ids depend on it).  Refinement re-reads the 5x5 box from L2.
//
// This header also holds the building blocks of the two persistent forms (nms_peaks_persist.cuh,
// nms_peaks_banded.cuh): the 8-neighbour test, the peak finisher, the scanners' pass 1 and their role constants.
#pragma once

#include "common.cuh"

namespace spg {

struct NmsArgs {
    const float *heat;
    int64_t img_stride, chan_stride;  // elements
    int H, W, band_rows, radius, use_bulk, image_base;
    float thr;                        // (float)thre1: torch compares in f32 (util.py:182)
    Workspace ws;
};

constexpr int kNmsThreads = 256;
constexpr int kNmsBufs = 3;  // band ring: two bands in flight while one is scanned

__device__ __forceinline__ bool nms_is_peak(const float *buf, int lo, int H, int W, int y, int x, float v, float thr) {
    // keep = (hmax == heat) & (heat >= thre); np.nonzero(heat * keep) drops exact zeros
    if (!(v >= thr) || v == 0.0f) return false;
#pragma unroll
    for (int dy = -1; dy <= 1; dy++) {
        const int yy = y + dy;
        if (yy < 0 || yy >= H) continue;  // reflect-pad-1 == window clipped to the image
        const float *row = buf + (size_t)(yy - lo) * W;
#pragma unroll
        for (int dx = -1; dx <= 1; dx++) {
            const int xx = x + dx;
            if (xx < 0 || xx >= W) continue;
            if (!(row[xx] <= v)) return false;
        }
    }
    return true;
}

// refine_centroid (utils/util.py:204-211) for an interior peak, box (2R+1)^2 read from L2.
// np.mgrid's first grid varies along ROWS and is the one added to x (axes swapped relative to intent; kept).
// Both sums follow numpy's pairwise order for n = (2R+1)^2 in [9, 81]: eight running accumulators over
// i = 0 .. n-2 (n-1 is a multiple of 8 for every odd square), combined as ((0+1)+(2+3))+((4+5)+(6+7)), then
// the last element.  Streaming into the accumulators keeps everything in registers.
template <int R>
__device__ __forceinline__ void refine_box(const float *__restrict__ plane, int W, int x, int y, double &rx, double &ry,
                                           float &sc) {
    constexpr int D = 2 * R + 1, N = D * D;
    if (N == 1) {  // radius 0: offsets are 0/b, the mean is the value itself
        const float b = plane[(size_t)y * W + x];
        const float s32 = 0.0f + b;
        rx = __dadd_rn((double)x, __ddiv_rn(__dmul_rn((double)b, 0.0), (double)s32));
        ry = __dadd_rn((double)y, __ddiv_rn(__dmul_rn((double)b, 0.0), (double)s32));
        sc = __fdiv_rn(s32, 1.0f);
        return;
    }
    float s[8];
    double ax[8], ay[8];
    float ts = 0.0f;
    double tx = 0.0, ty = 0.0;
#pragma unroll
    for (int i = 0; i < N; i++) {
        const int r = i / D - R, q = i % D - R;
        const float b = plane[(size_t)(y + r) * W + (x + q)];  // global (L2-hot) or shared memory
        const double wr = __dmul_rn((double)b, (double)r), wc = __dmul_rn((double)b, (double)q);
        if (i < 8) {
            s[i] = b; ax[i] = wr; ay[i] = wc;
        } else if (i < N - 1) {
            s[i & 7] = __fadd_rn(s[i & 7], b);
            ax[i & 7] = __dadd_rn(ax[i & 7], wr);
            ay[i & 7] = __dadd_rn(ay[i & 7], wc);
        } else {
            ts = b; tx = wr; ty = wc;
        }
    }
    const float s32 = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(s[0], s[1]), __fadd_rn(s[2], s[3])),
                                          __fadd_rn(__fadd_rn(s[4], s[5]), __fadd_rn(s[6], s[7]))), ts);
    const double sx = __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(ax[0], ax[1]), __dadd_rn(ax[2], ax[3])),
                                          __dadd_rn(__dadd_rn(ax[4], ax[5]), __dadd_rn(ax[6], ax[7]))), tx);
    const double sy = __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(ay[0], ay[1]), __dadd_rn(ay[2], ay[3])),
                                          __dadd_rn(__dadd_rn(ay[4], ay[5]), __dadd_rn(ay[6], ay[7]))), ty);
    rx = __dadd_rn((double)x, __ddiv_rn(sx, (double)s32));
    ry = __dadd_rn((double)y, __ddiv_rn(sy, (double)s32));
    sc = __fdiv_rn(s32, (float)N);  // score_box.mean() stays f32
}

// The 8-neighbour test of one float4 group (row y, columns x0 .. x0 + 3), with neighbours clamped to the image: a clamped
// neighbour is a pixel that is already inside the clipped 3x3 window (or the pixel itself), so the window max is
// unchanged.  `rows` is addressed by GLOBAL row index.  Peaks are appended to `list` (unordered) through `*cnt`.
__device__ __forceinline__ void nms_test_group(const float *rows, int y, int x0, int H, int W, float thr, int *cnt, uint32_t *list, int capP) {
    const float *rc = rows + (size_t)y * W;
    const float *ru = rows + (size_t)max(y - 1, 0) * W;
    const float *rd = rows + (size_t)min(y + 1, H - 1) * W;
    const float4 c4 = *reinterpret_cast<const float4 *>(rc + x0);
    const float4 u4 = *reinterpret_cast<const float4 *>(ru + x0);
    const float4 d4 = *reinterpret_cast<const float4 *>(rd + x0);
    const int xl = max(x0 - 1, 0), xr = min(x0 + 4, W - 1);
    const float U[6] = {ru[xl], u4.x, u4.y, u4.z, u4.w, ru[xr]};
    const float C[6] = {rc[xl], c4.x, c4.y, c4.z, c4.w, rc[xr]};
    const float D[6] = {rd[xl], d4.x, d4.y, d4.z, d4.w, rd[xr]};
#pragma unroll
    for (int e = 0; e < 4; e++) {
        const float v = C[e + 1];
        // keep = (hmax == heat) & (heat >= thre) (util.py:182); np.nonzero(heat * keep) drops exact zeros.
        // "all neighbours <= v" (not fmax) so that a NaN neighbour vetoes the peak like torch's max-pool
        const bool pk = (v >= thr) & (v != 0.0f) & (U[e] <= v) & (U[e + 1] <= v) & (U[e + 2] <= v) &
                        (C[e] <= v) & (C[e + 2] <= v) & (D[e] <= v) & (D[e + 1] <= v) & (D[e + 2] <= v);
        if (pk) {
            const int pos = atomicAdd(cnt, 1);
            if (pos < capP) list[pos] = (uint32_t)(y * W + x0 + e);
        }
    }
}

// Finishes the peak at row y, column x of `plane`: the border test, the refinement (util.py:201-211, from L2) and the
// four stores at output slot `out`.  R >= 0: the refinement radius (== a.radius) is a compile-time constant, so only
// one refine_box is compiled in; R < 0: a.radius is dispatched at run time.
template <int R = -1>
__device__ __forceinline__ void nms_finish_peak(const NmsArgs &a, const float *plane, int H, int W, size_t out, int y, int x) {
    const Workspace &ws = a.ws;
    const int r = R >= 0 ? R : a.radius;
    double rx, ry;
    float sc;
    uint32_t anchor = ((uint32_t)y << 16) | (uint32_t)x;
    if (y + r + 1 > H || y - r < 0 || x + r + 1 > W || x - r < 0) {
        rx = (double)x;  // util.py:201-202: the box leaves the image -> integer anchor, raw map value
        ry = (double)y;
        sc = plane[(size_t)y * W + x];
        anchor |= 0x80000000u;
    } else if constexpr (R >= 0) {
        refine_box<R>(plane, W, x, y, rx, ry, sc);  // util.py:204-211
    } else {
        switch (r) {  // util.py:204-211
            case 0: refine_box<0>(plane, W, x, y, rx, ry, sc); break;
            case 1: refine_box<1>(plane, W, x, y, rx, ry, sc); break;
            case 2: refine_box<2>(plane, W, x, y, rx, ry, sc); break;
            case 3: refine_box<3>(plane, W, x, y, rx, ry, sc); break;
            default: refine_box<4>(plane, W, x, y, rx, ry, sc); break;
        }
    }
    ws.peak_x[out] = rx;
    ws.peak_y[out] = ry;
    ws.peak_score[out] = sc;
    ws.peak_anchor[out] = anchor;
}

// Publishes the peak count of plane (image n, part c).
__device__ __forceinline__ void nms_publish_count(const NmsArgs &a, int n, int c, int total) {
    a.ws.peak_count[(size_t)n * a.ws.K + c] = total;
    if (total > a.ws.capP) atomicOr(&a.ws.status[n], kStPeakOverflow);
}

// ---- the persistent forms (nms_peaks_persist.cuh, nms_peaks_banded.cuh): one resident 1024-thread CTA per SM with the
// same roles -- a loader warp, scanner warps, finisher warps -- and a ring of peak lists between scanners and finishers
constexpr int kNmsPThreads = 1024;
constexpr int kNmsPFinishers = 3;
constexpr int kNmsPLists = 2 * kNmsPFinishers;
constexpr int kNmsPScanners = kNmsPThreads / 32 - 1 - kNmsPFinishers;  // 28
constexpr int kNmsPMaxIter = 5;  // 32-lane passes of pass 1 over a scanner's share of a plane or band

// Pass 1 of a persistent scanner: the float4 groups g = g0 + it * g_step + lane (it < ITER, g < g_end) of `data` that
// reach thre1 are queued in `wq`, warp-aggregated, in group order.  First only the votes (one load, three max, one
// compare, one ballot per 128 elements -- the common case is an empty mask), then the queue from the masks.  Returns the
// queue length (warp-uniform); the queue is visible to the whole warp.
template <int ITER>
__device__ __forceinline__ int nms_queue_groups(const float *data, int g0, int g_step, int g_end, float thr, int lane, uint16_t *wq) {
    uint32_t am[ITER];
#pragma unroll
    for (int it = 0; it < ITER; it++) {
        const int g = g0 + it * g_step + lane;
        bool act = false;
        if (g < g_end) {
            const float4 c4 = *reinterpret_cast<const float4 *>(data + 4 * (size_t)g);
            act = fmaxf(fmaxf(c4.x, c4.y), fmaxf(c4.z, c4.w)) >= thr;
        }
        am[it] = __ballot_sync(0xffffffffu, act);
    }
    int nq = 0;
#pragma unroll
    for (int it = 0; it < ITER; it++) {
        const uint32_t m = am[it];
        if (m) {  // warp-uniform
            if ((m >> lane) & 1u) wq[nq + __popc(m & ((1u << lane) - 1u))] = (uint16_t)(g0 + it * g_step + lane);
            nq += __popc(m);
        }
    }
    __syncwarp();
    return nq;
}

// A persistent finisher's share of plane `item` (= n_local * K + c): lane t takes peaks t, t + 32, ... of the unordered
// list, ranks each by raster index (= np.nonzero order, evaluate.py:193; indices are unique) and finishes it at its rank.
// R: as in nms_finish_peak.  w4_magic != 0: ceil(2^32 / (W / 4)), and every raster index / 4 is below 2^16, so the row
// is umulhi(index / 4, w4_magic) (exact there, as in the scanners); 0: the row is index / W.  staged != nullptr: the
// whole plane in shared memory, which the refinement reads instead of the plane in global memory (L2).
template <int R = -1>
__device__ __forceinline__ void nms_finish_plane(const NmsArgs &a, const uint32_t *list, int total, int item, int lane,
                                                 uint32_t w4_magic, const float *staged = nullptr) {
    const int K = a.ws.K, capP = a.ws.capP, W = a.W;
    const int n_local = item / K, c = item - n_local * K;
    const float *plane = staged ? staged : a.heat + (int64_t)n_local * a.img_stride + (int64_t)c * a.chan_stride;
    const int np = min(total, capP);
    const size_t out_base = ((size_t)(a.image_base + n_local) * K + c) * capP;
    for (int t = lane; t < np; t += 32) {
        const uint32_t mine = list[t];
        int rank = 0;
        for (int u = 0; u < np; u++) rank += list[u] < mine;
        const int y = w4_magic ? (int)__umulhi(mine >> 2, w4_magic) : (int)mine / W, x = (int)mine - y * W;
        nms_finish_peak<R>(a, plane, a.H, W, out_base + rank, y, x);
    }
    if (lane == 0) nms_publish_count(a, a.image_base + n_local, c, total);
}

// The per-plane schedule: the CTA finds the peaks of part c of image n_local of `a` (plane a.heat + n_local * img_stride
// + c * chan_stride, geometry a.H x a.W in bands of a.band_rows) and writes them to slot a.image_base + n_local.
__device__ __forceinline__ void nms_peaks_plane(const NmsArgs &a, int n_local, int c) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t bar[kNmsBufs];
    __shared__ int s_count;

    const Workspace &ws = a.ws;
    const int tid = threadIdx.x;
    const int n = a.image_base + n_local;
    const int H = a.H, W = a.W, br = a.band_rows;
    const float *plane = a.heat + (int64_t)n_local * a.img_stride + (int64_t)c * a.chan_stride;

    const int nb = (H + br - 1) / br;
    // one band (whole plane resident): a single buffer without halo rows; else two band buffers with a halo row each side
    const size_t band_floats = nb == 1 ? (size_t)H * W : (size_t)(br + 2) * W;
    const size_t buf_stride = (band_floats + 31) & ~(size_t)31;
    const int nbufs = min(nb, kNmsBufs);
    float *buf0 = reinterpret_cast<float *>(smem_raw);
    uint32_t *s_list = reinterpret_cast<uint32_t *>(buf0 + (size_t)nbufs * buf_stride);
    uint32_t *s_sorted = s_list + ws.capP;
    uint16_t *s_queue = reinterpret_cast<uint16_t *>(s_sorted + ws.capP);  // float4 groups of the band worth testing

    if (tid == 0) {
        s_count = 0;
        if (a.use_bulk) {
            for (int i = 0; i < kNmsBufs; i++) mbar_init(&bar[i], 1);
            fence_mbar_init();
        }
    }
    __syncthreads();

    auto band_lo = [&](int b) { return max(b * br - 1, 0); };
    auto band_hi = [&](int b) { return min((b + 1) * br + 1, H); };
    auto issue = [&](int b) {  // one thread: bulk copy rows [lo, hi) of the plane into ring buffer b % kNmsBufs
        const int lo = band_lo(b), hi = band_hi(b);
        const uint32_t bytes = (uint32_t)(hi - lo) * W * sizeof(float);
        mbar_expect_tx(&bar[b % kNmsBufs], bytes);
        bulk_g2s(buf0 + (size_t)(b % kNmsBufs) * buf_stride, plane + (size_t)lo * W, bytes, &bar[b % kNmsBufs]);
    };

    if (a.use_bulk && tid == 0)
        for (int b = 0; b < nbufs; b++) issue(b);

    for (int b = 0; b < nb; b++) {
        float *buf = a.use_bulk ? buf0 + (size_t)(b % kNmsBufs) * buf_stride : buf0;
        const int lo = band_lo(b), hi = band_hi(b);
        if (a.use_bulk) {
            mbar_wait(&bar[b % kNmsBufs], (b / kNmsBufs) & 1);
        } else {
            const int cnt = (hi - lo) * W;
            for (int i = tid; i < cnt; i += kNmsThreads) buf[i] = plane[(size_t)lo * W + i];
            __syncthreads();
        }
        const int y0 = b * br, y1 = min(y0 + br, H);
        if ((W & 3) == 0) {
            // Pass 1: float4 groups; a group is dropped with one compare when none of its values reaches thre1 (the
            // common case); the others are queued, warp-aggregated.  Pass 2 runs the 8-neighbour test densely over
            // the queue, so warps do not drag idle lanes through it.
            // Each warp owns a contiguous slice of the band's groups and a private queue, so the two passes need no
            // block barrier (neighbour rows are read-only in the band buffer).
            const int W4 = W >> 2;
            const int groups = (y1 - y0) * W4;
            const int lane = tid & 31, warp = tid >> 5;
            const int gpw = (groups + (kNmsThreads / 32) - 1) / (kNmsThreads / 32);  // groups per warp
            const int g_lo = warp * gpw, g_hi = min(g_lo + gpw, groups);
            uint16_t *wq = s_queue + g_lo;  // at most gpw entries
            int nq = 0;                     // warp-uniform
            for (int g0 = g_lo; g0 < g_hi; g0 += 32) {
                const int g = g0 + lane;
                bool act = false;
                if (g < g_hi) {
                    const float4 c4 = *reinterpret_cast<const float4 *>(buf + (size_t)(y0 - lo) * W + 4 * (size_t)g);
                    act = fmaxf(fmaxf(c4.x, c4.y), fmaxf(c4.z, c4.w)) >= a.thr;
                }
                const uint32_t am = __ballot_sync(0xffffffffu, act);
                if (act) wq[nq + __popc(am & ((1u << lane) - 1u))] = (uint16_t)g;
                nq += __popc(am);
            }
            __syncwarp();
            const float *rows = buf - (size_t)lo * W;  // addressed by global row index
            for (int q = lane; q < nq; q += 32) {
                const int g = wq[q];
                const int r = g / W4, xq = g - r * W4;
                nms_test_group(rows, y0 + r, 4 * xq, H, W, a.thr, &s_count, s_list, ws.capP);
            }
        } else {
            const int cnt = (y1 - y0) * W;
            for (int i = tid; i < cnt; i += kNmsThreads) {
                const int r = i / W, x = i - r * W;
                const int y = y0 + r;
                const float v = buf[(size_t)(y - lo) * W + x];
                if (nms_is_peak(buf, lo, H, W, y, x, v, a.thr)) {
                    const int pos = atomicAdd(&s_count, 1);
                    if (pos < ws.capP) s_list[pos] = (uint32_t)(y * W + x);
                }
            }
        }
        __syncthreads();  // band consumed: its buffer may be refilled, s_count/s_list visible
        if (a.use_bulk && tid == 0 && b + kNmsBufs < nb) issue(b + kNmsBufs);
    }

    const int total = s_count;
    const int np = min(total, ws.capP);
    // rank sort by raster index == np.nonzero order (evaluate.py:193); indices are unique
    for (int t = tid; t < np; t += kNmsThreads) {
        const uint32_t mine = s_list[t];
        int rank = 0;
        for (int u = 0; u < np; u++) rank += s_list[u] < mine;
        s_sorted[rank] = mine;
    }
    __syncthreads();
    const size_t out_base = ((size_t)n * ws.K + c) * ws.capP;
    for (int t = tid; t < np; t += kNmsThreads) {
        const int lin = (int)s_sorted[t], y = lin / W;
        nms_finish_peak(a, plane, H, W, out_base + t, y, lin - y * W);
    }
    if (tid == 0) nms_publish_count(a, n, c, total);
}

__global__ void __launch_bounds__(kNmsThreads, 4) nms_peaks_kernel(NmsArgs a) {
    nms_peaks_plane(a, blockIdx.x / a.ws.K, blockIdx.x % a.ws.K);
}

// ---- ragged batches: images of different sizes in one launch ----
// One image of a ragged launch: its plane base, channel stride and geometry, and the slot its results go to.
struct NmsImage {
    const float *heat;
    int64_t chan_stride;  // elements
    int H, W, band_rows, use_bulk, slot;
};
// Images per ragged launch; the descriptors travel as a kernel parameter (NmsArgs + 128 x 40 B, well inside the
// 32 764 bytes CUDA 12.1 allows), so a call returns with nothing of the caller's left to copy.
constexpr int kRaggedMaxImages = 128;
struct NmsRagged {
    NmsImage img[kRaggedMaxImages];
};

// Block b: image r.img[b / K], part b % K.  The host orders the images by plane size, largest first, so the longest
// CTAs enter the queue first; the order decides scheduling only.
__global__ void __launch_bounds__(kNmsThreads, 4) nms_peaks_ragged_kernel(NmsArgs a, const __grid_constant__ NmsRagged r) {
    const NmsImage &im = r.img[blockIdx.x / a.ws.K];
    NmsArgs b = a;
    b.heat = im.heat;
    b.img_stride = 0;
    b.chan_stride = im.chan_stride;
    b.H = im.H;
    b.W = im.W;
    b.band_rows = im.band_rows;
    b.use_bulk = im.use_bulk;
    b.image_base = im.slot;
    nms_peaks_plane(b, 0, blockIdx.x % a.ws.K);
}

inline size_t nms_smem_bytes(int band_rows, int H, int W, int capP) {
    const bool single = band_rows >= H;
    const size_t band_floats = ((single ? (size_t)H * W : (size_t)(band_rows + 2) * W) + 31) & ~(size_t)31;
    const size_t queue = (((size_t)std::min(band_rows, H) * W / 4 + 8) * sizeof(uint16_t) + 15) & ~(size_t)15;
    const int nb = single ? 1 : (H + band_rows - 1) / band_rows;
    return (size_t)std::min(nb, kNmsBufs) * band_floats * sizeof(float) + 2 * (size_t)capP * sizeof(uint32_t) + queue;
}

}  // namespace spg
