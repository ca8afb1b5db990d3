// postnet.cuh -- K0: the post-network stage of predict() (SURVEY.md §8 f-1), one fused kernel per scale.
//
// Replaces the body of the scale loop of predict() after the forward pass, /root/reference/evaluate.py:126-161:
//   split the two outputs (image, mirrored image) into body-part / keypoint channels        (:128-136)
//   flip ensemble: mirror the second output back, permute its channels, average            (:139-140)
//   cv2.resize(..., fx=stride, fy=stride, INTER_CUBIC)                                      (:143, :152)
//   angle != 0 (rotation search): cv2.warpAffine(..., rotate_matrix_reverse, (0, 0))       (:144, :153; postnet_rot_kernel)
//   crop the padding                                                                        (:148, :157)
//   cv2.resize(..., (image_w, image_h), INTER_CUBIC)                                        (:149, :158)
//   heatmap_avg += heatmap / n ; paf_avg += paf / n   (float64 accumulators, :160-161; find_peaks casts the
//   keypoint maps back to float32, :173)
// so that the maps the grouping kernels read are produced on the device, in the layout they stream
// (channel-first planes), and never visit the host.
//
// Arithmetic: OpenCV's generic bicubic path as restated -- and pinned to cv2 -- by oracle/postnet_port.py
// (coordinate (d + 0.5) * scale - 0.5 in double rounded to float, A = -0.75 coefficients in float32, taps clamped to
// the source, a float32 horizontal pass whose result is rounded to float32, then a float32 vertical pass; taps are
// multiplied and added left to right, one rounding per operation).  This translation unit is built with
// -fmad=false and the code spells out every *_rn operation, so the kernel's maps are BIT-IDENTICAL to the port's
// (tests/test_gpu_postnet.py), which in turn is within 2.8e-5 of cv2 (the IPP build in the reference's wheels is not
// bit-defined across hosts: DESIGN.md §8).
//
// One CTA computes one output tile of one channel of one image and runs the four separable passes through shared
// memory: source tile (flip-averaged while it is loaded) -> horizontal x stride -> vertical x stride (= the cropped
// intermediate the reference materialises at full size) -> horizontal to the image grid -> vertical to the image
// grid -> epilogue (scale by 1/n in float32, accumulate in float64, store).  HBM traffic is the network output once
// (x ~1.2 for tile halos) plus the output planes once; the 48 x Hp x Wp float32 intermediate never exists in memory.
#pragma once

#include <cuda_fp16.h>

#include "interp.cuh"

namespace spg {

constexpr int kPostThreads = 256;
constexpr int kPostTW = 64, kPostTH = 32;     // largest output tile
constexpr int kPostC1 = 96, kPostR1 = 48;     // capacity of the intermediate (cropped, x stride) tile (static shared memory <= 48 KB)
constexpr int kPostCS = 32, kPostRS = 20;     // capacity of the source tile (network resolution)
constexpr int kMaxNetChannels = 64;

constexpr int kPostMaxScales = 4;  // scales the stride-4 kernel fuses into one launch (more: one launch per group of 4)
struct PostScale {              // one entry of the scale loop (evaluate.py:90)
    const void *net;            // [N][2][C][h][w]: image, mirrored image (evaluate.py:116-126)
    int net_is_f16;             // 0: float32, 1: float16 (converted on load)
    long long img_stride, pair_stride, chan_stride;  // elements
    int h, w;                   // network output size
    int crop_h, crop_w;         // imageToTest size = padded size minus pad[2], pad[3] (pad[0] = pad[1] = 0 always)
    double sx2, sy2;            // source step per destination pixel of the resize to the image
};

// What every image of a launch shares.
struct PostArgs {
    int scale_index, n_scales;  // accumulate over the scale loop (:160-161)
    int n_fused;                // items (scales) summed inside ONE launch (stride 4 fuses up to kPostMaxScales; the generic
                                // and the rotated kernel take one); scale_index is the index of the first in the whole loop
    int n_out;                  // output channels handled: K keypoint + L body-part
    int K;                      // first K outputs are keypoint channels
    short src_chan[kMaxNetChannels];   // network channel of output c (keypoints: heat_chan0 + c; body parts: paf_chan0 + k)
    short flip_chan[kMaxNetChannels];  // network channel of the mirrored output that is averaged into output c
    int paf_is_f64;
    int nan_scrub;              // demo_image.py:179-180: NaN -> 0 after the accumulation
    int chan_chunk;             // stride-4 kernel: channels one CTA walks over (grid.y = ceil(n_out / chan_chunk))
    double sx1, sy1;            // source step per destination pixel of the x stride resize (the second resize's: sc[t])
};

// One image of a launch and the launch's items of it.  The per-launch kernels take one for all grid.z = N images of one
// size (pointers to slot 0; slot n is n planes further), the ragged kernels a table of them.
struct PostImage {
    PostScale sc[kPostMaxScales];  // the items of the launch, in the order of the scale loop (a.n_fused of them)
    int H, W;                   // image size = output size
    float *heat;                // [K][H][W] float32 (what find_peaks reads after its cast, evaluate.py:173)
    void *paf;                  // [L][H][W] float32 (single scale: the float64 values are exact float32) or float64
    double *heat_acc;           // [K][H][W] float64 scratch of sums that outlive a launch, or nullptr
    int tile_w, tile_h, tiles_x, tiles_y;
    int first_cta;              // ragged launches: the first CTA (blockIdx.x) of the image's tiles
    double rot[6];              // rotated items: the inverse of the warp matrix (x4 grid of the output -> of the input)
};

__device__ __forceinline__ float tap4(float a0, float a1, float a2, float a3, const float *c) {
    // taps summed left to right, every product and sum rounded to float32
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a0, c[0]), __fmul_rn(a1, c[1])), __fmul_rn(a2, c[2])), __fmul_rn(a3, c[3]));
}

struct AxisTab {  // per destination index of a tile: first tap (absolute source index, unclamped) + weights
    int s;
    float c[4];
};

__global__ void __launch_bounds__(kPostThreads) postnet_generic_kernel(PostArgs a, PostImage im) {
    __shared__ AxisTab t2x[kPostTW], t2y[kPostTH], t1x[kPostC1], t1y[kPostR1];
    __shared__ float s0[kPostRS * kPostCS];     // source tile, flip-averaged
    __shared__ float s1[kPostRS * kPostC1];     // after the horizontal x stride pass
    __shared__ float s2[kPostR1 * kPostC1];     // after the vertical x stride pass = the cropped intermediate
    __shared__ float s3[kPostR1 * kPostTW];     // after the horizontal pass of the second resize
    __shared__ int r_lo[4];                     // c_lo, r_lo of the intermediate tile; source col / row origin

    const int tid = threadIdx.x;
    const int tile = blockIdx.x, c = blockIdx.y, n = blockIdx.z;
    const int ty = tile / im.tiles_x, tx = tile - ty * im.tiles_x;
    const int ox0 = tx * im.tile_w, oy0 = ty * im.tile_h;
    const int tw = min(im.tile_w, im.W - ox0), th = min(im.tile_h, im.H - oy0);
    const PostScale &S = im.sc[0];
    const bool identity = S.crop_h == im.H && S.crop_w == im.W;  // second resize with scale 1: weights (0, 1, 0, 0)

    // ---- tables of the second resize for this tile's output columns / rows
    if (tid < tw) t2x[tid].s = axis_entry(ox0 + tid, S.sx2, t2x[tid].c);
    if (tid >= 64 && tid < 64 + th) t2y[tid - 64].s = axis_entry(oy0 + tid - 64, S.sy2, t2y[tid - 64].c);
    __syncthreads();
    if (tid == 0) {
        // crop-coordinate range the tile reads (taps clamped to the cropped array, :148-149)
        const int c_lo = identity ? ox0 : clampi(t2x[0].s, 0, S.crop_w - 1), c_hi = identity ? ox0 + tw - 1 : clampi(t2x[tw - 1].s + 3, 0, S.crop_w - 1);
        const int rr_lo = identity ? oy0 : clampi(t2y[0].s, 0, S.crop_h - 1), rr_hi = identity ? oy0 + th - 1 : clampi(t2y[th - 1].s + 3, 0, S.crop_h - 1);
        r_lo[0] = c_lo; r_lo[1] = c_hi - c_lo + 1;
        r_lo[2] = rr_lo; r_lo[3] = rr_hi - rr_lo + 1;
    }
    __syncthreads();
    const int c_lo = r_lo[0], C1 = r_lo[1], y_lo = r_lo[2], R1 = r_lo[3];
    // ---- tables of the first resize (x stride) for the intermediate columns / rows of the tile
    if (tid < C1) t1x[tid].s = axis_entry(c_lo + tid, a.sx1, t1x[tid].c);
    if (tid >= 128 && tid < 128 + R1) t1y[tid - 128].s = axis_entry(y_lo + tid - 128, a.sy1, t1y[tid - 128].c);
    __syncthreads();
    const int sc_lo = clampi(t1x[0].s, 0, S.w - 1), sc_hi = clampi(t1x[C1 - 1].s + 3, 0, S.w - 1);
    const int sr_lo = clampi(t1y[0].s, 0, S.h - 1), sr_hi = clampi(t1y[R1 - 1].s + 3, 0, S.h - 1);
    const int CS = sc_hi - sc_lo + 1, RS = sr_hi - sr_lo + 1;

    // ---- source tile: (out[c] + mirrored_out[flip(c)][:, ::-1]) / 2  (:139-140), float32
    {
        const long long base0 = (long long)n * S.img_stride + (long long)a.src_chan[c] * S.chan_stride;
        const long long base1 = (long long)n * S.img_stride + S.pair_stride + (long long)a.flip_chan[c] * S.chan_stride;
        for (int e = tid; e < RS * CS; e += kPostThreads) {
            const int i = e / CS, j = e - i * CS;
            const int y = sr_lo + i, x = sc_lo + j;
            float v0, v1;
            if (S.net_is_f16) {
                const __half *p = static_cast<const __half *>(S.net);
                v0 = __half2float(p[base0 + (long long)y * S.w + x]);
                v1 = __half2float(p[base1 + (long long)y * S.w + (S.w - 1 - x)]);
            } else {
                const float *p = static_cast<const float *>(S.net);
                v0 = p[base0 + (long long)y * S.w + x];
                v1 = p[base1 + (long long)y * S.w + (S.w - 1 - x)];
            }
            s0[i * kPostCS + j] = __fdiv_rn(__fadd_rn(v0, v1), 2.0f);
        }
    }
    __syncthreads();
    // ---- pass 1: horizontal x stride on every source row of the tile
    for (int e = tid; e < RS * C1; e += kPostThreads) {
        const int i = e / C1, X = e - i * C1;
        const AxisTab &t = t1x[X];
        const float *row = s0 + i * kPostCS - sc_lo;
        s1[i * kPostC1 + X] = tap4(row[clampi(t.s, 0, S.w - 1)], row[clampi(t.s + 1, 0, S.w - 1)], row[clampi(t.s + 2, 0, S.w - 1)],
                                   row[clampi(t.s + 3, 0, S.w - 1)], t.c);
    }
    __syncthreads();
    // ---- pass 2: vertical x stride -> the cropped intermediate (what the reference holds after :148 / :157)
    for (int e = tid; e < R1 * C1; e += kPostThreads) {
        const int Y = e / C1, X = e - Y * C1;
        const AxisTab &t = t1y[Y];
        const float *col = s1 + X - sr_lo * kPostC1;
        s2[Y * kPostC1 + X] = tap4(col[clampi(t.s, 0, S.h - 1) * kPostC1], col[clampi(t.s + 1, 0, S.h - 1) * kPostC1],
                                   col[clampi(t.s + 2, 0, S.h - 1) * kPostC1], col[clampi(t.s + 3, 0, S.h - 1) * kPostC1], t.c);
    }
    __syncthreads();
    // ---- pass 3: horizontal pass of the second resize (clamped to the cropped array)
    if (!identity) {
        for (int e = tid; e < R1 * tw; e += kPostThreads) {
            const int Y = e / tw, x = e - Y * tw;
            const AxisTab &t = t2x[x];
            const float *row = s2 + Y * kPostC1 - c_lo;
            s3[Y * kPostTW + x] = tap4(row[clampi(t.s, 0, S.crop_w - 1)], row[clampi(t.s + 1, 0, S.crop_w - 1)],
                                       row[clampi(t.s + 2, 0, S.crop_w - 1)], row[clampi(t.s + 3, 0, S.crop_w - 1)], t.c);
        }
        __syncthreads();
    }
    // ---- pass 4 + epilogue: vertical pass, / n in float32, float64 accumulation over the scale loop (:160-161)
    const float nf = (float)a.n_scales;
    const size_t plane = (size_t)im.H * im.W;
    const bool is_heat = c < a.K;
    const size_t pbase = is_heat ? ((size_t)n * a.K + c) * plane : ((size_t)n * (a.n_out - a.K) + (c - a.K)) * plane;
    const bool first = a.scale_index == 0, last = a.scale_index == a.n_scales - 1;
    for (int e = tid; e < th * tw; e += kPostThreads) {
        const int y = e / tw, x = e - y * tw;
        float v;
        if (identity) {
            v = s2[y * kPostC1 + x];
        } else {
            const AxisTab &t = t2y[y];
            const float *col = s3 + x - y_lo * kPostTW;
            v = tap4(col[clampi(t.s, 0, S.crop_h - 1) * kPostTW], col[clampi(t.s + 1, 0, S.crop_h - 1) * kPostTW],
                     col[clampi(t.s + 2, 0, S.crop_h - 1) * kPostTW], col[clampi(t.s + 3, 0, S.crop_h - 1) * kPostTW], t.c);
        }
        const size_t o = pbase + (size_t)(oy0 + y) * im.W + (ox0 + x);
        const float part = __fdiv_rn(v, nf);  // float32 array / Python int -> float32
        if (a.n_scales == 1) {  // avg = 0.0 + part: exact, the float64 value is the float32 one
            const float r = (a.nan_scrub && part != part) ? 0.0f : part;
            if (is_heat) im.heat[o] = r;
            else if (a.paf_is_f64) static_cast<double *>(im.paf)[o] = (double)r;
            else static_cast<float *>(im.paf)[o] = r;
        } else {
            double *acc = is_heat ? im.heat_acc : static_cast<double *>(im.paf);
            double s = __dadd_rn(first ? 0.0 : acc[o], (double)part);
            if (a.nan_scrub && s != s) s = 0.0;  // demo_image.py:179-180 scrubs after every scale
            acc[o] = s;
            if (is_heat && last) im.heat[o] = (float)s;  // find_peaks: heatmap_avg.astype(np.float32)
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// stride == 4 (the reference's model, utils/config: stride = 4): the x stride resize has only FOUR weight sets.
// (d + 0.5) / 4 - 0.5 = q + g_r for d = 4q + r, g_r in {-0.375, -0.125, 0.125, 0.375}: exact in float, so the weights of
// destination index d depend on r alone and its taps are source indices q-2..q+1 (r < 2) or q-1..q+2 (r >= 2).  One
// thread therefore loads FIVE source values and produces FOUR outputs (a float4 store), in both the horizontal and the
// vertical pass.  Everything that depends only on the tile POSITION -- the second resize's weights and tap offsets, the
// clamped row / column offsets of all four passes -- is computed once per CTA (per scale), and the CTA then walks over a
// chunk of CHANNELS of its tile (the first version rebuilt the tables for every (tile, channel) CTA: 40 % of its
// instructions were table set-up, 36 % per-row index arithmetic).
// The SCALE LOOP of predict() (:90, :160-161) runs inside the kernel: a thread keeps the float64 sums of its output
// pixels in registers while it works through the scales, so the averaged maps are written exactly once -- a launch per
// scale would read-modify-write 48 float64 planes per extra scale (3.6x the traffic at 3 scales).
// Same operations in the same order as the generic kernel: identical maps.
// Tile capacities of the stride-4 kernel: a full 64 x 32 output tile up to a second resize that halves the crop (the x2
// scale of the reference's multi-scale search): 64 * 2 + 13 <= 144 intermediate columns, 32 * 2 + 13 <= 80 rows; the source
// tile is a quarter of that plus the taps.  (The first version's 104 x 56 made the x2 scale cut the tile to 43 x 19: a third
// of the lanes idle in the passes of the second resize, and the per-(channel, scale) set-up paid for 817 pixels instead of 2048.)
constexpr int kPostF_C1 = 144, kPostF_R1 = 80;
constexpr int kPostF_Q = kPostF_C1 / 4, kPostF_P = kPostF_R1 / 4;
constexpr int kPostF_CS = 44, kPostF_RS = 28;   // source tile (network resolution)
struct PostTabs {
    float4 w2x[kPostTW], w2y[kPostTH];   // weights of the second resize per output column / row of the tile
    int4 o2x[kPostTW], o2y[kPostTH];     // its four tap offsets: columns of s2 (elements), rows of s3 (elements, x kPostTW)
    int o1x[kPostF_Q][5];                // pass 1: the five source columns of group q (elements of an s0 row)
    int o1y[kPostF_P][5];                // pass 2: the five source rows of group p (elements of s1, x kPostF_C1)
    float4 wph[4];                       // the four weight sets of the x4 resize
    int rng[8];
};
constexpr size_t postF_smem_bytes(int n_tabs) {
    return n_tabs * sizeof(PostTabs) + sizeof(float) * ((size_t)kPostF_RS * kPostF_CS + (size_t)kPostF_RS * kPostF_C1 +
                                                        (size_t)kPostF_R1 * kPostF_C1 + (size_t)kPostF_R1 * kPostTW);
}

// v / n for the n of the scale loop (float32 array / Python int, evaluate.py:160-161), correctly rounded like the division it
// replaces but in three instructions instead of ~14: with c = RN(1 / n), q0 = RN(v * c), r = v - q0 * n (exact in one FMA),
// q = RN(q0 + r * c) is RN(v / n) -- Markstein's correction step; checked against the exact quotient for every float32
// significand and n = 3, 5, 6, 7, 9 (powers of two are exact trivially).  Zeros keep their sign; values whose intermediates
// could leave the normal range (and every other n) take the division.
__device__ __forceinline__ float div_by_scales(float v, float nf, float rcp, bool small_n) {
    const float q0 = __fmul_rn(v, rcp);
    const float r = __fmaf_rn(-q0, nf, v);
    float q = __fmaf_rn(r, rcp, q0);
    const float av = fabsf(v);
    if (av == 0.0f) q = v;
    else if (!(small_n && av >= 0x1p-100f && av < 0x1p100f)) q = __fdiv_rn(v, nf);
    return q;
}

__device__ __forceinline__ float tap4w(float a0, float a1, float a2, float a3, const float4 &c) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a0, c.x), __fmul_rn(a1, c.y)), __fmul_rn(a2, c.z)), __fmul_rn(a3, c.w));
}

// ---- building blocks of postnet_kernel and postnet_rot_kernel: one definition each, called by both kernels in the same
// order.  Functions that end with a barrier say so; every thread of the CTA calls them.

// Second resize of the output tile at (ox0, oy0): per output column / row the weights and the first tap (absolute crop
// index, unclamped, in .x), and the four weight sets of the x4 resize.  Ends with a barrier.
__device__ __forceinline__ void post_tabs_resize2(PostTabs &T, const PostScale &S, int ox0, int oy0, int tw, int th, int tid) {
    if (tid < tw) {
        float cc[4];
        T.o2x[tid].x = axis_entry(ox0 + tid, S.sx2, cc);  // first tap (absolute crop column, unclamped) for now
        T.w2x[tid] = make_float4(cc[0], cc[1], cc[2], cc[3]);
    } else if (tid >= 64 && tid < 64 + th) {
        float cc[4];
        T.o2y[tid - 64].x = axis_entry(oy0 + tid - 64, S.sy2, cc);
        T.w2y[tid - 64] = make_float4(cc[0], cc[1], cc[2], cc[3]);
    } else if (tid >= 128 && tid < 132) {
        float cc[4];
        axis_entry(4 + (tid - 128), 0.25, cc);  // destination 4 + r: the same fraction as every 4q + r
        T.wph[tid - 128] = make_float4(cc[0], cc[1], cc[2], cc[3]);
    }
    __syncthreads();
}

// (one thread) the x4 groups that cover columns c_lo..c_hi and rows y_lo..y_hi of the x stride grid, widened to multiples
// of 4, and the source tile they read
__device__ __forceinline__ void post_tabs_range(PostTabs &T, const PostScale &S, int c_lo, int c_hi, int y_lo, int y_hi) {
    const int q_lo = c_lo >> 2, Q = (c_hi >> 2) - q_lo + 1, p_lo = y_lo >> 2, P = (y_hi >> 2) - p_lo + 1;
    const int sc_lo = max(q_lo - 2, 0), sc_hi = min(q_lo + Q + 1, S.w - 1);
    const int sr_lo = max(p_lo - 2, 0), sr_hi = min(p_lo + P + 1, S.h - 1);
    T.rng[0] = q_lo; T.rng[1] = Q; T.rng[2] = p_lo; T.rng[3] = P;
    T.rng[4] = sc_lo; T.rng[5] = sc_hi - sc_lo + 1; T.rng[6] = sr_lo; T.rng[7] = sr_hi - sr_lo + 1;
}

// Tap offsets of the four passes, clamps applied here once.  The second resize's are relative to (c_org, y_org), the crop
// position of element 0 of the buffer passes 3 and 4 read.  Ends with a barrier.
__device__ __forceinline__ void post_tabs_offsets(PostTabs &T, const PostScale &S, int tw, int th, int c_org, int y_org, int tid) {
    const int q_lo = T.rng[0], Q = T.rng[1], p_lo = T.rng[2], P = T.rng[3], sc_lo = T.rng[4], sr_lo = T.rng[6];
    if (tid < tw) {
        const int b = T.o2x[tid].x;
        T.o2x[tid] = make_int4(clampi(b, 0, S.crop_w - 1) - c_org, clampi(b + 1, 0, S.crop_w - 1) - c_org,
                               clampi(b + 2, 0, S.crop_w - 1) - c_org, clampi(b + 3, 0, S.crop_w - 1) - c_org);
    } else if (tid >= 64 && tid < 64 + th) {
        const int b = T.o2y[tid - 64].x;
        T.o2y[tid - 64] = make_int4((clampi(b, 0, S.crop_h - 1) - y_org) * kPostTW, (clampi(b + 1, 0, S.crop_h - 1) - y_org) * kPostTW,
                                    (clampi(b + 2, 0, S.crop_h - 1) - y_org) * kPostTW, (clampi(b + 3, 0, S.crop_h - 1) - y_org) * kPostTW);
    } else if (tid >= 128 && tid < 128 + Q) {
        const int qa = q_lo + tid - 128;
#pragma unroll
        for (int k = 0; k < 5; k++) T.o1x[tid - 128][k] = clampi(qa - 2 + k, 0, S.w - 1) - sc_lo;
    } else if (tid >= 192 && tid < 192 + P) {
        const int pa = p_lo + tid - 192;
#pragma unroll
        for (int k = 0; k < 5; k++) T.o1y[tid - 192][k] = (clampi(pa - 2 + k, 0, S.h - 1) - sr_lo) * kPostF_C1;
    }
    __syncthreads();
}

// T.rng as values: read once per (channel, scale) iteration, before the barriers that would force shared-memory re-reads
struct PostRange {
    int q_lo, Q, p_lo, P, sc_lo, CS, sr_lo, RS;
};
__device__ __forceinline__ PostRange post_range(const PostTabs &T) {
    return PostRange{T.rng[0], T.rng[1], T.rng[2], T.rng[3], T.rng[4], T.rng[5], T.rng[6], T.rng[7]};
}

constexpr int kPostNW = kPostThreads / 32;
constexpr int kPostKI = (kPostF_RS + kPostNW - 1) / kPostNW;  // source rows per warp
constexpr int kPostKJ = (kPostF_CS + 31) / 32;                // column passes per row
constexpr int kPostKY = kPostTH / kPostNW, kPostKX = kPostTW / 32;  // output pixels per thread: rows warp + NW * ky, columns lane + 32 * kx

// global loads of channel c's source tile (image and mirrored image) into registers
template <bool F16>
__device__ __forceinline__ void post_prefetch(float (&pv0)[kPostKI][kPostKJ], float (&pv1)[kPostKI][kPostKJ], const PostScale &S,
                                              const PostTabs &T, const PostArgs &a, int n, int c, int warp, int lane) {
    const int sc_lo = T.rng[4], CS = T.rng[5], sr_lo = T.rng[6], RS = T.rng[7];
    const long long base0 = (long long)n * S.img_stride + (long long)a.src_chan[c] * S.chan_stride + (long long)sr_lo * S.w + sc_lo;
    const long long base1 = (long long)n * S.img_stride + S.pair_stride + (long long)a.flip_chan[c] * S.chan_stride + (long long)sr_lo * S.w + (S.w - 1 - sc_lo);
#pragma unroll
    for (int ki = 0; ki < kPostKI; ki++) {
        const int i = warp + kPostNW * ki;
#pragma unroll
        for (int kj = 0; kj < kPostKJ; kj++) {
            const int j = lane + 32 * kj;
            if (i < RS && j < CS) {
                if (F16) {
                    const __half *p = static_cast<const __half *>(S.net);
                    pv0[ki][kj] = __half2float(p[base0 + (long long)i * S.w + j]);
                    pv1[ki][kj] = __half2float(p[base1 + (long long)i * S.w - j]);
                } else {
                    const float *p = static_cast<const float *>(S.net);
                    pv0[ki][kj] = p[base0 + (long long)i * S.w + j];
                    pv1[ki][kj] = p[base1 + (long long)i * S.w - j];
                }
            }
        }
    }
}

// source tile: (out[c] + mirrored_out[flip(c)][:, ::-1]) / 2  (:139-140), float32, from the prefetched registers
__device__ __forceinline__ void post_commit(float *s0, const float (&pv0)[kPostKI][kPostKJ], const float (&pv1)[kPostKI][kPostKJ],
                                            const PostRange &R, int warp, int lane) {
    const int CS = R.CS, RS = R.RS;
#pragma unroll
    for (int ki = 0; ki < kPostKI; ki++) {
        const int i = warp + kPostNW * ki;
#pragma unroll
        for (int kj = 0; kj < kPostKJ; kj++) {
            const int j = lane + 32 * kj;
            if (i < RS && j < CS) s0[i * kPostF_CS + j] = __fdiv_rn(__fadd_rn(pv0[ki][kj], pv1[ki][kj]), 2.0f);
        }
    }
}

// Passes 1 and 2: the x4 resize of the source tile s0 into the x4 groups R describes, s2 [4P][kPostF_C1], with the four
// weight sets W of T.wph.  Ends with a barrier.
__device__ __forceinline__ void post_x4_passes(const PostTabs &T, const PostRange &R, const float4 (&W)[4], const float *s0, float *s1,
                                               float *s2, int tid, int lane, int warp) {
    const int Q = R.Q, P = R.P, RS = R.RS;
    const float4 W0 = W[0], W1 = W[1], W2 = W[2], W3 = W[3];
    // ---- pass 1: horizontal x4 -- five source values in, four intermediate columns out.  A row's groups beyond the
    // 32nd (Q <= 36: the x2 scale has 35) do not get a second lane pass of their own: all rows' leftovers are dealt
    // to the CTA's threads four per row.
    auto h_item = [&](int i, int q) {
        const float *row = s0 + i * kPostF_CS;
        const int *o = T.o1x[q];
        const float v0 = row[o[0]], v1 = row[o[1]], v2 = row[o[2]], v3 = row[o[3]], v4 = row[o[4]];
        float4 r;
        r.x = tap4w(v0, v1, v2, v3, W0);
        r.y = tap4w(v0, v1, v2, v3, W1);
        r.z = tap4w(v1, v2, v3, v4, W2);
        r.w = tap4w(v1, v2, v3, v4, W3);
        *reinterpret_cast<float4 *>(s1 + i * kPostF_C1 + 4 * q) = r;
    };
    for (int i = warp; i < RS; i += kPostNW)
        if (lane < Q) h_item(i, lane);
    if (Q > 32) {
        static_assert(kPostF_Q <= 36 && kPostF_RS * 4 <= kPostThreads, "leftover groups: four per row, one thread each");
        const int i = tid >> 2, q = 32 + (tid & 3);
        if (i < RS && q < Q) h_item(i, q);
    }
    __syncthreads();
    // ---- pass 2: vertical x4 -> the x stride grid (what the reference holds after :143 / :152): five 16-byte loads in,
    // four rows of four columns out
    auto v_item = [&](int p, int x4) {
        const int *o = T.o1y[p];
        const float4 b0 = *reinterpret_cast<const float4 *>(s1 + o[0] + 4 * x4), b1 = *reinterpret_cast<const float4 *>(s1 + o[1] + 4 * x4),
                     b2 = *reinterpret_cast<const float4 *>(s1 + o[2] + 4 * x4), b3 = *reinterpret_cast<const float4 *>(s1 + o[3] + 4 * x4),
                     b4 = *reinterpret_cast<const float4 *>(s1 + o[4] + 4 * x4);
        float *dst = s2 + 4 * p * kPostF_C1 + 4 * x4;
        *reinterpret_cast<float4 *>(dst) = make_float4(tap4w(b0.x, b1.x, b2.x, b3.x, W0), tap4w(b0.y, b1.y, b2.y, b3.y, W0),
                                                       tap4w(b0.z, b1.z, b2.z, b3.z, W0), tap4w(b0.w, b1.w, b2.w, b3.w, W0));
        *reinterpret_cast<float4 *>(dst + kPostF_C1) = make_float4(tap4w(b0.x, b1.x, b2.x, b3.x, W1), tap4w(b0.y, b1.y, b2.y, b3.y, W1),
                                                                   tap4w(b0.z, b1.z, b2.z, b3.z, W1), tap4w(b0.w, b1.w, b2.w, b3.w, W1));
        *reinterpret_cast<float4 *>(dst + 2 * kPostF_C1) = make_float4(tap4w(b1.x, b2.x, b3.x, b4.x, W2), tap4w(b1.y, b2.y, b3.y, b4.y, W2),
                                                                       tap4w(b1.z, b2.z, b3.z, b4.z, W2), tap4w(b1.w, b2.w, b3.w, b4.w, W2));
        *reinterpret_cast<float4 *>(dst + 3 * kPostF_C1) = make_float4(tap4w(b1.x, b2.x, b3.x, b4.x, W3), tap4w(b1.y, b2.y, b3.y, b4.y, W3),
                                                                       tap4w(b1.z, b2.z, b3.z, b4.z, W3), tap4w(b1.w, b2.w, b3.w, b4.w, W3));
    };
    for (int p = warp; p < P; p += kPostNW)
        if (lane < Q) v_item(p, lane);
    if (Q > 32) {
        static_assert(kPostF_P * 4 <= kPostThreads, "leftover column groups: four per row group, one thread each");
        const int p = tid >> 2, x4 = 32 + (tid & 3);
        if (p < P && x4 < Q) v_item(p, x4);
    }
    __syncthreads();
}

// Pass 3: horizontal pass of the second resize over the crop rows the tile needs, s2 -> s3.  Ends with a barrier when it runs.
template <bool IDENT>
__device__ __forceinline__ void post_resize2_h(const PostTabs &T, const float *s2, float *s3, bool identity, int tw, int th, int lane, int warp) {
    if (!IDENT && !identity) {
        const int yr_lo = T.o2y[0].x / kPostTW, yr_hi = T.o2y[th - 1].w / kPostTW;
        int4 ox[kPostKX];     // this thread's columns are the same in every row: offsets and weights once per (channel, scale)
        float4 wx[kPostKX];
#pragma unroll
        for (int kx = 0; kx < kPostKX; kx++) {
            const int x = min(lane + 32 * kx, tw - 1);
            ox[kx] = T.o2x[x];
            wx[kx] = T.w2x[x];
        }
        for (int Y = yr_lo + warp; Y <= yr_hi; Y += kPostNW) {
            const float *row = s2 + Y * kPostF_C1;
#pragma unroll
            for (int kx = 0; kx < kPostKX; kx++)
                if (lane + 32 * kx < tw)
                    s3[Y * kPostTW + lane + 32 * kx] = tap4w(row[ox[kx].x], row[ox[kx].y], row[ox[kx].z], row[ox[kx].w], wx[kx]);
        }
        __syncthreads();
    }
}

// Where channel c of image n goes: one base pointer per dtype (32-bit offsets from it per thread; the dtype branches are
// block-uniform), and whether the values stored are float32.
struct PostOut {
    size_t pbase;
    float *f;
    double *d;
    bool store_f;
};
__device__ __forceinline__ PostOut post_out(const PostArgs &a, const PostImage &im, int n, int c, int ox0, int oy0, bool more_follow) {
    const size_t plane = (size_t)im.H * im.W;
    const bool is_heat = c < a.K;
    PostOut o;
    o.pbase = (is_heat ? ((size_t)n * a.K + c) * plane : ((size_t)n * (a.n_out - a.K) + (c - a.K)) * plane) + (size_t)oy0 * im.W + ox0;
    o.f = is_heat ? im.heat + o.pbase : static_cast<float *>(im.paf) + o.pbase;
    o.d = (is_heat ? im.heat_acc : static_cast<double *>(im.paf)) + (is_heat && im.heat_acc == nullptr ? 0 : o.pbase);
    o.store_f = is_heat ? !more_follow : !a.paf_is_f64;
    return o;
}

// continuing a scale loop longer than one launch: the float64 sums so far
template <bool SINGLE>
__device__ __forceinline__ void post_load_acc(double (&acc)[SINGLE ? 1 : kPostKY][SINGLE ? 1 : kPostKX], const PostArgs &a, const PostImage &im,
                                              int c, size_t pbase, int tw, int th, int lane, int warp) {
    if (!SINGLE && a.scale_index > 0) {
        const double *prev = c < a.K ? im.heat_acc : static_cast<const double *>(im.paf);
#pragma unroll
        for (int ky = 0; ky < kPostKY; ky++)
#pragma unroll
            for (int kx = 0; kx < kPostKX; kx++) {
                const int y = warp + kPostNW * ky, x = lane + 32 * kx;
                acc[SINGLE ? 0 : ky][SINGLE ? 0 : kx] = (y < th && x < tw) ? prev[pbase + (size_t)y * im.W + x] : 0.0;
            }
    }
}

// Pass 4 and epilogue: vertical pass of the second resize (s3; with an identity second resize the crop itself, s2),
// / n in float32, float64 sum over the scale loop (:160-161) in registers.  SINGLE: the maps are stored from here.
// (c_org, y_org) is the crop position of element 0 of s2.
template <bool SINGLE, bool IDENT>
__device__ __forceinline__ void post_resize2_v(double (&acc)[SINGLE ? 1 : kPostKY][SINGLE ? 1 : kPostKX], const PostTabs &T,
                                               const float *s2, const float *s3, bool identity, const PostArgs &a, const PostImage &im,
                                               const PostOut &out,
                                               int ox0, int oy0, int tw, int th, int c_org, int y_org, bool zero_start,
                                               float nf, float nf_rcp, bool nf_small, int lane, int warp) {
    float r1[SINGLE ? kPostKY : 1][SINGLE ? kPostKX : 1];  // single scale: the values this thread stores
#pragma unroll
    for (int ky = 0; ky < kPostKY; ky++) {
        const int y = warp + kPostNW * ky;
        if (y < th) {
            int4 o = make_int4(0, 0, 0, 0);
            float4 wy = make_float4(0.f, 1.f, 0.f, 0.f);
            if (!IDENT && !identity) {
                o = T.o2y[y];
                wy = T.w2y[y];
            }
            const float *idrow = s2 + (oy0 + y - y_org) * kPostF_C1 + (ox0 - c_org);
#pragma unroll
            for (int kx = 0; kx < kPostKX; kx++) {
                const int x = lane + 32 * kx;
                if (x < tw) {
                    float v;
                    if (IDENT) v = idrow[x];
                    else v = identity ? idrow[x] : tap4w(s3[o.x + x], s3[o.y + x], s3[o.z + x], s3[o.w + x], wy);
                    if (SINGLE) {  // avg = 0.0 + v / 1: the float64 value is this float32 one
                        r1[SINGLE ? ky : 0][SINGLE ? kx : 0] = (a.nan_scrub && v != v) ? 0.0f : v;  // demo_image.py:179-180
                    } else {
                        const float part = div_by_scales(v, nf, nf_rcp, nf_small);  // float32 array / Python int -> float32
                        double sacc = __dadd_rn(zero_start ? 0.0 : acc[SINGLE ? 0 : ky][SINGLE ? 0 : kx], (double)part);
                        if (a.nan_scrub && sacc != sacc) sacc = 0.0;  // demo_image.py:179-180 scrubs after every scale
                        acc[SINGLE ? 0 : ky][SINGLE ? 0 : kx] = sacc;
                    }
                }
            }
        }
    }
    if (SINGLE) {  // one block-uniform branch on the output type, then eight stores at constant offsets from one pointer
        const int o0 = warp * im.W + lane, dy = kPostNW * im.W;
        if (out.store_f) {
            float *op = out.f + o0;
#pragma unroll
            for (int ky = 0; ky < kPostKY; ky++)
#pragma unroll
                for (int kx = 0; kx < kPostKX; kx++)
                    if (warp + kPostNW * ky < th && lane + 32 * kx < tw) op[ky * dy + 32 * kx] = r1[SINGLE ? ky : 0][SINGLE ? kx : 0];
        } else {
            double *op = out.d + o0;
#pragma unroll
            for (int ky = 0; ky < kPostKY; ky++)
#pragma unroll
                for (int kx = 0; kx < kPostKX; kx++)
                    if (warp + kPostNW * ky < th && lane + 32 * kx < tw) op[ky * dy + 32 * kx] = (double)r1[SINGLE ? ky : 0][SINGLE ? kx : 0];
        }
    }
}

// the averaged maps, written once: keypoint maps as float32 (find_peaks' cast, :173), body parts float64 / float32
template <bool SINGLE>
__device__ __forceinline__ void post_store_acc(const double (&acc)[SINGLE ? 1 : kPostKY][SINGLE ? 1 : kPostKX], const PostImage &im,
                                               const PostOut &out, int tw, int th, int lane, int warp) {
    if (!SINGLE) {
#pragma unroll
        for (int ky = 0; ky < kPostKY; ky++) {
            const int y = warp + kPostNW * ky;
            const int orow = y * im.W;
#pragma unroll
            for (int kx = 0; kx < kPostKX; kx++) {
                const int x = lane + 32 * kx;
                if (y < th && x < tw) {
                    const double v = acc[SINGLE ? 0 : ky][SINGLE ? 0 : kx];
                    if (out.store_f) out.f[orow + x] = (float)v;
                    else out.d[orow + x] = v;
                }
            }
        }
    }
}

// SINGLE: one scale in the whole loop (the reference's default): no float64 sums, the maps are stored from pass 4.
// IDENT: every fused scale's second resize is the identity (crop == image: weights (0,1,0,0)) -- passes 3 and 4 fall away.
// F16: the network output is float16.
// One CTA: tile `tile` of image `im` (slot n of its output planes), channel chunk `chunk`.
template <bool SINGLE, bool IDENT, bool F16>
__device__ __forceinline__ void postnet_tile(const PostArgs &a, const PostImage &im, int tile, int chunk, int n) {
    constexpr int kTabs = SINGLE ? 1 : kPostMaxScales;
    extern __shared__ __align__(16) unsigned char post_smem[];
    PostTabs *TT = reinterpret_cast<PostTabs *>(post_smem);
    float *s0 = reinterpret_cast<float *>(post_smem + kTabs * sizeof(PostTabs));  // source tile, flip-averaged [RS][kPostF_CS]
    float *s1 = s0 + kPostF_RS * kPostF_CS;                               // after the horizontal x4 pass    [RS][kPostF_C1]
    float *s2 = s1 + kPostF_RS * kPostF_C1;                               // after the vertical x4 pass      [4P][kPostF_C1]
    float *s3 = s2 + kPostF_R1 * kPostF_C1;                               // after the 2nd resize's h. pass  [4P][kPostTW]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int c_begin = chunk * a.chan_chunk, c_end = min(c_begin + a.chan_chunk, a.n_out);
    const int ty = tile / im.tiles_x, tx = tile - ty * im.tiles_x;
    const int ox0 = tx * im.tile_w, oy0 = ty * im.tile_h;
    const int tw = min(im.tile_w, im.W - ox0), th = min(im.tile_h, im.H - oy0);

    // ---- once per CTA and scale: everything that depends on the tile position only
    for (int t = 0; t < a.n_fused; t++) {
        PostTabs &T = TT[t];
        const PostScale &S = im.sc[t];
        const bool identity = IDENT || (S.crop_h == im.H && S.crop_w == im.W);  // second resize with scale 1: weights (0, 1, 0, 0)
        post_tabs_resize2(T, S, ox0, oy0, tw, th, tid);
        if (tid == 0) {
            // crop-coordinate range the tile reads (taps clamped to the cropped array, :148-149)
            const int c_lo = identity ? ox0 : clampi(T.o2x[0].x, 0, S.crop_w - 1), c_hi = identity ? ox0 + tw - 1 : clampi(T.o2x[tw - 1].x + 3, 0, S.crop_w - 1);
            const int y_lo = identity ? oy0 : clampi(T.o2y[0].x, 0, S.crop_h - 1), y_hi = identity ? oy0 + th - 1 : clampi(T.o2y[th - 1].x + 3, 0, S.crop_h - 1);
            post_tabs_range(T, S, c_lo, c_hi, y_lo, y_hi);
        }
        __syncthreads();
        post_tabs_offsets(T, S, tw, th, 4 * T.rng[0], 4 * T.rng[2], tid);
    }
    const float nf = (float)a.n_scales, nf_rcp = __fdiv_rn(1.0f, nf);
    const bool nf_small = a.n_scales >= 2 && a.n_scales <= 9;
    const bool more_follow = a.scale_index + a.n_fused < a.n_scales;  // only with more than kPostMaxScales scales

    float pv0[kPostKI][kPostKJ], pv1[kPostKI][kPostKJ];
    if (c_begin < c_end) post_prefetch<F16>(pv0, pv1, im.sc[0], TT[0], a, n, c_begin, warp, lane);

    for (int c = c_begin; c < c_end; c++) {
        const PostOut out = post_out(a, im, n, c, ox0, oy0, more_follow);
        double acc[SINGLE ? 1 : kPostKY][SINGLE ? 1 : kPostKX];
        post_load_acc<SINGLE>(acc, a, im, c, out.pbase, tw, th, lane, warp);
        for (int t = 0; t < a.n_fused; t++) {
            const PostTabs &T = TT[t];
            const PostScale &S = im.sc[t];
            const bool identity = IDENT || (S.crop_h == im.H && S.crop_w == im.W);
            const PostRange R = post_range(T);
            const float4 W[4] = {T.wph[0], T.wph[1], T.wph[2], T.wph[3]};
            // ---- source tile.  Its global loads were issued one iteration ago (the chain load -> barrier -> four short
            // passes is latency bound otherwise); commit them, then put the next iteration's loads in flight under this
            // iteration's passes.
            post_commit(s0, pv0, pv1, R, warp, lane);
            __syncthreads();
            {
                int tn = t + 1, cn = c;
                if (tn == a.n_fused) { tn = 0; cn = c + 1; }
                if (cn < c_end) post_prefetch<F16>(pv0, pv1, im.sc[tn], TT[tn], a, n, cn, warp, lane);
            }
            post_x4_passes(T, R, W, s0, s1, s2, tid, lane, warp);  // -> the cropped intermediate (what the reference holds after :148 / :157)
            post_resize2_h<IDENT>(T, s2, s3, identity, tw, th, lane, warp);
            post_resize2_v<SINGLE, IDENT>(acc, T, s2, s3, identity, a, im, out, ox0, oy0, tw, th, 4 * R.q_lo, 4 * R.p_lo,
                                          a.scale_index == 0 && t == 0, nf, nf_rcp, nf_small, lane, warp);
            __syncthreads();  // s0..s3 are reused by the next scale / channel
        }
        post_store_acc<SINGLE>(acc, im, out, tw, th, lane, warp);
    }
}

template <bool SINGLE, bool IDENT, bool F16>
__global__ void __launch_bounds__(kPostThreads, 2) postnet_kernel(PostArgs a, PostImage im) {
    postnet_tile<SINGLE, IDENT, F16>(a, im, blockIdx.x, blockIdx.y, blockIdx.z);
}

// ---------------------------------------------------------------------------------------------------------------
// An item of the rotation search (evaluate.py:107-158, angle != 0), stride 4, one item per launch: between the x4 resize
// and the crop the maps go through cv2.warpAffine(map, rotate_matrix_reverse, (0, 0)), INTER_LINEAR, BORDER_CONSTANT 0,
// on the x4 grid (Hp x Wp = 4h x 4w, output grid = input grid).  The x4 maps still never exist in memory.  Per output tile:
//   1. the crop span [c_lo, c_hi] x [y_lo, y_hi] the tile's second resize reads (the tables postnet_kernel uses);
//   2. the box of the x4 grid whose values the warp of that span reads.  Box argument: pixel (x, y) reads the taps
//      (sx + j, sy + i), i, j in {0, 1}, with sx = ((rhe(1024 (m1 y + m2)) + 16 + rhe(1024 m0 x)) >> 5) >> 5.  The two
//      roundings and the +16 move 1024 * u (u = m0 x + m1 y + m2) by at most 17, so sx lies within one pixel of floor(u)
//      (likewise sy of v = m3 x + m4 y + m5).  u and v are affine, so over the span they take their extremes at its
//      corners: every tap lies in [floor(u_min) - 1, floor(u_max) + 2] x [floor(v_min) - 1, floor(v_max) + 2].  The box
//      adds one more pixel on each side against the rounding of the corner values themselves and is clipped to the grid
//      (taps outside the grid read 0 and need no value);
//   3. the box's x4 values into shared memory with the same passes as postnet_kernel, from a flip-averaged source tile;
//   4. the warp gathers the span from them (OpenCV's fixed point, bit for bit: oracle/postnet_rotation_port.py);
//   5. the second resize and the epilogue of postnet_kernel: / n in float32, float64 sums that continue through memory
//      between launches, keypoint maps cast to float32 by the last item, nan_scrub.
// The host picks a tile whose span and box fit the buffers (a rotation grows the box by at most sqrt(2) per axis).
constexpr int kPostR_R1 = 64;  // rows of the warped span (its columns: kPostF_C1)
constexpr size_t postR_smem_bytes() {
    return sizeof(PostTabs) + sizeof(float) * ((size_t)kPostF_RS * kPostF_CS + (size_t)kPostF_RS * kPostF_C1 +
                                               (size_t)kPostF_R1 * kPostF_C1 + (size_t)kPostR_R1 * kPostF_C1);
}
static_assert(kPostR_R1 * kPostTW <= kPostF_RS * (kPostF_CS + kPostF_C1), "pass 3's output fits where the source tile was");

// One CTA: tile `tile` of the rotated item of image `im` (slot n of its output planes), channel chunk `chunk`.
template <bool SINGLE, bool F16>
__device__ __forceinline__ void postnet_rot_tile(const PostArgs &a, const PostImage &im, int tile, int chunk, int n) {
    extern __shared__ __align__(16) unsigned char post_smem[];
    PostTabs &T = *reinterpret_cast<PostTabs *>(post_smem);
    float *s0 = reinterpret_cast<float *>(post_smem + sizeof(PostTabs));  // source tile, flip-averaged [RS][kPostF_CS]
    float *s1 = s0 + kPostF_RS * kPostF_CS;                   // after the horizontal x4 pass        [RS][kPostF_C1]
    float *su = s1 + kPostF_RS * kPostF_C1;                   // the box of the x4 grid              [4P][kPostF_C1]
    float *sr = su + kPostF_R1 * kPostF_C1;                   // the warped crop span                [kPostR_R1][kPostF_C1]
    float *s3 = s0;                                           // after the 2nd resize's h. pass      [kPostR_R1][kPostTW]
    __shared__ int span[4];                                   // c_lo, y_lo, columns, rows of the crop span
    __shared__ int colA[kPostF_C1], colB[kPostF_C1], rowX[kPostR_R1], rowY[kPostR_R1];  // fixed-point coordinate terms

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int c_begin = chunk * a.chan_chunk, c_end = min(c_begin + a.chan_chunk, a.n_out);
    const int ty = tile / im.tiles_x, tx = tile - ty * im.tiles_x;
    const int ox0 = tx * im.tile_w, oy0 = ty * im.tile_h;
    const int tw = min(im.tile_w, im.W - ox0), th = min(im.tile_h, im.H - oy0);
    const PostScale &S = im.sc[0];
    const bool identity = S.crop_h == im.H && S.crop_w == im.W;
    const int Wp = 4 * S.w, Hp = 4 * S.h;
    const double m0 = im.rot[0], m1 = im.rot[1], m2 = im.rot[2], m3 = im.rot[3], m4 = im.rot[4], m5 = im.rot[5];

    post_tabs_resize2(T, S, ox0, oy0, tw, th, tid);
    if (tid == 0) {
        const int c_lo = identity ? ox0 : clampi(T.o2x[0].x, 0, S.crop_w - 1), c_hi = identity ? ox0 + tw - 1 : clampi(T.o2x[tw - 1].x + 3, 0, S.crop_w - 1);
        const int y_lo = identity ? oy0 : clampi(T.o2y[0].x, 0, S.crop_h - 1), y_hi = identity ? oy0 + th - 1 : clampi(T.o2y[th - 1].x + 3, 0, S.crop_h - 1);
        span[0] = c_lo; span[1] = y_lo; span[2] = c_hi - c_lo + 1; span[3] = y_hi - y_lo + 1;
        double u_lo = INFINITY, u_hi = -INFINITY, v_lo = INFINITY, v_hi = -INFINITY;
        for (int k = 0; k < 4; k++) {
            const double x = (k & 1) ? c_hi : c_lo, y = (k & 2) ? y_hi : y_lo;
            const double u = m0 * x + m1 * y + m2, v = m3 * x + m4 * y + m5;
            u_lo = fmin(u_lo, u); u_hi = fmax(u_hi, u); v_lo = fmin(v_lo, v); v_hi = fmax(v_hi, v);
        }
        // clipped in double first: a box far outside the grid must not overflow the conversion
        auto clip = [](double e, int hi) { return (int)fmin(fmax(e, 0.0), (double)hi); };
        post_tabs_range(T, S, clip(floor(u_lo) - 2.0, Wp - 1), clip(floor(u_hi) + 3.0, Wp - 1), clip(floor(v_lo) - 2.0, Hp - 1),
                        clip(floor(v_hi) + 3.0, Hp - 1));
    }
    __syncthreads();
    const int c_lo = span[0], y_lo = span[1], C1 = span[2], R1 = span[3];
    // per column rhe(1024 m0 x), rhe(1024 m3 x); per row rhe(1024 (m1 y + m2)) + 16, rhe(1024 (m4 y + m5)) + 16
    // (warpAffine's adelta / bdelta and X0 / Y0; __double2int_rn rounds ties to even like cvRound)
    for (int i = tid; i < C1; i += kPostThreads) {
        const double x = (double)(c_lo + i);
        colA[i] = __double2int_rn(__dmul_rn(__dmul_rn(m0, x), 1024.0));
        colB[i] = __double2int_rn(__dmul_rn(__dmul_rn(m3, x), 1024.0));
    }
    for (int i = tid; i < R1; i += kPostThreads) {
        const double y = (double)(y_lo + i);
        rowX[i] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m1, y), m2), 1024.0)) + 16;
        rowY[i] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m4, y), m5), 1024.0)) + 16;
    }
    post_tabs_offsets(T, S, tw, th, c_lo, y_lo, tid);

    const float nf = (float)a.n_scales, nf_rcp = __fdiv_rn(1.0f, nf);
    const bool nf_small = a.n_scales >= 2 && a.n_scales <= 9;
    const bool more_follow = a.scale_index + 1 < a.n_scales;
    const PostRange R = post_range(T);
    const float4 W[4] = {T.wph[0], T.wph[1], T.wph[2], T.wph[3]};
    const int bx0 = 4 * R.q_lo, by0 = 4 * R.p_lo;

    float pv0[kPostKI][kPostKJ], pv1[kPostKI][kPostKJ];
    if (c_begin < c_end) post_prefetch<F16>(pv0, pv1, S, T, a, n, c_begin, warp, lane);
    for (int c = c_begin; c < c_end; c++) {
        const PostOut out = post_out(a, im, n, c, ox0, oy0, more_follow);
        double acc[SINGLE ? 1 : kPostKY][SINGLE ? 1 : kPostKX];
        post_load_acc<SINGLE>(acc, a, im, c, out.pbase, tw, th, lane, warp);
        post_commit(s0, pv0, pv1, R, warp, lane);
        __syncthreads();
        if (c + 1 < c_end) post_prefetch<F16>(pv0, pv1, S, T, a, n, c + 1, warp, lane);
        post_x4_passes(T, R, W, s0, s1, su, tid, lane, warp);
        // ---- the warp: the crop span from the box, taps outside the x4 grid read 0 (evaluate.py:144-146, :153-155)
        for (int e = tid; e < R1 * C1; e += kPostThreads) {
            const int Y = e / C1, X = e - Y * C1;
            sr[Y * kPostF_C1 + X] = warp_linear<1>(rowX[Y] + colA[X], rowY[Y] + colB[X], Wp, Hp, su, kPostF_C1, bx0, by0,
                                                   [](float v) { return v; });
        }
        __syncthreads();
        post_resize2_h<false>(T, sr, s3, identity, tw, th, lane, warp);
        post_resize2_v<SINGLE, false>(acc, T, sr, s3, identity, a, im, out, ox0, oy0, tw, th, c_lo, y_lo, a.scale_index == 0, nf,
                                      nf_rcp, nf_small, lane, warp);
        __syncthreads();  // s0 / s3, su and sr are reused by the next channel
        post_store_acc<SINGLE>(acc, im, out, tw, th, lane, warp);
    }
}

template <bool SINGLE, bool F16>
__global__ void __launch_bounds__(kPostThreads, 2) postnet_rot_kernel(PostArgs a, PostImage im) {
    postnet_rot_tile<SINGLE, F16>(a, im, blockIdx.x, blockIdx.y, blockIdx.z);
}

// ---------------------------------------------------------------------------------------------------------------
// The reference's default configuration -- ONE scale whose crop is the image (scale_search = [1.0] on an image that needs
// no second resize: evaluate.py:149 is the identity, weights (0, 1, 0, 0)) -- needs only the two x4 passes, and the vertical
// one can store straight to the maps.  This kernel is postnet_kernel<true, true, F16> with everything that does not
// depend on the channel hoisted out of the channel loop: a thread keeps its five clamped tap offsets of either pass, the
// four weight sets and its global offsets in registers, so a channel costs it the source loads, one item of the
// horizontal pass (6 shared loads, 56 flops, two 16-byte shared stores) and one of the vertical pass (five 16-byte shared
// loads, 112 flops, four 16-byte global stores: 16 output pixels) -- ~16 instructions per output pixel instead of ~80.
// Same operations in the same order on every value: identical maps.
constexpr int kPostI_TW = 128, kPostI_TH = 32;      // output tile
constexpr int kPostI_Q = kPostI_TW / 4, kPostI_P = kPostI_TH / 4;
constexpr int kPostI_RS = kPostI_P + 4, kPostI_CS = kPostI_Q + 4;  // source tile (network resolution): groups p-2 .. p+2
constexpr int kPostI_S0 = kPostI_CS;                // row stride of the source tile in shared memory
constexpr int kPostI_LD = (kPostI_RS * kPostI_CS + kPostThreads - 1) / kPostThreads;  // source elements per thread

// One CTA: tile `tile` of image `im` (slot n of its output planes), channel chunk `chunk`.
template <bool F16>
__device__ __forceinline__ void postnet_x4_ident_tile(const PostArgs &a, const PostImage &im, int tile, int chunk, int n) {
    __shared__ float s0[2][kPostI_RS * kPostI_S0];                  // source tile, flip-averaged
    __shared__ __align__(16) float s1[2][kPostI_RS * kPostI_TW];   // after the horizontal pass
    __shared__ int s_o1x[kPostI_Q + 1][5], s_o1y[kPostI_P][5];
    __shared__ float4 s_wph[4];

    const int tid = threadIdx.x;
    const PostScale &S = im.sc[0];
    const int c_begin = chunk * a.chan_chunk, c_end = min(c_begin + a.chan_chunk, a.n_out);
    const int ty = tile / im.tiles_x, tx = tile - ty * im.tiles_x;
    const int ox0 = tx * kPostI_TW, oy0 = ty * kPostI_TH;
    const int tw = min(kPostI_TW, im.W - ox0), th = min(kPostI_TH, im.H - oy0);
    // crop columns ox0 .. ox0 + tw - 1 = intermediate groups q_lo .. q_lo + Q - 1 (ox0, oy0 are multiples of 4)
    const int q_lo = ox0 >> 2, Q = ((ox0 + tw - 1) >> 2) - q_lo + 1, p_lo = oy0 >> 2, P = ((oy0 + th - 1) >> 2) - p_lo + 1;
    const int sc_lo = max(q_lo - 2, 0), sc_hi = min(q_lo + Q + 1, S.w - 1), sr_lo = max(p_lo - 2, 0), sr_hi = min(p_lo + P + 1, S.h - 1);
    const int CS = sc_hi - sc_lo + 1, RS = sr_hi - sr_lo + 1;
    if (tid <= Q && tid <= kPostI_Q) {  // (one entry past the last group: the pair (q, q + 1) of pass 1 reads it)
#pragma unroll
        for (int k = 0; k < 5; k++) s_o1x[tid][k] = clampi(q_lo + tid - 2 + k, 0, S.w - 1) - sc_lo;
    } else if (tid >= 64 && tid < 64 + P) {
#pragma unroll
        for (int k = 0; k < 5; k++) s_o1y[tid - 64][k] = (clampi(p_lo + tid - 64 - 2 + k, 0, S.h - 1) - sr_lo) * kPostI_TW;
    } else if (tid >= 96 && tid < 100) {
        float cc[4];
        axis_entry(4 + (tid - 96), 0.25, cc);  // destination 4 + r: the same fraction as every 4q + r
        s_wph[tid - 96] = make_float4(cc[0], cc[1], cc[2], cc[3]);
    }
    __syncthreads();
    const float4 W0 = s_wph[0], W1 = s_wph[1], W2 = s_wph[2], W3 = s_wph[3];
    // pass 1 item of this thread: source row i1, the two groups q1, q1 + 1 (six source values in, eight columns out)
    const int i1 = tid >> 4, q1 = 2 * (tid & 15);
    const bool act1 = i1 < RS && q1 < Q;
    int h0 = 0, h1 = 0, h2 = 0, h3 = 0, h4 = 0, h5 = 0;
    if (act1) {
        const int b = i1 * kPostI_S0;
        h0 = b + s_o1x[q1][0]; h1 = b + s_o1x[q1][1]; h2 = b + s_o1x[q1][2]; h3 = b + s_o1x[q1][3]; h4 = b + s_o1x[q1][4];
        h5 = b + s_o1x[q1 + 1][4];
    }
    const int d1 = i1 * kPostI_TW + 4 * q1;
    // pass 2 item: row group p2, columns 4 * x2 .. 4 * x2 + 3 (five 16-byte loads in, four rows of four columns out)
    const int p2 = tid >> 5, x2 = tid & 31;
    const bool act2 = p2 < P && 4 * x2 < tw;
    int v0 = 0, v1 = 0, v2 = 0, v3 = 0, v4 = 0;
    if (act2) {
        v0 = s_o1y[p2][0] + 4 * x2; v1 = s_o1y[p2][1] + 4 * x2; v2 = s_o1y[p2][2] + 4 * x2; v3 = s_o1y[p2][3] + 4 * x2; v4 = s_o1y[p2][4] + 4 * x2;
    }
    // 16-byte stores need all of the tile's columns and 16-byte aligned rows (W a multiple of 4; float64 rows: always then)
    const bool vec = tw == kPostI_TW && (im.W & 3) == 0;
    // source elements of this thread (row-major over the RS x CS tile)
    long long g0[kPostI_LD], g1[kPostI_LD];
    int sdst[kPostI_LD];
    bool actl[kPostI_LD];
#pragma unroll
    for (int u = 0; u < kPostI_LD; u++) {
        const int e = tid + kPostThreads * u;
        const int i = e / CS, j = e - i * CS;
        actl[u] = i < RS;
        sdst[u] = i * kPostI_S0 + j;
        g0[u] = (long long)n * S.img_stride + (long long)(sr_lo + i) * S.w + sc_lo + j;
        g1[u] = (long long)n * S.img_stride + S.pair_stride + (long long)(sr_lo + i) * S.w + (S.w - 1 - sc_lo) - j;
    }
    float pv0[kPostI_LD], pv1[kPostI_LD];
    auto prefetch = [&](int c) {
        const long long c0 = (long long)a.src_chan[c] * S.chan_stride, c1 = (long long)a.flip_chan[c] * S.chan_stride;
#pragma unroll
        for (int u = 0; u < kPostI_LD; u++) {
            if (actl[u]) {
                if (F16) {
                    const __half *p = static_cast<const __half *>(S.net);
                    pv0[u] = __half2float(p[g0[u] + c0]);
                    pv1[u] = __half2float(p[g1[u] + c1]);
                } else {
                    const float *p = static_cast<const float *>(S.net);
                    pv0[u] = p[g0[u] + c0];
                    pv1[u] = p[g1[u] + c1];
                }
            }
        }
    };
    const size_t plane = (size_t)im.H * im.W;
    const size_t othread = (size_t)(oy0 + 4 * p2) * im.W + ox0 + 4 * x2;  // first output of the pass-2 item
    // One barrier per channel: the interval between two barriers runs the horizontal pass of channel c (source tile buffer
    // `buf` -> s1[buf]), the vertical pass + stores of channel c - 1 (s1[buf ^ 1]), commits channel c + 1's source tile (loaded
    // one interval ago) to the other s0 buffer and puts channel c + 2's loads in flight.
    auto commit = [&](int b) {  // (out[c] + mirrored_out[flip(c)][:, ::-1]) / 2  (:139-140), float32
#pragma unroll
        for (int u = 0; u < kPostI_LD; u++)
            if (actl[u]) s0[b][sdst[u]] = __fdiv_rn(__fadd_rn(pv0[u], pv1[u]), 2.0f);
    };
    if (c_begin < c_end) {
        prefetch(c_begin);
        commit(0);
        if (c_begin + 1 < c_end) prefetch(c_begin + 1);
    }
    __syncthreads();
    int buf = 0;
    for (int c = c_begin; c <= c_end; c++, buf ^= 1) {
        // ---- pass 1: horizontal x4
        if (act1 && c < c_end) {
            const float a0 = s0[buf][h0], a1 = s0[buf][h1], a2 = s0[buf][h2], a3 = s0[buf][h3], a4 = s0[buf][h4], a5 = s0[buf][h5];
            float4 r, t;
            r.x = tap4w(a0, a1, a2, a3, W0);
            r.y = tap4w(a0, a1, a2, a3, W1);
            r.z = tap4w(a1, a2, a3, a4, W2);
            r.w = tap4w(a1, a2, a3, a4, W3);
            t.x = tap4w(a1, a2, a3, a4, W0);
            t.y = tap4w(a1, a2, a3, a4, W1);
            t.z = tap4w(a2, a3, a4, a5, W2);
            t.w = tap4w(a2, a3, a4, a5, W3);
            *reinterpret_cast<float4 *>(s1[buf] + d1) = r;
            *reinterpret_cast<float4 *>(s1[buf] + d1 + 4) = t;
        }
        // ---- pass 2: vertical x4, stored straight to the maps (single scale: avg = 0.0 + v / 1 is the float32 value itself)
        if (act2 && c > c_begin) {
            const float *s1b = s1[buf ^ 1];
            const int cp = c - 1;
            const float4 b0 = *reinterpret_cast<const float4 *>(s1b + v0), b1 = *reinterpret_cast<const float4 *>(s1b + v1),
                         b2 = *reinterpret_cast<const float4 *>(s1b + v2), b3 = *reinterpret_cast<const float4 *>(s1b + v3),
                         b4 = *reinterpret_cast<const float4 *>(s1b + v4);
            float4 r[4];
            r[0] = make_float4(tap4w(b0.x, b1.x, b2.x, b3.x, W0), tap4w(b0.y, b1.y, b2.y, b3.y, W0), tap4w(b0.z, b1.z, b2.z, b3.z, W0), tap4w(b0.w, b1.w, b2.w, b3.w, W0));
            r[1] = make_float4(tap4w(b0.x, b1.x, b2.x, b3.x, W1), tap4w(b0.y, b1.y, b2.y, b3.y, W1), tap4w(b0.z, b1.z, b2.z, b3.z, W1), tap4w(b0.w, b1.w, b2.w, b3.w, W1));
            r[2] = make_float4(tap4w(b1.x, b2.x, b3.x, b4.x, W2), tap4w(b1.y, b2.y, b3.y, b4.y, W2), tap4w(b1.z, b2.z, b3.z, b4.z, W2), tap4w(b1.w, b2.w, b3.w, b4.w, W2));
            r[3] = make_float4(tap4w(b1.x, b2.x, b3.x, b4.x, W3), tap4w(b1.y, b2.y, b3.y, b4.y, W3), tap4w(b1.z, b2.z, b3.z, b4.z, W3), tap4w(b1.w, b2.w, b3.w, b4.w, W3));
            if (a.nan_scrub) {  // demo_image.py:179-180
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    r[k].x = r[k].x != r[k].x ? 0.0f : r[k].x; r[k].y = r[k].y != r[k].y ? 0.0f : r[k].y;
                    r[k].z = r[k].z != r[k].z ? 0.0f : r[k].z; r[k].w = r[k].w != r[k].w ? 0.0f : r[k].w;
                }
            }
            const bool is_heat = cp < a.K;
            const size_t pbase = (is_heat ? ((size_t)n * a.K + cp) * plane : ((size_t)n * (a.n_out - a.K) + (cp - a.K)) * plane) + othread;
            if (is_heat || !a.paf_is_f64) {
                float *of = (is_heat ? im.heat : static_cast<float *>(im.paf)) + pbase;
                if (vec) {
#pragma unroll
                    for (int k = 0; k < 4; k++)
                        if (4 * p2 + k < th) *reinterpret_cast<float4 *>(of + (size_t)k * im.W) = r[k];
                } else {
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        if (4 * p2 + k < th) {
                            const float e[4] = {r[k].x, r[k].y, r[k].z, r[k].w};
#pragma unroll
                            for (int x = 0; x < 4; x++)
                                if (4 * x2 + x < tw) of[(size_t)k * im.W + x] = e[x];
                        }
                    }
                }
            } else {
                double *od = static_cast<double *>(im.paf) + pbase;
                if (vec) {
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        if (4 * p2 + k < th) {
                            double2 *q = reinterpret_cast<double2 *>(od + (size_t)k * im.W);
                            q[0] = make_double2((double)r[k].x, (double)r[k].y);
                            q[1] = make_double2((double)r[k].z, (double)r[k].w);
                        }
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        if (4 * p2 + k < th) {
                            const float e[4] = {r[k].x, r[k].y, r[k].z, r[k].w};
#pragma unroll
                            for (int x = 0; x < 4; x++)
                                if (4 * x2 + x < tw) od[(size_t)k * im.W + x] = (double)e[x];
                        }
                    }
                }
            }
        }
        if (c + 1 < c_end) {
            commit(buf ^ 1);
            if (c + 2 < c_end) prefetch(c + 2);
        }
        __syncthreads();
    }
}

template <bool F16>
__global__ void __launch_bounds__(kPostThreads, 4) postnet_x4_ident_kernel(PostArgs a, PostImage im) {
    postnet_x4_ident_tile<F16>(a, im, blockIdx.x, blockIdx.y, blockIdx.z);
}

// ---------------------------------------------------------------------------------------------------------------
// Ragged batches (predict() for a batch of images of different sizes, with one item or several items -- the
// multi-scale and rotation search -- each): every image has the same items (one product(multiplier, rotate_angle)), so
// a launch covers one group of items -- up to kPostMaxScales fused unrotated items, or one item when any is rotated --
// for many images.  grid.x walks the images' tiles back to back, grid.y the channel chunks (one chunk size per launch).
// The float64 sums of the items in one launch stay in registers (postnet_tile); sums that outlive a launch go through
// each image's own keypoint scratch (PostImage::heat_acc) and its float64 body-part planes.  Each CTA runs the
// per-launch kernel's body on its image's geometry: every image gets exactly the maps spg_postnet_rotated gives it
// alone.  Images per launch: as many descriptors as fit next to PostArgs in the kernel parameters.
constexpr int kPostTableImages = (int)((kParamBytes - sizeof(PostArgs) - 8) / sizeof(PostImage));
struct PostTable {
    int n;                                  // images of this launch
    PostImage img[kPostTableImages];        // first_cta increasing
};
static_assert(sizeof(PostArgs) + sizeof(PostTable) <= kParamBytes, "a launch's parameters fit the kernel-parameter limit");

template <bool F16>
__global__ void __launch_bounds__(kPostThreads, 4) postnet_x4_ident_ragged_kernel(PostArgs a, const __grid_constant__ PostTable r) {
    const PostImage &im = ragged_member(r, blockIdx.x);
    postnet_x4_ident_tile<F16>(a, im, blockIdx.x - im.first_cta, blockIdx.y, 0);
}

// The four-phase body as two kernels, one item per image and fused items, so that spg_stage_kernel's names (the kernels'
// own) tell the two schedules apart.
template <bool F16>
__global__ void __launch_bounds__(kPostThreads, 2) postnet_ragged_kernel(PostArgs a, const __grid_constant__ PostTable r) {
    const PostImage &im = ragged_member(r, blockIdx.x);
    postnet_tile<true, false, F16>(a, im, blockIdx.x - im.first_cta, blockIdx.y, 0);
}

template <bool IDENT, bool F16>
__global__ void __launch_bounds__(kPostThreads, 2) postnet_items_ragged_kernel(PostArgs a, const __grid_constant__ PostTable r) {
    const PostImage &im = ragged_member(r, blockIdx.x);
    postnet_tile<false, IDENT, F16>(a, im, blockIdx.x - im.first_cta, blockIdx.y, 0);
}

template <bool SINGLE, bool F16>
__global__ void __launch_bounds__(kPostThreads, 2) postnet_rot_ragged_kernel(PostArgs a, const __grid_constant__ PostTable r) {
    const PostImage &im = ragged_member(r, blockIdx.x);
    postnet_rot_tile<SINGLE, F16>(a, im, blockIdx.x - im.first_cta, blockIdx.y, 0);
}

}  // namespace spg
