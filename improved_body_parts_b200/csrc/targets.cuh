// targets.cuh -- training samples on the device: the reference data server's Transformer.transform and
// Heatmapper.create_heatmaps (py_cocodata_server/py_data_transformer.py:112-184, py_data_heatmapper.py:50-97) for a batch
// of samples of different source sizes and person counts.
//
// targets_warp_kernel: per sample, the uint8 BGR source through cv2.warpAffine(img, M, dsize, INTER_LINEAR,
// BORDER_CONSTANT, border) and the table of np.float32(u8) / 255. into an HWC float32 image; mask_miss and mask_all
// through the same warp (their own border values) and cv2.resize(..., INTER_AREA) by the integer factor `stride`, then the
// table.  OpenCV's uint8 warp is fixed point: the coordinates of warp_linear (warp_coords / warp_tap), then short weights
// 32 * (32 - ay)(32 - ax) ... summing to 2^15, the four taps combined in int (taps outside the source read the border
// value) and (sum + 2^14) >> 15.  INTER_AREA by an integer factor is OpenCV's fast-area arithmetic (area_u8): (box sum
// + 2) >> 2 at stride 2, else rint(float32(box sum) * float32(1 / stride^2)), ties to even.  A mask pixel is the box of
// stride x stride warped pixels it consumes, so the full-size masks are never written.
//
// targets_maps_kernel: per sample the [L + K + 2][h][w] float32 target, every value written once by one thread:
//   body-part channels 0..L-1: the reference's distances() Gaussian of every visible limb (both ends v < 2) whose box
//     covers the pixel, accumulated acc = f32(f64(acc) + g) in person order and averaged in float32;
//   keypoint channels L..L+K-1: the max of outer(exp_y, exp_x) over the visible joints whose window covers the pixel,
//     exp = (float)exp((double)arg) of the float32 argument (DESIGN.md §4: numpy's float32 exp is not correctly rounded);
//   channel L+K: cv2.erode(mask_all, ones(3, 3)) -- the 3x3 min, neighbours outside the map ignored;
//   channel L+K+1: the max over the keypoint channels, recomputed from the joints rather than read back, so the kernel
//     needs no ordering between its CTAs;
//   every channel then clip(0, 1) (NaN kept, as np.clip).
// A CTA owns kTgtThreads consecutive pixels of one channel of one sample.  It walks the sample's joints or limbs in
// chunks of kTgtThreads, one per thread: each computes its window or box as the reference does (f32 division, round
// ties-to-even, the off-map skips and the clip at 0 and at the map), and the ones that reach the CTA's rows are compacted
// into shared memory in person order; every thread then runs its pixel over the list.  Windows are clipped in double
// before any conversion to int, so coordinates up to +-FLT_MAX give empty windows and no overflow.
//
// targets_tint_kernel (below the warp): the colour distortion, in place on the uint8 sources before the warp.
//
// The launches are ragged like prenet.cuh: a member table (one sample each) travels as a __grid_constant__ kernel
// parameter and a CTA finds its member by binary search over first_cta (ragged_member).
#pragma once

#include "interp.cuh"

namespace spg {

constexpr int kTgtThreads = 256;
constexpr int kTgtWarps = kTgtThreads / 32;

// what every member of a launch shares: the spg_target_params of the call, resolved
struct TgtCommon {
    int stride;
    int out_h, out_w;              // warped image rows / columns
    int map_h, map_w;              // out_h / stride, out_w / stride
    int half;                      // gaussian_size / 2
    int border[5];                 // image B, G, R; mask_miss; mask_all
    float kp_ds2;                  // float32(2 sigma^2): the keypoint Gaussian's divisor
    float paf_thre;                // float32(paf_thre)
    double paf_ds2;                // 2 paf_sigma^2
    double limb_thre;              // limb_gaussian_thre
    float lut[256];                // np.float32(u8) / 255.
};

// ---- warp ----------------------------------------------------------------------------------------------------------
struct TgtWarpMember {
    const unsigned char *src, *miss, *all;   // [h][w][3], [h][w], [h][w]
    long long src_stride, mask_stride;       // bytes between rows
    float *img_out, *miss_out, *all_out;     // [out_h][out_w][3], [map_h][map_w] x 2
    double rot[6];                           // the inverse of M: output pixel -> source
    int h, w;
    int img_ctas;                            // CTAs of the image part; the mask part follows
    int first_cta;
};
constexpr int kTgtWarpMax = (int)((kParamBytes - sizeof(TgtCommon) - 8) / sizeof(TgtWarpMember));
struct TgtWarpRagged {
    TgtCommon c;
    int n;
    TgtWarpMember img[kTgtWarpMax];   // first_cta increasing
};
static_assert(sizeof(TgtWarpRagged) <= kParamBytes, "a launch's parameters fit the kernel-parameter limit");

// one channel of warpAffine's uint8 INTER_LINEAR at tap t: int sum of the four taps with weights summing to 2^15
__device__ __forceinline__ int warp_u8(const WarpTap &t, const unsigned char *g, long long pitch, int cs, int w, int h, int border) {
    const bool x0in = t.sx >= 0 && t.sx < w, x1in = t.sx + 1 >= 0 && t.sx + 1 < w;
    const bool y0in = t.sy >= 0 && t.sy < h, y1in = t.sy + 1 >= 0 && t.sy + 1 < h;
    const unsigned char *u = g + (long long)t.sy * pitch + (long long)t.sx * cs;
    const int v00 = (y0in && x0in) ? u[0] : border, v01 = (y0in && x1in) ? u[cs] : border;
    const int v10 = (y1in && x0in) ? u[pitch] : border, v11 = (y1in && x1in) ? u[pitch + cs] : border;
    const int gx = 32 - t.ax, gy = 32 - t.ay;
    const int acc = v00 * (32 * gy * gx) + v01 * (32 * gy * t.ax) + v10 * (32 * t.ay * gx) + v11 * (32 * t.ay * t.ax);
    return (acc + (1 << 14)) >> 15;
}

// cv2.resize(INTER_AREA)'s uint8 value of a box sum s by the integer factor f (f^2 <= 2^24): the 2 x 2 path's
// (s + 2) >> 2 (ties up), else the generic fast-area path's saturate_cast<uchar>(s * (1.f / f^2)) -- an int sum, a float32
// reciprocal and product, rounded ties to even.  The product is not always the correctly rounded quotient (f = 22, 34, ...).
__device__ __forceinline__ int area_u8(int s, int f) {
    if (f == 2) return (s + 2) >> 2;
    const int v = __float2int_rn(__fmul_rn(__int2float_rn(s), __fdiv_rn(1.0f, (float)(f * f))));
    return min(max(v, 0), 255);
}

__global__ void __launch_bounds__(kTgtThreads) targets_warp_kernel(const __grid_constant__ TgtWarpRagged r) {
    const TgtWarpMember &a = ragged_member(r, (int)blockIdx.x);
    const TgtCommon &c = r.c;
    const int cta = (int)blockIdx.x - a.first_cta;
    if (cta < a.img_ctas) {  // one output pixel of the image per thread
        const int p = cta * kTgtThreads + (int)threadIdx.x;
        if (p >= c.out_h * c.out_w) return;
        const int y = p / c.out_w, x = p - y * c.out_w;
        int xs, ys;
        warp_coords(a.rot, x, y, xs, ys);
        const WarpTap t = warp_tap(xs, ys);
        float *o = a.img_out + (long long)p * 3;
#pragma unroll
        for (int ch = 0; ch < 3; ch++) o[ch] = c.lut[warp_u8(t, a.src + ch, a.src_stride, 3, a.w, a.h, c.border[ch])];
        return;
    }
    // one pixel of both masks per thread: the area box of stride x stride warped pixels
    const int p = (cta - a.img_ctas) * kTgtThreads + (int)threadIdx.x;
    if (p >= c.map_h * c.map_w) return;
    const int my = p / c.map_w, mx = p - my * c.map_w;
    int s_miss = 0, s_all = 0;
    for (int dy = 0; dy < c.stride; dy++)
        for (int dx = 0; dx < c.stride; dx++) {
            int xs, ys;
            warp_coords(a.rot, mx * c.stride + dx, my * c.stride + dy, xs, ys);
            const WarpTap t = warp_tap(xs, ys);
            s_miss += warp_u8(t, a.miss, a.mask_stride, 1, a.w, a.h, c.border[3]);
            s_all += warp_u8(t, a.all, a.mask_stride, 1, a.w, a.h, c.border[4]);
        }
    a.miss_out[p] = c.lut[area_u8(s_miss, c.stride)];
    a.all_out[p] = c.lut[area_u8(s_all, c.stride)];
}

// ---- colour distortion -----------------------------------------------------------------------------------------------
// targets_tint_kernel: Transformer.distort_color (py_data_transformer.py:97-110) in place on uint8 BGR sources, before
// targets_warp_kernel reads them.  A separate pass rather than part of the warp's tap reads: the warp stays as it is
// (untinted samples cannot move, its border value stays untinted as in the reference), and the pass costs one read and
// one write of the tinted sources.  Per pixel:
//   cv2.cvtColor(COLOR_BGR2HSV), uint8: integer arithmetic on the 2^12 fixed-point tables sdiv / hdiv (shared memory,
//     computed per CTA: no quotient is a tie, so the integer rounding below is cvRound's);
//   the draws minus (10, 20, 20) added, clamped to [0, 179], [0, 255], [0, 255];
//   cv2.cvtColor(COLOR_HSV2BGR), uint8: float32 with the two fused multiply-adds OpenCV's vector code has (the build has
//     -fmad=false, so only the written __fmaf_rn fuse), then x * 255 truncated -- or rounded to nearest even in the last
//     width % row_block columns of every row, which OpenCV's scalar tail handles (DESIGN.md §4).
// A thread owns kTintPix consecutive pixels of one row: 16-byte accesses when the group's address is 16-byte aligned,
// 4-byte when 4-byte aligned, bytes otherwise (a row's last group, odd pitches).
constexpr int kTintPix = 16;
constexpr int kTintWords = kTintPix * 3 / 4;

struct TgtTintMember {
    unsigned char *image;    // [h][w][3], rows row_stride bytes apart; tinted in place
    long long row_stride;
    int h, w;
    int dh, ds, dv;          // the draws minus 10, 20, 20
    int tail;                // first rounded column: w - w % row_block
    int groups;              // kTintPix-pixel groups per row
    int first_cta;
};
constexpr int kTgtTintMax = (int)((kParamBytes - 16) / sizeof(TgtTintMember));
struct TgtTintRagged {
    int n;
    TgtTintMember img[kTgtTintMax];   // first_cta increasing
};
static_assert(sizeof(TgtTintRagged) <= kParamBytes, "a launch's parameters fit the kernel-parameter limit");

// the HSV -> BGR table entry k of [V, V(1-S), V(1-S hh), V(1-S(1-hh))] without dynamic indexing into registers
__device__ __forceinline__ float tint_pick(int k, float t0, float t1, float t2, float t3) {
    return k == 0 ? t0 : (k == 1 ? t1 : (k == 2 ? t2 : t3));
}

// one pixel (b, g, r) in place
__device__ __forceinline__ void tint_pixel(const int *sdiv, const int *hdiv, const TgtTintMember &a, bool round, int &b, int &g, int &r) {
    int v = max(max(b, g), r);
    const int diff = v - min(min(b, g), r);
    int s = (diff * sdiv[v] + (1 << 11)) >> 12;
    const int vr = -(int)(v == r), vg = -(int)(v == g);
    int h = (vr & (g - b)) + (~vr & ((vg & (b - r + 2 * diff)) + (~vg & (r - g + 4 * diff))));
    h = (h * hdiv[diff] + (1 << 11)) >> 12;
    h += h < 0 ? 180 : 0;
    h = min(max(h + a.dh, 0), 179);
    s = min(max(s + a.ds, 0), 255);
    v = min(max(v + a.dv, 0), 255);
    const float S = __fmul_rn((float)s, 1.f / 255.f), V = __fmul_rn((float)v, 1.f / 255.f);
    float hh = __fmul_rn((float)h, 6.f / 180.f);
    if (hh >= 6.f) hh = __fsub_rn(hh, 6.f);
    const float fl = floorf(hh);
    const int sector = (int)fl;  // 0..5
    hh = __fsub_rn(hh, fl);
    // S == 0 needs no case of its own: every entry is then exactly V
    const float t0 = V, t1 = __fmul_rn(V, __fsub_rn(1.f, S)), t2 = __fmul_rn(V, __fmaf_rn(-S, hh, 1.f)),
                t3 = __fmul_rn(V, __fmaf_rn(-S, __fsub_rn(1.f, hh), 1.f));
    // cv2's sector table {1,3,0},{1,0,2},{3,0,1},{0,2,1},{0,1,3},{2,1,0}, one 2-bit entry per sector and channel
    const int sh = 2 * sector;
    const float fb = __fmul_rn(tint_pick((0x835 >> sh) & 3, t0, t1, t2, t3), 255.f);
    const float fg = __fmul_rn(tint_pick((0x583 >> sh) & 3, t0, t1, t2, t3), 255.f);
    const float fr = __fmul_rn(tint_pick((0x358 >> sh) & 3, t0, t1, t2, t3), 255.f);
    b = min(max(round ? __float2int_rn(fb) : __float2int_rz(fb), 0), 255);
    g = min(max(round ? __float2int_rn(fg) : __float2int_rz(fg), 0), 255);
    r = min(max(round ? __float2int_rn(fr) : __float2int_rz(fr), 0), 255);
}

__global__ void __launch_bounds__(kTgtThreads) targets_tint_kernel(const __grid_constant__ TgtTintRagged r) {
    __shared__ int sdiv[256], hdiv[256];
    for (int i = threadIdx.x; i < 256; i += kTgtThreads) {  // round((255 << 12) / i), round((180 << 12) / (6 i))
        sdiv[i] = i ? (2 * (255 << 12) + i) / (2 * i) : 0;
        hdiv[i] = i ? (2 * (180 << 12) + 6 * i) / (12 * i) : 0;
    }
    __syncthreads();
    const TgtTintMember &a = ragged_member(r, (int)blockIdx.x);
    const long long q = (long long)((int)blockIdx.x - a.first_cta) * kTgtThreads + threadIdx.x;
    if (q >= (long long)a.h * a.groups) return;
    const int y = (int)(q / a.groups), x0 = (int)(q - (long long)y * a.groups) * kTintPix;
    const int np = min(kTintPix, a.w - x0);
    unsigned char *p = a.image + (long long)y * a.row_stride + (long long)x0 * 3;
    const unsigned long long addr = (unsigned long long)p;
    unsigned int wd[kTintWords];
    const bool full = np == kTintPix, v16 = full && (addr & 15) == 0, v4 = full && (addr & 3) == 0;
    if (v16) {
#pragma unroll
        for (int k = 0; k < kTintWords / 4; k++) {
            const uint4 u = reinterpret_cast<const uint4 *>(p)[k];
            wd[4 * k] = u.x; wd[4 * k + 1] = u.y; wd[4 * k + 2] = u.z; wd[4 * k + 3] = u.w;
        }
    } else if (v4) {
#pragma unroll
        for (int k = 0; k < kTintWords; k++) wd[k] = reinterpret_cast<const unsigned int *>(p)[k];
    } else {
#pragma unroll
        for (int k = 0; k < kTintWords; k++) {
            unsigned int u = 0;
#pragma unroll
            for (int j = 0; j < 4; j++) u |= (4 * k + j < 3 * np ? (unsigned int)p[4 * k + j] : 0u) << (8 * j);
            wd[k] = u;
        }
    }
#pragma unroll
    for (int i = 0; i < kTintPix; i++) {
        if (i >= np) continue;
        int c[3];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) c[ch] = (wd[(3 * i + ch) >> 2] >> (8 * ((3 * i + ch) & 3))) & 255;
        tint_pixel(sdiv, hdiv, a, x0 + i >= a.tail, c[0], c[1], c[2]);
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
            const int k = (3 * i + ch) >> 2, sft = 8 * ((3 * i + ch) & 3);
            wd[k] = (wd[k] & ~(255u << sft)) | ((unsigned int)c[ch] << sft);
        }
    }
    if (v16) {
#pragma unroll
        for (int k = 0; k < kTintWords / 4; k++)
            reinterpret_cast<uint4 *>(p)[k] = make_uint4(wd[4 * k], wd[4 * k + 1], wd[4 * k + 2], wd[4 * k + 3]);
    } else if (v4) {
#pragma unroll
        for (int k = 0; k < kTintWords; k++) reinterpret_cast<unsigned int *>(p)[k] = wd[k];
    } else {
#pragma unroll
        for (int k = 0; k < 3 * kTintPix; k++)
            if (k < 3 * np) p[k] = (unsigned char)(wd[k >> 2] >> (8 * (k & 3)));
    }
}

// ---- ground-truth maps ---------------------------------------------------------------------------------------------
struct TgtMapsMember {
    const float *joints;      // [n_persons][K][3] float32 (x, y, v)
    const float *mask_all;    // [map_h][map_w]
    float *labels;            // [L + K + 2][map_h][map_w]
    int n_persons;
    int tiles;                // CTAs per channel: ceil(map_h * map_w / kTgtThreads)
    int first_cta;
};
constexpr int kTgtMapsMax = (int)((kParamBytes - sizeof(TgtCommon) - sizeof(int16_t) * kMaxLimbs * 2 - 32) / sizeof(TgtMapsMember));
struct TgtMapsRagged {
    TgtCommon c;
    int K, L;
    int16_t limbs[kMaxLimbs * 2];     // [L][2] (from, to): the handle's limb table
    int n;
    TgtMapsMember img[kTgtMapsMax];   // first_cta increasing
};
static_assert(sizeof(TgtMapsRagged) <= kParamBytes, "a launch's parameters fit the kernel-parameter limit");

// a window [x0, x1) x [y0, y1) of the map and what the pixels inside it need
struct TgtItem {
    int x0, x1, y0, y1;
    float jx, jy;             // keypoints: the joint; limbs: xD, yD (float32 x2 - x1, y2 - y1)
    double ax, ay, den;       // limbs: x1, y1, norm2 + 1e-6
};

// [lo, hi) clipped to [0, n) in double (no int overflow for any finite input): false when empty.  A NaN bound (a NaN
// joint coordinate) is empty too, as +-inf ones are: fmax / fmin would replace it by the map's edge.
__device__ __forceinline__ bool tgt_clip(double lo, double hi, int n, int &a, int &b) {
    if (isnan(lo) || isnan(hi)) return false;
    lo = fmax(lo, 0.0);
    hi = fmin(hi, (double)n);
    if (!(lo < hi)) return false;
    a = (int)lo;
    b = (int)hi;
    return true;
}

// keypoint window of joint (x, y): round(x / stride) -+ gaussian_size // 2, f32 division, ties to even
__device__ __forceinline__ bool tgt_joint_item(const TgtCommon &c, float x, float y, TgtItem &it) {
    const double rx = (double)rintf(__fdiv_rn(x, (float)c.stride)), ry = (double)rintf(__fdiv_rn(y, (float)c.stride));
    it.jx = x;
    it.jy = y;
    return tgt_clip(rx - c.half, rx + c.half + 1, c.map_w, it.x0, it.x1) && tgt_clip(ry - c.half, ry + c.half + 1, c.map_h, it.y0, it.y1);
}

// body-part box of a limb (x1, y1) -> (x2, y2), and the terms of distances() that do not depend on the pixel
__device__ __forceinline__ bool tgt_limb_item(const TgtCommon &c, float x1, float y1, float x2, float y2, TgtItem &it) {
    const float dx = __fsub_rn(x2, x1), dy = __fsub_rn(y2, y1);
    const float dnorm = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
    if (dnorm == 0.0f) return false;  // the reference prints and skips
    const float s = (float)c.stride;
    const float mnx = x1 < x2 ? x1 : x2, mxx = x1 < x2 ? x2 : x1;
    const float mny = y1 < y2 ? y1 : y2, mxy = y1 < y2 ? y2 : y1;
    const double lx = rintf(__fdiv_rn(__fsub_rn(mnx, c.paf_thre), s)), hx = rintf(__fdiv_rn(__fadd_rn(mxx, c.paf_thre), s));
    const double ly = rintf(__fdiv_rn(__fsub_rn(mny, c.paf_thre), s)), hy = rintf(__fdiv_rn(__fadd_rn(mxy, c.paf_thre), s));
    if (!tgt_clip(lx, hx + 1, c.map_w, it.x0, it.x1) || !tgt_clip(ly, hy + 1, c.map_h, it.y0, it.y1)) return false;
    it.jx = dx;
    it.jy = dy;
    it.ax = (double)x1;
    it.ay = (double)y1;
    it.den = __dadd_rn(__dsqrt_rn((double)dnorm), 1e-6);
    return true;
}

// distances(): the limb's Gaussian at the grid point (X, Y), then the <= thresh -> 0.01 floor
__device__ __forceinline__ double tgt_limb_value(const TgtCommon &c, const TgtItem &it, double X, double Y) {
    const double detaX = __dsub_rn(it.ax, X), detaY = __dsub_rn(it.ay, Y);
    double d = __dsub_rn(__dmul_rn((double)it.jx, detaY), __dmul_rn(detaX, (double)it.jy));
    d = fabs(__ddiv_rn(d, it.den));
    const double g = exp(__ddiv_rn(-__dmul_rn(d, d), c.paf_ds2));
    return g <= c.limb_thre ? 0.01 : g;
}

// exp(-((grid - x)^2) / 2 sigma^2) of one axis, float32 argument, exp in double rounded once to float32
__device__ __forceinline__ float tgt_kp_axis(const TgtCommon &c, int i, float x) {
    const float g = (float)(i * c.stride) + (0.5f * (float)c.stride - 0.5f);  // i * stride + stride / 2 - 0.5, exact
    const float d = __fsub_rn(g, x);
    return __double2float_rn(exp((double)__fdiv_rn(-__fmul_rn(d, d), c.kp_ds2)));
}

__global__ void __launch_bounds__(kTgtThreads) targets_maps_kernel(const __grid_constant__ TgtMapsRagged r) {
    __shared__ TgtItem list[kTgtThreads];
    __shared__ int warp_count[kTgtWarps];
    const TgtMapsMember &a = ragged_member(r, (int)blockIdx.x);
    const TgtCommon &c = r.c;
    const int K = r.K, L = r.L;
    const int cta = (int)blockIdx.x - a.first_cta;
    const int ch = cta / a.tiles, tile = cta - ch * a.tiles;
    const int n_pix = c.map_h * c.map_w;
    const int p = tile * kTgtThreads + (int)threadIdx.x;
    const bool live = p < n_pix;
    const int py = live ? p / c.map_w : 0, px = live ? p - py * c.map_w : 0;
    float *out = a.labels + (long long)ch * n_pix;

    if (ch == L + K) {  // cv2.erode(mask_all, ones(3, 3)): out-of-map neighbours are ignored
        if (!live) return;
        float m = a.mask_all[p];
        for (int yy = max(py - 1, 0); yy <= min(py + 1, c.map_h - 1); yy++)
            for (int xx = max(px - 1, 0); xx <= min(px + 1, c.map_w - 1); xx++) m = fminf(m, a.mask_all[yy * c.map_w + xx]);
        out[p] = m < 0.0f ? 0.0f : (m > 1.0f ? 1.0f : m);
        return;
    }

    // the rows this CTA's pixels span: items are kept when their window reaches them
    const int row_lo = (tile * kTgtThreads) / c.map_w, row_hi = min((tile * kTgtThreads + kTgtThreads - 1) / c.map_w, c.map_h - 1);
    const bool limb = ch < L;
    const int fr = limb ? r.limbs[2 * ch] : 0, to = limb ? r.limbs[2 * ch + 1] : 0;
    const int n_items = ch == L + K + 1 ? a.n_persons * K : a.n_persons;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double X = (double)(px * c.stride) + (0.5 * c.stride - 0.5), Y = (double)(py * c.stride) + (0.5 * c.stride - 0.5);
    float kp = 0.0f, acc = 0.0f, cnt = 0.0f;

    for (int base = 0; base < n_items; base += kTgtThreads) {
        const int i = base + (int)threadIdx.x;
        TgtItem it;
        bool keep = false;
        if (i < n_items) {
            if (limb) {
                const float *f = a.joints + ((long long)i * K + fr) * 3, *t = a.joints + ((long long)i * K + to) * 3;
                if (f[2] < 2.0f && t[2] < 2.0f) keep = tgt_limb_item(c, f[0], f[1], t[0], t[1], it);
            } else {
                const int part = ch == L + K + 1 ? i % K : ch - L, person = ch == L + K + 1 ? i / K : i;
                const float *j = a.joints + ((long long)person * K + part) * 3;
                if (j[2] < 2.0f) keep = tgt_joint_item(c, j[0], j[1], it);
            }
            keep = keep && it.y1 > row_lo && it.y0 <= row_hi;
        }
        // ordered compaction: the kept items of the chunk in item (= person) order
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_count[warp] = __popc(b);
        __syncthreads();
        int off = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kTgtWarps; w++) {
            off += w < warp ? warp_count[w] : 0;
            total += warp_count[w];
        }
        if (keep) list[off + __popc(b & ((1u << lane) - 1u))] = it;
        __syncthreads();
        if (live) {
            for (int k = 0; k < total; k++) {
                const TgtItem &q = list[k];
                if (px < q.x0 || px >= q.x1 || py < q.y0 || py >= q.y1) continue;
                if (limb) {
                    acc = __double2float_rn(__dadd_rn((double)acc, tgt_limb_value(c, q, X, Y)));
                    cnt = __fadd_rn(cnt, 1.0f);
                } else {
                    kp = fmaxf(kp, __fmul_rn(tgt_kp_axis(c, py, q.jy), tgt_kp_axis(c, px, q.jx)));
                }
            }
        }
        __syncthreads();
    }
    if (!live) return;
    float v = limb ? (cnt > 0.0f ? __fdiv_rn(acc, cnt) : acc) : kp;
    out[p] = v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v);
}

}  // namespace spg
