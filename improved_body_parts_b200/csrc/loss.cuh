// loss.cuh -- the training loss on the device: the reference's MultiTaskLoss (models/loss_model.py:22-81, 133-161: the
// multi-scale focal L2 with gamma = 1, alpha = beta = 0) and MultiTaskLossParallel's L2 (models/loss_model_parallel.py:
// 19-75, 120-139), forward and gradient, for nstack <= 8 stacks x 5 scales of predictions.
//
// Ground truth of scale j (the predictions' scale j is (H >> j) x (W >> j) of the H x W targets):
//   labels: F.adaptive_avg_pool2d -- CUDA torch's row-major sequential float32 sum over the 2^j x 2^j window, then
//     `sum / kH / kW` (not a hierarchical 2 x 2 pyramid: that gives other bits);
//   mask:   F.interpolate(bilinear, align_corners=False) -- the identity at j = 0; for j >= 1 every weight is exactly 0.5
//     and CUDA torch combines the four taps as 0.5 (0.5 a + 0.5 b) + 0.5 (0.5 c + 0.5 d).  Focal: then `< 0.5 -> 0`,
//     times w_bkg on channel C - 2 and times w_heat on channels heat_start..bkg_start-1.  L2: the raw interpolation.
// Per element, s the prediction (as float32), gt, m the mask above, d = s - gt:
//   focal: st = gt >= 0.01f ? s : 1 - s, u = 1 - st, factor = |u|, term = ((d d) factor) m
//   l2:    term = (d d) m
// and its gradient, autograd's chain in float32: gA = G m; pa = (gA factor) (2 d); pb = (gA (d d)) sign(u), negated
// when st = s; grad = pa + pb (l2: grad = gA (2 d)).  G of (scale j, stack k) is autograd's chain outermost first,
// ((((g / B) / sum_sw) sw_j) / sum_nw) nw_k, where CUDA torch divides by a host scalar b as a multiply by
// (float)(1.0 / b).  Built with -fmad=false like the rest of the library: no contraction can move a bit.
//
// One CTA per (sample, channel, band of kLossBand scale-0 rows): it stages the band's labels and mask in shared memory,
// builds both pyramids there (scale j's band is kLossBand >> j rows), then streams the band's pixels of all nstack x 5
// prediction tensors: thread t owns the groups of kLossVec consecutive elements t, t + kLossThreads, ... of a band, read
// with one vector access when the tensor's rows allow it, so the order of a thread's sum never depends on alignment.
//   loss_forward_kernel:  per (scale, stack) a float64 sum of the float32 terms per thread, reduced over the CTA in a
//     fixed order into one partial per CTA; the last CTA to finish (a ticket the caller owns, reset by that CTA) adds the
//     partials in a fixed order, rounds each sum to float32 and combines them into the loss in the reference's order of
//     float32 operations.  Nothing depends on the SM count: the bits repeat from run to run and from card to card.
//   loss_backward_kernel: every prediction's gradient written once, recomputed from the inputs and *grad_output (a
//     device scalar): no state from the forward.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace spg {

constexpr int kLossThreads = 256;
constexpr int kLossWarps = kLossThreads / 32;
constexpr int kLossBand = 16;       // scale-0 rows per CTA: the coarsest scale's pooling window
constexpr int kLossScales = 5;
constexpr int kLossMaxStacks = 8;
constexpr int kLossSlots = kLossScales * kLossMaxStacks;
constexpr int kLossVec = 4;         // elements per group: 16 bytes of float32, 8 of bfloat16 / float16

struct LossPred {
    const void *data;               // [B][>= C][H >> j][W >> j], unit column stride
    void *grad;                     // backward only
    long long bs, cs, rs;           // data strides in elements
    long long gbs, gcs, grs;        // grad strides in elements
    int vec;                        // rows of data (and grad) take kLossVec-element vector accesses
};

struct LossArgs {
    const float *labels;            // [B][C][H][W]
    const float *mask;              // [B][1][H][W]
    float *sums;                    // forward: [5][nstack]
    float *loss;                    // forward: the scalar
    double *partial;                // forward: [5 * nstack][gridDim.x], the call's own
    unsigned int *ticket;           // forward: CTAs done, the call's own; 0 on entry, left 0 by the last CTA
    const float *grad_output;       // backward
    int focal, nstack, B, C, H, W, heat_start, bkg_start, bands;
    float w_bkg, w_heat;            // channel C - 2; channels heat_start..bkg_start-1
    float nw[kLossMaxStacks], sw[kLossScales];
    float inv_batch, inv_sw, inv_nw;  // float32 reciprocals of the batch divisor, sum(sw), sum(nw)
    LossPred pred[kLossSlots];      // [k * 5 + j]: pred_tuple[k][j]
};

__host__ __device__ constexpr int loss_level_offset(int W, int j) {  // floats before level j of a staged pyramid
    return j == 0 ? 0 : loss_level_offset(W, j - 1) + (kLossBand >> (j - 1)) * (W >> (j - 1));
}
// floats of one staged pyramid, rounded up to 16 bytes so that the mask's pyramid after it takes float4 stores
__host__ __device__ constexpr int loss_pyramid_floats(int W) { return (loss_level_offset(W, kLossScales) + 3) & ~3; }
__host__ __device__ constexpr size_t loss_smem_bytes(int W) { return 2 * sizeof(float) * (size_t)loss_pyramid_floats(W); }

__device__ __forceinline__ float loss_ld(const float *p) { return *p; }
__device__ __forceinline__ float loss_ld(const __nv_bfloat16 *p) { return __bfloat162float(*p); }
__device__ __forceinline__ float loss_ld(const __half *p) { return __half2float(*p); }
__device__ __forceinline__ void loss_st(float *p, float v) { *p = v; }
__device__ __forceinline__ void loss_st(__nv_bfloat16 *p, float v) { *p = __float2bfloat16_rn(v); }
__device__ __forceinline__ void loss_st(__half *p, float v) { *p = __float2half_rn(v); }
// kLossVec elements at once: one 16-byte access of float32, one 8-byte access of two packed pairs otherwise
__device__ __forceinline__ void loss_ld4(const float *p, float *v) {
    const float4 q = *reinterpret_cast<const float4 *>(p);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
}
__device__ __forceinline__ void loss_st4(float *p, const float *v) { *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]); }
template <typename T2, typename T>
__device__ __forceinline__ void loss_ld4_pairs(const T *p, float *v) {
    const uint2 q = *reinterpret_cast<const uint2 *>(p);
    T2 lo, hi;
    memcpy(&lo, &q.x, 4);
    memcpy(&hi, &q.y, 4);
    v[0] = loss_ld(&lo.x); v[1] = loss_ld(&lo.y); v[2] = loss_ld(&hi.x); v[3] = loss_ld(&hi.y);
}
__device__ __forceinline__ void loss_ld4(const __nv_bfloat16 *p, float *v) { loss_ld4_pairs<__nv_bfloat162>(p, v); }
__device__ __forceinline__ void loss_ld4(const __half *p, float *v) { loss_ld4_pairs<__half2>(p, v); }
__device__ __forceinline__ void loss_st4(__nv_bfloat16 *p, const float *v) {
    const __nv_bfloat162 lo = __floats2bfloat162_rn(v[0], v[1]), hi = __floats2bfloat162_rn(v[2], v[3]);
    uint2 q;
    memcpy(&q.x, &lo, 4);
    memcpy(&q.y, &hi, 4);
    *reinterpret_cast<uint2 *>(p) = q;
}
__device__ __forceinline__ void loss_st4(__half *p, const float *v) {
    const __half2 lo = __floats2half2_rn(v[0], v[1]), hi = __floats2half2_rn(v[2], v[3]);
    uint2 q;
    memcpy(&q.x, &lo, 4);
    memcpy(&q.y, &hi, 4);
    *reinterpret_cast<uint2 *>(p) = q;
}

// scale j >= 1 of both pyramids at pixel p of the band, from scale 0
template <int J>
__device__ __forceinline__ void loss_pool(float *gt, float *mk, int W, int p) {
    constexpr int K = 1 << J;
    const int Wj = W >> J, y = p / Wj, x = p - y * Wj;
    const float *g = gt + y * K * W + x * K;
    float s = 0.0f;
#pragma unroll
    for (int r = 0; r < K; r++)
#pragma unroll
        for (int q = 0; q < K; q++) s = __fadd_rn(s, g[r * W + q]);
    gt[loss_level_offset(W, J) + p] = __fdiv_rn(__fdiv_rn(s, (float)K), (float)K);
    const float *m = mk + (y * K + K / 2 - 1) * W + x * K + K / 2 - 1;
    const float top = __fadd_rn(__fmul_rn(0.5f, m[0]), __fmul_rn(0.5f, m[1]));
    const float bot = __fadd_rn(__fmul_rn(0.5f, m[W]), __fmul_rn(0.5f, m[W + 1]));
    mk[loss_level_offset(W, J) + p] = __fadd_rn(__fmul_rn(0.5f, top), __fmul_rn(0.5f, bot));
}

// the CTA's (sample, channel, band); stages and builds both pyramids, the mask thresholded and weighted for the channel
__device__ __forceinline__ void loss_stage(const LossArgs &a, float *gt, float *mk, int &b, int &c, int &band) {
    band = (int)(blockIdx.x % (unsigned)a.bands);
    c = (int)((blockIdx.x / (unsigned)a.bands) % (unsigned)a.C);
    b = (int)(blockIdx.x / ((unsigned)a.bands * (unsigned)a.C));
    const int W = a.W, n0 = kLossBand * W / 4;
    const float4 *lab = reinterpret_cast<const float4 *>(a.labels + (((long long)b * a.C + c) * a.H + (long long)band * kLossBand) * W);
    const float4 *msk = reinterpret_cast<const float4 *>(a.mask + ((long long)b * a.H + (long long)band * kLossBand) * W);
    for (int i = threadIdx.x; i < n0; i += kLossThreads) {
        reinterpret_cast<float4 *>(gt)[i] = lab[i];
        reinterpret_cast<float4 *>(mk)[i] = msk[i];
    }
    __syncthreads();
    // the coarsest level's long sums first, so that they start with the CTA
    const int n4 = W >> 4, n3 = 2 * (W >> 3), n2 = 4 * (W >> 2), n1 = 8 * (W >> 1);
    for (int q = threadIdx.x; q < n4 + n3 + n2 + n1; q += kLossThreads) {
        if (q < n4) loss_pool<4>(gt, mk, W, q);
        else if (q < n4 + n3) loss_pool<3>(gt, mk, W, q - n4);
        else if (q < n4 + n3 + n2) loss_pool<2>(gt, mk, W, q - n4 - n3);
        else loss_pool<1>(gt, mk, W, q - n4 - n3 - n2);
    }
    __syncthreads();
    if (a.focal) {
        const bool bkg = c == a.C - 2, heat = c >= a.heat_start && c < a.bkg_start;
        for (int i = threadIdx.x; i < loss_level_offset(W, kLossScales); i += kLossThreads) {
            float m = mk[i] < 0.5f ? 0.0f : mk[i];
            if (bkg) m = __fmul_rn(m, a.w_bkg);
            if (heat) m = __fmul_rn(m, a.w_heat);
            mk[i] = m;
        }
        __syncthreads();
    }
}

__device__ __forceinline__ float loss_term(bool focal, float s, float gt, float m) {
    const float d = __fsub_rn(s, gt), d2 = __fmul_rn(d, d);
    if (!focal) return __fmul_rn(d2, m);
    const float st = gt >= 0.01f ? s : __fsub_rn(1.0f, s);
    return __fmul_rn(__fmul_rn(d2, fabsf(__fsub_rn(1.0f, st))), m);
}

__device__ __forceinline__ float loss_grad(bool focal, float s, float gt, float m, float G) {
    const float d = __fsub_rn(s, gt), gA = __fmul_rn(G, m), d2x = __fmul_rn(2.0f, d);
    if (!focal) return __fmul_rn(gA, d2x);
    const bool pos = gt >= 0.01f;
    const float u = __fsub_rn(1.0f, pos ? s : __fsub_rn(1.0f, s));
    const float pa = __fmul_rn(__fmul_rn(gA, fabsf(u)), d2x);
    const float sgn = u > 0.0f ? 1.0f : (u < 0.0f ? -1.0f : 0.0f);
    const float pb = __fmul_rn(__fmul_rn(gA, __fmul_rn(d, d)), sgn);
    return __fadd_rn(pa, pos ? -pb : pb);
}

// one band of one prediction tensor (scale j): forward returns this thread's float64 sum, backward writes the gradient
template <typename T, bool BWD>
__device__ __forceinline__ double loss_band(const LossArgs &a, const LossPred &p, int j, int b, int c, int band,
                                            const float *gt, const float *mk, float G) {
    const int Wj = a.W >> j, rows = kLossBand >> j, n = rows * Wj;
    const long long y0 = (long long)band * rows;
    const T *src = static_cast<const T *>(p.data) + b * p.bs + c * p.cs + y0 * p.rs;
    T *dst = BWD ? static_cast<T *>(p.grad) + b * p.gbs + c * p.gcs + y0 * p.grs : nullptr;
    gt += loss_level_offset(a.W, j);
    mk += loss_level_offset(a.W, j);
    const bool focal = a.focal != 0;
    double acc = 0.0;
    for (int e0 = kLossVec * (int)threadIdx.x; e0 < n; e0 += kLossVec * kLossThreads) {
        float s[kLossVec], out[kLossVec];
        if (p.vec) {  // Wj % kLossVec == 0: the group is one aligned piece of one row
            const int r = e0 / Wj;
            loss_ld4(src + r * p.rs + (e0 - r * Wj), s);
        } else {
#pragma unroll
            for (int i = 0; i < kLossVec; i++) {
                const int e = e0 + i, r = e / Wj;
                s[i] = e < n ? loss_ld(src + r * p.rs + (e - r * Wj)) : 0.0f;
            }
        }
#pragma unroll
        for (int i = 0; i < kLossVec; i++) {
            if (e0 + i >= n) break;
            if (BWD) out[i] = loss_grad(focal, s[i], gt[e0 + i], mk[e0 + i], G);
            else acc = __dadd_rn(acc, (double)loss_term(focal, s[i], gt[e0 + i], mk[e0 + i]));
        }
        if (BWD) {
            if (p.vec) {
                const int r = e0 / Wj;
                loss_st4(dst + r * p.grs + (e0 - r * Wj), out);
            } else {
#pragma unroll
                for (int i = 0; i < kLossVec; i++) {
                    const int e = e0 + i, r = e / Wj;
                    if (e < n) loss_st(dst + r * p.grs + (e - r * Wj), out[i]);
                }
            }
        }
    }
    return acc;
}

// lane 0 gets the warp's sum, in a fixed order
__device__ __forceinline__ double loss_warp_sum(double v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, off));
    return v;
}

template <typename T>
__global__ void __launch_bounds__(kLossThreads) loss_forward_kernel(const __grid_constant__ LossArgs a) {
    extern __shared__ float4 loss_smem[];
    __shared__ double red[kLossSlots][kLossWarps];
    __shared__ int last;
    float *gt = reinterpret_cast<float *>(loss_smem), *mk = gt + loss_pyramid_floats(a.W);
    int b, c, band;
    loss_stage(a, gt, mk, b, c, band);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nsum = kLossScales * a.nstack;
    for (int j = 0; j < kLossScales; j++)
        for (int k = 0; k < a.nstack; k++) {
            const double v = loss_warp_sum(loss_band<T, false>(a, a.pred[k * kLossScales + j], j, b, c, band, gt, mk, 0.0f));
            if (lane == 0) red[j * a.nstack + k][warp] = v;
        }
    __syncthreads();
    const unsigned ctas = gridDim.x;
    if ((int)threadIdx.x < nsum) {
        double s = 0.0;
        for (int w = 0; w < kLossWarps; w++) s = __dadd_rn(s, red[threadIdx.x][w]);
        a.partial[(size_t)threadIdx.x * ctas + blockIdx.x] = s;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(a.ticket, 1u) == ctas - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    // the last CTA: every sum over the CTAs in a fixed order
    for (int q = 0; q < nsum; q++) {
        double v = 0.0;
        for (unsigned i = threadIdx.x; i < ctas; i += kLossThreads) v = __dadd_rn(v, __ldcg(a.partial + (size_t)q * ctas + i));
        v = loss_warp_sum(v);
        if (lane == 0) red[q][warp] = v;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    // the reference's float32 combination: Python sum() from 0 over the stacks and then the scales
    float total = 0.0f;
    for (int j = 0; j < kLossScales; j++) {
        float acc = 0.0f;
        for (int k = 0; k < a.nstack; k++) {
            double s = 0.0;
            for (int w = 0; w < kLossWarps; w++) s = __dadd_rn(s, red[j * a.nstack + k][w]);
            const float f = __double2float_rn(s);
            a.sums[j * a.nstack + k] = f;
            acc = __fadd_rn(acc, __fmul_rn(f, a.nw[k]));
        }
        total = __fadd_rn(total, __fmul_rn(__fmul_rn(acc, a.inv_nw), a.sw[j]));
    }
    a.loss[0] = __fmul_rn(__fmul_rn(total, a.inv_sw), a.inv_batch);
    *a.ticket = 0u;
}

template <typename T>
__global__ void __launch_bounds__(kLossThreads) loss_backward_kernel(const __grid_constant__ LossArgs a) {
    extern __shared__ float4 loss_smem[];
    float *gt = reinterpret_cast<float *>(loss_smem), *mk = gt + loss_pyramid_floats(a.W);
    int b, c, band;
    loss_stage(a, gt, mk, b, c, band);
    const float g = __fmul_rn(__fmul_rn(*a.grad_output, a.inv_batch), a.inv_sw);
    for (int j = 0; j < kLossScales; j++) {
        const float gj = __fmul_rn(__fmul_rn(g, a.sw[j]), a.inv_nw);
        for (int k = 0; k < a.nstack; k++)
            loss_band<T, true>(a, a.pred[k * kLossScales + j], j, b, c, band, gt, mk, __fmul_rn(gj, a.nw[k]));
    }
}

}  // namespace spg
