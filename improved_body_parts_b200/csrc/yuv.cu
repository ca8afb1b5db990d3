// yuv.cu -- yuv_to_bgr_kernel (spg_yuv_to_bgr; yuv.cuh describes it) and its launch, a translation unit of its own.
#include "yuv.cuh"

namespace spg {

// OpenCV's ITUR_BT_601_* constants (modules/imgproc/src/color_yuv.simd.hpp), shift 20
constexpr int kYuvCY = 1220542, kYuvCUB = 2116026, kYuvCUG = -409993, kYuvCVG = -852492, kYuvCVR = 1673527;
constexpr int kYuvShift = 20;

__device__ __forceinline__ unsigned char yuv_sat(int v) { return (unsigned char)min(max(v >> kYuvShift, 0), 255); }

// one pixel of luma Y with the chroma terms of its block
__device__ __forceinline__ void yuv_pixel(int Y, int buv, int guv, int ruv, unsigned char *o) {
    const int y = max(0, Y - 16) * kYuvCY;
    o[0] = yuv_sat(y + buv);
    o[1] = yuv_sat(y + guv);
    o[2] = yuv_sat(y + ruv);
}

__global__ void __launch_bounds__(kYuvThreads) yuv_to_bgr_kernel(const __grid_constant__ YuvRagged r) {
    const YuvMember &m = ragged_member(r, (int)blockIdx.x);
    const long long q = (long long)((int)blockIdx.x - m.first_cta) * kYuvThreads + threadIdx.x;
    const bool packed = m.format == SPG_YUV_YUYV;
    if (q >= (long long)(packed ? m.h : m.h / 2) * m.units) return;
    const int by = (int)(q / m.units), bx = (int)(q - (long long)by * m.units);
    int u, v, Y[4];
    if (packed) {
        const unsigned char *p = m.plane[0] + by * m.pitch[0] + 4LL * bx;
        Y[0] = p[0], u = p[1], Y[1] = p[2], v = p[3];
    } else {
        const unsigned char *y0 = m.plane[0] + 2LL * by * m.pitch[0] + 2LL * bx, *y1 = y0 + m.pitch[0];
        Y[0] = y0[0], Y[1] = y0[1], Y[2] = y1[0], Y[3] = y1[1];
        if (m.format == SPG_YUV_NV12) {
            const unsigned char *c = m.plane[1] + by * m.pitch[1] + 2LL * bx;
            u = c[0], v = c[1];
        } else {
            u = m.plane[1][by * m.pitch[1] + bx];
            v = m.plane[2][by * m.pitch[2] + bx];
        }
    }
    const int uu = u - 128, vv = v - 128, half = 1 << (kYuvShift - 1);
    const int ruv = half + kYuvCVR * vv, guv = half + kYuvCVG * vv + kYuvCUG * uu, buv = half + kYuvCUB * uu;
    unsigned char *o = m.out + (packed ? by : 2LL * by) * m.out_pitch + 6LL * bx;
    yuv_pixel(Y[0], buv, guv, ruv, o);
    yuv_pixel(Y[1], buv, guv, ruv, o + 3);
    if (!packed) {
        yuv_pixel(Y[2], buv, guv, ruv, o + m.out_pitch);
        yuv_pixel(Y[3], buv, guv, ruv, o + m.out_pitch + 3);
    }
}

cudaError_t yuv_launch(unsigned grid, cudaStream_t st, const YuvRagged &r) {
    yuv_to_bgr_kernel<<<grid, kYuvThreads, 0, st>>>(r);
    return cudaGetLastError();
}

}  // namespace spg
