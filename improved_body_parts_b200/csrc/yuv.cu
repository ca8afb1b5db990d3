// yuv.cu -- spg_yuv_to_bgr and its kernel, yuv_to_bgr_kernel (yuv.cuh describes it).
#include "runtime.cuh"

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

}  // namespace spg

using namespace spg;

extern "C" {

int spg_yuv_to_bgr(spg_handle *h, const spg_yuv_member *members, int32_t n, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (n < 0 || (n > 0 && !members)) return fail(h, SPG_E_INVALID, "members is NULL or n negative");
    std::vector<YuvMember> ms((size_t)n);
    std::vector<long long> ctas((size_t)n);
    for (int i = 0; i < n; i++) {  // validate every member before the first launch
        const spg_yuv_member &s = members[i];
        const int H = s.height, W = s.width, f = s.format;
        if (f != SPG_YUV_NV12 && f != SPG_YUV_I420 && f != SPG_YUV_YUYV)
            return fail(h, SPG_E_INVALID, "member %d: format %d is not SPG_YUV_NV12, SPG_YUV_I420 or SPG_YUV_YUYV", i, f);
        if (s.reserved != 0) return fail(h, SPG_E_INVALID, "member %d: reserved must be 0", i);
        if (H < 1 || W < 1 || H > 32767 || W > 32767) return fail(h, SPG_E_INVALID, "member %d: frame %dx%d outside [1, 32767]", i, H, W);
        if (W % 2 != 0 || (f != SPG_YUV_YUYV && H % 2 != 0))
            return fail(h, SPG_E_INVALID, "member %d: a %s frame needs an even %s (got %dx%d)", i, f == SPG_YUV_YUYV ? "YUYV" : "4:2:0",
                        f == SPG_YUV_YUYV ? "width" : "height and width", H, W);
        const int n_planes = f == SPG_YUV_NV12 ? 2 : (f == SPG_YUV_I420 ? 3 : 1);
        const long long row[3] = {f == SPG_YUV_YUYV ? 2LL * W : W, f == SPG_YUV_NV12 ? W : W / 2, W / 2};
        YuvMember m{};
        for (int k = 0; k < n_planes; k++) {
            if (!s.planes[k]) return fail(h, SPG_E_INVALID, "member %d: plane %d is NULL", i, k);
            if (s.pitches[k] < row[k])
                return fail(h, SPG_E_INVALID, "member %d: plane %d's pitch %lld is below its row's %lld bytes", i, k,
                            (long long)s.pitches[k], row[k]);
            m.plane[k] = s.planes[k];
            m.pitch[k] = s.pitches[k];
        }
        if (!s.out) return fail(h, SPG_E_INVALID, "member %d: out is NULL", i);
        if (s.out_pitch < 3LL * W)
            return fail(h, SPG_E_INVALID, "member %d: out_pitch %lld is below the row's %lld bytes", i, (long long)s.out_pitch, 3LL * W);
        m.out = s.out;
        m.out_pitch = s.out_pitch;
        m.format = f;
        m.h = H;
        m.w = W;
        m.units = W / 2;
        ms[i] = m;
        ctas[i] = ((long long)(f == SPG_YUV_YUYV ? H : H / 2) * m.units + kYuvThreads - 1) / kYuvThreads;
    }
    if (ms.empty()) return SPG_OK;
    std::vector<RaggedRange> ranges;
    std::vector<int> first;
    int rc;
    if ((rc = deal_ragged(h, ctas, kYuvTableMax, "member", nullptr, ranges, first))) return rc;
    DeviceGuard guard(h->device);
    YuvRagged table{};
    for (const RaggedRange &g : ranges) {
        fill_table(table, ms, first, g);
        if ((rc = launch(h, kStageYuv, "yuv_to_bgr_kernel", yuv_to_bgr_kernel, dim3(g.ctas), kYuvThreads, 0,
                         static_cast<cudaStream_t>(stream), table)))
            return rc;
    }
    return SPG_OK;
}

}  // extern "C"
