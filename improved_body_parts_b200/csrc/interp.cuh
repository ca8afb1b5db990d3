// interp.cuh -- OpenCV's interpolation arithmetic shared by the pre-network (prenet.cuh), post-network (postnet.cuh) and
// training-sample (targets.cuh) kernels: the bicubic coefficients of cv2.resize and the fixed-point taps of
// cv2.warpAffine's INTER_LINEAR.  Every product and sum is rounded as OpenCV rounds it (the translation unit is built with
// -fmad=false).
#pragma once

#include "common.cuh"

namespace spg {

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

// interpolateCubic (imgproc/src/resize.cpp), float32, exactly oracle/postnet_port.py::cubic_coeffs
__device__ __forceinline__ void cubic_coeffs(float x, float c[4]) {
    const float A = -0.75f;
    const float x1 = __fadd_rn(x, 1.0f);
    c[0] = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x1), __fmul_rn(5.0f, A)), x1), __fmul_rn(8.0f, A)), x1), __fmul_rn(4.0f, A));
    const float a2 = __fadd_rn(A, 2.0f), a3 = __fadd_rn(A, 3.0f);
    c[1] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(a2, x), a3), x), x), 1.0f);
    const float y = __fsub_rn(1.0f, x);
    c[2] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(a2, y), a3), y), y), 1.0f);
    c[3] = __fsub_rn(__fsub_rn(__fsub_rn(1.0f, c[0]), c[1]), c[2]);
}

// destination index d of an axis -> first tap (s - 1, unclamped) and the four weights
__device__ __forceinline__ int axis_entry(int d, double scale, float c[4]) {
    const float f = (float)__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5);  // fx = (float)((dx+0.5)*scale_x - 0.5)
    const float fl = floorf(f);
    cubic_coeffs(__fsub_rn(f, fl), c);
    return (int)fl - 1;
}

// One destination pixel of warpAffine's INTER_LINEAR (imgproc/src/imgwarp.cpp) on a w x h grid: (xs, ys) are its source
// coordinates in OpenCV's fixed point, X0 + adelta and Y0 + bdelta (1/1024 px, the +16 rounding term included).  The grid's
// value (y, x) is val(g[(y - y0) * pitch + (x - x0) * CS]); taps outside the grid read 0 (BORDER_CONSTANT) and are never
// loaded.  Every product and sum is rounded to float32, left to right.  Shared by the inverse warp of the maps
// (postnet_rot_kernel) and the forward warp of the input image (prenet.cuh).
// (xs, ys) -> the top-left tap (sx, sy) and the 1/32 px fractions (ax, ay) of warpAffine's INTER_TAB_SIZE table; shared
// with the uint8 tap combine of the training-sample warp (targets.cuh)
struct WarpTap {
    int sx, sy, ax, ay;
};
__device__ __forceinline__ WarpTap warp_tap(int xs, int ys) {
    const int xf = xs >> 5, yf = ys >> 5;
    return {clampi(xf >> 5, -32768, 32767), clampi(yf >> 5, -32768, 32767), xf & 31, yf & 31};  // saturate_cast<short>
}
// warpAffine's fixed-point source coordinates (X0 + adelta, Y0 + bdelta, the +16 rounding term included) of destination
// pixel (x, y) under the inverted matrix m (rounded ties-to-even like cvRound)
__device__ __forceinline__ void warp_coords(const double m[6], int x, int y, int &xs, int &ys) {
    const double xd = (double)x, yd = (double)y;
    xs = __double2int_rn(__dmul_rn(__dmul_rn(m[0], xd), 1024.0)) + __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], yd), m[2]), 1024.0)) + 16;
    ys = __double2int_rn(__dmul_rn(__dmul_rn(m[3], xd), 1024.0)) + __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], yd), m[5]), 1024.0)) + 16;
}
template <int CS, typename T, typename Val>
__device__ __forceinline__ float warp_linear(int xs, int ys, int w, int h, const T *g, int pitch, int x0, int y0, const Val &val) {
    const WarpTap t = warp_tap(xs, ys);
    const int sx = t.sx, sy = t.sy;
    const float fx = __fmul_rn((float)t.ax, 0.03125f), fy = __fmul_rn((float)t.ay, 0.03125f);
    const float gx = __fsub_rn(1.0f, fx), gy = __fsub_rn(1.0f, fy);
    const bool x0in = sx >= 0 && sx < w, x1in = sx + 1 >= 0 && sx + 1 < w;
    const bool y0in = sy >= 0 && sy < h, y1in = sy + 1 >= 0 && sy + 1 < h;
    const T *u = g + (sy - y0) * pitch + (sx - x0) * CS;
    const float t00 = (y0in && x0in) ? val(u[0]) : 0.0f, t01 = (y0in && x1in) ? val(u[CS]) : 0.0f;
    const float t10 = (y1in && x0in) ? val(u[pitch]) : 0.0f, t11 = (y1in && x1in) ? val(u[pitch + CS]) : 0.0f;
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(t00, __fmul_rn(gy, gx)), __fmul_rn(t01, __fmul_rn(gy, fx))),
                               __fmul_rn(t10, __fmul_rn(fy, gx))), __fmul_rn(t11, __fmul_rn(fy, fx)));
}

}  // namespace spg
