// prenet.cuh -- the input side of predict() (the pre-network stage): per (scale, angle) item, the [2][Hp][Wp][3] float32
// pair the network receives, from the uint8 BGR image.
//
// Replaces the body of the item loop of predict() before the forward pass, the reference's evaluate.py:98-121:
//   cv2.resize(image, (0, 0), fx=scale, fy=scale, INTER_CUBIC)           (:98)
//   util.padRightDownCorner(..., max_downsample, padValue)                (:99-100)
//   np.float32(padded / 255)                                              (:105)
//   angle != 0: cv2.warpAffine(input_img, rotate_matrix, (0, 0))         (:108-111; INTER_LINEAR, BORDER_CONSTANT 0)
//   the image and its mirror, concatenated                                (:116-119)
//
// Arithmetic: OpenCV's generic uint8 bicubic path as restated by oracle/prenet_port.py::resize_cubic_u8 (the IPP build
// in the reference's wheels differs from it by at most 1 LSB in some pixels; DESIGN.md §4): float32 coefficients at
// (d + 0.5) / fx - 0.5 converted to short as rint(c * 2048), taps clamped to the image, an exact integer horizontal pass,
// and a vertical pass that is float32 without contraction (S0*b0 + (S1*b1 + (S2*b2 + S3*b3)), b = beta * 2^-22, rounded
// ties-to-even) on the first (W1 * 3) / 8 * 8 values of an interleaved row -- VResizeCubicVec_32s8u's 8-lane groups -- and
// the integer (sum S*beta + 2^21) >> 22 on the rest.  A resize to the source's own size is a copy.  The byte -> float
// conversion is a table of the float32 roundings of i / 255 in double; the warp is warp_linear, the fixed-point tap of
// postnet_rot_kernel, on the padded grid (taps outside it read 0, not the pad value).  The pair is bit-identical to the
// port's (tests/test_gpu_prenet.py).
//
// The stage is ragged: a launch covers many members -- one (scale, angle) item of one source image each -- whose
// sources and padded sizes may all differ.  Each member has a descriptor (PreMember) in a table that travels as the
// kernel parameter; grid.x walks each member's CTAs (one per kPreThreads pixels of one padded row) back to back, and a
// CTA finds its member by binary search over the table's first_cta (ragged_member).  A CTA belongs to one member.
// Unrotated members are one launch of prenet_kernel<false>: a thread computes one padded pixel straight from the source
// and stores it to the image and to the mirror.  Rotated members first write their padded uint8 images to the handle's
// scratch grid (prenet_resize_kernel); prenet_kernel<true> then warps from the grid.  Every output float is stored once.
#pragma once

#include "interp.cuh"

namespace spg {

constexpr int kPreThreads = 128;
constexpr int kPreLanes = 8;  // values per vector iteration of VResizeCubicVec_32s8u (v_int16 at the SSE baseline)

// One member: one item of one source image.
struct PreMember {
    const unsigned char *src;      // the source: h rows of w x 3 bytes
    unsigned char *grid;           // rotated members: [Hp][Wp][3] the padded uint8 image (the handle's scratch)
    float *out;                    // [2][Hp][Wp][3]
    long long row_stride;          // bytes
    double scale;                  // 1 / fx, either axis
    double rot[6];                 // rotated members: the inverse of the forward matrix (output pixel -> padded grid)
    int h, w;                      // source size
    int H1, W1;                    // resized size (imageToTest)
    int Hp, Wp;                    // padded size
    int copy;                      // H1 == h and W1 == w: cv2.resize copies
    int n_body;                    // values of an interleaved resized row on the vector path: (W1 * 3) / 8 * 8
    int pad_value;
    int tiles_x;                   // CTAs per padded row: ceil(Wp / kPreThreads)
    int first_cta;                 // the member's first grid.x position in its launch
};

constexpr int kPreMaxMembers = (int)((kParamBytes - 8) / sizeof(PreMember));
struct PreRagged {
    int n;                                // members of this launch
    PreMember img[kPreMaxMembers];        // first_cta increasing
};
static_assert(sizeof(PreRagged) <= kParamBytes, "a launch's parameters fit the kernel-parameter limit");

// the member of CTA blockIdx.x and the pixel (y, x) of its padded image this thread computes
__device__ __forceinline__ const PreMember &prenet_member(const PreRagged &r, int &y, int &x) {
    const PreMember &a = ragged_member(r, (int)blockIdx.x);
    const int cta = (int)blockIdx.x - a.first_cta;
    y = cta / a.tiles_x;
    x = (cta - y * a.tiles_x) * kPreThreads + (int)threadIdx.x;
    return a;
}

// byte -> float32(byte / 255), the quotient rounded in double and then to float32 as numpy does
__device__ __forceinline__ void prenet_lut(float *lut) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = __double2float_rn(__ddiv_rn((double)i, 255.0));
    __syncthreads();
}

// pixel (y, x) of the padded uint8 image of `img`: the resized image's or the pad value
__device__ __forceinline__ void prenet_pixel(const PreMember &a, const unsigned char *img, int y, int x, int v[3]) {
    if (y >= a.H1 || x >= a.W1) {
        v[0] = v[1] = v[2] = a.pad_value;
        return;
    }
    if (a.copy) {
        const unsigned char *p = img + (long long)y * a.row_stride + 3 * x;
        v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
        return;
    }
    float c[4];
    int ax[4], by[4], col[4];
    const int x0 = axis_entry(x, a.scale, c);
#pragma unroll
    for (int k = 0; k < 4; k++) {
        ax[k] = __float2int_rn(__fmul_rn(c[k], 2048.0f));  // saturate_cast<short>(c * INTER_RESIZE_COEF_SCALE)
        col[k] = 3 * clampi(x0 + k, 0, a.w - 1);
    }
    const int y0 = axis_entry(y, a.scale, c);
#pragma unroll
    for (int k = 0; k < 4; k++) by[k] = __float2int_rn(__fmul_rn(c[k], 2048.0f));
    int S[4][3];  // horizontal pass of the four source rows: exact
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const unsigned char *row = img + (long long)clampi(y0 + r, 0, a.h - 1) * a.row_stride;
#pragma unroll
        for (int ch = 0; ch < 3; ch++)
            S[r][ch] = row[col[0] + ch] * ax[0] + row[col[1] + ch] * ax[1] + row[col[2] + ch] * ax[2] + row[col[3] + ch] * ax[3];
    }
    float b[4];
#pragma unroll
    for (int k = 0; k < 4; k++) b[k] = __fmul_rn((float)by[k], 2.384185791015625e-07f);  // beta * 2^-22, exact
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
        if (3 * x + ch < a.n_body) {  // vector body: float32, nested from the right, no FMA
            float t = __fmul_rn((float)S[3][ch], b[3]);
            t = __fadd_rn(__fmul_rn((float)S[2][ch], b[2]), t);
            t = __fadd_rn(__fmul_rn((float)S[1][ch], b[1]), t);
            t = __fadd_rn(__fmul_rn((float)S[0][ch], b[0]), t);
            v[ch] = clampi(__float2int_rn(t), 0, 255);
        } else {  // scalar tail: FixedPtCast<int, uchar, 22>
            const int acc = S[0][ch] * by[0] + S[1][ch] * by[1] + S[2][ch] * by[2] + S[3][ch] * by[3];
            v[ch] = clampi((acc + (1 << 21)) >> 22, 0, 255);
        }
    }
}

// rotated members: the padded uint8 image into the scratch grid
__global__ void __launch_bounds__(kPreThreads) prenet_resize_kernel(const __grid_constant__ PreRagged r) {
    int y, x;
    const PreMember &a = prenet_member(r, y, x);
    if (x >= a.Wp) return;
    int v[3];
    prenet_pixel(a, a.src, y, x, v);
    unsigned char *g = a.grid + ((long long)y * a.Wp + x) * 3;
    g[0] = (unsigned char)v[0]; g[1] = (unsigned char)v[1]; g[2] = (unsigned char)v[2];
}

// one pixel of the pair per thread: stored to the image at (y, x) and to the mirror at (y, Wp - 1 - x)
template <bool ROT>
__global__ void __launch_bounds__(kPreThreads) prenet_kernel(const __grid_constant__ PreRagged r) {
    __shared__ float lut[256];
    prenet_lut(lut);
    int y, x;
    const PreMember &a = prenet_member(r, y, x);
    if (x >= a.Wp) return;
    float f[3];
    if (ROT) {
        // warpAffine's adelta / bdelta and X0 / Y0 (rounded ties-to-even like cvRound), as postnet_rot_kernel
        int xs, ys;
        warp_coords(a.rot, x, y, xs, ys);
#pragma unroll
        for (int ch = 0; ch < 3; ch++)
            f[ch] = warp_linear<3>(xs, ys, a.Wp, a.Hp, a.grid + ch, 3 * a.Wp, 0, 0, [&](unsigned char v) { return lut[v]; });
    } else {
        int v[3];
        prenet_pixel(a, a.src, y, x, v);
        f[0] = lut[v[0]]; f[1] = lut[v[1]]; f[2] = lut[v[2]];
    }
    float *o = a.out + ((long long)y * a.Wp + x) * 3;
    float *m = a.out + ((long long)(a.Hp + y) * a.Wp + (a.Wp - 1 - x)) * 3;
    o[0] = f[0]; o[1] = f[1]; o[2] = f[2];
    m[0] = f[0]; m[1] = f[1]; m[2] = f[2];
}

}  // namespace spg
