// jpeg.cu -- the JPEG decoder's kernels for spg_jpeg_decode_ragged (jpeg.cuh describes them, jpeg_kernels.cuh holds
// them) and their launch, a translation unit of their own.
#define JPEG_KERNEL(name) name##_kernel
#define JPEG_MEMBER(r) ragged_member(r, (int)blockIdx.x)
#define JPEG_FRAME_EXIT(past)
#define JPEG_INTERVAL_END(m) m.seg_len
#include "jpeg_kernels.cuh"

namespace spg {

const char *const kJpegKernelName[kJpegKernels] = {"jpeg_count_kernel", "jpeg_prefix_kernel", "jpeg_pack_kernel", "jpeg_interval_kernel",
                                                   "jpeg_sync_kernel", "jpeg_fixup_kernel", "jpeg_write_kernel",
                                                   "jpeg_dc_kernel", "jpeg_idct_kernel", "jpeg_color_kernel",
                                                   "jpeg_count_frame_kernel", "jpeg_prefix_frame_kernel", "jpeg_pack_frame_kernel",
                                                   "jpeg_interval_frame_kernel", "jpeg_sync_frame_kernel",
                                                   "jpeg_fixup_frame_kernel", "jpeg_write_frame_kernel"};

cudaError_t jpeg_launch(JpegKernel k, unsigned grid, cudaStream_t st, const JpegRagged &r) {
    if (k >= kJpegCountFrame) return jpeg_frame_launch(k, grid, st, r);
    void (*const kern[kJpegCountFrame])(JpegRagged) = {jpeg_count_kernel, jpeg_prefix_kernel, jpeg_pack_kernel, jpeg_interval_kernel,
                                                    jpeg_sync_kernel,  jpeg_fixup_kernel, jpeg_write_kernel,
                                                    jpeg_dc_kernel,    jpeg_idct_kernel,  jpeg_color_kernel};
    kern[k]<<<grid, kJpegBlock[k], 0, st>>>(r);
    return cudaGetLastError();
}

}  // namespace spg

