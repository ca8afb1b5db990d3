// jpeg_frame.cu -- the frame form of the JPEG decoder's count to write kernels (spg_jpeg_decode_frames; jpeg_kernels.cuh
// holds their source), compiled with the frame macros in a unit of their own; jpeg.cu launches them by kJpegFrameKernels.
#include "jpeg.cuh"

namespace spg {

// The member of a frame launch holds capacities where a ragged member holds the file's values: seg_len is the scan bytes
// the scratch was carved for, and the grids cover that many.  The frame's segment and length come from its device record,
// and the chunk and subsequence counts follow from them as spg_jpeg_decode_ragged computes them on the host.  A length
// outside [0, capacity] decodes as an empty segment, which the decode flags SPG_JPEG_CORRUPT; no byte past the frame's
// own segment or unstuffed stream is read, whatever an earlier, longer frame left in the buffers.
__device__ __forceinline__ JpegMember jpeg_framed(const JpegMember &cap) {
    JpegMember m = cap;
    const long long len = cap.rec->scan_length;
    const int n = len >= 0 && len <= cap.seg_len ? (int)len : 0;
    m.seg = cap.rec->data + cap.rec->scan_offset;
    m.seg_len = n;
    m.n_chunks = max(1, (n + kJpegChunk - 1) / kJpegChunk);
    m.n_subs = m.restart ? 0 : max(1, (int)((8ll * n + kJpegSubBits - 1) / kJpegSubBits));
    return m;
}

}  // namespace spg

#define JPEG_FRAME_FORM
#define JPEG_KERNEL(name) name##_frame_kernel
#define JPEG_MEMBER(r) jpeg_framed(ragged_member(r, (int)blockIdx.x))
#define JPEG_FRAME_EXIT(past) \
    if (past) return;
// starts[] entries a malformed frame's pack left unwritten hold an earlier frame's offsets: an interval is bounded by this
// frame's unstuffed length, which the pack writes whatever the data
#define JPEG_INTERVAL_END(m) m.starts[m.n_intervals]
#include "jpeg_kernels.cuh"

namespace spg {

void (*const kJpegFrameKernels[kJpegKernels - kJpegCountFrame])(JpegRagged) = {
    jpeg_count_frame_kernel, jpeg_prefix_frame_kernel, jpeg_pack_frame_kernel, jpeg_interval_frame_kernel,
    jpeg_sync_frame_kernel,  jpeg_fixup_frame_kernel,  jpeg_write_frame_kernel};

}  // namespace spg
