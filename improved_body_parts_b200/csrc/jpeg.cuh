// jpeg.cuh -- cv2.imread's JPEG decode on the device (include/spgroup.h "JPEG decoding"): baseline / extended-sequential
// Huffman files, a batch of any sizes per launch.  spg_jpeg_parse (host) has checked the headers and built the Huffman
// decoding tables; the kernels here run, for every image of the call at once:
//
//   jpeg_count_kernel / jpeg_prefix_kernel /
//   jpeg_pack_kernel                       the entropy-coded segment unstuffed (0xFF 0x00 -> 0xFF, fill bytes and
//                                          markers dropped) into one contiguous stream, and the restart intervals' start
//                                          offsets: a parallel compaction, 4 KiB of the segment per CTA, with one CTA
//                                          per image scanning the chunks' counts in between.
//   jpeg_interval_kernel                   images with restart intervals: one thread decodes one interval (independent
//                                          by construction: byte aligned, DC predictors reset).
//   jpeg_sync_kernel / jpeg_fixup_kernel /  images without: the self-synchronising subsequence decode (Klein & Wiseman
//   jpeg_write_kernel                      2003; Weissenberger & Schmidt, ICPP 2018).  The stream is cut into
//                                          kJpegSubBits-bit subsequences, one per thread.  A thread decodes its own from a
//                                          guessed state (bit position, block of the MCU, coefficient index) and runs on to
//                                          the first symbol boundary past its end: its exit state.  Rounds inside the CTA
//                                          re-decode a subsequence from its predecessor's exit until no exit changes; the
//                                          fix-up kernel carries the true state across the CTA boundaries (a thread per
//                                          boundary, in rounds) and scans the per-subsequence block counts into output
//                                          offsets; the write kernel decodes each subsequence once more from its true
//                                          entry and stores the coefficients.
//   jpeg_dc_kernel                         the DC predictions: a segmented scan of the DC differences per component, reset
//                                          at every restart interval.
//   jpeg_idct_kernel                       dequantisation and libjpeg's islow IDCT, one block per thread, into component
//                                          planes of whole blocks.
//   jpeg_color_kernel                      fancy upsampling, YCbCr -> BGR (or grey -> BGR) and the EXIF orientation, one
//                                          output pixel per thread, written straight into the caller's image.
//
// Every read of the segment is bounded by its length, every block index by the image's block count, whatever the record
// holds.  A stream that does not decode the way libjpeg decodes a well-formed file (a code not in the table, a coefficient
// index past 63, bits or blocks running out) sets SPG_JPEG_CORRUPT; a block outside the range where libjpeg-turbo's SIMD
// and C IDCTs agree sets SPG_JPEG_RANGE (DESIGN.md §4).  The launches are ragged like prenet.cuh: the member table travels
// as a __grid_constant__ parameter and a CTA finds its image by binary search over first_cta (ragged_member).
//
// The frame form (spg_jpeg_decode_frame: one frame, recorded into a CUDA graph and replayed for every frame of one format)
// runs the same count to write kernels with grids sized for a capacity in scan bytes; they read the frame's segment
// address and length from its device record at run time, and the CTAs past the frame's work return (jpeg_kernels.cuh).
//
// jpeg.cu compiles the kernels and holds the host code; jpeg_frame.cu compiles the frame form's kernels with the frame
// macros, in a module of their own, and exports them as kJpegFrameKernels.  This header is what the two share.
#pragma once

#include "../../include/spgroup.h"
#include "common.cuh"

namespace spg {

constexpr int kJpegChunk = 4096;           // segment bytes per CTA of the unstuffing kernels
constexpr int kJpegPackThreads = 256;      // 16 bytes each
#ifndef SPG_JPEG_SUB_BITS
#define SPG_JPEG_SUB_BITS 1024
#endif
constexpr int kJpegSubBits = SPG_JPEG_SUB_BITS;  // bits per subsequence (DESIGN.md §3; the Makefile's jpeg_variants)
constexpr int kJpegSubThreads = 128;       // subsequences per CTA of the subsequence kernels
constexpr int kJpegThreads = 256;          // the other kernels
constexpr int kJpegStOk = 0, kJpegStCorrupt = 11, kJpegStRange = 12;  // SPG_JPEG_OK / _CORRUPT / _RANGE

// One subsequence's states: entry and exit (bit position; u << 8 | k), the blocks whose DC it decodes from its entry, and
// (after the fix-up) the index of the first of them.
struct JpegSub {
    int entry_pos, entry_uk, exit_pos, exit_uk, n, base;
};

// One image of a call (of spg_jpeg_decode_frame: seg is unused, seg_len, n_chunks and n_subs are the capacity's).
struct JpegMember {
    const spg_jpeg_record *rec;     // device copy of the record (tables)
    const unsigned char *seg;       // the entropy-coded segment
    int seg_len;
    int n_chunks;                   // ceil(seg_len / kJpegChunk)
    unsigned char *packed;          // the unstuffed stream (<= seg_len bytes)
    int *chunk_counts;              // [n_chunks][2]: kept bytes, restart markers
    int *starts;                    // [n_intervals + 1]: interval starts in packed; the last entry is the stream length
    JpegSub *subs;                  // [n_subs] (images without restart intervals)
    short *coef;                    // [total_blocks][64], MCU order, natural order within a block
    unsigned char *plane[3];        // component planes of whole blocks, plane_w[c] bytes per row
    int plane_w[3];
    unsigned char *out;             // [out_h][out_w][3]
    int *status;
    int n_subs, total_blocks;
    int frame_h, frame_w, out_h, out_w, orientation;
    int n_comp, hs, vs, mcus_x, mcus_y, bpm, restart, n_intervals;
    int first_cta;
};
constexpr int kJpegTableMax = (int)((kParamBytes - 8) / sizeof(JpegMember));
struct JpegRagged {
    int n;
    JpegMember img[kJpegTableMax];  // first_cta increasing
};

// The decoder's kernels, in launch order, and their block sizes; then the frame form's count to write kernels, which read
// the segment's address and length from the device record (spg_jpeg_decode_frame; the DC, IDCT and colour kernels are
// the ragged ones).
enum JpegKernel : int { kJpegCount, kJpegPrefix, kJpegPack, kJpegInterval, kJpegSync, kJpegFixup, kJpegWrite, kJpegDc, kJpegIdct, kJpegColor,
                        kJpegCountFrame, kJpegPrefixFrame, kJpegPackFrame, kJpegIntervalFrame, kJpegSyncFrame, kJpegFixupFrame,
                        kJpegWriteFrame, kJpegKernels };
constexpr int kJpegBlock[kJpegKernels] = {kJpegPackThreads, kJpegPackThreads, kJpegPackThreads, kJpegThreads, kJpegSubThreads, kJpegThreads,
                                          kJpegSubThreads, kJpegThreads, kJpegThreads, kJpegThreads,
                                          kJpegPackThreads, kJpegPackThreads, kJpegPackThreads, kJpegThreads, kJpegSubThreads, kJpegThreads,
                                          kJpegSubThreads};
// the frame form's kernels, kJpegCountFrame to kJpegWriteFrame (jpeg_frame.cu)
extern void (*const kJpegFrameKernels[kJpegKernels - kJpegCountFrame])(JpegRagged);

}  // namespace spg
