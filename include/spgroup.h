/*
 * spgroup.h -- C ABI of the H100-native keypoint-grouping path (libspgroup.so).
 *
 * Drop-in boundary for SimplePose's post-network grouping stage.  The reference
 * (hellojialee/Improved-Body-Parts) has no plugin/FFI layer: the boundary is three module-level
 * Python functions called back to back at evaluate.py:509-511 plus two helpers in
 * utils/util.py.  Each entry point below names the reference interface it replaces; INTEGRATION.md
 * shows the ctypes binding a maintainer adds to evaluate.py.
 *
 * Conventions
 *   - plain C: opaque handle, POD structs, raw pointers and sizes; no torch / C++ types.
 *   - every function returns 0 (SPG_OK) or a negative SPG_E_* code; spg_last_error() gives a message.
 *   - device pointers are raw CUDA device addresses in the handle's device's primary context;
 *     `stream` is a cudaStream_t passed as void* (NULL = default stream).  Kernel launches are
 *     asynchronous on that stream; the *_download_* / spg_group_host calls synchronise it.
 *   - maps are channel-first float planes with contiguous rows (pixel stride 1, row stride W);
 *     image and channel strides are given in ELEMENTS.  The network's raw [N,50,h,w] tensor can be
 *     passed directly with channel offsets 0 (body parts) / 30 (keypoints), config/config.py:101-103.
 *   - no CPU fallback exists: without a usable sm_90 device spg_create fails.
 *   - per-image problems (capacity overflows, an out-of-range sample index where the reference would
 *     raise IndexError) are reported in the status word of that image, never by exceptions.
 */
#ifndef SPGROUP_H_
#define SPGROUP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SPG_ABI_VERSION 3

enum {
    SPG_OK = 0,
    SPG_E_INVALID = -1,   /* bad argument (shape, capacity, alignment, null pointer) */
    SPG_E_CUDA = -2,      /* a CUDA runtime call failed; see spg_last_error          */
    SPG_E_NO_DEVICE = -3, /* no CUDA device / not an sm_90 part                      */
    SPG_E_STATE = -4,     /* stage called before the stage that feeds it             */
    SPG_E_CAPTURE = -5    /* the call would have to grow a scratch buffer while its stream is capturing a */
                          /* CUDA graph: reserve it first (spg_reserve_frame); nothing was enqueued      */
};

/* per-image status bits (spg_download_status) */
enum {
    SPG_ST_PEAK_OVERFLOW = 1u << 0,  /* a part class had more peaks than max_peaks_per_part      */
    SPG_ST_CAND_OVERFLOW = 1u << 1,  /* a limb had more surviving candidates than max_cands      */
    SPG_ST_ROW_OVERFLOW = 1u << 2,   /* person assembly needed more than max_person_rows rows    */
    SPG_ST_SAMPLE_INDEX = 1u << 3,   /* a line sample fell outside the map: the reference would  */
                                     /* raise IndexError at evaluate.py:235                      */
    SPG_ST_ASSERT = 1u << 4,         /* the reference would raise at evaluate.py:437-439         */
    SPG_ST_WIRE_OVERFLOW = 1u << 5,  /* more persons than the wire record holds (rows beyond are dropped) */
    SPG_ST_NONFINITE = 1u << 6,      /* a limb pair has a non-finite length (an end point with a NaN or infinite  */
                                     /* coordinate, from a non-finite map value inside its refinement box): the   */
                                     /* reference would raise ValueError / OverflowError at evaluate.py:226       */
    SPG_ST_NAN_PRIORITY = 1u << 7    /* a limb with two or more candidates has one with a NaN priority (a border */
                                     /* peak with a NaN score, or +inf + -inf): the reference's sort at           */
                                     /* evaluate.py:259 orders unordered keys, which is not reproduced            */
};

/* dtype of the body-part planes.  predict() accumulates them in float64 (evaluate.py:86,161); with a single scale
 * (the reference's default, utils/config:26) every float64 value is exactly a float32 one, so the planes can be STORED
 * as float32 and evaluated with the float64 arithmetic the reference applies: SPG_F32_AS_F64 -- half the HBM traffic,
 * bit-identical results to SPG_F64 planes holding the same values.  SPG_F16 is accepted for network outputs and loss
 * predictions only, SPG_BF16 for loss predictions only. */
enum { SPG_F32 = 0, SPG_F64 = 1, SPG_F32_AS_F64 = 2, SPG_F16 = 3, SPG_BF16 = 4 };

typedef struct spg_handle spg_handle;

/* Skeleton + capacities.  Mirrors config/config.py:52-126 (runtime data, not compile-time). */
typedef struct spg_config {
    int32_t abi_version;        /* SPG_ABI_VERSION */
    int32_t device;             /* CUDA device ordinal */
    int32_t n_parts;            /* K: keypoint channels used (18; evaluate.py:175,187) */
    int32_t n_limbs;            /* L: body-part channels (30; config.py:94-96) */
    const int32_t *limbs;       /* [L][2] (from_part, to_part) = limbs_conn */
    int32_t n_out_joints;       /* 17 COCO joints */
    const int32_t *out_from_part; /* [n_out_joints] part index feeding each output joint (inverse of dt_gt_mapping, config.py:117) */
    int32_t max_batch;          /* images resident per call */
    int32_t max_h, max_w;       /* largest map */
    int32_t max_peaks_per_part; /* <= 128 */
    int32_t max_cands_per_limb; /* surviving candidates kept per (image, limb) */
    int32_t max_person_rows;    /* <= 128; rows of `subset` alive or dead during assembly */
} spg_config;

/* Grouping hyper-parameters: the reference's `params` dict (utils/config:17-28) plus the two literals of
 * the final prune (evaluate.py:493). */
typedef struct spg_params {
    double thre1, thre2, connect_ration, len_rate, connection_tole, min_mean_score;
    int32_t mid_num, offset_radius, remove_recon, min_parts;
    /* demo_image.py's inlined copy of the grouping code differs from evaluate.py in two decisions (SURVEY 3.2); both 0
     * for evaluate.py.  With min_parts = 4 (demo_image.py:533) they give the demo's behaviour. */
    int32_t crit1_strict;       /* 1: `count >  connect_ration*n` (demo_image.py:288) instead of `>=` (evaluate.py:246) */
    int32_t refresh_len_check;  /* 1: the same-B refresh also requires len_rate*maxlen > len (demo_image.py:414-415)   */
} spg_params;

/* Device-resident results of the last call, for consumers that stay on the GPU (NCCL gather, benchmarks).
 * All arrays are indexed [image][...] with the capacities of spg_config. */
typedef struct spg_device_view {
    int32_t max_batch, n_parts, n_limbs, n_out_joints, cap_peaks, cap_cands, cap_rows;
    /* peaks: [N][K][cap_peaks] */
    const double *peak_x, *peak_y;     /* refined coordinates (util.py:204-211) */
    const float *peak_score;
    const uint32_t *peak_anchor;       /* (y << 16) | x integer anchor; bit 31 = border peak (integer coords, util.py:201-202) */
    const int32_t *peak_count;         /* [N][K] true count (may exceed cap -> status bit) */
    /* connections: [N][L][cap_peaks] in greedy acceptance order (evaluate.py:263-270) */
    const uint32_t *conn_ij;           /* (i << 16) | j */
    const double *conn_score, *conn_norm;
    const int32_t *conn_count;         /* [N][L]; -1 = special_k (evaluate.py:272-274) */
    const int32_t *cand_count;         /* [N][L] candidates that passed both criteria (evaluate.py:252) */
    const int32_t *surv_count;         /* [N][L] pairs that survived the scoring kernel's conservative screen (diagnostic) */
    /* persons */
    const double *subset;              /* [N][cap_rows][K+2][2] after the prune (evaluate.py:491-496) */
    const int32_t *n_persons;          /* [N] */
    const double *people_xy;           /* [N][cap_rows][n_out_joints][2] (evaluate.py:523-539) */
    const double *people_score;        /* [N][cap_rows]  1 - 1/total (evaluate.py:541) */
    const uint32_t *status;            /* [N] SPG_ST_* bits */
} spg_device_view;

/* ---- lifetime -------------------------------------------------------------------------------- */
int spg_create(const spg_config *cfg, spg_handle **out);
void spg_destroy(spg_handle *h);
const char *spg_last_error(const spg_handle *h); /* h may be NULL: last creation error */
int spg_abi_version(void);
int spg_get_device_view(const spg_handle *h, spg_device_view *out);

/* ---- whole path: replaces the three calls at evaluate.py:509-511 ------------------------------ */
/* device inputs already resident; asynchronous on `stream` */
int spg_group_batch(spg_handle *h, const float *heat_dev, int64_t heat_image_stride, int64_t heat_chan_stride,
                    const void *paf_dev, int32_t paf_dtype, int64_t paf_image_stride, int64_t paf_chan_stride,
                    int32_t n_images, int32_t height, int32_t width, double image_extent,
                    const spg_params *params, void *stream);

/* One image of a ragged call: its own maps, size and extent.  evaluate.py groups every validation image at its own
 * resolution (process(), evaluate.py:501-543), so a batch of them has no common size. */
typedef struct spg_image_maps {
    const float *heat;          /* [>=K][H][W] float32, rows contiguous, planes heat_chan_stride elements apart */
    const void *paf;            /* [>=L][H][W] of the call's paf_dtype, planes paf_chan_stride elements apart   */
    int64_t heat_chan_stride, paf_chan_stride;
    int32_t height, width;
    double image_extent;        /* this image's oriImg.shape[0] (evaluate.py:510) */
} spg_image_maps;

/* peaks -> connections -> people for n_images maps of different sizes; image i's results in slot i, equal to what
 * spg_group_batch returns for that image alone (the candidate arrays aside: they are unordered).  Every image is
 * validated before the first launch; SPG_E_INVALID names the first bad one.  Asynchronous on `stream`; `images` may be
 * reused as soon as the call returns.  Wire output and the armed wire signal apply as for spg_group_batch. */
int spg_group_ragged(spg_handle *h, const spg_image_maps *images, int32_t n_images, int32_t paf_dtype,
                     const spg_params *params, void *stream);

/* ---- the capacity-free tier: one image whatever its number of peaks, candidates and persons ---------------------
 * The calls above hold at most max_peaks_per_part peaks per part (<= 128), max_cands_per_limb candidates per limb and
 * max_person_rows rows (<= 128); an image past one of them gets SPG_ST_PEAK_OVERFLOW / SPG_ST_CAND_OVERFLOW /
 * SPG_ST_ROW_OVERFLOW and undefined outputs.  spg_group_unbounded regroups such an image with every list sized from the
 * image itself, bit-identical to the reference as the bounded path is: peaks -> connections -> people of `image` (its
 * maps, size and image_extent) on `stream`.  The host sizes each stage's tables from the previous stage's counts, so the
 * call synchronises `stream` three times; the tables belong to the handle, grow on demand and live until spg_destroy.
 * The tier's status word carries SPG_ST_SAMPLE_INDEX, SPG_ST_ASSERT, SPG_ST_NONFINITE and SPG_ST_NAN_PRIORITY as the
 * bounded path sets them, never a capacity bit.  Its own limits -- at most 65535 peaks per part ((i, j) of a connection are packed in 16 bits each), 32767
 * accepted connections per image (the person table has one row per connection) and 2^31 - 1 candidates -- and a failed
 * allocation make the call return an error, never undefined output.  Maps: 2 <= height, width <= 32767; the handle's
 * max_h / max_w do not apply. */
int spg_group_unbounded(spg_handle *h, const spg_image_maps *image, int32_t paf_dtype, const spg_params *params,
                        void *stream);
typedef struct spg_unbounded_sizes {
    int32_t cap_peaks;  /* peak arrays are [K][cap_peaks], connection arrays [L][cap_peaks] */
    int32_t cap_rows;   /* person arrays are [cap_rows][...] */
    int32_t n_persons;  /* persons after the prune */
    uint32_t status;    /* SPG_ST_* bits of the image */
} spg_unbounded_sizes;
/* The last spg_group_unbounded call's results, laid out as the spg_download_* arrays of ONE image with the tier's sizes:
 * peak_count [K], x / y / score / anchor [K][cap_peaks], conn_count / cand_count [L], ij / conn_score / conn_norm
 * [L][cap_peaks], subset [cap_rows][K+2][2], people_xy [cap_rows][J][2], people_score [cap_rows].  `sizes` is always
 * filled; NULL arrays are skipped, so a first call with NULL arrays gives the sizes to allocate.  Synchronises `stream`.
 * SPG_E_STATE before the first successful spg_group_unbounded. */
int spg_download_unbounded(spg_handle *h, spg_unbounded_sizes *sizes, int32_t *peak_count, double *x, double *y,
                           float *score, uint32_t *anchor, int32_t *conn_count, int32_t *cand_count, uint32_t *ij,
                           double *conn_score, double *conn_norm, double *subset, double *people_xy,
                           double *people_score, void *stream);

/* host inputs (pinned for full overlap; pageable works): H2D in chunks overlapped with the kernels, results
 * copied back into the caller's arrays (any of which may be NULL).  Synchronous.
 *   heat_host [N][K][H][W] f32, paf_host [N][L][H][W] f32|f64
 *   out_n_persons [N], out_people_xy [N][cap_rows][J][2], out_people_score [N][cap_rows], out_status [N] */
int spg_group_host(spg_handle *h, const float *heat_host, const void *paf_host, int32_t paf_dtype,
                   int32_t n_images, int32_t height, int32_t width, double image_extent,
                   const spg_params *params, int32_t *out_n_persons, double *out_people_xy,
                   double *out_people_score, uint32_t *out_status);

/* pinned host memory for spg_group_host callers that do not have their own */
int spg_host_alloc(void **ptr, uint64_t bytes);
int spg_host_free(void *ptr);

/* ---- post-network stage: the scale loop of predict() after the forward pass, evaluate.py:126-161 ----------- */
/* One entry per (scale) of params['scale_search']: the network's output for a batch of image pairs
 * [N][2][C][h][w] (image, mirrored image; evaluate.py:116-126), device memory, float32 or float16. */
typedef struct spg_postnet_scale {
    const void *net_out;
    int32_t dtype;                  /* SPG_F32 | SPG_F16 */
    int64_t image_stride, pair_stride, chan_stride; /* elements; rows are contiguous (row stride w) */
    int32_t h, w;                   /* network output size = padded input size / stride */
    int32_t crop_h, crop_w;         /* imageToTest size: padded size minus pad[2] / pad[3] (evaluate.py:148) */
} spg_postnet_scale;
typedef struct spg_postnet_desc {
    int32_t n_scales;               /* items: len(multiplier) * len(rotate_angle), in product() order (scale-major) */
    const spg_postnet_scale *scales;
    int32_t stride;                 /* model_params['stride'] (4) */
    int32_t paf_chan0, heat_chan0;  /* first body-part / keypoint channel of the network output (0 / 30, config.py:101-103) */
    const int32_t *flip_paf_ord;    /* [n_limbs]  config.py:121-124 */
    const int32_t *flip_heat_ord;   /* [n_parts] */
    int32_t nan_scrub;              /* demo_image.py:179-180: NaN -> 0 in the averaged maps (evaluate.py: 0) */
} spg_postnet_desc;
/* flip ensemble (:139-140) + cv2.resize x stride (:143,152) + crop (:148,157) + cv2.resize to the image (:149,158) +
 * float64 average over the scales (:160-161), fused, writing the channel-first planes the grouping kernels stream:
 *   heat_out [N][n_parts][H][W] float32 (the cast of evaluate.py:173 applied),
 *   paf_out  [N][n_limbs][H][W] SPG_F64, or SPG_F32 when n_scales == 1 (then pass SPG_F32_AS_F64 to the grouping calls).
 * Interpolation follows OpenCV's generic bicubic path (A = -0.75) operation for operation in float32. */
int spg_postnet(spg_handle *h, const spg_postnet_desc *desc, int32_t n_images, int32_t height, int32_t width,
                float *heat_out, void *paf_out, int32_t paf_dtype, void *stream);
/* The rotation search (rotation_search != [0], evaluate.py:107-158): per item, whether its x stride maps go through
 * cv2.warpAffine(map, matrix, (0, 0)) (INTER_LINEAR, BORDER_CONSTANT 0) before the crop.  The warp follows OpenCV's
 * fixed-point algorithm bit for bit.  Rotated items need stride 4. */
typedef struct spg_postnet_rotation {
    int32_t apply;      /* 0: angle == 0, the item is not warped (evaluate.py:115,144,153); 1: warped */
    int32_t reserved;   /* 0 */
    double matrix[6];   /* row-major 2x3 matrix evaluate.py passes to cv2.warpAffine for the maps (rotate_matrix_reverse) */
} spg_postnet_rotation;
/* spg_postnet with rot [desc->n_scales] (NULL: no item is rotated; spg_postnet is this call with NULL). */
int spg_postnet_rotated(spg_handle *h, const spg_postnet_desc *desc, const spg_postnet_rotation *rot,
                        int32_t n_images, int32_t height, int32_t width, float *heat_out, void *paf_out,
                        int32_t paf_dtype, void *stream);
/* Ragged batches: predict()'s post-network stage for images of different sizes in one call, one item per image (a single
 * scale, no rotation: the reference's default, utils/config).  What the images share: */
typedef struct spg_postnet_common {
    int32_t stride;                 /* model_params['stride']: must be 4 */
    int32_t paf_chan0, heat_chan0;  /* as spg_postnet_desc */
    const int32_t *flip_paf_ord;    /* [n_limbs] */
    const int32_t *flip_heat_ord;   /* [n_parts] */
    int32_t nan_scrub;              /* as spg_postnet_desc */
    int32_t net_dtype;              /* SPG_F32 | SPG_F16: the dtype of every image's network output */
} spg_postnet_common;
/* One image: the network's output for its pair and where its maps go. */
typedef struct spg_postnet_image {
    const void *net_out;            /* [2][C][h][w] (image, mirrored image), rows contiguous (row stride w) */
    int64_t pair_stride, chan_stride; /* elements */
    int32_t h, w;                   /* network output size = padded input size / 4 */
    int32_t crop_h, crop_w;         /* imageToTest size (evaluate.py:148) */
    int32_t height, width;          /* image size = map size */
    float *heat_out;                /* [n_parts][height][width] float32, 16-byte aligned */
    void *paf_out;                  /* [n_limbs][height][width] of the call's paf_dtype, 16-byte aligned */
} spg_postnet_image;
/* Image i's maps equal those spg_postnet gives for it alone (n_scales = 1).  paf_dtype: SPG_F32 (float32 storage of the
 * float64 values, as for a single scale: pass SPG_F32_AS_F64 to the grouping calls) or SPG_F64.  Every image is validated
 * before the first launch; SPG_E_INVALID names the first bad one.  Asynchronous on `stream` (never synchronises);
 * `images` may be reused as soon as the call returns. */
int spg_postnet_ragged(spg_handle *h, const spg_postnet_common *common, const spg_postnet_image *images,
                       int32_t n_images, int32_t paf_dtype, void *stream);
/* Ragged batches with several items per image: the multi-scale and rotation search (scale_search, rotation_search) for
 * images of different sizes in one call.  items [n_images][n_items] in product(multiplier, rotate_angle) order: the
 * items of one image share height, width, heat_out and paf_out.  rot [n_images][n_items] as spg_postnet_rotated's, or
 * NULL (no item rotated); item t is rotated in every image or in none.  Image i's maps equal those spg_postnet_rotated
 * gives for it alone.  paf_dtype SPG_F64, or SPG_F32 for n_items == 1.  Validation, asynchrony and reuse of `items` /
 * `rot` as spg_postnet_ragged; the handle's float64 keypoint scratch grows on demand to the batch's sum of
 * n_parts * height * width when the sums outlive a launch (more than 4 items, or a rotated one). */
int spg_postnet_ragged_items(spg_handle *h, const spg_postnet_common *common, const spg_postnet_image *items,
                             const spg_postnet_rotation *rot, int32_t n_images, int32_t n_items, int32_t paf_dtype,
                             void *stream);

/* ---- pre-network stage: the item loop of predict() before the forward pass, evaluate.py:94-121 ------------ */
/* One (scale, angle) item of product(multiplier, rotate_angle) (evaluate.py:90). */
typedef struct spg_prenet_item {
    double scale;               /* fx = fy of cv2.resize, after the 2600 / 3800 clamp (evaluate.py:94-96) */
    int32_t rotate;             /* 0: angle == 0, no warp; 1: cv2.warpAffine(input_img, matrix, (0, 0)) (:108-111) */
    int32_t reserved;           /* 0 */
    double matrix[6];           /* row-major 2x3 FORWARD matrix evaluate.py:109 passes to warpAffine (rotate_matrix) */
    float *out;                 /* [n_images][2][Hp][Wp][3] float32: the image, then its mirror (:116-119) */
    int64_t out_image_stride;   /* elements between images (>= 2 * Hp * Wp * 3 when n_images > 1) */
} spg_prenet_item;
/* image_dev [n_images][height][width][3] uint8 (BGR as read), rows of width * 3 contiguous bytes row_stride bytes apart,
 * images image_stride bytes apart.  Per item: cv2.resize(image, (0, 0), fx=scale, fy=scale, INTER_CUBIC) to
 * H1 = cvRound(height * scale) x W1 = cvRound(width * scale) (:98), padded below / right with pad_value to
 * Hp x Wp, multiples of max_downsample (:99-100), divided by 255 in float32 (:105), warped for rotate = 1 (the padded
 * grid, taps outside it read 0) and mirrored.  The resize follows OpenCV's GENERIC uint8 path bit for bit (the IPP build
 * differs by at most 1 LSB); the warp follows its fixed-point algorithm bit for bit.  The library computes the geometry;
 * the host inverts the matrix in warpAffine's operation order.  Asynchronous on `stream`; a handle-owned scratch grid
 * for rotated items grows on demand and lives until spg_destroy. */
int spg_prenet(spg_handle *h, const uint8_t *image_dev, int64_t image_stride, int64_t row_stride, int32_t n_images,
               int32_t height, int32_t width, int32_t max_downsample, int32_t pad_value, const spg_prenet_item *items,
               int32_t n_items, void *stream);
/* One member of a ragged pre-network call: one (scale, angle) item of one image. */
typedef struct spg_prenet_member {
    const uint8_t *image;       /* [height][width][3] uint8 device image (BGR as read), rows row_stride bytes apart */
    int64_t row_stride;         /* >= width * 3 */
    int32_t height, width;
    double scale;               /* as spg_prenet_item */
    int32_t rotate;             /* as spg_prenet_item */
    int32_t reserved;           /* 0 */
    double matrix[6];           /* as spg_prenet_item */
    float *out;                 /* [2][Hp][Wp][3] float32: the image, then its mirror */
} spg_prenet_member;
/* spg_prenet for members of different image sizes, scales and angles in one call (a batch of images of different sizes,
 * each with its own items): member i's pair equals the one spg_prenet gives for that image and item alone.  Every member
 * is validated before the first launch (spg_prenet's rules per member; SPG_E_INVALID names the first bad one as
 * "member i").  Asynchronous on `stream`; `members` may be reused as soon as the call returns.  The scratch grid of
 * rotated members grows on demand to the total of Hp * Wp * 3 bytes of the rotated members of one launch (up to a few
 * hundred members). */
int spg_prenet_ragged(spg_handle *h, int32_t max_downsample, int32_t pad_value, const spg_prenet_member *members,
                      int32_t n_members, void *stream);

/* ---- frames recorded into a CUDA graph ---------------------------------------------------------------------------
 * spg_prenet, spg_postnet / spg_postnet_rotated and spg_group_batch (with or without spg_set_wire_output) can be
 * recorded on a stream that is capturing a CUDA graph: they neither synchronise nor read device data back, and every
 * choice they make (kernel, tiling, shared memory) depends on their arguments alone.  A call made while its stream
 * captures never allocates: if it would have to grow one of the handle's scratch buffers it returns SPG_E_CAPTURE before
 * enqueueing anything, and the capture, the stream and the handle stay usable.  The persistent limb scorer's item queue
 * is zeroed by a memset node ahead of its kernel in a captured call on a handle that spg_reserve_frame prepared, so
 * every replay starts from the same state.
 *
 * spg_reserve_frame grows, outside any capture, every scratch buffer one frame needs: an image of height x width
 * through spg_prenet with `items` (their scale, rotate, reserved and matrix fields; out is not read) and
 * max_downsample, then through spg_postnet_rotated with one scale per item at `stride` and a rotation wherever the item
 * has rotate = 1.  The handle's max_batch sizes the post-network sums as spg_postnet_rotated does.  *moved (may be NULL)
 * is set to 1 when a buffer had to be reallocated, which invalidates graphs captured earlier from this handle's calls
 * (they hold the old address), else to 0.  Synchronous; must not be called while any stream of the device captures.
 *
 * spg_jpeg_decode_frame (below) is the JPEG decode of one frame in a form that can be recorded: its graph serves every
 * frame of one format, and spg_jpeg_reserve_frame grows its scratch for a format and a capacity ahead of the capture,
 * with *moved as here.  spg_yuv_to_bgr (below) can be recorded as it is: it has no scratch to reserve. */
int spg_reserve_frame(spg_handle *h, int32_t height, int32_t width, int32_t max_downsample, const spg_prenet_item *items,
                      int32_t n_items, int32_t stride, int32_t *moved);
/* Several frames in one graph (a tick): spg_prenet_ragged, spg_postnet_ragged_items and spg_group_ragged (with or without
 * spg_set_wire_output) can be recorded as the calls above can.  They neither synchronise nor copy from the host: their
 * member tables travel as kernel parameters.  spg_group_ragged allocates nothing (its workspace is the handle's,
 * max_batch images); the other two grow a scratch buffer only through the rule above.  spg_reserve_frames grows, outside
 * any capture, what one tick needs: members [n_images][n_items] in product(multiplier, rotate_angle) order, as
 * spg_prenet_ragged takes them (every member of image i reads an image of its height x width; image, out and row_stride
 * are not read), then spg_postnet_ragged_items over those images with n_items items (rotated where the member is) and
 * spg_group_ragged over n_images <= max_batch images.  *moved as for spg_reserve_frame.  Synchronous; must not be called
 * while any stream of the device captures. */
int spg_reserve_frames(spg_handle *h, int32_t max_downsample, const spg_prenet_member *members, int32_t n_images,
                       int32_t n_items, int32_t *moved);

/* ---- YUV frames: cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420 / _YUYV) ----------------------------------------- */
enum {
    SPG_YUV_NV12 = 1,  /* planes[0] Y [height][width], planes[1] interleaved U, V [height / 2][width] */
    SPG_YUV_I420 = 2,  /* planes[0] Y [height][width], planes[1] U and planes[2] V [height / 2][width / 2] */
    SPG_YUV_YUYV = 3   /* planes[0] Y0 U Y1 V [height][2 * width] (packed 4:2:2) */
};
/* One frame of spg_yuv_to_bgr: its planes (device memory, rows pitches[k] bytes apart; the planes a format does not use
 * are not read) and its [height][width][3] uint8 BGR output (device, rows out_pitch bytes apart). */
typedef struct spg_yuv_member {
    int32_t format;             /* SPG_YUV_NV12, SPG_YUV_I420 or SPG_YUV_YUYV */
    int32_t height, width;      /* even for NV12 and I420; width even for YUYV (cv2 refuses the others) */
    int32_t reserved;           /* 0 */
    const uint8_t *planes[3];
    int64_t pitches[3];         /* >= each plane's row bytes */
    uint8_t *out;
    int64_t out_pitch;          /* >= 3 * width */
} spg_yuv_member;
/* Per member, OpenCV's integer BT.601 limited-range conversion, bit for bit with cv2.cvtColor: with y = max(0, Y - 16)
 * * 1220542 and r = 1 << 19, B = (y + r + 2116026 (U - 128)) >> 20, G = (y + r - 409993 (U - 128) - 852492 (V - 128))
 * >> 20 and R = (y + r + 1673527 (V - 128)) >> 20, each saturated to [0, 255]; a 2x2 block (4:2:0) or a 2x1 pair (4:2:2)
 * shares its U and V.  Every member is validated before the first launch (SPG_E_INVALID names the first bad one as
 * "member i").  Asynchronous on `stream`; `members` may be reused as soon as the call returns.  The call allocates
 * nothing and never synchronises, and its launches depend on the members alone, so it can be recorded into a CUDA graph
 * (see "frames recorded into a CUDA graph") and replayed with new contents in the same planes. */
int spg_yuv_to_bgr(spg_handle *h, const spg_yuv_member *members, int32_t n, void *stream);

/* ---- tracking people across a stream's frames: OKS association of each frame's people with the stream's tracks ------
 * A stream (one camera or one video) keeps a table of at most SPG_TRACK_SLOTS tracks in caller-owned device memory; a
 * zero-filled table is empty, with its id counter at 0.  A track holds its id, its age (frames of its stream since it
 * was last matched) and its last pose, 17 COCO joints as a wire record row stores them. */
#define SPG_TRACK_SLOTS 128
typedef struct spg_track {
    int64_t id;
    int32_t age;
    int32_t live;               /* 0: the slot is free */
    double xy[17][2];
    uint64_t present;           /* bit g: joint g was found (as a wire record row's mask) */
} spg_track;
typedef struct spg_track_table {
    int64_t next_id;            /* the id the stream's next track takes: ids are unique within a stream */
    int64_t reserved;
    spg_track tracks[SPG_TRACK_SLOTS];
} spg_track_table;
/* One frame of spg_track_frames; every address is device memory, read or written when the launch runs. */
typedef struct spg_track_frame {
    const void *record;         /* the frame's wire record, spg_wire_record_bytes(h) bytes (the handle's wire rows) */
    const int32_t *stream;      /* the frame's table index in [0, n_tables), or -1: the frame is skipped */
    const int32_t *jpeg_status; /* NULL, or the frame's decode_status: a value other than SPG_JPEG_OK makes the */
                                /* frame unobserved                                                            */
    int64_t *ids;               /* [wire rows]: the first n_persons get the id of each row's person, or -1 */
    double *oks;                /* NULL, or [SPG_TRACK_SLOTS][wire rows]: OKS of each live track (by slot) with */
                                /* each person of an observed frame, as matched; other entries are not written */
} spg_track_frame;
/* Per frame, in order (several frames of one stream in one call are taken in call order):
 *   1. the OKS of each live track with each of the record's first n_persons persons: COCO's keypoint sigmas
 *      (cocoeval.py's kpt_oks_sigmas), the track's pose as ground truth; T = its joints present with finite x and y,
 *      area = max((xmax - xmin) * (ymax - ymin), 1) over T; per joint of T present and finite in the person
 *      e = (dx^2 + dy^2) / (2 sigma)^2 / area / 2 in float64 in that order, OKS = sum of exp(-e) in joint order / |T|
 *      (0 when T is empty); a joint of T the person lacks counts in |T| and adds nothing;
 *   2. greedy matching over the pairs with OKS >= oks_threshold: highest OKS first, ties to the lower track id, then to
 *      the lower person row, a pair taken when both members are free;
 *   3. a matched track takes the person's pose and age 0; the person gets the track's id;
 *   4. every other live track ages by 1 and is dropped when its age exceeds max_age;
 *   5. in row order, each unmatched person starts a track with the stream's next id in the lowest free slot, or, in a
 *      full table, in place of the track of largest age (ties: smallest id).
 * A frame whose record has a status bit, or whose jpeg_status is not SPG_JPEG_OK, is unobserved: only step 4 runs and
 * its persons get -1.  A skipped frame (stream -1) changes no table; its persons get -1.  The handle must have 17 output
 * joints; oks_threshold is finite and max_age >= 0.  One CTA per stream of the call, from the first frame of it.
 * Asynchronous on `stream`; allocates nothing and never synchronises, and its launches depend on n alone, so it can be
 * recorded into a CUDA graph and replayed with new records, stream indices and statuses at the same addresses.  Frames
 * may be reused as soon as the call returns. */
int spg_track_frames(spg_handle *h, const spg_track_frame *frames, int32_t n, spg_track_table *tables, int32_t n_tables,
                     double oks_threshold, int32_t max_age, void *stream);

/* ---- smoothing tracked people's keypoints: a One-Euro filter (Casiez, Roussel and Vogel, CHI 2012) per track and joint
 * A stream keeps a table of SPG_TRACK_SLOTS filter slots in caller-owned device memory, keyed by track id (the ids
 * spg_track_frames writes); a zero-filled table is empty.  A slot holds a track's filter state per joint. */
typedef struct spg_smooth_slot {
    int64_t id;                 /* the track id the slot holds */
    int64_t last;               /* the table's clock when the slot was last used */
    int32_t live;               /* 0: the slot is free */
    uint32_t mask;              /* bit g: joint g has state */
    double joint[17][5];        /* per joint xh, yh, dxh, dyh, tj: the filtered position and speed, and its time */
} spg_smooth_slot;
typedef struct spg_smooth_table {
    int64_t clock;              /* frames of the stream seen so far */
    int64_t reserved;
    spg_smooth_slot slots[SPG_TRACK_SLOTS];
} spg_smooth_table;
/* One frame of spg_smooth_frames; every address is device memory, read or written when the launch runs. */
typedef struct spg_smooth_frame {
    const void *record;         /* the frame's wire record, spg_wire_record_bytes(h) bytes (the handle's wire rows) */
    const int32_t *stream;      /* the frame's table index in [0, n_tables), or -1: the frame is skipped */
    const int64_t *ids;         /* [wire rows]: the track id of each of the first n_persons rows, or -1 */
    const double *time;         /* the frame's time in seconds */
    double *xy;                 /* [wire rows][17][2]: the first n_persons rows are written */
} spg_smooth_frame;
/* All arithmetic is float64, one rounding per operation in the order written, no fused multiply-add; TWO_PI =
 * 6.283185307179586.  Per frame of a stream, in call order (several frames of one stream in one call are taken in call
 * order):
 *   1. the table's clock advances;
 *   2. each person with id >= 0 finds the live slot holding its id; a person whose slot an earlier row of the frame
 *      holds (a repeated id) is passed through raw;
 *   3. in row order, each person with id >= 0 and no slot takes the lowest free slot or, in a full table, the slot not
 *      used by this frame of smallest last (ties: the lowest index), whose state is reset (mask and joints 0); a person
 *      whose id an earlier row of the frame took, or who finds no slot (more than SPG_TRACK_SLOTS ids in one frame), is
 *      passed through raw;
 *   4. used slots get last = clock;
 *   5. per joint of a person with a slot: the joint is used when the row's presence mask has it and its x and y are
 *      finite; over the used joints sc = ((xmax - xmin) + (ymax - ymin)) / 2, then sc = sc if sc > 1.0 else 1.0.  A used joint without
 *      state (its mask bit clear) or whose dt = t - tj is not positive and finite takes xh = x, yh = y, dxh = dyh = 0,
 *      tj = t and sets its mask bit; otherwise
 *        vx = (x - xh) / dt / sc, vy = (y - yh) / dt / sc, ad = 1 / (1 + 1 / (TWO_PI * d_cutoff * dt)),
 *        dxh = ad * vx + (1 - ad) * dxh, dyh = ad * vy + (1 - ad) * dyh, fc = min_cutoff + beta * sqrt(dxh * dxh +
 *        dyh * dyh), a = 1 / (1 + 1 / (TWO_PI * fc * dt)), xh = a * x + (1 - a) * xh, yh = a * y + (1 - a) * yh, tj = t.
 *      A used joint's output is (xh, yh); every other joint's is the row's (x, y), and its state is left alone.
 * People with id -1 are passed through raw and change nothing.  A skipped frame (stream -1) changes no table; its rows
 * are passed through raw.  The handle must have 17 output joints; min_cutoff > 0, d_cutoff > 0 and beta >= 0, all
 * finite.  One CTA per stream of the call, from the first frame of it.  Asynchronous on `stream`; allocates nothing and
 * never synchronises, and its launches depend on n alone, so it can be recorded into a CUDA graph and replayed with new
 * records, ids, stream indices and times at the same addresses.  Frames may be reused as soon as the call returns. */
int spg_smooth_frames(spg_handle *h, const spg_smooth_frame *frames, int32_t n, spg_smooth_table *tables, int32_t n_tables,
                      double min_cutoff, double beta, double d_cutoff, void *stream);

/* ---- training samples: the reference data server's Transformer.transform and Heatmapper.create_heatmaps ------
 * (py_cocodata_server/py_data_transformer.py:112-184, py_data_heatmapper.py:50-97).  What a call's samples share, the
 * reference's CanonicalConfig / TransformationParams: */
typedef struct spg_target_params {
    int32_t stride;             /* config.stride: the map is the warped image / stride (must divide out_h and out_w; */
                                /* at most 2901, so that a mask box sum of 255 * stride^2 fits an int)              */
    int32_t gaussian_size;      /* Heatmapper.gaussian_size: a keypoint window is round(x / stride) +- gaussian_size // 2 */
    int32_t out_h, out_w;       /* warped image rows / columns: warpAffine's dsize (config.height, config.width) is */
                                /* (columns, rows), so out_h = config.width and out_w = config.height                 */
    double sigma;               /* transform_params.sigma: keypoint Gaussian */
    double paf_sigma;           /* transform_params.paf_sigma: body-part Gaussian */
    double limb_gaussian_thre;  /* body-part values <= this become 0.01 */
    double paf_thre;            /* transform_params.paf_thre: the body-part box's margin in image pixels */
    int32_t border_image[3];    /* warpAffine's borderValue for the image: (124, 127, 127) */
    int32_t border_mask_miss;   /* 255 */
    int32_t border_mask_all;    /* 0 */
    int32_t reserved;           /* 0 */
} spg_target_params;
/* One sample of spg_targets_warp: device sources and outputs. */
typedef struct spg_target_sample {
    const uint8_t *image;       /* [height][width][3] uint8 (BGR as read), rows image_row_stride bytes apart */
    const uint8_t *mask_miss;   /* [height][width] uint8, rows mask_row_stride bytes apart */
    const uint8_t *mask_all;    /* [height][width] uint8, rows mask_row_stride bytes apart */
    int64_t image_row_stride, mask_row_stride;
    int32_t height, width;
    double matrix[6];           /* the row-major 2x3 matrix AugmentSelection.affine returns (source -> output) */
    float *image_out;           /* [out_h][out_w][3] float32 */
    float *mask_miss_out;       /* [out_h / stride][out_w / stride] float32 */
    float *mask_all_out;        /* [out_h / stride][out_w / stride] float32 */
} spg_target_sample;
/* Per sample: cv2.warpAffine(image, matrix, (out_w, out_h), INTER_LINEAR, BORDER_CONSTANT, border_image) / 255. as
 * float32, and each mask through the same warp (its own border value), cv2.resize(..., INTER_AREA) by the integer factor
 * stride and / 255.  The warp follows OpenCV's uint8 fixed-point algorithm bit for bit; the area resize follows its
 * fast-area arithmetic on the int box sum s: (s + 2) >> 2 at stride 2, else saturate_cast<uchar>(s * (1.f / stride^2)),
 * a float32 product rounded ties to even (not always the correctly rounded s / stride^2: strides 22, 34, 44, ...).  The
 * full-size warped masks are never stored.  Every sample is validated before the first launch (SPG_E_INVALID names the first bad one).
 * Asynchronous on `stream` (never synchronises); `samples` may be reused as soon as the call returns. */
int spg_targets_warp(spg_handle *h, const spg_target_params *params, const spg_target_sample *samples, int32_t n_samples,
                     void *stream);
/* One sample of spg_targets_maps. */
typedef struct spg_target_joints {
    const float *joints;        /* [n_persons][n_parts][3] float32 device (x, y, v) in output pixels; v < 2 is visible */
                                /* (v NaN is not); a visible joint may have any coordinates: one that is NaN or     */
                                /* +-inf, or so large that its window misses the map, draws no keypoint, and a limb */
                                /* with a NaN end draws nothing.  A limb with an infinite end, or whose length      */
                                /* overflows float32, draws the reference's expressions' values (NaN or 1.0 in its  */
                                /* box, as the numpy port computes them).  targets.py refuses non-finite visible    */
                                /* joints, as the reference's int(round(x)) does.                                   */
    int32_t n_persons;          /* any count >= 0 */
    int32_t reserved;           /* 0 */
    const float *mask_all;      /* [out_h / stride][out_w / stride] float32 device: spg_targets_warp's mask_all_out */
    float *labels;              /* [n_limbs + n_parts + 2][out_h / stride][out_w / stride] float32 */
} spg_target_joints;
/* Per sample, Heatmapper.create_heatmaps: body-part channels 0..L-1 (the handle's limb table), keypoint channels
 * L..L+K-1, cv2.erode(mask_all, ones(3, 3)) in channel L+K and the max of the keypoint channels in channel L+K+1, clipped
 * to [0, 1].  Each value is written once.  Validation, asynchrony and reuse of `samples` as spg_targets_warp. */
int spg_targets_maps(spg_handle *h, const spg_target_params *params, const spg_target_joints *samples, int32_t n_samples,
                     void *stream);
/* One sample of spg_targets_tint: a uint8 BGR source tinted in place, and the reference's three draws. */
typedef struct spg_target_tint {
    uint8_t *image;             /* [height][width][3] uint8 device, rows row_stride bytes apart */
    int64_t row_stride;         /* >= 3 * width */
    int32_t height, width;
    int32_t hue, saturation, value;  /* np.random.randint(21), randint(81), randint(61): applied as -10, -20, -20 */
    int32_t row_block;          /* >= 1: OpenCV's HSV->BGR vector block (32 with AVX-512): the last width % row_block */
                                /* pixels of every row are rounded to nearest, the others truncated                  */
} spg_target_tint;
/* Per sample, Transformer.distort_color (py_data_transformer.py:97-110) in place: cv2.cvtColor(COLOR_BGR2HSV), the
 * draws minus (10, 20, 20) added and clamped to [0, 179] / [0, 255] / [0, 255], cv2.cvtColor(COLOR_HSV2BGR), bit for bit
 * with OpenCV's uint8 algorithms.  Run it on the sources before spg_targets_warp reads them.  Validation (draws in range,
 * row_stride, NULL image, row_block), asynchrony and reuse of `samples` as spg_targets_warp. */
int spg_targets_tint(spg_handle *h, const spg_target_tint *samples, int32_t n_samples, void *stream);

/* ---- training loss: the reference's MultiTaskLoss (models/loss_model.py:22-81, 133-161) and MultiTaskLossParallel's
 * L2 (models/loss_model_parallel.py:19-75, 120-139) over nstack x 5 prediction tensors ------------------------------ */
enum {
    SPG_LOSS_FOCAL = 0,  /* MultiTaskLoss: focal L2 (gamma 1, alpha = beta = 0), mask thresholded at 0.5 and weighted */
    SPG_LOSS_L2 = 1      /* MultiTaskLossParallel: plain L2 with the interpolated mask; no batch division            */
};
typedef struct spg_loss_params {
    int32_t mode;                /* SPG_LOSS_FOCAL | SPG_LOSS_L2 */
    int32_t nstack;              /* 1..8 */
    int32_t batch, channels, height, width;  /* of the targets: labels [B][C][H][W], mask_miss [B][1][H][W]; H and W */
                                 /* multiples of 16; scale j of every stack is (H >> j) x (W >> j)                   */
    int32_t heat_start, bkg_start;  /* focal: channels heat_start..bkg_start-1 take keypoint_task_weight */
    double multi_task_weight;    /* focal: channel C - 2's mask weight */
    double keypoint_task_weight; /* focal */
    double nstack_weight[8];     /* [nstack] */
    double scale_weight[5];
    double batch_divisor;        /* focal: opt.batch_size; l2: 1 */
    double scale_weight_sum;     /* sum(scale_weight) as Python sums it */
    double nstack_weight_sum;    /* sum(nstack_weight) */
} spg_loss_params;
/* One prediction tensor, pred_tuple[k][j] at index k * 5 + j: [B][>= C][H >> j][W >> j] with unit column stride.  The
 * loss reads channels 0..C-1.  Strides are in elements.  grad is written by spg_loss_backward only, with its own strides,
 * in the same dtype. */
typedef struct spg_loss_pred {
    const void *data;
    void *grad;
    int64_t batch_stride, chan_stride, row_stride;
    int64_t grad_batch_stride, grad_chan_stride, grad_row_stride;
} spg_loss_pred;
/* Bytes of float64 partial sums spg_loss_forward needs for `params`: 8 x 5 x nstack x batch x channels x height / 16
 * (one per (scale, stack) and CTA); -1 when params is NULL or its nstack, batch, channels or height is out of range. */
int64_t spg_loss_workspace_bytes(const spg_loss_params *params);
/* The loss of the predictions `preds` (nstack * 5 records, `pred_dtype` SPG_F32 | SPG_BF16 | SPG_F16, all the same)
 * against labels (float32 [B][C][H][W]) and mask_miss (float32 [B][1][H][W]), both contiguous and 16-byte aligned:
 * stack_sums [5][nstack] float32 device (the per-stack sums the reference prints, float64 accumulation rounded once) and
 * *loss float32 device (combined from those sums in the reference's order of float32 operations).  A low-precision
 * prediction is the reference applied to its float32 value.  The call's workspace is the caller's: `ticket` one uint32
 * device word that is 0 when the call starts (the call leaves it 0 again, so calls in order on one stream may share it)
 * and `partials` spg_loss_workspace_bytes(params) device bytes, 8-byte aligned, needing no initial value.  Calls with
 * workspaces of their own may run concurrently on different streams, and a call captured in a CUDA graph keeps
 * pointing at the workspace it was given.  Every argument is validated before the first launch (SPG_E_INVALID names the
 * bad one); asynchronous on `stream`; allocates nothing; `params` and `preds` may be reused on return. */
int spg_loss_forward(spg_handle *h, const spg_loss_params *params, const float *mask_miss, const float *labels,
                     const spg_loss_pred *preds, int32_t pred_dtype, float *stack_sums, float *loss, uint32_t *ticket,
                     double *partials, void *stream);
/* Every prediction's gradient of (*grad_output, a float32 device scalar) x loss, written once into preds[i].grad in the
 * prediction's dtype (the float32 gradient rounded once).  Recomputed from the inputs: independent of any forward call.
 * Validation, asynchrony and reuse as spg_loss_forward; needs no workspace and allocates nothing. */
int spg_loss_backward(spg_handle *h, const spg_loss_params *params, const float *mask_miss, const float *labels,
                      const spg_loss_pred *preds, int32_t pred_dtype, const float *grad_output, void *stream);

/* ---- keypoint evaluation: pycocotools' COCOeval(iouType='keypoints') evaluate() and accumulate() (evaluate.py:617-619)
 * on packed device arrays.  A unit is one (category, image) pair, u = category * n_images + image, in the sorted order
 * of params.catIds and params.imgIds.  Every array below is a device array; counts are element counts. -------------- */
typedef struct spg_coco_params {
    const double *iou_thrs;  /* [n_iou]: params.iouThrs */
    const double *rec_thrs;  /* [n_rec]: params.recThrs */
    const double *area_rng;  /* [n_area][2]: params.areaRng */
    const int32_t *max_dets; /* [n_max_dets]: params.maxDets, ascending (evaluate() sorts them); a detection counts */
                             /* for max_dets[m] below that rank and below its unit's kept count                   */
    const double *kpt_vars;  /* [n_kpt]: (params.kpt_oks_sigmas * 2) ** 2 as numpy computes it */
    int32_t n_iou, n_rec, n_area, n_max_dets, n_kpt;  /* n_kpt 1..128 */
} spg_coco_params;
typedef struct spg_coco_data {
    int32_t n_images, n_cats;
    int32_t n_gt, n_dt;   /* ground truths and detections, each grouped by unit, in annotation order within a unit */
    int32_t n_kept;       /* sum over units of min(detections, max_dets[n_max_dets - 1]) */
    int32_t n_ious;       /* sum over units of min(detections, max_dets[n_max_dets - 1]) x ground truths */
    const int32_t *gt_start, *dt_start, *kept_start, *iou_start;  /* [n_units + 1]: each unit's first entry */
    const int32_t *dt_unit;  /* [n_dt] */
    const double *gt_kpts;   /* [n_gt][n_kpt][3] */
    const double *gt_bbox;   /* [n_gt][4] */
    const double *gt_area;   /* [n_gt] */
    const int64_t *gt_id;    /* [n_gt] */
    const uint8_t *gt_flags; /* [n_gt]: SPG_COCO_IGNORE | SPG_COCO_CROWD */
    const double *dt_kpts;   /* [n_dt][n_kpt][3] */
    const double *dt_area, *dt_score;  /* [n_dt] */
    const int64_t *dt_id;    /* [n_dt] */
} spg_coco_data;
enum {
    SPG_COCO_IGNORE = 1, /* _prepare's gt['ignore']: iscrowd or num_keypoints == 0 */
    SPG_COCO_CROWD = 2   /* int(gt['iscrowd']) != 0 */
};
/* evaluate()'s results, which accumulate() reads. */
typedef struct spg_coco_eval {
    double *ious;          /* [n_ious]: per unit its [kept][gts] OKS matrix (computeOks), rows in score order */
    int32_t *dt_order;     /* [n_dt]: per unit, its detections' indices sorted by descending score (stable) */
    int32_t *dt_rank;      /* [n_dt]: each detection's position in its unit's dt_order */
    int32_t *cat_order;    /* [n_dt]: per category, its detections in image order stably sorted by descending score */
    int32_t *gt_order;     /* [n_area][n_gt]: per unit, its ground truths' indices in evaluateImg's order */
    uint8_t *gt_ignore;    /* [n_area][n_gt]: evalImgs' gtIgnore, in gt_order */
    int64_t *gt_matches;   /* [n_area][n_iou][n_gt]: gtMatches (the matched detection's id, or 0), in gt_order */
    int64_t *dt_matches;   /* [n_area][n_iou][n_kept]: dtMatches (the matched ground truth's id, or 0), in dt_order */
    uint8_t *dt_ignore;    /* [n_area][n_iou][n_kept]: dtIgnore */
} spg_coco_eval;
/* computeOks and evaluateImg for every unit, area range and threshold.  Sorts use NaN-last keys with -0.0 == 0.0 and
 * keep ties in input order, as numpy's mergesort.  Every count and product of counts must fit in int32; arguments are
 * validated before the first launch.  Asynchronous on `stream`; the handle's sort scratch grows on demand, so calls on
 * one handle must not run concurrently on different streams. */
int spg_coco_evaluate(spg_handle *h, const spg_coco_params *params, const spg_coco_data *data, const spg_coco_eval *eval,
                      void *stream);
/* accumulate() from spg_coco_evaluate's results with the same params and data: precision and scores
 * [n_iou][n_rec][n_cats][n_area][n_max_dets] and recall [n_iou][n_cats][n_area][n_max_dets], float64; -1 where a
 * (category, area range) has no ground truth that is not ignored.  Asynchronous; the scratch grows on demand. */
int spg_coco_accumulate(spg_handle *h, const spg_coco_params *params, const spg_coco_data *data, const spg_coco_eval *eval,
                        double *precision, double *recall, double *scores, void *stream);

/* ---- JPEG decoding: what cv2.imread(path) returns for the validation images (evaluate.py:502), on the device ---------
 * Baseline and extended-sequential Huffman files (SOF0 / SOF1) with 8-bit samples, 8- or 16-bit quantisation tables, one
 * component (returned as BGR, as IMREAD_COLOR does) or three YCbCr components in one interleaved scan with luma sampling
 * 1x1, 2x1, 1x2 or 2x2 and 1x1 chroma, with or without restart intervals, any APPn / COM segments, and the EXIF
 * orientation OpenCV applies.  The output equals OpenCV 4.x with libjpeg-turbo's default decode (islow IDCT, fancy
 * upsampling) bit for bit.  Every other file is refused with a reason, for the caller to read with cv2. */
enum {
    SPG_JPEG_OK = 0,
    SPG_JPEG_NOT_JPEG = 1,   /* no SOI marker */
    SPG_JPEG_TRUNCATED = 2,  /* a segment or the entropy-coded data runs past the end of the buffer, or no EOI */
    SPG_JPEG_PROCESS = 3,    /* progressive, lossless, arithmetic-coded or hierarchical */
    SPG_JPEG_PRECISION = 4,  /* samples other than 8-bit */
    SPG_JPEG_COLOR = 5,      /* not 1 or 3 components, or 3 that libjpeg treats as RGB (Adobe transform 0, ids 'R','G','B') */
    SPG_JPEG_SAMPLING = 6,   /* sampling other than luma 1x1 / 2x1 / 1x2 / 2x2 with 1x1 chroma */
    SPG_JPEG_SCAN = 7,       /* more than one scan, a scan without every component in frame order, or Ss/Se/Ah/Al */
    SPG_JPEG_TABLES = 8,     /* a missing or invalid quantisation or Huffman table */
    SPG_JPEG_MALFORMED = 9,  /* a length, count or marker libjpeg rejects or treats as corrupt */
    SPG_JPEG_EXIF = 10,      /* an EXIF block whose orientation cannot be read the way OpenCV reads it */
    SPG_JPEG_CORRUPT = 11,   /* decoder: a bad Huffman code, a coefficient index past 63, too few bits or blocks */
    SPG_JPEG_RANGE = 12      /* decoder: a block outside the range where libjpeg-turbo's SIMD and C islow IDCTs agree */
};
/* A decoding table of one Huffman table. */
typedef struct spg_jpeg_huff {
    uint16_t lookup[512];    /* the next 9 bits -> (code length << 8) | symbol; 0: the code is longer than 9 bits */
    int32_t maxcode[18];     /* [l]: the largest code of length l (1..16), -1 when there is none */
    int32_t valoff[18];      /* [l]: symbols[code + valoff[l]] is the symbol of a code of length l */
    uint8_t symbols[256];
} spg_jpeg_huff;
/* One parsed file.  spg_jpeg_parse fills everything down to `ac`; the caller sets the last three fields for
 * spg_jpeg_decode_ragged. */
typedef struct spg_jpeg_record {
    int32_t status;          /* SPG_JPEG_OK, or why the file is refused (the fields below are then unspecified) */
    int32_t orientation;     /* EXIF orientation 1..8 (1 when absent) */
    int32_t height, width;   /* the decoded image: after the orientation */
    int32_t frame_height, frame_width;  /* as coded (SOF) */
    int32_t n_components;    /* 1 or 3 */
    int32_t h_samp, v_samp;  /* luma sampling factors; chroma is 1x1 (1 and 1 for one component) */
    int32_t mcus_x, mcus_y;  /* MCU columns and rows */
    int32_t blocks_per_mcu;  /* h_samp * v_samp + 2, or 1 */
    int32_t restart_interval;  /* MCUs per restart interval; 0: none */
    int32_t n_intervals;     /* ceil(mcus_x * mcus_y / restart_interval), or 1 */
    int64_t scan_offset;     /* the entropy-coded data: its first byte in the file */
    int64_t scan_length;     /* its bytes, up to the 0xFF that starts EOI (restart markers and stuffing included) */
    uint16_t quant[3][64];   /* per component, natural (row-major) order */
    spg_jpeg_huff dc[3], ac[3];  /* per component */
    const uint8_t *data;     /* device: the file's bytes (at least scan_offset + scan_length of them) */
    uint8_t *out;            /* device: [height][width][3] uint8 BGR */
    int32_t *decode_status;  /* device: set to SPG_JPEG_OK, SPG_JPEG_CORRUPT or SPG_JPEG_RANGE by the decode */
} spg_jpeg_record;
/* Host only (no device, no handle): parse `size` bytes at `data` into *record.  Every length and count is checked
 * against the buffer; nothing outside it is read.  Returns SPG_OK with record->status saying whether the file can be
 * decoded on the device, or SPG_E_INVALID for a NULL record, a negative size or NULL data with a positive size. */
int spg_jpeg_parse(const uint8_t *data, int64_t size, spg_jpeg_record *record);
/* Decode n files parsed with status SPG_JPEG_OK into their `out` images, every image of the call in each launch.  Each
 * record's decode_status gets SPG_JPEG_OK, or SPG_JPEG_CORRUPT / SPG_JPEG_RANGE for an image whose data the device
 * path cannot reproduce cv2 on: its `out` is then unspecified and the file is for cv2.  Records are validated before
 * the first launch (SPG_E_INVALID names the first bad one).  Asynchronous on `stream`; `records` may be reused on
 * return.  The handle's scratch (the unstuffed data, coefficients and planes) grows on demand, so calls on one handle
 * must not run concurrently on different streams. */
int spg_jpeg_decode_ragged(spg_handle *h, const spg_jpeg_record *records, int32_t n, void *stream);
/* The decode of one frame, which can be recorded into a CUDA graph (see "frames recorded into a CUDA graph") and replayed
 * for every frame of one format.  The format is what the recorded launches depend on: frame height and width, component
 * count, luma sampling, restart interval and EXIF orientation, taken from the host record `format` (validated as
 * spg_jpeg_decode_ragged validates a record; its `out` and `decode_status` are the frame's output and status).  The rest
 * is read on the device when the launches run, from `device_record` (a device copy of the frame's parsed record): the
 * bytes at `data`, the scan's offset and length, the quantisation and Huffman tables.  The grids cover max_scan_bytes of
 * entropy-coded data, 1 .. 2^28 - 1; a frame whose scan_length exceeds it gets SPG_JPEG_CORRUPT, and no byte past a
 * frame's own data is read, whatever an earlier, longer frame left in the buffers.  The frame's image and status are
 * those spg_jpeg_decode_ragged gives.  Asynchronous on `stream`; never synchronises or allocates while `stream`
 * captures: a scratch buffer too small then returns SPG_E_CAPTURE with nothing enqueued.  The calls of one handle share
 * its scratch, so they must run in stream order. */
int spg_jpeg_decode_frame(spg_handle *h, const spg_jpeg_record *device_record, const spg_jpeg_record *format,
                          int64_t max_scan_bytes, void *stream);
/* Grow, outside any capture, the scratch spg_jpeg_decode_frame needs for `format` and max_scan_bytes; *moved (may be
 * NULL) as for spg_reserve_frame: 1 when the buffer was reallocated, which invalidates graphs that recorded this handle's
 * JPEG frame decodes.  Synchronous; must not be called while any stream of the device captures. */
int spg_jpeg_reserve_frame(spg_handle *h, const spg_jpeg_record *format, int64_t max_scan_bytes, int32_t *moved);
/* spg_jpeg_decode_frame for n frames in each launch (spg_jpeg_decode_frame is this call with n = 1): member i has its own
 * format formats[i] (host), its own capacity capacities[i] in scan bytes (host) and its own device record
 * device_records[i] (a device array of n records).  Interval and subsequence members mix in one call.  Each member's
 * grids cover its capacity; its CTAs past its own chunk or subsequence count return at once; a member whose scan_length
 * exceeds its capacity gets SPG_JPEG_CORRUPT and no byte past a member's own data is read.  Each member's image and
 * status equal those spg_jpeg_decode_ragged gives.  Asynchronous, capture rules and stream order as
 * spg_jpeg_decode_frame. */
int spg_jpeg_decode_frames(spg_handle *h, const spg_jpeg_record *device_records, const spg_jpeg_record *formats,
                           const int64_t *capacities, int32_t n, void *stream);
/* Grow, outside any capture, the scratch spg_jpeg_decode_frames needs for these n formats and capacities; *moved as for
 * spg_jpeg_reserve_frame (which is this call with n = 1). */
int spg_jpeg_reserve_frames(spg_handle *h, const spg_jpeg_record *formats, const int64_t *capacities, int32_t n,
                            int32_t *moved);

/* ---- stage entry points (stage-wise parity; each consumes the previous stage's device state) ---- */
/* find_peaks: evaluate.py:169-203 = util.keypoint_heatmap_nms (utils/util.py:177-183) + util.refine_centroid (:186-211) */
int spg_nms_peaks(spg_handle *h, const float *heat_dev, int64_t image_stride, int64_t chan_stride,
                  int32_t n_images, int32_t height, int32_t width, const spg_params *params, void *stream);
/* find_connections, scoring half: evaluate.py:211-255 (every candidate pair of every limb) */
int spg_limb_score(spg_handle *h, const void *paf_dev, int32_t paf_dtype, int64_t image_stride,
                   int64_t chan_stride, int32_t n_images, int32_t height, int32_t width, double image_extent,
                   const spg_params *params, void *stream);
/* find_connections, matching half: evaluate.py:259-274 (stable sort by priority + greedy assignment) */
int spg_limb_match(spg_handle *h, int32_t n_images, const spg_params *params, void *stream);
/* find_people + process() tail: evaluate.py:279-498 and :523-543 */
int spg_assemble(spg_handle *h, int32_t n_images, const spg_params *params, void *stream);
/* the two previous stages fused in one kernel (one CTA per image: matcher warps feed the assembler warp limb by limb
 * through shared memory); what spg_group_batch / spg_group_host run.  Same outputs as the two calls back to back. */
int spg_match_assemble(spg_handle *h, int32_t n_images, const spg_params *params, void *stream);

/* ---- host <-> device state transfer for the stage-wise drop-in functions ---------------------- */
/* peaks of ONE image, part-major flat arrays as the reference's all_peaks flattens (evaluate.py:283):
 * part_count[K], x[n], y[n], score[n] with n = sum(part_count); image_index selects the slot */
int spg_upload_peaks(spg_handle *h, int32_t image_index, const int32_t *part_count, const double *x, const double *y,
                     const float *score, void *stream);
/* connections of ONE image: conn_count[L] (-1 = special), rows concatenated over limbs:
 * ij[m][2] (indices inside candA/candB), score[m], norm[m] */
int spg_upload_connections(spg_handle *h, int32_t image_index, const int32_t *conn_count, const int32_t *ij,
                           const double *score, const double *norm, void *stream);

/* downloads synchronise `stream`.  Arrays are dense with the handle's capacities; NULL pointers are skipped. */
int spg_download_peaks(spg_handle *h, int32_t n_images, int32_t *peak_count /*[N][K]*/, double *x, double *y,
                       float *score, uint32_t *anchor /*[N][K][cap_peaks] each*/, void *stream);
int spg_download_connections(spg_handle *h, int32_t n_images, int32_t *conn_count /*[N][L]*/,
                             int32_t *cand_count /*[N][L]*/, uint32_t *ij, double *score,
                             double *norm /*[N][L][cap_peaks] each*/, void *stream);
int spg_download_people(spg_handle *h, int32_t n_images, int32_t *n_persons /*[N]*/,
                        double *subset /*[N][cap_rows][K+2][2]*/, double *people_xy /*[N][cap_rows][J][2]*/,
                        double *people_score /*[N][cap_rows]*/, void *stream);
int spg_download_status(spg_handle *h, int32_t n_images, uint32_t *status /*[N]*/, void *stream);

/* ---- wire records: what leaves the GPU (format_results, evaluate.py:563-582) ------------------------------- */
/* One fixed-stride record per image: an 8-byte header followed by `rows` person rows of (2*n_out_joints + 2)
 * 8-byte words -- x0,y0,...,x16,y16 (doubles, COCO order, evaluate.py:523-539), the person score 1 - 1/total
 * (double, :541), and a uint64 presence mask (bit g set: joint g was found; clear: the reference's `X, Y = 0, 0`
 * placeholder, :531) -- i.e. exactly the payload format_results turns into {"keypoints": [x,y,v]*17, "score": s}
 * (v = x>0 or y>0).
 * Only the first n_persons rows are written; the rest of the slot is never touched, so when the record lives in
 * another GPU's memory only live rows cross NVLink. */
typedef struct spg_wire_header {
    int32_t n_persons;
    uint32_t status; /* SPG_ST_* bits of the image */
} spg_wire_header;
/* bytes of one image's record for this handle: 8 + wire_rows * (2*n_out_joints + 2) * 8 */
int64_t spg_wire_record_bytes(const spg_handle *h);
/* Direct the assemble stage to ALSO emit wire records: image i of a call goes to
 * (char*)wire_dev + (first_record + i) * spg_wire_record_bytes().  `wire_dev` may be local device memory or PEER
 * memory (another GPU's buffer opened with spg_wire_open: the records then travel over NVLink as the kernel stores
 * them -- the gather of the person lists fused into the kernel that produces them, no collective kernel).
 * wire_rows <= max_person_rows caps the rows per record (SPG_ST_WIRE_OVERFLOW).  NULL switches wire output off. */
int spg_set_wire_output(spg_handle *h, void *wire_dev, int64_t first_record, int32_t wire_rows);

/* Arm the NEXT single-launch assemble stage (spg_assemble / spg_match_assemble / spg_group_batch; not spg_group_host,
 * which launches per chunk) to publish its own completion: the CTA that finishes last release-stores `value` into
 * *word_dev (local or peer memory) after every record of the launch has been stored -- the producer's "my records
 * have landed" without a separate signalling kernel.  One shot; NULL disarms.  Needs spg_set_wire_output. */
int spg_arm_wire_signal(spg_handle *h, uint64_t *word_dev, uint64_t value);

/* ---- peer memory + stream-ordered signalling for the NVLink gather (no NCCL in the data path) ------------ */
/* A sink is plain device memory that other processes (one per GPU) can map: create it on the owner, send the
 * 64-byte handle to the peers by any means (torch.distributed), open it there.  Zero-filled on creation. */
int spg_wire_create(int32_t device, uint64_t bytes, void **dev_ptr, unsigned char ipc_handle[64]);
int spg_wire_open(int32_t device, const unsigned char ipc_handle[64], void **peer_ptr);
int spg_wire_close(void *peer_ptr);
int spg_wire_destroy(int32_t device, void *dev_ptr);
/* release-store `value` into a 64-bit word (local or peer memory) once everything earlier on `stream` has
 * completed: a one-thread kernel (fence.sys + st.release.sys).  The producer's "my records have landed". */
int spg_wire_signal(int32_t device, uint64_t *word_dev, uint64_t value, void *stream);
/* the same value into up to 32 words (each local or peer memory) with ONE launch: the consumer's acknowledgement to all ranks */
int spg_wire_signal_many(int32_t device, uint64_t *const *words_dev, int32_t n_words, uint64_t value, void *stream);
/* make `stream` wait until *word_dev >= value.  `word_dev` must be LOCAL device memory: the wait is a stream
 * memory operation (cuStreamWaitValue64), executed by the copy/compute front end -- no kernel sits on an SM
 * spinning, so it cannot collide with the persistent kernels that own every SM.  */
int spg_wire_wait(int32_t device, const uint64_t *word_dev, uint64_t value, void *stream);

/* number of kernel launches issued by this handle since creation (bench.py's gpu_launches) */
int64_t spg_launch_count(const spg_handle *h);
/* name of the kernel variant the last launch of a stage used (0 nms_peaks, 1 limb_score, 2 limb_match, 3 assemble,
 * 4 post-network stage, 5 pre-network stage, 6 training samples, 7 training loss, 8 keypoint evaluation, 9 JPEG decode,
 * 10 YUV conversion, 11 tracking, 12 smoothing);
 * "" before the first launch.  Profiling aid: lets bench.py label its per-kernel numbers with the ncu kernel name. */
const char *spg_stage_kernel(const spg_handle *h, int32_t stage);

#ifdef __cplusplus
}
#endif
#endif /* SPGROUP_H_ */
