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

#define SPG_ABI_VERSION 2

enum {
    SPG_OK = 0,
    SPG_E_INVALID = -1,   /* bad argument (shape, capacity, alignment, null pointer) */
    SPG_E_CUDA = -2,      /* a CUDA runtime call failed; see spg_last_error          */
    SPG_E_NO_DEVICE = -3, /* no CUDA device / not an sm_90 part                      */
    SPG_E_STATE = -4      /* stage called before the stage that feeds it             */
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

/* ---- training samples: the reference data server's Transformer.transform and Heatmapper.create_heatmaps ------
 * (py_cocodata_server/py_data_transformer.py:112-184, py_data_heatmapper.py:50-97).  What a call's samples share, the
 * reference's CanonicalConfig / TransformationParams: */
typedef struct spg_target_params {
    int32_t stride;             /* config.stride: the map is the warped image / stride (must divide out_h and out_w) */
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
 * stride and / 255.  The warp and the area resize follow OpenCV's uint8 algorithms bit for bit; the full-size warped masks
 * are never stored.  Every sample is validated before the first launch (SPG_E_INVALID names the first bad one).
 * Asynchronous on `stream` (never synchronises); `samples` may be reused as soon as the call returns. */
int spg_targets_warp(spg_handle *h, const spg_target_params *params, const spg_target_sample *samples, int32_t n_samples,
                     void *stream);
/* One sample of spg_targets_maps. */
typedef struct spg_target_joints {
    const float *joints;        /* [n_persons][n_parts][3] float32 device (x, y, v) in output pixels; v < 2 is visible */
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
/* The loss of the predictions `preds` (nstack * 5 records, `pred_dtype` SPG_F32 | SPG_BF16 | SPG_F16, all the same)
 * against labels (float32 [B][C][H][W]) and mask_miss (float32 [B][1][H][W]), both contiguous and 16-byte aligned:
 * stack_sums [5][nstack] float32 device (the per-stack sums the reference prints, float64 accumulation rounded once) and
 * *loss float32 device (combined from those sums in the reference's order of float32 operations).  A low-precision
 * prediction is the reference applied to its float32 value.  Every argument is validated before the first launch
 * (SPG_E_INVALID names the bad one); asynchronous on `stream`; `params` and `preds` may be reused on return.  The
 * handle's partial-sum buffer grows on demand (a call with no larger shape than an earlier one allocates nothing); calls
 * on one handle must not run concurrently on different streams. */
int spg_loss_forward(spg_handle *h, const spg_loss_params *params, const float *mask_miss, const float *labels,
                     const spg_loss_pred *preds, int32_t pred_dtype, float *stack_sums, float *loss, void *stream);
/* Every prediction's gradient of (*grad_output, a float32 device scalar) x loss, written once into preds[i].grad in the
 * prediction's dtype (the float32 gradient rounded once).  Recomputed from the inputs: independent of any forward call.
 * Validation, asynchrony and reuse as spg_loss_forward; allocates nothing. */
int spg_loss_backward(spg_handle *h, const spg_loss_params *params, const float *mask_miss, const float *labels,
                      const spg_loss_pred *preds, int32_t pred_dtype, const float *grad_output, void *stream);

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
 * 4 post-network stage, 5 pre-network stage, 6 training samples, 7 training loss);
 * "" before the first launch.  Profiling aid: lets bench.py label its per-kernel numbers with the ncu kernel name. */
const char *spg_stage_kernel(const spg_handle *h, int32_t stage);

#ifdef __cplusplus
}
#endif
#endif /* SPGROUP_H_ */
