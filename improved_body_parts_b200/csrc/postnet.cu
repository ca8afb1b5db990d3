// postnet.cu -- the post-network stage (postnet.cuh: the network output resized, averaged over the scales and the
// mirror pair, and rotated back), the pre-network stage (prenet.cuh: the network input resized, padded and rotated) and
// the frame reservations that size both stages' scratch before a CUDA graph captures them.
#include "runtime.cuh"

#include <cmath>
#include <cstdio>

#include "postnet.cuh"
#include "prenet.cuh"

using namespace spg;

extern "C" {

// ---- post-network stage ------------------------------------------------------------------------
int spg_postnet(spg_handle *h, const spg_postnet_desc *d, int32_t n, int32_t H, int32_t W, float *heat_out, void *paf_out,
                int32_t paf_dtype, void *stream) {
    return spg_postnet_rotated(h, d, nullptr, n, H, W, heat_out, paf_out, paf_dtype, stream);
}

// Channels per CTA: a CTA builds its tile's tables once and walks over a chunk of channels -- as many as still leave
// ~ctas_per_sm CTAs per SM over `tiles` tiles (a few resident: several waves).  ctas_per_sm 0: one channel per CTA.
static int post_chan_chunk(const spg_handle *h, int n_out, long long tiles, int ctas_per_sm) {
    const int n_chunks = ctas_per_sm == 0 ? n_out
                                          : (int)std::min<long long>(n_out, std::max<long long>(1, ((long long)h->sm_count * ctas_per_sm + tiles - 1) / tiles));
    return (n_out + n_chunks - 1) / n_chunks;
}

static int postnet_grid(spg_handle *h, PostArgs &a, const PostImage &im, int n, int ctas_per_sm, dim3 *grid) {
    const long long tiles = (long long)im.tiles_x * im.tiles_y;
    if (tiles > 0x7fffffffLL || n > 65535) return fail(h, SPG_E_INVALID, "postnet grid too large");
    a.chan_chunk = post_chan_chunk(h, a.n_out, tiles * n, ctas_per_sm);
    *grid = dim3((unsigned)tiles, (unsigned)((a.n_out + a.chan_chunk - 1) / a.chan_chunk), (unsigned)n);
    return SPG_OK;
}

// CTAs per SM the channel chunks aim at: the identity kernel (4 resident per SM) and the four-phase kernels (2 resident)
constexpr int kPostIdentCtasPerSm = 32, kPostCtasPerSm = 16;

// output tile of the four-phase kernels: as large as the shared-memory tiles of the intermediate / source allow
static int post_tile_dim(double s2, double s1, int cap1, int cap0, int maxd, double margin) {
    const double c1 = std::min((double)cap1, ((double)cap0 - 7.0) / s1) - margin;  // intermediate span allowed
    return std::max(1, std::min(maxd, (int)(c1 / std::max(s2, 1e-6))));
}

// one item's network output and the steps of its resize to the H x W image
static PostScale post_scale(const void *net, int dtype, int64_t img_stride, int64_t pair_stride, int64_t chan_stride, int h, int w,
                            int crop_h, int crop_w, int H, int W) {
    PostScale s{};
    s.net = net; s.net_is_f16 = dtype == SPG_F16;
    s.img_stride = img_stride; s.pair_stride = pair_stride; s.chan_stride = chan_stride;
    s.h = h; s.w = w; s.crop_h = crop_h; s.crop_w = crop_w;
    // cv2.resize(dsize): inv_scale = dst/src, scale = 1/inv_scale (two roundings, as OpenCV)
    s.sx2 = 1.0 / ((double)W / (double)crop_w);
    s.sy2 = 1.0 / ((double)H / (double)crop_h);
    return s;
}

// A scale's or an item's network output (`what` names it in the error): present, float32 or float16, and its crop
// inside the h x w output up-sampled by `stride`
static int check_net_out(spg_handle *h, const char *what, const void *net, int dtype, int hn, int wn, int crop_h, int crop_w,
                         int stride) {
    if (!net) return fail(h, SPG_E_INVALID, "%s: net_out is NULL", what);
    if (dtype != SPG_F32 && dtype != SPG_F16) return fail(h, SPG_E_INVALID, "%s: network output must be SPG_F32 or SPG_F16", what);
    if (hn < 1 || wn < 1 || crop_h < 1 || crop_w < 1 || crop_h > hn * stride || crop_w > wn * stride)
        return fail(h, SPG_E_INVALID, "%s: crop %dx%d does not fit the up-sampled %dx%d output", what, crop_h, crop_w, hn * stride,
                    wn * stride);
    return SPG_OK;
}

// A rotation entry: apply 0 or 1, reserved 0 and a finite matrix.  `what` names the entry in the error and `apply` its
// apply field.
static int check_rotation(spg_handle *h, const char *what, const char *apply, const spg_postnet_rotation &r) {
    if ((r.apply != 0 && r.apply != 1) || r.reserved != 0)
        return fail(h, SPG_E_INVALID, "%s: %s must be 0 or 1 and reserved 0", what, apply);
    for (int k = 0; k < 6; k++)
        if (!std::isfinite(r.matrix[k])) return fail(h, SPG_E_INVALID, "%s: matrix entry %d is not finite", what, k);
    return SPG_OK;
}

// The arguments every launch of a call shares: the output channels (K keypoint, then L body part) and the network
// channels each one averages, validated; the scale count, NaN scrub, body-part dtype and the x stride resize's step.
static int post_common(spg_handle *h, int stride, int n_scales, int paf_chan0, int heat_chan0, const int32_t *flip_paf_ord,
                       const int32_t *flip_heat_ord, int nan_scrub, int paf_dtype, PostArgs &a) {
    const Workspace &ws = h->ws;
    if (ws.K + ws.L > kMaxNetChannels) return fail(h, SPG_E_INVALID, "too many channels for postnet");
    a.n_out = ws.K + ws.L; a.K = ws.K;
    for (int c = 0; c < ws.K; c++) {
        if (flip_heat_ord[c] < 0 || flip_heat_ord[c] >= ws.K) return fail(h, SPG_E_INVALID, "flip_heat_ord[%d] out of range", c);
        a.src_chan[c] = (short)(heat_chan0 + c);
        a.flip_chan[c] = (short)(heat_chan0 + flip_heat_ord[c]);
    }
    for (int k = 0; k < ws.L; k++) {
        if (flip_paf_ord[k] < 0 || flip_paf_ord[k] >= ws.L) return fail(h, SPG_E_INVALID, "flip_paf_ord[%d] out of range", k);
        a.src_chan[ws.K + k] = (short)(paf_chan0 + k);
        a.flip_chan[ws.K + k] = (short)(paf_chan0 + flip_paf_ord[k]);
    }
    a.n_scales = n_scales; a.nan_scrub = nan_scrub != 0; a.paf_is_f64 = paf_dtype == SPG_F64;
    a.sx1 = 1.0 / (double)stride; a.sy1 = a.sx1;  // cv2.resize(fx = stride): scale = 1/fx
    return SPG_OK;
}

// The kernel families of the post-network stage (PostPlan::family), each with its per-launch and its ragged kernels by
// template flags [single][ident][f16] (nullptr: not instantiated), under the names spg_stage_kernel reports (the ragged
// ones by [single]).
enum : int { kPostIdent, kPostFourPhase, kPostRotated, kPostGeneric };
struct PostKernels {
    const char *name;
    void (*fn[2][2][2])(PostArgs, PostImage);
    const char *ragged_name[2];
    void (*ragged[2][2][2])(PostArgs, PostTable);
};
static const PostKernels kPostKernels[4] = {
    {"postnet_x4_ident_kernel", {{}, {{}, {postnet_x4_ident_kernel<false>, postnet_x4_ident_kernel<true>}}},
     {"", "postnet_x4_ident_ragged_kernel"}, {{}, {{}, {postnet_x4_ident_ragged_kernel<false>, postnet_x4_ident_ragged_kernel<true>}}}},
    {"postnet_kernel",
     {{{postnet_kernel<false, false, false>, postnet_kernel<false, false, true>}, {postnet_kernel<false, true, false>, postnet_kernel<false, true, true>}},
      {{postnet_kernel<true, false, false>, postnet_kernel<true, false, true>}, {}}},
     {"postnet_items_ragged_kernel", "postnet_ragged_kernel"},
     {{{postnet_items_ragged_kernel<false, false>, postnet_items_ragged_kernel<false, true>},
       {postnet_items_ragged_kernel<true, false>, postnet_items_ragged_kernel<true, true>}},
      {{postnet_ragged_kernel<false>, postnet_ragged_kernel<true>}, {}}}},
    {"postnet_rot_kernel",
     {{{postnet_rot_kernel<false, false>, postnet_rot_kernel<false, true>}, {}}, {{postnet_rot_kernel<true, false>, postnet_rot_kernel<true, true>}, {}}},
     {"postnet_rot_ragged_kernel", "postnet_rot_ragged_kernel"},
     {{{postnet_rot_ragged_kernel<false, false>, postnet_rot_ragged_kernel<false, true>}, {}},
      {{postnet_rot_ragged_kernel<true, false>, postnet_rot_ragged_kernel<true, true>}, {}}}},
    {"postnet_generic_kernel", {{{postnet_generic_kernel}}}, {}, {}},
};

struct PostPlan {
    int family;
    bool single, ident, f16;  // the kernel's template flags (kPostKernels[family].fn)
    int tile_w, tile_h;
    int ctas_per_sm;          // target of the channel chunk (post_chan_chunk)
    size_t smem;              // dynamic shared memory
};

// The schedule of one launch over the n_fused items of image im (im.sc, im.H x im.W; a rotated item: im.rot).
// `single`: one scale in the whole scale loop; `item` names the item in the error.
static int plan_post(spg_handle *h, const PostImage &im, int n_fused, bool single, int stride, bool rotated, int item, PostPlan *pl) {
    const PostScale *sc = im.sc;
    const int H = im.H, W = im.W;
    const double *rot = rotated ? im.rot : nullptr;
    const double s1 = 1.0 / (double)stride;  // PostArgs::sx1 (post_common)
    if (stride != 4) {
        *pl = PostPlan{kPostGeneric, false, false, false, post_tile_dim(sc[0].sx2, s1, kPostC1, kPostCS, kPostTW, 7.0),
                       post_tile_dim(sc[0].sy2, s1, kPostR1, kPostRS, kPostTH, 7.0), 0, 0};
        return SPG_OK;
    }
    const PostScale &S = sc[0];
    if (rot) {
        // the largest tile (up to 64 x 32) whose crop span and rotated box fit the kernel's buffers: a span of cw x ch
        // crop pixels reads a box of |m0| cw + |m1| ch (+ 7, the box's margins) columns of the x4 grid, and its x4
        // groups add up to two more
        const bool ident = S.crop_h == H && S.crop_w == W;
        auto fits = [&](int tw, int th) {
            const double cw = ident ? tw : tw * S.sx2 + 5.0, ch = ident ? th : th * S.sy2 + 5.0;
            const double bw = std::fabs(rot[0]) * cw + std::fabs(rot[1]) * ch + 7.0;
            const double bh = std::fabs(rot[3]) * cw + std::fabs(rot[4]) * ch + 7.0;
            return cw <= kPostF_C1 && ch <= kPostR_R1 && bw / 4.0 + 2.0 <= kPostF_Q && bh / 4.0 + 2.0 <= kPostF_P;
        };
        int tw = kPostTW, th = kPostTH;
        while (!fits(tw, th) && (tw > 1 || th > 1)) {
            if (tw * S.sx2 >= th * S.sy2 && tw > 1) tw--;
            else if (th > 1) th--;
            else tw--;
        }
        if (!fits(tw, th)) return fail(h, SPG_E_INVALID, "rotation %d: the crop is too large for the image to warp it", item);
        *pl = PostPlan{kPostRotated, single, false, S.net_is_f16 != 0, tw, th, kPostCtasPerSm, postR_smem_bytes()};
        return SPG_OK;
    }
    bool ident = true, any16 = false, all16 = true;
    for (int t = 0; t < n_fused; t++) {
        ident = ident && sc[t].crop_h == H && sc[t].crop_w == W;
        any16 = any16 || sc[t].net_is_f16;
        all16 = all16 && sc[t].net_is_f16;
    }
    if (any16 != all16) return fail(h, SPG_E_INVALID, "the network outputs of all scales must have the same dtype");
    if (single && ident) {  // the reference's default: its own kernel (two passes, per-thread state hoisted)
        *pl = PostPlan{kPostIdent, true, true, all16, kPostI_TW, kPostI_TH, kPostIdentCtasPerSm, 0};
        return SPG_OK;
    }
    *pl = PostPlan{kPostFourPhase, single, ident, all16, kPostTW, kPostTH, kPostCtasPerSm, postF_smem_bytes(single ? 1 : kPostMaxScales)};
    for (int t = 0; t < n_fused; t++) {  // as large as every scale's second resize allows
        pl->tile_w = std::min(pl->tile_w, post_tile_dim(sc[t].sx2, s1, kPostF_C1, kPostF_CS, kPostTW, 13.0));
        pl->tile_h = std::min(pl->tile_h, post_tile_dim(sc[t].sy2, s1, kPostF_R1, kPostF_RS, kPostTH, 13.0));
    }
    return SPG_OK;
}

// Completes image im's descriptor for one group of n_fused items, whose scales, size, output planes and float64 sums the
// caller has set: the inverse of a rotated item's warp matrix (rot: the forward matrix, nullptr: not rotated) and the
// tiling plan_post picks for the image alone.
static int post_image(spg_handle *h, PostImage &im, int n_fused, bool single, int stride, const double *rot, int item, PostPlan *pl) {
    if (rot) invert_affine(rot, im.rot);
    int rc;
    if ((rc = plan_post(h, im, n_fused, single, stride, rot != nullptr, item, pl))) return rc;
    im.tile_w = pl->tile_w;
    im.tile_h = pl->tile_h;
    im.tiles_x = (im.W + im.tile_w - 1) / im.tile_w;
    im.tiles_y = (im.H + im.tile_h - 1) / im.tile_h;
    return SPG_OK;
}

int spg_postnet_rotated(spg_handle *h, const spg_postnet_desc *d, const spg_postnet_rotation *rot, int32_t n, int32_t H, int32_t W,
                        float *heat_out, void *paf_out, int32_t paf_dtype, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (!d || !d->scales || d->n_scales < 1 || !d->flip_paf_ord || !d->flip_heat_ord) return fail(h, SPG_E_INVALID, "postnet descriptor incomplete");
    bool any_rot = false;
    int rc;
    char what[32];
    for (int t = 0; rot && t < d->n_scales; t++) {
        snprintf(what, sizeof what, "rotation %d", t);
        if ((rc = check_rotation(h, what, "apply", rot[t]))) return rc;
        if (rot[t].apply && d->stride != 4) return fail(h, SPG_E_INVALID, "rotation %d: rotated items need stride 4", t);
        any_rot = any_rot || rot[t].apply;
    }
    if ((!heat_out || !paf_out) && n > 0) return fail(h, SPG_E_INVALID, "heat_out/paf_out is NULL");
    if (paf_dtype != SPG_F32 && paf_dtype != SPG_F64) return fail(h, SPG_E_INVALID, "paf_dtype must be SPG_F32 or SPG_F64");
    if (paf_dtype == SPG_F32 && d->n_scales != 1)
        return fail(h, SPG_E_INVALID, "float32 body-part planes hold the reference's float64 values only for a single scale");
    if (d->stride < 1 || d->stride > 16) return fail(h, SPG_E_INVALID, "stride outside [1,16]");
    if ((rc = check_dims(h, n, H, W))) return rc;
    if (n == 0) return SPG_OK;
    const Workspace &ws = h->ws;
    // validate every scale and fill the common arguments
    PostArgs a{};
    if ((rc = post_common(h, d->stride, d->n_scales, d->paf_chan0, d->heat_chan0, d->flip_paf_ord, d->flip_heat_ord, d->nan_scrub,
                          paf_dtype, a)))
        return rc;
    DeviceGuard guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (d->n_scales > 1 && (d->stride != 4 || d->n_scales > kPostMaxScales || any_rot)) {  // float64 keypoint sums that outlive a launch
        if ((rc = grow_on(h, h->heat_acc, (size_t)h->cfg.max_batch * ws.K * H * W * sizeof(double), st, "the float64 keypoint sums")))
            return rc;
    }
    for (int t = 0; t < d->n_scales; t++) {
        const spg_postnet_scale &sc = d->scales[t];
        snprintf(what, sizeof what, "scale %d", t);
        if ((rc = check_net_out(h, what, sc.net_out, sc.dtype, sc.h, sc.w, sc.crop_h, sc.crop_w, d->stride))) return rc;
    }
    // At stride 4 the scale loop runs INSIDE the kernel (groups of kPostMaxScales): one tile geometry for all fused scales.
    // With a rotated item, or at another stride, every item is a launch of its own, in item order; the float64 sums
    // continue through memory.
    const int group = d->stride == 4 && !any_rot ? kPostMaxScales : 1;
    for (int t0 = 0; t0 < d->n_scales; t0 += group) {
        a.n_fused = std::min(group, d->n_scales - t0);
        a.scale_index = t0;
        PostImage im{};
        for (int t = 0; t < a.n_fused; t++) {
            const spg_postnet_scale &sc = d->scales[t0 + t];
            im.sc[t] = post_scale(sc.net_out, sc.dtype, sc.image_stride, sc.pair_stride, sc.chan_stride, sc.h, sc.w, sc.crop_h, sc.crop_w, H, W);
        }
        im.H = H; im.W = W; im.heat = heat_out; im.paf = paf_out; im.heat_acc = static_cast<double *>(h->heat_acc.p);
        PostPlan pl;
        dim3 grid;
        if ((rc = post_image(h, im, a.n_fused, d->n_scales == 1, d->stride, any_rot && rot[t0].apply ? rot[t0].matrix : nullptr, t0, &pl)) ||
            (rc = postnet_grid(h, a, im, n, pl.ctas_per_sm, &grid)))
            return rc;
        const PostKernels &k = kPostKernels[pl.family];
        if ((rc = launch(h, kStagePostnet, k.name, k.fn[pl.single][pl.ident][pl.f16], grid, kPostThreads, pl.smem, st, a, im))) return rc;
    }
    return SPG_OK;
}

// Ragged batches, over items[n][n_items] and rot (NULL, or one entry per item): spg_postnet_rotated's schedule for every
// image at once.  The items go in groups -- kPostMaxScales fused unrotated items, or one item per group when any is
// rotated -- and within a group each image goes in the family and tile plan_post picks for it alone.  A group's images
// are bucketed by kernel, identity family first, and each bucket's images go largest first into its launches' tables
// (deal_ragged), with one channel chunk for all its launches.
static int postnet_ragged(spg_handle *h, const spg_postnet_common *cm, const spg_postnet_image *items,
                          const spg_postnet_rotation *rot, int32_t n, int32_t n_items, int32_t paf_dtype, void *stream) {
    if (!h) return SPG_E_INVALID;
    int rc;
    if ((rc = check_batch(h, n))) return rc;
    if (n > 0 && (!items || n_items < 1)) return fail(h, SPG_E_INVALID, "items is NULL or n_items %d below 1", n_items);
    if (!cm || !cm->flip_paf_ord || !cm->flip_heat_ord) return fail(h, SPG_E_INVALID, "postnet common descriptor incomplete");
    if (cm->stride != 4) return fail(h, SPG_E_INVALID, "the ragged post-network stage needs stride 4 (got %d)", cm->stride);
    if (cm->net_dtype != SPG_F32 && cm->net_dtype != SPG_F16) return fail(h, SPG_E_INVALID, "network output must be SPG_F32 or SPG_F16");
    if (paf_dtype != SPG_F32 && paf_dtype != SPG_F64) return fail(h, SPG_E_INVALID, "paf_dtype must be SPG_F32 or SPG_F64");
    if (paf_dtype == SPG_F32 && n_items > 1)
        return fail(h, SPG_E_INVALID, "float32 body-part planes hold the reference's float64 values only for a single item");
    PostArgs a{};
    if ((rc = post_common(h, 4, std::max(n_items, 1), cm->paf_chan0, cm->heat_chan0, cm->flip_paf_ord, cm->flip_heat_ord,
                          cm->nan_scrub, paf_dtype, a)))
        return rc;
    // validate every image and item before the first launch; errors name "image i", or "image i item t" of several items
    char what[48];
    auto name = [&](int i, int t) {
        if (n_items == 1) snprintf(what, sizeof what, "image %d", i);
        else snprintf(what, sizeof what, "image %d item %d", i, t);
        return what;
    };
    bool any_rot = false;
    for (int i = 0; rot && i < n; i++) {
        for (int t = 0; t < n_items; t++) {
            const spg_postnet_rotation &r = rot[(size_t)i * n_items + t];
            if ((rc = check_rotation(h, name(i, t), "rotation apply", r))) return rc;
            if (r.apply != rot[t].apply)
                return fail(h, SPG_E_INVALID, "%s: rotated in some images and not in others (one rotation_search per call)", name(i, t));
            any_rot = any_rot || r.apply;
        }
    }
    const int max_h = std::min(h->cfg.max_h, 32767), max_w = std::min(h->cfg.max_w, 32767);
    std::vector<size_t> acc_off((size_t)n);  // each image's float64 keypoint sums in the handle's scratch
    size_t acc_total = 0;
    for (int i = 0; i < n; i++) {
        const spg_postnet_image &im = items[(size_t)i * n_items];
        for (int t = 0; t < n_items; t++) {
            const spg_postnet_image &it = items[(size_t)i * n_items + t];
            if (!it.heat_out || !it.paf_out) return fail(h, SPG_E_INVALID, "%s: heat_out/paf_out is NULL", name(i, t));
            if (it.height != im.height || it.width != im.width || it.heat_out != im.heat_out || it.paf_out != im.paf_out)
                return fail(h, SPG_E_INVALID, "%s: height/width/heat_out/paf_out differ from the image's item 0", name(i, t));
            if ((rc = check_net_out(h, name(i, t), it.net_out, cm->net_dtype, it.h, it.w, it.crop_h, it.crop_w, 4))) return rc;
            if (it.pair_stride < 0 || it.chan_stride < 0) return fail(h, SPG_E_INVALID, "%s: negative stride", name(i, t));
        }
        // the kernels store rows of 4 values with 16-byte stores (postnet_x4_ident_tile)
        if ((reinterpret_cast<uintptr_t>(im.heat_out) & 15) || (reinterpret_cast<uintptr_t>(im.paf_out) & 15))
            return fail(h, SPG_E_INVALID, "image %d: heat_out/paf_out must be 16-byte aligned", i);
        if (im.height < 2 || im.width < 2 || im.height > max_h || im.width > max_w)
            return fail(h, SPG_E_INVALID, "image %d: map %dx%d outside [2, %dx%d]", i, im.height, im.width, max_h, max_w);
        acc_off[i] = acc_total;
        acc_total += (size_t)h->ws.K * im.height * im.width;
    }
    if (n == 0) return SPG_OK;
    // the schedule of every launch, planned (and checked) before the first one: per item group, one launch list per kernel
    struct Bucket {
        int t0, n_fused;
        PostPlan plan;
        long long tiles;
        std::vector<std::pair<int, PostImage>> imgs;  // (image, its descriptor)
        std::vector<PostImage> ms;                    // the descriptors in launch order, dealt into ranges
        std::vector<RaggedRange> ranges;
        std::vector<int> first_cta;
    };
    std::vector<Bucket> buckets;
    const int per_group = any_rot ? 1 : kPostMaxScales;
    DeviceGuard guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double *acc = nullptr;
    if (n_items > 1 && (n_items > kPostMaxScales || any_rot)) {  // float64 keypoint sums that outlive a launch
        if ((rc = grow_on(h, h->heat_acc, acc_total * sizeof(double), st, "the float64 keypoint sums"))) return rc;
        acc = static_cast<double *>(h->heat_acc.p);
    }
    for (int t0 = 0; t0 < n_items; t0 += per_group) {
        const int nf = std::min(per_group, n_items - t0);
        const bool rotated = any_rot && rot[t0].apply;
        const size_t first = buckets.size();
        for (int i = 0; i < n; i++) {
            const spg_postnet_image &im = items[(size_t)i * n_items];
            PostImage d{};
            for (int t = 0; t < nf; t++) {
                const spg_postnet_image &it = items[(size_t)i * n_items + t0 + t];
                d.sc[t] = post_scale(it.net_out, cm->net_dtype, 0, it.pair_stride, it.chan_stride, it.h, it.w, it.crop_h, it.crop_w,
                                     im.height, im.width);
            }
            d.H = im.height; d.W = im.width; d.heat = im.heat_out; d.paf = im.paf_out;
            d.heat_acc = acc ? acc + acc_off[i] : nullptr;
            PostPlan pl;
            if ((rc = post_image(h, d, nf, n_items == 1, 4, rotated ? rot[(size_t)i * n_items + t0].matrix : nullptr, t0, &pl)))
                return fail(h, rc, "%s: %s", name(i, t0), std::string(h->err).c_str());
            size_t b = first;
            while (b < buckets.size() && !(buckets[b].plan.family == pl.family && buckets[b].plan.single == pl.single &&
                                           buckets[b].plan.ident == pl.ident))
                b++;
            if (b == buckets.size()) buckets.push_back(Bucket{t0, nf, pl, 0, {}, {}, {}, {}});
            buckets[b].imgs.emplace_back(i, d);
            buckets[b].tiles += (long long)d.tiles_x * d.tiles_y;
        }
        // identity family first; the buckets of fused or rotated items are of one family each and keep their order
        std::stable_sort(buckets.begin() + first, buckets.end(), [](const Bucket &x, const Bucket &y) {
            return x.plan.family < y.plan.family;
        });
    }
    // each bucket's images largest first, dealt into its launches' tables
    for (Bucket &b : buckets) {
        std::stable_sort(b.imgs.begin(), b.imgs.end(), [](const std::pair<int, PostImage> &x, const std::pair<int, PostImage> &y) {
            return (int64_t)x.second.H * x.second.W > (int64_t)y.second.H * y.second.W;
        });
        std::vector<int> ids;
        std::vector<long long> ctas;
        for (const auto &e : b.imgs) {
            ids.push_back(e.first);
            b.ms.push_back(e.second);
            ctas.push_back((long long)e.second.tiles_x * e.second.tiles_y);
        }
        if ((rc = deal_ragged(h, ctas, kPostTableImages, "image", ids.data(), b.ranges, b.first_cta))) return rc;
    }
    PostTable r{};
    for (const Bucket &b : buckets) {
        const PostKernels &k = kPostKernels[b.plan.family];
        a.n_fused = b.n_fused;
        a.scale_index = b.t0;
        a.chan_chunk = post_chan_chunk(h, a.n_out, b.tiles, b.plan.ctas_per_sm);
        const unsigned chunks = (unsigned)((a.n_out + a.chan_chunk - 1) / a.chan_chunk);
        for (const RaggedRange &g : b.ranges) {
            fill_table(r, b.ms, b.first_cta, g);
            if ((rc = launch(h, kStagePostnet, k.ragged_name[b.plan.single], k.ragged[b.plan.single][b.plan.ident][b.plan.f16],
                             dim3(g.ctas, chunks), kPostThreads, b.plan.smem, st, a, r)))
                return rc;
        }
    }
    return SPG_OK;
}

int spg_postnet_ragged(spg_handle *h, const spg_postnet_common *cm, const spg_postnet_image *images, int32_t n, int32_t paf_dtype,
                       void *stream) {
    if (h && !images && n > 0) return fail(h, SPG_E_INVALID, "images is NULL");
    return postnet_ragged(h, cm, images, nullptr, n, 1, paf_dtype, stream);
}

int spg_postnet_ragged_items(spg_handle *h, const spg_postnet_common *cm, const spg_postnet_image *items,
                             const spg_postnet_rotation *rot, int32_t n, int32_t n_items, int32_t paf_dtype, void *stream) {
    return postnet_ragged(h, cm, items, rot, n, n_items, paf_dtype, stream);
}

// ---- pre-network stage -------------------------------------------------------------------------
namespace {

// One member's descriptor: the checks every item of spg_prenet and every member of spg_prenet_ragged passes (`what` and
// `index` name it in the error) and the geometry of cv2.resize and util.padRightDownCorner.  The caller sets src and
// row_stride.
int prenet_member(spg_handle *h, const char *what, int index, int height, int width, int max_downsample, int pad_value,
                  double scale, int rotate, int reserved, const double *matrix, float *out, PreMember &a) {
    if (!std::isfinite(scale) || !(scale > 0)) return fail(h, SPG_E_INVALID, "%s %d: scale must be finite and positive", what, index);
    if ((rotate != 0 && rotate != 1) || reserved != 0)
        return fail(h, SPG_E_INVALID, "%s %d: rotate must be 0 or 1 and reserved 0", what, index);
    for (int k = 0; k < 6; k++)
        if (!std::isfinite(matrix[k])) return fail(h, SPG_E_INVALID, "%s %d: matrix entry %d is not finite", what, index, k);
    const double rh = (double)height * scale, rw = (double)width * scale;  // dsize = saturate_cast<int>(size * fx)
    if (!(rh < 32767.5 && rw < 32767.5)) return fail(h, SPG_E_INVALID, "%s %d: padded image above 32767 pixels a side", what, index);
    a = PreMember{};
    a.H1 = (int)std::nearbyint(rh);
    a.W1 = (int)std::nearbyint(rw);
    if (a.H1 < 1 || a.W1 < 1) return fail(h, SPG_E_INVALID, "%s %d: the resized image is empty (%dx%d)", what, index, a.H1, a.W1);
    a.Hp = (a.H1 + max_downsample - 1) / max_downsample * max_downsample;
    a.Wp = (a.W1 + max_downsample - 1) / max_downsample * max_downsample;
    if (a.Hp > 32767 || a.Wp > 32767 || (long long)a.Hp * a.Wp * 3 > 0x7fffffffLL)
        return fail(h, SPG_E_INVALID, "%s %d: padded image %dx%d above 32767 pixels a side or 2^31 values", what, index, a.Hp, a.Wp);
    if (!out) return fail(h, SPG_E_INVALID, "%s %d: out is NULL", what, index);
    a.h = height; a.w = width;
    a.copy = a.H1 == height && a.W1 == width;  // cv2.resize: dsize == ssize is a copy
    a.n_body = a.W1 * 3 / kPreLanes * kPreLanes;
    a.pad_value = pad_value;
    a.scale = 1.0 / scale;  // resize keeps scale = 1 / inv_scale, not src / dst
    a.out = out;
    a.tiles_x = (a.Wp + kPreThreads - 1) / kPreThreads;
    if (rotate) invert_affine(matrix, a.rot);
    return SPG_OK;
}

// The launches of validated members: the unrotated ones in prenet_kernel<false> launches, then the rotated ones, each
// launch of them a prenet_resize_kernel, which writes every member's padded uint8 image to its own part of the handle's
// scratch grid (grown to the largest launch's total), and a prenet_kernel<true> that warps from it.  Every launch is
// planned and checked before the first.
int prenet_launch(spg_handle *h, const std::vector<PreMember> &ms, const std::vector<char> &rotated, cudaStream_t st) {
    struct Group {
        std::vector<PreMember> ms;
        std::vector<RaggedRange> ranges;
        std::vector<int> first_cta;
    } groups[2];
    size_t grid_need = 0;
    int rc;
    for (int rot = 0; rot < 2; rot++) {
        Group &gr = groups[rot];
        std::vector<int> ids;
        std::vector<long long> ctas;
        for (int i = 0; i < (int)ms.size(); i++) {
            if (rotated[i] != rot) continue;
            ids.push_back(i);
            gr.ms.push_back(ms[i]);
            ctas.push_back((long long)ms[i].tiles_x * ms[i].Hp);
        }
        if ((rc = deal_ragged(h, ctas, kPreMaxMembers, "member", ids.data(), gr.ranges, gr.first_cta))) return rc;
        for (const RaggedRange &g : gr.ranges) {
            size_t bytes = 0;
            for (size_t k = g.begin; rot && k < g.end; k++) bytes += (size_t)gr.ms[k].Hp * gr.ms[k].Wp * 3;
            grid_need = std::max(grid_need, bytes);
        }
    }
    if ((rc = grow_on(h, h->pre_grid, grid_need, st, "the rotated items' padded images"))) return rc;
    PreRagged r{};
    for (int rot = 0; rot < 2; rot++) {
        for (const RaggedRange &g : groups[rot].ranges) {
            fill_table(r, groups[rot].ms, groups[rot].first_cta, g);
            const dim3 grid(g.ctas);
            if (rot) {
                size_t at = 0;  // the range's padded images back to back in the scratch grid
                for (int k = 0; k < r.n; k++) {
                    r.img[k].grid = static_cast<unsigned char *>(h->pre_grid.p) + at;
                    at += (size_t)r.img[k].Hp * r.img[k].Wp * 3;
                }
                if ((rc = launch(h, kStagePrenet, "prenet_resize_kernel", prenet_resize_kernel, grid, kPreThreads, 0, st, r)) ||
                    (rc = launch(h, kStagePrenet, "prenet_kernel<true>", prenet_kernel<true>, grid, kPreThreads, 0, st, r)))
                    return rc;
            } else if ((rc = launch(h, kStagePrenet, "prenet_kernel<false>", prenet_kernel<false>, grid, kPreThreads, 0, st, r))) {
                return rc;
            }
        }
    }
    return SPG_OK;
}

int check_prenet_common(spg_handle *h, int32_t max_downsample, int32_t pad_value) {
    if (max_downsample < 1 || max_downsample > 32767) return fail(h, SPG_E_INVALID, "max_downsample %d outside [1, 32767]", max_downsample);
    if (pad_value < 0 || pad_value > 255) return fail(h, SPG_E_INVALID, "pad_value %d outside [0, 255]", pad_value);
    return SPG_OK;
}

}  // namespace

int spg_prenet_ragged(spg_handle *h, int32_t max_downsample, int32_t pad_value, const spg_prenet_member *members,
                      int32_t n_members, void *stream) {
    if (!h) return SPG_E_INVALID;
    int rc;
    if ((rc = check_prenet_common(h, max_downsample, pad_value))) return rc;
    if (n_members < 0 || (n_members > 0 && !members)) return fail(h, SPG_E_INVALID, "members is NULL or n_members negative");
    // validate every member before the first launch
    std::vector<PreMember> ms((size_t)n_members);
    std::vector<char> rotated((size_t)n_members);
    for (int i = 0; i < n_members; i++) {
        const spg_prenet_member &m = members[i];
        if (m.height < 1 || m.width < 1 || m.height > 32767 || m.width > 32767)
            return fail(h, SPG_E_INVALID, "member %d: image %dx%d outside [1, 32767]", i, m.height, m.width);
        if (!m.image) return fail(h, SPG_E_INVALID, "member %d: image is NULL", i);
        if (m.row_stride < 3LL * m.width) return fail(h, SPG_E_INVALID, "member %d: row_stride below width * 3", i);
        if ((rc = prenet_member(h, "member", i, m.height, m.width, max_downsample, pad_value, m.scale, m.rotate, m.reserved,
                                m.matrix, m.out, ms[i])))
            return rc;
        ms[i].src = m.image;
        ms[i].row_stride = m.row_stride;
        rotated[i] = (char)m.rotate;
    }
    if (n_members == 0) return SPG_OK;
    DeviceGuard guard(h->device);
    return prenet_launch(h, ms, rotated, static_cast<cudaStream_t>(stream));
}

// n_images x n_items members of one image size on the ragged path
int spg_prenet(spg_handle *h, const uint8_t *image, int64_t image_stride, int64_t row_stride, int32_t n, int32_t height,
               int32_t width, int32_t max_downsample, int32_t pad_value, const spg_prenet_item *items, int32_t n_items,
               void *stream) {
    if (!h) return SPG_E_INVALID;
    if (n < 0 || n > 65535) return fail(h, SPG_E_INVALID, "n_images %d outside [0, 65535]", n);
    if (height < 1 || width < 1 || height > 32767 || width > 32767)
        return fail(h, SPG_E_INVALID, "image %dx%d outside [1, 32767]", height, width);
    int rc;
    if ((rc = check_prenet_common(h, max_downsample, pad_value))) return rc;
    if (n_items < 0 || (n_items > 0 && !items)) return fail(h, SPG_E_INVALID, "items is NULL or n_items negative");
    if (n > 0 && !image) return fail(h, SPG_E_INVALID, "image_dev is NULL");
    if (row_stride < 3LL * width || image_stride < 0) return fail(h, SPG_E_INVALID, "row_stride below width * 3 or image_stride negative");
    // validate every item before the first launch
    std::vector<PreMember> ms;
    std::vector<char> rotated;
    ms.reserve((size_t)n * n_items);
    rotated.reserve((size_t)n * n_items);
    for (int t = 0; t < n_items; t++) {
        const spg_prenet_item &it = items[t];
        PreMember a;
        if ((rc = prenet_member(h, "item", t, height, width, max_downsample, pad_value, it.scale, it.rotate, it.reserved, it.matrix,
                                it.out, a)))
            return rc;
        const long long pair = 2LL * a.Hp * a.Wp * 3;
        if (n > 1 && it.out_image_stride < pair)
            return fail(h, SPG_E_INVALID, "item %d: out_image_stride %lld below the pair's %lld elements", t, (long long)it.out_image_stride, pair);
        a.row_stride = row_stride;
        for (int i = 0; i < n; i++) {
            ms.push_back(a);
            ms.back().src = image + (int64_t)i * image_stride;
            ms.back().out = it.out + (int64_t)i * it.out_image_stride;
            rotated.push_back((char)it.rotate);
        }
    }
    if (ms.empty()) return SPG_OK;
    DeviceGuard guard(h->device);
    return prenet_launch(h, ms, rotated, static_cast<cudaStream_t>(stream));
}

int spg_reserve_frame(spg_handle *h, int32_t height, int32_t width, int32_t max_downsample, const spg_prenet_item *items,
                      int32_t n_items, int32_t stride, int32_t *moved) {
    if (!h) return SPG_E_INVALID;
    if (moved) *moved = 0;
    int rc;
    if ((rc = check_prenet_common(h, max_downsample, 0))) return rc;
    if (n_items < 1 || !items) return fail(h, SPG_E_INVALID, "items is NULL or n_items %d below 1", n_items);
    if (stride < 1 || stride > 16) return fail(h, SPG_E_INVALID, "stride outside [1,16]");
    if ((rc = check_dims(h, 1, height, width))) return rc;
    // spg_prenet's scratch grid: the padded images of the rotated items, which one launch holds at most
    size_t grid = 0;
    bool any_rot = false;
    for (int t = 0; t < n_items; t++) {
        const spg_prenet_item &it = items[t];
        PreMember a;
        float out;  // the geometry does not read the output
        if ((rc = prenet_member(h, "item", t, height, width, max_downsample, 0, it.scale, it.rotate, it.reserved, it.matrix, &out, a)))
            return rc;
        if (it.rotate) grid += (size_t)a.Hp * a.Wp * 3;
        any_rot = any_rot || it.rotate;
    }
    // spg_postnet_rotated's float64 keypoint sums, when they outlive a launch
    size_t acc = 0;
    if (n_items > 1 && (stride != 4 || n_items > kPostMaxScales || any_rot))
        acc = (size_t)h->cfg.max_batch * h->ws.K * height * width * sizeof(double);
    if (moved) *moved = grid > h->pre_grid.bytes || acc > h->heat_acc.bytes;  // set before a failed growth too
    h->frames_reserved = true;
    DeviceGuard guard(h->device);
    if ((rc = grow(h, h->pre_grid, grid))) return rc;
    return grow(h, h->heat_acc, acc);
}

int spg_reserve_frames(spg_handle *h, int32_t max_downsample, const spg_prenet_member *members, int32_t n_images,
                       int32_t n_items, int32_t *moved) {
    if (!h) return SPG_E_INVALID;
    if (moved) *moved = 0;
    int rc;
    if ((rc = check_prenet_common(h, max_downsample, 0))) return rc;
    if (!members || n_images < 1 || n_items < 1)
        return fail(h, SPG_E_INVALID, "members is NULL, or n_images %d or n_items %d below 1", n_images, n_items);
    // spg_postnet_ragged_items and spg_group_ragged hold the batch in the handle's max_batch-sized workspace
    if ((rc = check_batch(h, n_images))) return rc;
    // spg_prenet_ragged's scratch grid: at most every rotated member's padded image in one launch; then
    // spg_postnet_ragged_items' float64 keypoint sums, when they outlive a launch
    size_t grid = 0, acc = 0;
    bool any_rot = false;
    for (int i = 0; i < n_images; i++) {
        const spg_prenet_member &im = members[(size_t)i * n_items];
        if ((rc = check_dims(h, 1, im.height, im.width))) return fail(h, rc, "image %d: %s", i, std::string(h->err).c_str());
        for (int t = 0; t < n_items; t++) {
            const int k = i * n_items + t;
            const spg_prenet_member &m = members[k];
            if (m.height != im.height || m.width != im.width)
                return fail(h, SPG_E_INVALID, "member %d: its image size differs from its image's first member", k);
            PreMember a;
            float out;  // the geometry does not read the output
            if ((rc = prenet_member(h, "member", k, m.height, m.width, max_downsample, 0, m.scale, m.rotate, m.reserved, m.matrix,
                                    &out, a)))
                return rc;
            if (m.rotate) grid += (size_t)a.Hp * a.Wp * 3;
            any_rot = any_rot || m.rotate;
        }
        acc += (size_t)h->ws.K * im.height * im.width * sizeof(double);
    }
    if (!(n_items > 1 && (n_items > kPostMaxScales || any_rot))) acc = 0;
    if (moved) *moved = grid > h->pre_grid.bytes || acc > h->heat_acc.bytes;  // set before a failed growth too
    h->frames_reserved = true;
    DeviceGuard guard(h->device);
    if ((rc = grow(h, h->pre_grid, grid))) return rc;
    return grow(h, h->heat_acc, acc);
}

}  // extern "C"
