// train.cu -- the training side: a batch's samples (targets.cuh: the augmentation warp, the colour distortion, the
// masks and the ground-truth maps) and the multi-scale loss with its gradient (loss.cuh).
#include "runtime.cuh"

#include <cmath>

#include "loss.cuh"
#include "targets.cuh"

using namespace spg;

namespace {

// The training-sample launches (spg_targets_warp / spg_targets_maps / spg_targets_tint): sample i takes ctas[i] CTAs,
// each launch has its member table as the parameter.
template <class R, class M>
int launch_samples(spg_handle *h, const char *name, void (*kern)(R), R &r, const std::vector<M> &ms, const std::vector<long long> &ctas,
                   cudaStream_t st) {
    if (ms.empty()) return SPG_OK;
    std::vector<RaggedRange> ranges;
    std::vector<int> first;
    int rc;
    if ((rc = deal_ragged(h, ctas, sizeof(r.img) / sizeof(r.img[0]), "sample", nullptr, ranges, first))) return rc;
    DeviceGuard guard(h->device);
    for (const RaggedRange &g : ranges) {
        fill_table(r, ms, first, g);
        if ((rc = launch(h, kStageTargets, name, kern, dim3(g.ctas), kTgtThreads, 0, st, r))) return rc;
    }
    return SPG_OK;
}

}  // namespace

extern "C" {

// ---- training samples --------------------------------------------------------------------------
namespace {

// the parameters every sample of a call shares, checked and resolved
int targets_common(spg_handle *h, const spg_target_params *p, TgtCommon &c) {
    if (!p) return fail(h, SPG_E_INVALID, "params is NULL");
    if (p->stride < 1 || p->out_h < 1 || p->out_w < 1 || p->out_h > 32767 || p->out_w > 32767)
        return fail(h, SPG_E_INVALID, "stride %d or output %dx%d outside [1, 32767]", p->stride, p->out_h, p->out_w);
    if (p->out_h % p->stride || p->out_w % p->stride)
        return fail(h, SPG_E_INVALID, "stride %d does not divide the output %dx%d", p->stride, p->out_h, p->out_w);
    // a mask pixel's box sum of up to 255 * stride^2 bytes is an int, as in OpenCV's area resize
    if (255LL * p->stride * p->stride > 0x7fffffffLL)
        return fail(h, SPG_E_INVALID, "stride %d: a mask box sum of 255 * stride^2 overflows int (stride <= 2901)", p->stride);
    if (p->gaussian_size < 0 || p->gaussian_size > 32767) return fail(h, SPG_E_INVALID, "gaussian_size %d outside [0, 32767]", p->gaussian_size);
    if (!std::isfinite(p->sigma) || !(p->sigma > 0) || !std::isfinite(p->paf_sigma) || !(p->paf_sigma > 0))
        return fail(h, SPG_E_INVALID, "sigma and paf_sigma must be finite and positive");
    if (!std::isfinite(p->limb_gaussian_thre) || !std::isfinite(p->paf_thre))
        return fail(h, SPG_E_INVALID, "limb_gaussian_thre and paf_thre must be finite");
    const int border[5] = {p->border_image[0], p->border_image[1], p->border_image[2], p->border_mask_miss, p->border_mask_all};
    for (int k = 0; k < 5; k++)
        if (border[k] < 0 || border[k] > 255) return fail(h, SPG_E_INVALID, "border value %d outside [0, 255]", border[k]);
    if (p->reserved != 0) return fail(h, SPG_E_INVALID, "reserved must be 0");
    c = TgtCommon{};
    c.stride = p->stride;
    c.out_h = p->out_h;
    c.out_w = p->out_w;
    c.map_h = p->out_h / p->stride;
    c.map_w = p->out_w / p->stride;
    c.half = p->gaussian_size / 2;
    for (int k = 0; k < 5; k++) c.border[k] = border[k];
    c.kp_ds2 = (float)(2.0 * p->sigma * p->sigma);          // np.array([2 * sigma * sigma]).astype(np.float32)
    c.paf_thre = (float)p->paf_thre;                        // float32 coordinate - paf_thre stays float32
    c.paf_ds2 = 2.0 * (p->paf_sigma * p->paf_sigma);        // 2 * sigma ** 2
    c.limb_thre = p->limb_gaussian_thre;
    for (int i = 0; i < 256; i++) c.lut[i] = (float)i / 255.0f;  // np.float32(u8) / 255.: a float32 division
    return SPG_OK;
}

}  // namespace

int spg_targets_warp(spg_handle *h, const spg_target_params *params, const spg_target_sample *samples, int32_t n, void *stream) {
    if (!h) return SPG_E_INVALID;
    int rc;
    TgtWarpRagged r{};
    if ((rc = targets_common(h, params, r.c))) return rc;
    if (n < 0 || (n > 0 && !samples)) return fail(h, SPG_E_INVALID, "samples is NULL or n_samples negative");
    const long long img_px = (long long)r.c.out_h * r.c.out_w, map_px = (long long)r.c.map_h * r.c.map_w;
    std::vector<TgtWarpMember> ms((size_t)n);
    for (int i = 0; i < n; i++) {  // validate every sample before the first launch
        const spg_target_sample &s = samples[i];
        if (s.height < 1 || s.width < 1 || s.height > 32767 || s.width > 32767)
            return fail(h, SPG_E_INVALID, "sample %d: source %dx%d outside [1, 32767]", i, s.height, s.width);
        if (!s.image || !s.mask_miss || !s.mask_all || !s.image_out || !s.mask_miss_out || !s.mask_all_out)
            return fail(h, SPG_E_INVALID, "sample %d: a source or output pointer is NULL", i);
        if (s.image_row_stride < 3LL * s.width || s.mask_row_stride < s.width)
            return fail(h, SPG_E_INVALID, "sample %d: a row stride is below the row's bytes", i);
        for (int k = 0; k < 6; k++)
            if (!std::isfinite(s.matrix[k])) return fail(h, SPG_E_INVALID, "sample %d: matrix entry %d is not finite", i, k);
        TgtWarpMember &a = ms[i];
        a.src = s.image; a.miss = s.mask_miss; a.all = s.mask_all;
        a.src_stride = s.image_row_stride; a.mask_stride = s.mask_row_stride;
        a.img_out = s.image_out; a.miss_out = s.mask_miss_out; a.all_out = s.mask_all_out;
        invert_affine(s.matrix, a.rot);
        a.h = s.height; a.w = s.width;
        a.img_ctas = (int)((img_px + kTgtThreads - 1) / kTgtThreads);
    }
    const long long per_sample = (img_px + kTgtThreads - 1) / kTgtThreads + (map_px + kTgtThreads - 1) / kTgtThreads;
    return launch_samples(h, "targets_warp_kernel", targets_warp_kernel, r, ms, std::vector<long long>((size_t)n, per_sample),
                          static_cast<cudaStream_t>(stream));
}

int spg_targets_maps(spg_handle *h, const spg_target_params *params, const spg_target_joints *samples, int32_t n, void *stream) {
    if (!h) return SPG_E_INVALID;
    int rc;
    TgtMapsRagged r{};
    if ((rc = targets_common(h, params, r.c))) return rc;
    if (n < 0 || (n > 0 && !samples)) return fail(h, SPG_E_INVALID, "samples is NULL or n_samples negative");
    r.K = h->ws.K;
    r.L = h->ws.L;
    for (int k = 0; k < 2 * r.L; k++) r.limbs[k] = h->ws.limbs[k];
    const long long map_px = (long long)r.c.map_h * r.c.map_w;
    const int tiles = (int)((map_px + kTgtThreads - 1) / kTgtThreads);
    const long long channels = r.L + r.K + 2;
    std::vector<TgtMapsMember> ms((size_t)n);
    for (int i = 0; i < n; i++) {  // validate every sample before the first launch
        const spg_target_joints &s = samples[i];
        if (s.n_persons < 0 || (long long)s.n_persons * r.K > 0x7fffffffLL - kTgtThreads)
            return fail(h, SPG_E_INVALID, "sample %d: n_persons %d outside [0, 2^31 / n_parts)", i, s.n_persons);
        if (s.reserved != 0) return fail(h, SPG_E_INVALID, "sample %d: reserved must be 0", i);
        if ((s.n_persons > 0 && !s.joints) || !s.mask_all || !s.labels)
            return fail(h, SPG_E_INVALID, "sample %d: joints, mask_all or labels is NULL", i);
        ms[i] = TgtMapsMember{s.joints, s.mask_all, s.labels, s.n_persons, tiles, 0};
    }
    return launch_samples(h, "targets_maps_kernel", targets_maps_kernel, r, ms, std::vector<long long>((size_t)n, channels * tiles),
                          static_cast<cudaStream_t>(stream));
}

int spg_targets_tint(spg_handle *h, const spg_target_tint *samples, int32_t n, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (n < 0 || (n > 0 && !samples)) return fail(h, SPG_E_INVALID, "samples is NULL or n_samples negative");
    TgtTintRagged r{};
    std::vector<TgtTintMember> ms((size_t)n);
    std::vector<long long> ctas((size_t)n);
    for (int i = 0; i < n; i++) {  // validate every sample before the first launch
        const spg_target_tint &s = samples[i];
        if (s.height < 1 || s.width < 1 || s.height > 32767 || s.width > 32767)
            return fail(h, SPG_E_INVALID, "sample %d: source %dx%d outside [1, 32767]", i, s.height, s.width);
        if (!s.image) return fail(h, SPG_E_INVALID, "sample %d: image is NULL", i);
        if (s.row_stride < 3LL * s.width) return fail(h, SPG_E_INVALID, "sample %d: row_stride %lld is below the row's bytes", i, (long long)s.row_stride);
        if (s.hue < 0 || s.hue > 20 || s.saturation < 0 || s.saturation > 80 || s.value < 0 || s.value > 60)
            return fail(h, SPG_E_INVALID, "sample %d: draws (%d, %d, %d) outside [0, 20] x [0, 80] x [0, 60]", i, s.hue, s.saturation, s.value);
        if (s.row_block < 1) return fail(h, SPG_E_INVALID, "sample %d: row_block %d below 1", i, s.row_block);
        const int groups = (s.width + kTintPix - 1) / kTintPix;
        ms[i] = TgtTintMember{s.image, s.row_stride, s.height, s.width, s.hue - 10, s.saturation - 20, s.value - 20,
                              s.width - s.width % s.row_block, groups, 0};
        ctas[i] = ((long long)s.height * groups + kTgtThreads - 1) / kTgtThreads;
    }
    return launch_samples(h, "targets_tint_kernel", targets_tint_kernel, r, ms, ctas, static_cast<cudaStream_t>(stream));
}

// ---- training loss -----------------------------------------------------------------------------
namespace {

// the loss kernels per prediction dtype, with the names spg_stage_kernel reports
struct LossKernels {
    int dtype;
    size_t esz;
    void (*fwd)(LossArgs), (*bwd)(LossArgs);
    const char *fwd_name, *bwd_name;
};
const LossKernels kLossKernels[] = {
    {SPG_F32, 4, loss_forward_kernel<float>, loss_backward_kernel<float>, "loss_forward_kernel<float>", "loss_backward_kernel<float>"},
    {SPG_BF16, 2, loss_forward_kernel<__nv_bfloat16>, loss_backward_kernel<__nv_bfloat16>, "loss_forward_kernel<bf16>",
     "loss_backward_kernel<bf16>"},
    {SPG_F16, 2, loss_forward_kernel<__half>, loss_backward_kernel<__half>, "loss_forward_kernel<f16>", "loss_backward_kernel<f16>"},
};

bool aligned(const void *p, size_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// everything a loss launch needs, validated: the kernels, the arguments, the grid and the dynamic shared memory
int loss_setup(spg_handle *h, const spg_loss_params *p, const float *mask, const float *labels, const spg_loss_pred *preds,
               int32_t dtype, bool backward, const LossKernels *&kern, LossArgs &a, long long &ctas, size_t &smem) {
    if (!p) return fail(h, SPG_E_INVALID, "params is NULL");
    if (p->mode != SPG_LOSS_FOCAL && p->mode != SPG_LOSS_L2) return fail(h, SPG_E_INVALID, "mode %d is not SPG_LOSS_FOCAL or SPG_LOSS_L2", p->mode);
    if (p->nstack < 1 || p->nstack > kLossMaxStacks) return fail(h, SPG_E_INVALID, "nstack %d outside [1, %d]", p->nstack, kLossMaxStacks);
    if (p->batch < 1 || p->channels < (p->mode == SPG_LOSS_FOCAL ? 2 : 1))
        return fail(h, SPG_E_INVALID, "targets: batch %d or channels %d too small", p->batch, p->channels);
    if (p->height < kLossBand || p->width < kLossBand || p->height % kLossBand || p->width % kLossBand || p->height > 32767 || p->width > 32767)
        return fail(h, SPG_E_INVALID, "targets: map %dx%d is not a multiple of %d in [%d, 32767]", p->height, p->width, kLossBand, kLossBand);
    if (p->mode == SPG_LOSS_FOCAL && (p->heat_start < 0 || p->heat_start > p->bkg_start || p->bkg_start > p->channels))
        return fail(h, SPG_E_INVALID, "heat_start %d / bkg_start %d outside 0 <= heat_start <= bkg_start <= %d", p->heat_start, p->bkg_start, p->channels);
    if (!labels || !aligned(labels, 16)) return fail(h, SPG_E_INVALID, "labels is NULL or not 16-byte aligned");
    if (!mask || !aligned(mask, 16)) return fail(h, SPG_E_INVALID, "mask_miss is NULL or not 16-byte aligned");
    kern = nullptr;
    for (const LossKernels &k : kLossKernels)
        if (k.dtype == dtype) kern = &k;
    if (!kern) return fail(h, SPG_E_INVALID, "pred_dtype %d is not SPG_F32, SPG_BF16 or SPG_F16", dtype);
    if (!preds) return fail(h, SPG_E_INVALID, "preds is NULL");
    // the forward kernel's room bounds both directions, so that forward and backward admit the same widths
    smem = loss_smem_bytes(p->width);
    const size_t room = smem_room(h, kern->fwd);
    if (smem > room) return fail(h, SPG_E_INVALID, "targets: map width %d needs %zu B of shared memory (limit %zu)", p->width, smem, room);
    const int bands = p->height / kLossBand;
    ctas = (long long)p->batch * p->channels * bands;
    if (ctas > 0x7fffffffLL) return fail(h, SPG_E_INVALID, "targets: %lld CTAs are above grid.x's 2^31 - 1", ctas);
    a = LossArgs{};
    a.labels = labels;
    a.mask = mask;
    a.focal = p->mode == SPG_LOSS_FOCAL;
    a.nstack = p->nstack;
    a.B = p->batch; a.C = p->channels; a.H = p->height; a.W = p->width;
    a.heat_start = a.focal ? p->heat_start : 0;
    a.bkg_start = a.focal ? p->bkg_start : 0;
    a.bands = bands;
    a.w_bkg = (float)p->multi_task_weight;
    a.w_heat = (float)p->keypoint_task_weight;
    for (int k = 0; k < p->nstack; k++) a.nw[k] = (float)p->nstack_weight[k];
    for (int j = 0; j < kLossScales; j++) a.sw[j] = (float)p->scale_weight[j];
    // CUDA torch divides a float32 tensor by a host scalar b as a multiply by its reciprocal taken in float64 and
    // rounded to float32, (float)(1.0 / b): not 1.0f / (float)b, which differs for b = 3.9 or 4.9
    a.inv_batch = (float)(1.0 / p->batch_divisor);
    a.inv_sw = (float)(1.0 / p->scale_weight_sum);
    a.inv_nw = (float)(1.0 / p->nstack_weight_sum);
    const size_t vb = kLossVec * kern->esz;
    for (int k = 0; k < p->nstack; k++)
        for (int j = 0; j < kLossScales; j++) {
            const spg_loss_pred &q = preds[k * kLossScales + j];
            const int i = k * kLossScales + j;
            if (!q.data || (backward && !q.grad))
                return fail(h, SPG_E_INVALID, "prediction %d (stack %d, scale %d): %s is NULL", i, k, j, q.data ? "grad" : "data");
            if (q.batch_stride < 0 || q.chan_stride < 0 || q.row_stride < 0 ||
                (backward && (q.grad_batch_stride < 0 || q.grad_chan_stride < 0 || q.grad_row_stride < 0)))
                return fail(h, SPG_E_INVALID, "prediction %d (stack %d, scale %d): negative stride", i, k, j);
            if (!aligned(q.data, kern->esz) || (backward && !aligned(q.grad, kern->esz)))
                return fail(h, SPG_E_INVALID, "prediction %d (stack %d, scale %d): not aligned to its dtype", i, k, j);
            const long long v = kLossVec;
            bool vec = (p->width >> j) % kLossVec == 0 && aligned(q.data, vb) && q.batch_stride % v == 0 && q.chan_stride % v == 0 &&
                       q.row_stride % v == 0;
            if (backward)
                vec = vec && aligned(q.grad, vb) && q.grad_batch_stride % v == 0 && q.grad_chan_stride % v == 0 && q.grad_row_stride % v == 0;
            a.pred[i] = LossPred{q.data, backward ? q.grad : nullptr, q.batch_stride, q.chan_stride, q.row_stride,
                                 q.grad_batch_stride, q.grad_chan_stride, q.grad_row_stride, (int)vec};
        }
    return SPG_OK;
}

}  // namespace

int64_t spg_loss_workspace_bytes(const spg_loss_params *p) {
    if (!p || p->nstack < 1 || p->nstack > kLossMaxStacks || p->batch < 1 || p->channels < 1 || p->height < kLossBand ||
        p->height % kLossBand)
        return -1;
    return (int64_t)sizeof(double) * kLossScales * p->nstack * p->batch * p->channels * (p->height / kLossBand);
}

int spg_loss_forward(spg_handle *h, const spg_loss_params *params, const float *mask_miss, const float *labels,
                     const spg_loss_pred *preds, int32_t pred_dtype, float *stack_sums, float *loss, uint32_t *ticket,
                     double *partials, void *stream) {
    if (!h) return SPG_E_INVALID;
    const LossKernels *kern;
    LossArgs a;
    long long ctas;
    size_t smem;
    int rc;
    DeviceGuard guard(h->device);  // loss_setup reads the kernels' attributes on the handle's device
    if ((rc = loss_setup(h, params, mask_miss, labels, preds, pred_dtype, false, kern, a, ctas, smem))) return rc;
    if (!stack_sums || !loss) return fail(h, SPG_E_INVALID, "stack_sums or loss is NULL");
    if (!ticket || !aligned(ticket, sizeof(uint32_t))) return fail(h, SPG_E_INVALID, "ticket is NULL or not 4-byte aligned");
    if (!partials || !aligned(partials, sizeof(double))) return fail(h, SPG_E_INVALID, "partials is NULL or not 8-byte aligned");
    a.ticket = ticket;
    a.partial = partials;
    a.sums = stack_sums;
    a.loss = loss;
    return launch(h, kStageLoss, kern->fwd_name, kern->fwd, dim3((unsigned)ctas), kLossThreads, smem, static_cast<cudaStream_t>(stream), a);
}

int spg_loss_backward(spg_handle *h, const spg_loss_params *params, const float *mask_miss, const float *labels,
                      const spg_loss_pred *preds, int32_t pred_dtype, const float *grad_output, void *stream) {
    if (!h) return SPG_E_INVALID;
    const LossKernels *kern;
    LossArgs a;
    long long ctas;
    size_t smem;
    int rc;
    DeviceGuard guard(h->device);  // loss_setup reads the kernels' attributes on the handle's device
    if ((rc = loss_setup(h, params, mask_miss, labels, preds, pred_dtype, true, kern, a, ctas, smem))) return rc;
    if (!grad_output) return fail(h, SPG_E_INVALID, "grad_output is NULL");
    a.grad_output = grad_output;
    return launch(h, kStageLoss, kern->bwd_name, kern->bwd, dim3((unsigned)ctas), kLossThreads, smem, static_cast<cudaStream_t>(stream), a);
}

}  // extern "C"
