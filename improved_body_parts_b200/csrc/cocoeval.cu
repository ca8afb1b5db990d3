// cocoeval.cu -- COCOeval's keypoint evaluation on the device (cocoeval.cuh): OKS, matching and the precision
// accumulation, with the CUB radix sorts that order the detections.
#include "runtime.cuh"

#include "cocoeval.cuh"

using namespace spg;

extern "C" {

// ---- keypoint evaluation -----------------------------------------------------------------------
namespace {

constexpr long long kInt32Max = 0x7fffffffLL;

// the parameters and data both COCO entry points take, checked: counts, products of counts that index an array, and
// the pointers of every array the kernels read
int coco_check(spg_handle *h, const spg_coco_params *p, const spg_coco_data *d, const spg_coco_eval *e) {
    if (!p || !d || !e) return fail(h, SPG_E_INVALID, "params, data or eval is NULL");
    if (p->n_iou < 1 || p->n_rec < 1 || p->n_area < 1 || p->n_max_dets < 1)
        return fail(h, SPG_E_INVALID, "n_iou %d, n_rec %d, n_area %d, n_max_dets %d: each must be >= 1", p->n_iou, p->n_rec, p->n_area,
                    p->n_max_dets);
    if (p->n_kpt < 1 || p->n_kpt > kCocoMaxKpt) return fail(h, SPG_E_INVALID, "n_kpt %d outside [1, %d]", p->n_kpt, kCocoMaxKpt);
    if (!p->iou_thrs || !p->rec_thrs || !p->area_rng || !p->max_dets || !p->kpt_vars) return fail(h, SPG_E_INVALID, "a params table is NULL");
    if (d->n_images < 0 || d->n_cats < 0 || d->n_gt < 0 || d->n_dt < 0 || d->n_kept < 0 || d->n_ious < 0 || d->n_kept > d->n_dt)
        return fail(h, SPG_E_INVALID, "negative count, or n_kept %d above n_dt %d", d->n_kept, d->n_dt);
    const long long units = (long long)d->n_images * d->n_cats;
    const long long A = p->n_area, T = p->n_iou, M = p->n_max_dets;
    struct Product {
        const char *what;
        long long n;
    };
    for (const Product &q : {Product{"units + 1", units + 1}, Product{"gt_matches", A * T * d->n_gt}, Product{"dt_matches", A * T * d->n_kept},
                             Product{"match warps", units * A * T}, Product{"accumulate CTAs", d->n_cats * A * M * T},
                             Product{"accumulate scratch", A * M * T * d->n_dt}, Product{"precision", T * p->n_rec * d->n_cats * A * M},
                             Product{"gt_kpts", (long long)d->n_gt * p->n_kpt * 3}, Product{"dt_kpts", (long long)d->n_dt * p->n_kpt * 3}})
        if (q.n > kInt32Max) return fail(h, SPG_E_INVALID, "%s: %lld entries are above 2^31 - 1", q.what, q.n);
    if (!d->gt_start || !d->dt_start || !d->kept_start || !d->iou_start) return fail(h, SPG_E_INVALID, "a start table is NULL");
    if (d->n_gt && (!d->gt_kpts || !d->gt_bbox || !d->gt_area || !d->gt_id || !d->gt_flags)) return fail(h, SPG_E_INVALID, "a gt array is NULL");
    if (d->n_dt && (!d->dt_unit || !d->dt_kpts || !d->dt_area || !d->dt_score || !d->dt_id)) return fail(h, SPG_E_INVALID, "a dt array is NULL");
    if ((d->n_ious && !e->ious) || (d->n_dt && (!e->dt_order || !e->dt_rank || !e->cat_order)) ||
        (d->n_gt && (!e->gt_order || !e->gt_ignore || !e->gt_matches)) || (d->n_kept && (!e->dt_matches || !e->dt_ignore)))
        return fail(h, SPG_E_INVALID, "an eval array is NULL");
    return SPG_OK;
}

// blocks of a grid-stride loop over n entries
unsigned coco_blocks(spg_handle *h, long long n) {
    return (unsigned)std::max(1LL, std::min((n + kCocoThreads - 1) / kCocoThreads, (long long)h->sm_count * 8));
}

int bits_for(long long n) {  // the radix bits a key below n needs
    int b = 1;
    while (b < 32 && (1LL << b) < n) b++;
    return b;
}

}  // namespace

int spg_coco_evaluate(spg_handle *h, const spg_coco_params *params, const spg_coco_data *data, const spg_coco_eval *eval,
                      void *stream) {
    if (!h) return SPG_E_INVALID;
    int rc;
    if ((rc = coco_check(h, params, data, eval))) return rc;
    const spg_coco_params &p = *params;
    const spg_coco_data &d = *data;
    const spg_coco_eval &e = *eval;
    DeviceGuard guard(h->device);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int n = d.n_dt;
    const long long units = (long long)d.n_images * d.n_cats;
    if (n > 0) {
        // the detections by score, then two stable sorts of that order: by unit (computeOks' and evaluateImg's order)
        // and by category (accumulate's order, images in sorted order within equal scores)
        size_t b64 = 0, b32 = 0;
        SPG_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, b64, (const unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                                    (const int32_t *)nullptr, (int32_t *)nullptr, n, 0, 64, st));
        SPG_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, b32, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const int32_t *)nullptr,
                                                    (int32_t *)nullptr, n, 0, 32, st));
        const size_t tmp_bytes = std::max(b64, b32);
        auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
        const size_t nk = up(sizeof(unsigned long long) * n), ni = up(sizeof(int32_t) * n);
        if ((rc = grow(h, h->coco_sort, 2 * nk + 4 * ni + tmp_bytes))) return rc;
        unsigned char *base = static_cast<unsigned char *>(h->coco_sort.p);
        auto *key = reinterpret_cast<unsigned long long *>(base), *key_out = reinterpret_cast<unsigned long long *>(base + nk);
        auto *val = reinterpret_cast<int32_t *>(base + 2 * nk), *by_score = reinterpret_cast<int32_t *>(base + 2 * nk + ni);
        // the 32-bit keys reuse the 64-bit key buffers
        auto *unit_key = reinterpret_cast<uint32_t *>(key), *cat_key = unit_key + n, *key32_out = reinterpret_cast<uint32_t *>(key_out);
        void *tmp = base + 2 * nk + 4 * ni;
        size_t tb = tmp_bytes;
        const unsigned blocks = coco_blocks(h, n);
        if ((rc = launch(h, kStageCoco, "coco_keys_kernel", coco_keys_kernel, blocks, kCocoThreads, 0, st, d, key, val))) return rc;
        SPG_CUDA(h, cub::DeviceRadixSort::SortPairs(tmp, tb, key, key_out, val, by_score, n, 0, 64, st));
        if ((rc = launch(h, kStageCoco, "coco_group_keys_kernel", coco_group_keys_kernel, blocks, kCocoThreads, 0, st, d,
                         (const int32_t *)by_score, unit_key, cat_key)))
            return rc;
        tb = tmp_bytes;
        SPG_CUDA(h, cub::DeviceRadixSort::SortPairs(tmp, tb, unit_key, key32_out, by_score, e.dt_order, n, 0, bits_for(units), st));
        tb = tmp_bytes;
        SPG_CUDA(h, cub::DeviceRadixSort::SortPairs(tmp, tb, cat_key, key32_out, by_score, e.cat_order, n, 0, bits_for(d.n_cats), st));
        if ((rc = launch(h, kStageCoco, "coco_rank_kernel", coco_rank_kernel, blocks, kCocoThreads, 0, st, d, e))) return rc;
    }
    if (d.n_ious > 0 &&
        (rc = launch(h, kStageCoco, "coco_oks_kernel", coco_oks_kernel, coco_blocks(h, d.n_ious), kCocoThreads, 0, st, p, d, e)))
        return rc;
    const long long warps = units * p.n_area * p.n_iou;
    if (warps > 0 && (rc = launch(h, kStageCoco, "coco_match_kernel", coco_match_kernel, (unsigned)((warps + kCocoWarps - 1) / kCocoWarps),
                                  kCocoThreads, 0, st, p, d, e)))
        return rc;
    return SPG_OK;
}

int spg_coco_accumulate(spg_handle *h, const spg_coco_params *params, const spg_coco_data *data, const spg_coco_eval *eval,
                        double *precision, double *recall, double *scores, void *stream) {
    if (!h) return SPG_E_INVALID;
    int rc;
    if ((rc = coco_check(h, params, data, eval))) return rc;
    const spg_coco_params &p = *params;
    const spg_coco_data &d = *data;
    const long long ctas = (long long)d.n_cats * p.n_area * p.n_max_dets * p.n_iou;
    if (ctas == 0) return SPG_OK;
    if (!precision || !recall || !scores) return fail(h, SPG_E_INVALID, "precision, recall or scores is NULL");
    DeviceGuard guard(h->device);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t entries = std::max<size_t>((size_t)p.n_area * p.n_max_dets * p.n_iou * d.n_dt, 1);
    const size_t ni = (sizeof(int32_t) * entries + 255) & ~(size_t)255;
    if ((rc = grow(h, h->coco_acc, 2 * ni + sizeof(double) * entries))) return rc;
    unsigned char *base = static_cast<unsigned char *>(h->coco_acc.p);
    return launch(h, kStageCoco, "coco_accumulate_kernel", coco_accumulate_kernel, (unsigned)ctas, kCocoThreads, 0, st, p, d, *eval,
                  precision, recall, scores, reinterpret_cast<int32_t *>(base), reinterpret_cast<int32_t *>(base + ni),
                  reinterpret_cast<double *>(base + 2 * ni));
}

}  // extern "C"
