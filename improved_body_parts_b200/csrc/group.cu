// group.cu -- the grouping pass (include/spgroup.h): the kernel tables and schedules of peak finding and limb scoring,
// the launchers of the stage-wise, batch, ragged and host-buffer entry points (the chunked pipeline: H2D copy of chunk
// c+1 overlapped with the kernels of chunk c on two streams), the state transfer used by the stage-wise drop-in
// functions, the wire output of the assemble kernels, and the capacity-free tier (group_unbounded.cuh).
#include "runtime.cuh"

#include <cstdint>

#include "assemble.cuh"
#include "group_unbounded.cuh"
#include "limb_match.cuh"
#include "limb_score.cuh"
#include "limb_score_persist.cuh"
#include "match_assemble.cuh"
#include "nms_peaks.cuh"
#include "nms_peaks_persist.cuh"
#include "nms_peaks_banded.cuh"

using namespace spg;

namespace {

int check_params(spg_handle *h, const spg_params *p) {
    if (!p) return fail(h, SPG_E_INVALID, "params is NULL");
    if (p->offset_radius < 0 || p->offset_radius > kMaxRefineRadius)
        return fail(h, SPG_E_INVALID, "offset_radius %d outside [0, %d]", p->offset_radius, kMaxRefineRadius);
    if (p->mid_num < 1) return fail(h, SPG_E_INVALID, "mid_num must be >= 1");
    return SPG_OK;
}

// the dtype of the body-part planes: an index into kScoreKernels
int check_dtype(spg_handle *h, int dtype) {
    if (dtype != SPG_F32 && dtype != SPG_F64 && dtype != SPG_F32_AS_F64)
        return fail(h, SPG_E_INVALID, "paf_dtype must be SPG_F32, SPG_F64 or SPG_F32_AS_F64");
    return SPG_OK;
}

// The limb-scoring kernels for one dtype of body-part planes, with the names spg_stage_kernel reports.  Index 0 of a
// pair samples the planes through L2, index 1 stages each plane in shared memory.
struct ScoreKernels {
    size_t esz;  // bytes per plane element
    void (*item[2])(ScoreArgs);
    const char *item_name[2];
    void (*ragged[2])(ScoreArgs, ScoreRagged);
    const char *ragged_name[2];
    void (*persist)(ScoreArgs, int, unsigned int *);  // f32 planes only
    const char *persist_name;
};

static_assert(SPG_F32 == 0 && SPG_F64 == 1 && SPG_F32_AS_F64 == 2, "kScoreKernels is indexed by the dtype");
const ScoreKernels kScoreKernels[3] = {
    {4, {limb_score_kernel<float, false>, limb_score_kernel<float, true>},
     {"limb_score_kernel<float,false>", "limb_score_kernel<float,true>"},
     {limb_score_ragged_kernel<float, false>, limb_score_ragged_kernel<float, true>},
     {"limb_score_ragged_kernel<float,false>", "limb_score_ragged_kernel<float,true>"},
     limb_score_persist_kernel<float>, "limb_score_persist_kernel<float>"},
    {8, {limb_score_kernel<double, false>, limb_score_kernel<double, true>},
     {"limb_score_kernel<double,false>", "limb_score_kernel<double,true>"},
     {limb_score_ragged_kernel<double, false>, limb_score_ragged_kernel<double, true>},
     {"limb_score_ragged_kernel<double,false>", "limb_score_ragged_kernel<double,true>"},
     nullptr, ""},
    {4, {limb_score_kernel<float, false, double>, limb_score_kernel<float, true, double>},
     {"limb_score_kernel<float,false,double>", "limb_score_kernel<float,true,double>"},
     {limb_score_ragged_kernel<float, false, double>, limb_score_ragged_kernel<float, true, double>},
     {"limb_score_ragged_kernel<float,false,double>", "limb_score_ragged_kernel<float,true,double>"},
     limb_score_persist_kernel<double>, "limb_score_persist_kernel<double>"},
};

// one kernel per refinement radius (check_params: 0 .. kMaxRefineRadius)
void (*const kNmsPersistKernels[])(NmsArgs, int) = {nms_peaks_persist_kernel<0>, nms_peaks_persist_kernel<1>, nms_peaks_persist_kernel<2>,
                                                    nms_peaks_persist_kernel<3>, nms_peaks_persist_kernel<4>};
static_assert(kMaxRefineRadius == 4, "one nms_peaks_persist_kernel instantiation per radius");

// ---- schedules: the kernel, band rows, bulk-copy flag and shared memory a stage uses for planes of one geometry ----
// `persistent` allows the persistent kernels (one resident CTA per SM over a ring of plane or band slots; SPG_PERSIST=0
// turns them off).  Ragged launches pass false: their CTAs take the plane geometry per image, which only the per-plane
// kernels do.
struct NmsPlan {
    enum { kPersist, kBanded, kBands } kind;
    int band_rows, use_bulk;
    size_t smem;
    NmsBanding bg;
};

// `image` >= 0 names the image of a ragged call in the error; `radius` picks the persistent kernel's instantiation
int plan_nms(spg_handle *h, const float *heat, int64_t img_stride, int64_t chan_stride, int H, int W, bool persistent, int radius,
             int image, NmsPlan *pl) {
    const int capP = h->ws.capP;
    *pl = NmsPlan{};
    pl->use_bulk = (W % 4 == 0) && (img_stride % 4 == 0) && (chan_stride % 4 == 0) && ((reinterpret_cast<uintptr_t>(heat) & 15) == 0);
    const bool persist = persistent && h->persist && pl->use_bulk;
    if (persist && nms_persist_smem_bytes(H, W, capP) <= smem_room(h, kNmsPersistKernels[radius]) && (size_t)H * W / 4 < 65536 &&
        (size_t)H * W * sizeof(float) < (1u << 20) &&
        ((size_t)H * W / 4 + kNmsPScanners - 1) / kNmsPScanners <= (size_t)32 * kNmsPMaxIter) {
        // one resident CTA per SM: loader, 28 scanners, 3 finishers over a ring of 3 plane slots
        pl->kind = NmsPlan::kPersist;
        pl->smem = nms_persist_smem_bytes(H, W, capP);
        return SPG_OK;
    }
    // The bands are sized 1 KB below the opt-in limit, which covers the kernel's static barriers.  The room alone would
    // change the slot count of some planes that fit either way, so it only caps that budget.
    if (persist) pl->bg = nms_banding(H, W, capP, std::min(h->smem_optin - 1024, smem_room(h, nms_peaks_banded_kernel)));
    if (pl->bg.slots >= kNmsBTeams) {
        // planes that do not fit three times: the same roles over a ring of ~17 KB band slots, four scanner teams
        pl->kind = NmsPlan::kBanded;
        pl->band_rows = pl->bg.band_rows;
        pl->smem = pl->bg.smem;
        return SPG_OK;
    }
    // bands of ~16 KB through a ring of 3 buffers: two bands in flight per CTA while one is scanned, 4 CTAs per SM
    pl->kind = NmsPlan::kBands;
    pl->band_rows = std::max(4, std::min(H, 4096 / W));
    pl->smem = nms_smem_bytes(pl->band_rows, H, W, capP);
    const size_t room = std::min(smem_room(h, nms_peaks_kernel), smem_room(h, nms_peaks_ragged_kernel));  // either launches the plan
    if (pl->smem <= room) return SPG_OK;
    if (image < 0)
        return fail(h, SPG_E_INVALID, "map width %d needs %zu B of shared memory per band (limit %zu)", W, pl->smem, room);
    return fail(h, SPG_E_INVALID, "image %d: map width %d needs %zu B of shared memory per band (limit %zu)", image, W, pl->smem,
                room);
}

struct ScorePlan {
    enum { kSampled, kStaged, kPersist } kind;  // kSampled and kStaged index the pairs of ScoreKernels
    size_t smem;
};

// the room of a kind of limb-scoring kernel: the plan must fit its per-plane and its ragged launch alike
size_t score_room(spg_handle *h, const ScoreKernels &k, int kind) {
    return std::min(smem_room(h, k.item[kind]), smem_room(h, k.ragged[kind]));
}

ScorePlan plan_score(spg_handle *h, const ScoreKernels &k, const void *paf, int64_t img_stride, int64_t chan_stride, int H, int W,
                     bool persistent) {
    const int capP = h->ws.capP;
    const size_t plane_bytes = (size_t)H * W * k.esz;
    const bool aligned = (plane_bytes % 16 == 0) && ((img_stride * k.esz) % 16 == 0) && ((chan_stride * k.esz) % 16 == 0) &&
                         ((reinterpret_cast<uintptr_t>(paf) & 15) == 0) && plane_bytes < (1u << 20);
    if (persistent && h->persist && k.persist && aligned && capP <= kPersistMaxCapP &&
        persist_smem_bytes(plane_bytes, capP) <= smem_room(h, k.persist))
        return {ScorePlan::kPersist, persist_smem_bytes(plane_bytes, capP)};  // one resident CTA per SM walking a ring of 3 plane slots (loader / screeners / scorers)
    const size_t staged = score_smem_bytes(plane_bytes, capP);
    if (aligned && staged <= score_room(h, k, ScorePlan::kStaged)) return {ScorePlan::kStaged, staged};
    return {ScorePlan::kSampled, score_smem_bytes(0, capP)};  // plane larger than shared memory (or unaligned): sample through L2
}

// ---- kernel arguments from the parameters; the launchers add the planes and the image range ----
NmsArgs nms_args(const spg_handle *h, const spg_params *p) {
    NmsArgs a{};
    a.radius = p->offset_radius;
    a.thr = (float)p->thre1;
    a.ws = h->ws;
    return a;
}

ScoreArgs score_args(const spg_handle *h, const spg_params *p) {
    ScoreArgs a{};
    a.mid_num = p->mid_num;
    a.thre2 = p->thre2;
    a.connect_ration = p->connect_ration;
    a.screen = h->screen;
    a.crit1_strict = p->crit1_strict != 0;
    a.exact_warps = h->exact_warps;
    a.ws = h->ws;
    return a;
}

// Arguments of the assemble stage (stand-alone or fused with the matcher); use_bulk is set by the caller.
AssembleArgs assemble_args(const spg_handle *h, int base, int n, const spg_params *p) {
    AssembleArgs a{};
    a.n_images = n;
    a.image_base = base;
    a.len_rate = p->len_rate;
    a.connection_tole = p->connection_tole;
    a.min_mean_score = p->min_mean_score;
    a.remove_recon = p->remove_recon;
    a.min_parts = p->min_parts;
    a.refresh_len_check = p->refresh_len_check != 0;
    a.wire_flag = h->armed_flag; a.wire_flag_value = h->armed_value; a.done_counter = h->done_counter;
    a.ws = h->ws;
    a.ws.wire_first += base;  // records are indexed by the image's position in the call
    return a;
}

// ---- stage launchers on absolute image range [base, base+n) with chunk-local input pointers ----
int launch_nms(spg_handle *h, const float *heat, int64_t img_stride, int64_t chan_stride, int base, int n, int H, int W,
               const spg_params *p, cudaStream_t st) {
    if (n == 0) return SPG_OK;
    NmsPlan pl;
    int rc;
    if ((rc = plan_nms(h, heat, img_stride, chan_stride, H, W, true, p->offset_radius, -1, &pl))) return rc;
    NmsArgs a = nms_args(h, p);
    a.heat = heat;
    a.img_stride = img_stride;
    a.chan_stride = chan_stride;
    a.H = H;
    a.W = W;
    a.band_rows = pl.band_rows;
    a.use_bulk = pl.use_bulk;
    a.image_base = base;
    const int items = n * h->ws.K;
    switch (pl.kind) {
        case NmsPlan::kPersist:
            return launch(h, kStageNms, "nms_peaks_persist_kernel", kNmsPersistKernels[a.radius], std::min(items, h->sm_count),
                          kNmsPThreads, pl.smem, st, a, items);
        case NmsPlan::kBanded:
            return launch(h, kStageNms, "nms_peaks_banded_kernel", nms_peaks_banded_kernel, std::min(items, h->sm_count), kNmsPThreads,
                          pl.smem, st, a, items, pl.bg.slots, pl.bg.n_bands);
        default:
            return launch(h, kStageNms, "nms_peaks_kernel", nms_peaks_kernel, items, kNmsThreads, pl.smem, st, a);
    }
}

int launch_score(spg_handle *h, const void *paf, int dtype, int64_t img_stride, int64_t chan_stride, int base, int n, int H,
                 int W, double extent, const spg_params *p, cudaStream_t st) {
    if (n == 0) return SPG_OK;
    const ScoreKernels &k = kScoreKernels[dtype];
    ScoreArgs a = score_args(h, p);
    a.paf = paf;
    a.img_stride = img_stride;
    a.chan_stride = chan_stride;
    a.H = H;
    a.W = W;
    a.image_base = base;
    a.image_extent = extent;
    h->cand_dtype = dtype;
    const ScorePlan pl = plan_score(h, k, paf, img_stride, chan_stride, H, W, true);
    const int grid = n * h->ws.L;
    if (pl.kind == ScorePlan::kPersist) {
        // The kernel leaves its queue at 0 for the next launch on the same stream.  spg_group_host's chunks run on the
        // handle's two streams and may overlap, so the second stream has a queue of its own.
        unsigned int *queue = h->score_queue + (st == h->streams[1] ? 2 : 0);
        // On a handle prepared for capture (spg_reserve_frame), a captured call also zeroes it with a memset node, so
        // that every replay of the graph starts from 0 whatever ran on the handle between replays.  Other handles never
        // ask the stream.
        bool capturing = false;
        int rc;
        if (h->frames_reserved && (rc = stream_capturing(h, st, &capturing))) return rc;
        if (capturing) SPG_CUDA(h, cudaMemsetAsync(queue, 0, 2 * sizeof(unsigned int), st));
        return launch(h, kStageScore, k.persist_name, k.persist, std::min(grid, h->sm_count), kPersistThreads, pl.smem, st, a, grid,
                      queue);
    }
    return launch(h, kStageScore, k.item_name[pl.kind], k.item[pl.kind], grid, kScoreThreads, pl.smem, st, a);
}

int launch_match(spg_handle *h, int base, int n, cudaStream_t st) {
    if (n == 0) return SPG_OK;
    MatchArgs a{};
    a.n_images = n;
    a.image_base = base;
    a.keys_valid = h->cand_dtype == SPG_F32;
    a.ws = h->ws;
    const int warps = n * h->ws.L;
    const int blocks = (warps * 32 + kMatchThreads - 1) / kMatchThreads;
    return launch(h, kStageMatch, "limb_match_kernel", limb_match_kernel, blocks, kMatchThreads, 0, st, a);
}

int launch_assemble(spg_handle *h, int base, int n, const spg_params *p, cudaStream_t st) {
    if (n == 0) return SPG_OK;
    AssembleArgs a = assemble_args(h, base, n, p);
    h->armed_flag = nullptr;  // one shot
    a.use_bulk = ((size_t)h->ws.L * h->ws.capP * sizeof(uint32_t)) % 16 == 0;  // bulk copies move multiples of 16 bytes
    const size_t smem = assemble_smem_bytes(h->ws.K, h->ws.capP, h->ws.capR) + assemble_conn_bytes(h->ws.L, h->ws.capP);
    const size_t room = smem_room(h, assemble_kernel);
    if (smem > room) return fail(h, SPG_E_INVALID, "capacities need %zu B of shared memory in assemble (limit %zu)", smem, room);
    return launch(h, kStageAssemble, "assemble_kernel", assemble_kernel, n, kAssembleThreads, smem, st, a);
}

int launch_match_assemble(spg_handle *h, int base, int n, const spg_params *p, cudaStream_t st) {
    if (n == 0) return SPG_OK;
    AssembleArgs a = assemble_args(h, base, n, p);
    a.use_bulk = ((size_t)h->ws.K * h->ws.capP * sizeof(float)) % 16 == 0;  // bulk copies move multiples of 16 bytes
    const size_t smem = match_assemble_smem_bytes(h->ws.K, h->ws.L, h->ws.capP, h->ws.capR, h->ma_warps);
    if (smem > smem_room(h, match_assemble_kernel)) {  // very large capacities: the two stand-alone kernels need less shared memory
        int rc;
        if ((rc = launch_match(h, base, n, st))) return rc;
        return launch_assemble(h, base, n, p, st);  // consumes the armed signal itself
    }
    h->armed_flag = nullptr;  // one shot
    h->stage_kernel[kStageAssemble] = "";
    return launch(h, kStageMatch, "match_assemble_kernel", match_assemble_kernel, n, 32 * (1 + h->ma_warps), smem, st, a,
                  h->cand_dtype == SPG_F32);
}

// persons from the scored candidates: the fused kernel, or the matcher and the assembler back to back (SPG_FUSE_MA=0)
int launch_people(spg_handle *h, int base, int n, const spg_params *p, cudaStream_t st) {
    if (h->fuse_ma) return launch_match_assemble(h, base, n, p, st);
    int rc;
    if ((rc = launch_match(h, base, n, st))) return rc;
    return launch_assemble(h, base, n, p, st);
}

int run_all(spg_handle *h, const float *heat, int64_t his, int64_t hcs, const void *paf, int dtype, int64_t pis, int64_t pcs,
            int base, int n, int H, int W, double extent, const spg_params *p, cudaStream_t st) {
    int rc;
    SPG_CUDA(h, cudaMemsetAsync(h->ws.status + base, 0, sizeof(uint32_t) * (size_t)n, st));
    if ((rc = launch_nms(h, heat, his, hcs, base, n, H, W, p, st))) return rc;
    if ((rc = launch_score(h, paf, dtype, pis, pcs, base, n, H, W, extent, p, st))) return rc;
    return launch_people(h, base, n, p, st);
}

// [dtype][write]: the scoring kernel for the plane's storage / arithmetic types (kScoreKernels' dtype order)
void (*const kUbScoreKernels[3][2])(UbArgs, ScoreArgs) = {
    {ub_score_kernel<float, float, false>, ub_score_kernel<float, float, true>},
    {ub_score_kernel<double, double, false>, ub_score_kernel<double, double, true>},
    {ub_score_kernel<float, double, false>, ub_score_kernel<float, double, true>},
};

}  // namespace

int spg::check_score_room(spg_handle *h) {
    for (const ScoreKernels &k : kScoreKernels)
        if (score_smem_bytes(0, h->ws.capP) > score_room(h, k, ScorePlan::kSampled))
            return fail(h, SPG_E_INVALID, "max_peaks_per_part %d needs %zu B of shared memory in limb scoring (limit %zu)", h->ws.capP,
                        score_smem_bytes(0, h->ws.capP), score_room(h, k, ScorePlan::kSampled));
    return SPG_OK;
}

extern "C" {

// The clock trace lives in this unit's module, with the kernels that write it.
#ifdef SPG_TRACE  // development builds only (make trace): the clock trace of the first CTAs of the last launches
int spg_trace_read(unsigned long long *out, size_t n_words, int clear) {
    const size_t n = std::min(n_words, (size_t)spg::kTraceCtas * spg::kTraceSlots);
    if (cudaMemcpyFromSymbol(out, spg::g_spg_trace, n * sizeof(unsigned long long)) != cudaSuccess) return -1;
    if (clear) {
        void *p = nullptr;
        if (cudaGetSymbolAddress(&p, spg::g_spg_trace) != cudaSuccess) return -1;
        if (cudaMemset(p, 0, sizeof(spg::g_spg_trace)) != cudaSuccess) return -1;
    }
    return 0;
}
// (start, exit) %globaltimer pairs of the first kTraceSpanCtas CTAs of the traced launches (SPG_TR_CTA_*)
int spg_trace_read_spans(unsigned long long *out, size_t n_words, int clear) {
    const size_t n = std::min(n_words, (size_t)2 * spg::kTraceSpanCtas);
    if (cudaMemcpyFromSymbol(out, spg::g_spg_cta_span, n * sizeof(unsigned long long)) != cudaSuccess) return -1;
    if (clear) {
        void *p = nullptr;
        if (cudaGetSymbolAddress(&p, spg::g_spg_cta_span) != cudaSuccess) return -1;
        if (cudaMemset(p, 0, sizeof(spg::g_spg_cta_span)) != cudaSuccess) return -1;
    }
    return 0;
}
#endif

// ---- wire records: the assemble kernels' output and its stream-ordered signal -----------------------------------
int64_t spg_wire_record_bytes(const spg_handle *h) {
    if (!h) return 0;
    const int rows = h->ws.wire_rows > 0 ? h->ws.wire_rows : h->ws.capR;
    return 8 + (int64_t)rows * (2 * h->ws.J + 2) * (int64_t)sizeof(double);
}

int spg_set_wire_output(spg_handle *h, void *wire_dev, int64_t first_record, int32_t wire_rows) {
    if (!h) return SPG_E_INVALID;
    if (!wire_dev) {
        h->ws.wire = nullptr;
        h->ws.wire_first = 0;
        return SPG_OK;
    }
    if (wire_rows < 1 || wire_rows > h->ws.capR) return fail(h, SPG_E_INVALID, "wire_rows %d outside [1, max_person_rows=%d]", wire_rows, h->ws.capR);
    if (first_record < 0) return fail(h, SPG_E_INVALID, "first_record is negative");
    if ((reinterpret_cast<uintptr_t>(wire_dev) & 7) != 0) return fail(h, SPG_E_INVALID, "wire buffer must be 8-byte aligned");
    if ((size_t)wire_rows * (2 * h->ws.J + 2) * sizeof(double) > assemble_conn_bytes(h->ws.L, h->ws.capP))
        return fail(h, SPG_E_INVALID, "wire_rows %d do not fit the assemble kernel's staging area", wire_rows);
    h->ws.wire = static_cast<unsigned char *>(wire_dev);
    h->ws.wire_first = first_record;
    h->ws.wire_rows = wire_rows;
    return SPG_OK;
}

int spg_arm_wire_signal(spg_handle *h, uint64_t *word_dev, uint64_t value) {
    if (!h) return SPG_E_INVALID;
    if (!word_dev) {
        h->armed_flag = nullptr;
        return SPG_OK;
    }
    if (!h->ws.wire) return fail(h, SPG_E_STATE, "spg_arm_wire_signal needs a wire output (spg_set_wire_output) first");
    if (!h->done_counter) {
        DeviceGuard guard(h->device);
        SPG_CUDA(h, cudaMalloc(&h->done_counter, sizeof(unsigned int)));
        SPG_CUDA(h, cudaMemset(h->done_counter, 0, sizeof(unsigned int)));
    }
    h->armed_flag = reinterpret_cast<unsigned long long *>(word_dev);
    h->armed_value = value;
    return SPG_OK;
}

// ---- stages ------------------------------------------------------------------------------------
int spg_nms_peaks(spg_handle *h, const float *heat, int64_t image_stride, int64_t chan_stride, int32_t n, int32_t H, int32_t W,
                  const spg_params *p, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (!heat && n > 0) return fail(h, SPG_E_INVALID, "heat_dev is NULL");
    int rc;
    if ((rc = check_dims(h, n, H, W)) || (rc = check_params(h, p))) return rc;
    DeviceGuard guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SPG_CUDA(h, cudaMemsetAsync(h->ws.status, 0, sizeof(uint32_t) * (size_t)n, st));
    if ((rc = launch_nms(h, heat, image_stride, chan_stride, 0, n, H, W, p, st))) return rc;
    h->stage = 1;
    return SPG_OK;
}

int spg_limb_score(spg_handle *h, const void *paf, int32_t dtype, int64_t image_stride, int64_t chan_stride, int32_t n, int32_t H,
                   int32_t W, double extent, const spg_params *p, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (!paf && n > 0) return fail(h, SPG_E_INVALID, "paf_dev is NULL");
    int rc;
    if ((rc = check_dtype(h, dtype))) return rc;
    if (h->stage < 1) return fail(h, SPG_E_STATE, "spg_limb_score needs peaks (spg_nms_peaks or spg_upload_peaks) first");
    if ((rc = check_dims(h, n, H, W)) || (rc = check_params(h, p))) return rc;
    DeviceGuard guard(h->device);
    if ((rc = launch_score(h, paf, dtype, image_stride, chan_stride, 0, n, H, W, extent, p, static_cast<cudaStream_t>(stream)))) return rc;
    h->stage = std::max(h->stage, 2);
    return SPG_OK;
}

int spg_limb_match(spg_handle *h, int32_t n, const spg_params *p, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (h->stage < 2) return fail(h, SPG_E_STATE, "spg_limb_match needs spg_limb_score first");
    int rc;
    if ((rc = check_batch(h, n)) || (rc = check_params(h, p))) return rc;
    DeviceGuard guard(h->device);
    if ((rc = launch_match(h, 0, n, static_cast<cudaStream_t>(stream)))) return rc;
    h->stage = std::max(h->stage, 3);
    return SPG_OK;
}

int spg_assemble(spg_handle *h, int32_t n, const spg_params *p, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (h->stage < 3) return fail(h, SPG_E_STATE, "spg_assemble needs connections (spg_limb_match or spg_upload_connections) first");
    int rc;
    if ((rc = check_batch(h, n)) || (rc = check_params(h, p))) return rc;
    DeviceGuard guard(h->device);
    if ((rc = launch_assemble(h, 0, n, p, static_cast<cudaStream_t>(stream)))) return rc;
    h->stage = 4;
    return SPG_OK;
}

int spg_match_assemble(spg_handle *h, int32_t n, const spg_params *p, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (h->stage < 2) return fail(h, SPG_E_STATE, "spg_match_assemble needs spg_limb_score first");
    int rc;
    if ((rc = check_batch(h, n)) || (rc = check_params(h, p))) return rc;
    DeviceGuard guard(h->device);
    if ((rc = launch_match_assemble(h, 0, n, p, static_cast<cudaStream_t>(stream)))) return rc;
    h->stage = 4;
    return SPG_OK;
}

int spg_group_batch(spg_handle *h, const float *heat, int64_t his, int64_t hcs, const void *paf, int32_t dtype, int64_t pis, int64_t pcs,
                    int32_t n, int32_t H, int32_t W, double extent, const spg_params *p, void *stream) {
    if (!h) return SPG_E_INVALID;
    if ((!heat || !paf) && n > 0) return fail(h, SPG_E_INVALID, "heat_dev/paf_dev is NULL");
    int rc;
    if ((rc = check_dtype(h, dtype)) || (rc = check_dims(h, n, H, W)) || (rc = check_params(h, p))) return rc;
    DeviceGuard guard(h->device);
    if ((rc = run_all(h, heat, his, hcs, paf, dtype, pis, pcs, 0, n, H, W, extent, p, static_cast<cudaStream_t>(stream)))) return rc;
    h->stage = 4;
    return SPG_OK;
}

// ---- ragged batches --------------------------------------------------------------------------------
// K1 and K2a run their per-plane schedules with the geometry taken per image from descriptors passed as kernel
// parameters; match_assemble reads no geometry and runs as for spg_group_batch.  Images go into each launch largest
// plane first (longest job first over the CTA queue); every CTA writes to its image's own slot.
int spg_group_ragged(spg_handle *h, const spg_image_maps *images, int32_t n, int32_t dtype, const spg_params *p, void *stream) {
    if (!h) return SPG_E_INVALID;
    int rc;
    if ((rc = check_batch(h, n))) return rc;
    if (!images && n > 0) return fail(h, SPG_E_INVALID, "images is NULL");
    if ((rc = check_dtype(h, dtype)) || (rc = check_params(h, p))) return rc;
    const Workspace &ws = h->ws;
    const ScoreKernels &k = kScoreKernels[dtype];
    const int max_h = std::min(h->cfg.max_h, 32767), max_w = std::min(h->cfg.max_w, 32767);
    DeviceGuard guard(h->device);  // the plans read the kernels' attributes on the handle's device
    // validate every image before the first launch
    std::vector<int> order((size_t)n);
    NmsPlan np;
    for (int i = 0; i < n; i++) {
        const spg_image_maps &im = images[i];
        if (!im.heat || !im.paf) return fail(h, SPG_E_INVALID, "image %d: heat/paf is NULL", i);
        if (im.height < 2 || im.width < 2 || im.height > max_h || im.width > max_w)
            return fail(h, SPG_E_INVALID, "image %d: map %dx%d outside [2, %dx%d]", i, im.height, im.width, max_h, max_w);
        if ((rc = plan_nms(h, im.heat, 0, im.heat_chan_stride, im.height, im.width, false, 0, i, &np))) return rc;
        order[i] = i;
    }
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) {
        return (int64_t)images[x].height * images[x].width > (int64_t)images[y].height * images[y].width;
    });
    std::vector<NmsImage> nms;
    std::vector<ScoreImage> staged, sampled;
    size_t nms_smem = 0, staged_smem = 0;
    nms.reserve(n);
    for (int i : order) {
        const spg_image_maps &im = images[i];
        const int H = im.height, W = im.width;
        plan_nms(h, im.heat, 0, im.heat_chan_stride, H, W, false, 0, i, &np);  // succeeded in the validation above
        NmsImage d{};
        d.heat = im.heat; d.chan_stride = im.heat_chan_stride; d.H = H; d.W = W; d.band_rows = np.band_rows; d.use_bulk = np.use_bulk; d.slot = i;
        nms_smem = std::max(nms_smem, np.smem);
        nms.push_back(d);
        ScoreImage s{};
        s.paf = im.paf; s.chan_stride = im.paf_chan_stride; s.image_extent = im.image_extent; s.H = H; s.W = W; s.slot = i;
        const ScorePlan sp = plan_score(h, k, im.paf, 0, im.paf_chan_stride, H, W, false);
        if (sp.kind == ScorePlan::kStaged) {
            staged.push_back(s);
            staged_smem = std::max(staged_smem, sp.smem);
        } else {
            sampled.push_back(s);
        }
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SPG_CUDA(h, cudaMemsetAsync(ws.status, 0, sizeof(uint32_t) * (size_t)n, st));
    if (n == 0) return SPG_OK;
    // `per` CTAs (its parts or limbs) per image; the kernels find an image at blockIdx.x / per
    auto per_image = [&](int stage, const char *name, auto kern, auto &r, int per, int block, size_t smem, const auto &args,
                         const auto &imgs) {
        std::vector<RaggedRange> ranges;
        std::vector<int> first;
        int rc2 = deal_ragged(h, std::vector<long long>(imgs.size(), per), sizeof(r.img) / sizeof(r.img[0]), "image", nullptr, ranges, first);
        for (size_t j = 0; rc2 == SPG_OK && j < ranges.size(); j++) {
            std::copy(imgs.begin() + ranges[j].begin, imgs.begin() + ranges[j].end, r.img);
            rc2 = launch(h, stage, name, kern, dim3(ranges[j].ctas), block, smem, st, args, r);
        }
        return rc2;
    };
    NmsRagged nr{};
    ScoreRagged sr{};
    if ((rc = per_image(kStageNms, "nms_peaks_ragged_kernel", nms_peaks_ragged_kernel, nr, ws.K, kNmsThreads, nms_smem, nms_args(h, p), nms)))
        return rc;
    h->cand_dtype = dtype;
    const ScoreArgs sa = score_args(h, p);
    if ((rc = per_image(kStageScore, k.ragged_name[1], k.ragged[1], sr, ws.L, kScoreThreads, staged_smem, sa, staged)) ||
        (rc = per_image(kStageScore, k.ragged_name[0], k.ragged[0], sr, ws.L, kScoreThreads, score_smem_bytes(0, ws.capP), sa, sampled)) ||
        (rc = launch_people(h, 0, n, p, st)))
        return rc;
    h->stage = 4;
    return SPG_OK;
}

int spg_group_host(spg_handle *h, const float *heat_host, const void *paf_host, int32_t dtype, int32_t n, int32_t H, int32_t W,
                   double extent, const spg_params *p, int32_t *out_n, double *out_xy, double *out_score, uint32_t *out_status) {
    if (!h) return SPG_E_INVALID;
    if ((!heat_host || !paf_host) && n > 0) return fail(h, SPG_E_INVALID, "heat_host/paf_host is NULL");
    int rc;
    if ((rc = check_dtype(h, dtype)) || (rc = check_dims(h, n, H, W)) || (rc = check_params(h, p))) return rc;
    DeviceGuard guard(h->device);
    const Workspace &ws = h->ws;
    const size_t plane = (size_t)H * W;
    const size_t heat_img = (size_t)ws.K * plane * sizeof(float), paf_img = (size_t)ws.L * plane * kScoreKernels[dtype].esz;
    // chunk so that copy(c+1) overlaps kernels(c); keep at least ~8 chunks for large batches
    const int chunk = std::max(1, std::min(n, std::max(8, n / 8)));
    if ((rc = grow(h, h->in_heat, 2 * (size_t)chunk * heat_img)) || (rc = grow(h, h->in_paf, 2 * (size_t)chunk * paf_img))) return rc;
    const size_t RSJ = (size_t)ws.capR * ws.J * 2;
    int ci = 0;
    for (int base = 0; base < n; base += chunk, ci++) {
        const int m = std::min(chunk, n - base);
        cudaStream_t st = h->streams[ci & 1];
        unsigned char *dh = static_cast<unsigned char *>(h->in_heat.p) + (size_t)(ci & 1) * chunk * heat_img;
        unsigned char *dp = static_cast<unsigned char *>(h->in_paf.p) + (size_t)(ci & 1) * chunk * paf_img;
        // stream order protects the staging buffers: chunk ci reuses the buffers of chunk ci-2 on the same stream
        SPG_CUDA(h, cudaMemcpyAsync(dh, reinterpret_cast<const unsigned char *>(heat_host) + (size_t)base * heat_img, (size_t)m * heat_img, cudaMemcpyHostToDevice, st));
        SPG_CUDA(h, cudaMemcpyAsync(dp, static_cast<const unsigned char *>(paf_host) + (size_t)base * paf_img, (size_t)m * paf_img, cudaMemcpyHostToDevice, st));
        if ((rc = run_all(h, reinterpret_cast<const float *>(dh), (int64_t)ws.K * plane, (int64_t)plane, dp, dtype, (int64_t)ws.L * plane,
                          (int64_t)plane, base, m, H, W, extent, p, st)))
            return rc;
        if (out_n) SPG_CUDA(h, cudaMemcpyAsync(out_n + base, ws.n_persons + base, sizeof(int32_t) * m, cudaMemcpyDeviceToHost, st));
        if (out_xy && ws.J) SPG_CUDA(h, cudaMemcpyAsync(out_xy + (size_t)base * RSJ, ws.people_xy + (size_t)base * RSJ, sizeof(double) * RSJ * m, cudaMemcpyDeviceToHost, st));
        if (out_score) SPG_CUDA(h, cudaMemcpyAsync(out_score + (size_t)base * ws.capR, ws.people_score + (size_t)base * ws.capR, sizeof(double) * ws.capR * m, cudaMemcpyDeviceToHost, st));
        if (out_status) SPG_CUDA(h, cudaMemcpyAsync(out_status + base, ws.status + base, sizeof(uint32_t) * m, cudaMemcpyDeviceToHost, st));
    }
    SPG_CUDA(h, cudaStreamSynchronize(h->streams[0]));
    SPG_CUDA(h, cudaStreamSynchronize(h->streams[1]));
    h->stage = 4;
    return SPG_OK;
}

// ---- state transfer ------------------------------------------------------------------------------
int spg_upload_peaks(spg_handle *h, int32_t img, const int32_t *part_count, const double *x, const double *y, const float *score, void *stream) {
    if (!h || !part_count) return SPG_E_INVALID;
    if (img < 0 || img >= h->cfg.max_batch) return fail(h, SPG_E_INVALID, "image_index out of range");
    DeviceGuard guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Workspace &ws = h->ws;
    // the image's dense [K][capP] tables are laid out on the host and go up in three copies + the counters
    const size_t KP = (size_t)ws.K * ws.capP;
    std::vector<double> dx(KP, 0.0), dy(KP, 0.0);
    std::vector<float> ds(KP, 0.0f);
    size_t off = 0;
    for (int c = 0; c < ws.K; c++) {
        const int m = part_count[c];
        if (m < 0 || m > ws.capP) return fail(h, SPG_E_INVALID, "part %d has %d peaks; capacity is %d", c, m, ws.capP);
        if (m && (!x || !y || !score)) return fail(h, SPG_E_INVALID, "peak arrays are NULL");
        for (int q = 0; q < m; q++) {
            dx[(size_t)c * ws.capP + q] = x[off + q];
            dy[(size_t)c * ws.capP + q] = y[off + q];
            ds[(size_t)c * ws.capP + q] = score[off + q];
        }
        off += m;
    }
    const size_t dst = (size_t)img * KP;
    SPG_CUDA(h, cudaMemcpyAsync(ws.peak_x + dst, dx.data(), sizeof(double) * KP, cudaMemcpyHostToDevice, st));
    SPG_CUDA(h, cudaMemcpyAsync(ws.peak_y + dst, dy.data(), sizeof(double) * KP, cudaMemcpyHostToDevice, st));
    SPG_CUDA(h, cudaMemcpyAsync(ws.peak_score + dst, ds.data(), sizeof(float) * KP, cudaMemcpyHostToDevice, st));
    SPG_CUDA(h, cudaMemcpyAsync(ws.peak_count + (size_t)img * ws.K, part_count, sizeof(int32_t) * ws.K, cudaMemcpyHostToDevice, st));
    SPG_CUDA(h, cudaMemsetAsync(ws.status + img, 0, sizeof(uint32_t), st));
    SPG_CUDA(h, cudaStreamSynchronize(st));  // the host arrays are temporaries: one synchronisation per image
    h->stage = std::max(h->stage, 1);
    return SPG_OK;
}

int spg_upload_connections(spg_handle *h, int32_t img, const int32_t *conn_count, const int32_t *ij, const double *score, const double *norm, void *stream) {
    if (!h || !conn_count) return SPG_E_INVALID;
    if (img < 0 || img >= h->cfg.max_batch) return fail(h, SPG_E_INVALID, "image_index out of range");
    DeviceGuard guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Workspace &ws = h->ws;
    // dense [L][capP] tables built on the host: three copies + the counters and ONE synchronisation per image
    // (round 1 synchronised once per limb -- up to 30 host round trips per image)
    const size_t LP = (size_t)ws.L * ws.capP;
    std::vector<uint32_t> dij(LP, 0u);
    std::vector<double> dsc(LP, 0.0), dnm(LP, 0.0);
    size_t off = 0;
    for (int k = 0; k < ws.L; k++) {
        const int m = conn_count[k];
        if (m > ws.capP) return fail(h, SPG_E_INVALID, "limb %d has %d connections; capacity is %d", k, m, ws.capP);
        if (m <= 0) continue;
        if (!ij || !score || !norm) return fail(h, SPG_E_INVALID, "connection arrays are NULL");
        for (int r = 0; r < m; r++) {
            const int32_t i = ij[(off + r) * 2], j = ij[(off + r) * 2 + 1];
            if (i < 0 || j < 0 || i >= ws.capP || j >= ws.capP) return fail(h, SPG_E_INVALID, "connection index out of range");
            dij[(size_t)k * ws.capP + r] = ((uint32_t)i << 16) | (uint32_t)j;
            dsc[(size_t)k * ws.capP + r] = score[off + r];
            dnm[(size_t)k * ws.capP + r] = norm[off + r];
        }
        off += m;
    }
    const size_t dst = (size_t)img * LP;
    SPG_CUDA(h, cudaMemcpyAsync(ws.conn_ij + dst, dij.data(), sizeof(uint32_t) * LP, cudaMemcpyHostToDevice, st));
    SPG_CUDA(h, cudaMemcpyAsync(ws.conn_score + dst, dsc.data(), sizeof(double) * LP, cudaMemcpyHostToDevice, st));
    SPG_CUDA(h, cudaMemcpyAsync(ws.conn_norm + dst, dnm.data(), sizeof(double) * LP, cudaMemcpyHostToDevice, st));
    SPG_CUDA(h, cudaMemcpyAsync(ws.conn_count + (size_t)img * ws.L, conn_count, sizeof(int32_t) * ws.L, cudaMemcpyHostToDevice, st));
    SPG_CUDA(h, cudaStreamSynchronize(st));
    h->stage = std::max(h->stage, 3);
    return SPG_OK;
}

#define SPG_D2H(dst, src, count)                                                                                          \
    do {                                                                                                                  \
        if (dst) SPG_CUDA(h, cudaMemcpyAsync((dst), (src), sizeof(*(dst)) * (size_t)(count), cudaMemcpyDeviceToHost, st)); \
    } while (0)

int spg_download_peaks(spg_handle *h, int32_t n, int32_t *peak_count, double *x, double *y, float *score, uint32_t *anchor, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (const int rc = check_batch(h, n)) return rc;
    DeviceGuard guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Workspace &ws = h->ws;
    const size_t m = (size_t)n * ws.K * ws.capP;
    SPG_D2H(peak_count, ws.peak_count, (size_t)n * ws.K);
    SPG_D2H(x, ws.peak_x, m);
    SPG_D2H(y, ws.peak_y, m);
    SPG_D2H(score, ws.peak_score, m);
    SPG_D2H(anchor, ws.peak_anchor, m);
    SPG_CUDA(h, cudaStreamSynchronize(st));
    return SPG_OK;
}

int spg_download_connections(spg_handle *h, int32_t n, int32_t *conn_count, int32_t *cand_count, uint32_t *ij, double *score, double *norm, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (const int rc = check_batch(h, n)) return rc;
    DeviceGuard guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Workspace &ws = h->ws;
    const size_t m = (size_t)n * ws.L * ws.capP;
    SPG_D2H(conn_count, ws.conn_count, (size_t)n * ws.L);
    SPG_D2H(cand_count, ws.cand_count, (size_t)n * ws.L);
    SPG_D2H(ij, ws.conn_ij, m);
    SPG_D2H(score, ws.conn_score, m);
    SPG_D2H(norm, ws.conn_norm, m);
    SPG_CUDA(h, cudaStreamSynchronize(st));
    return SPG_OK;
}

int spg_download_people(spg_handle *h, int32_t n, int32_t *n_persons, double *subset, double *people_xy, double *people_score, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (const int rc = check_batch(h, n)) return rc;
    DeviceGuard guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Workspace &ws = h->ws;
    SPG_D2H(n_persons, ws.n_persons, (size_t)n);
    SPG_D2H(subset, ws.subset, (size_t)n * ws.capR * (ws.K + 2) * 2);
    SPG_D2H(people_xy, ws.people_xy, (size_t)n * ws.capR * ws.J * 2);
    SPG_D2H(people_score, ws.people_score, (size_t)n * ws.capR);
    SPG_CUDA(h, cudaStreamSynchronize(st));
    return SPG_OK;
}

int spg_download_status(spg_handle *h, int32_t n, uint32_t *status, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (const int rc = check_batch(h, n)) return rc;
    DeviceGuard guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SPG_D2H(status, h->ws.status, (size_t)n);
    SPG_CUDA(h, cudaStreamSynchronize(st));
    return SPG_OK;
}

}  // extern "C"

// ---- the capacity-free tier (group_unbounded.cuh) ------------------------------------------------------------------
extern "C" {

int spg_group_unbounded(spg_handle *h, const spg_image_maps *im, int32_t dtype, const spg_params *p, void *stream) {
    if (!h) return SPG_E_INVALID;
    h->ub_valid = false;
    int rc;
    if (!im || !im->heat || !im->paf) return fail(h, SPG_E_INVALID, "image maps or their heat/paf are NULL");
    if ((rc = check_dtype(h, dtype)) || (rc = check_params(h, p))) return rc;
    const int H = im->height, W = im->width;
    if (H < 2 || W < 2 || H > 32767 || W > 32767) return fail(h, SPG_E_INVALID, "map %dx%d outside [2, 32767x32767]", H, W);
    DeviceGuard guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int K = h->ws.K, L = h->ws.L, J = h->ws.J;
    Workspace ws = h->ws;  // skeleton of the handle, arrays of the tier
    ws.max_batch = 1;
    ws.capC = 0;
    ws.surv_count = nullptr;
    ws.wire = nullptr;
    ws.wire_first = 0;
    ws.wire_rows = 0;
    int64_t *seg_off = nullptr;
    if ((rc = carve(h, h->ub_small, [&](Carver &c) {
             ws.peak_count = c.take<int32_t>(K);
             ws.status = c.take<uint32_t>(1);
             ws.n_persons = c.take<int32_t>(1);
             ws.conn_count = c.take<int32_t>(L);
             ws.cand_count = c.take<int32_t>(L);
             seg_off = c.take<int64_t>(L + 1);
         })))
        return rc;
    UbArgs u{};
    u.heat = im->heat;
    u.paf = im->paf;
    u.heat_chan_stride = im->heat_chan_stride;
    u.paf_chan_stride = im->paf_chan_stride;
    u.H = H;
    u.W = W;
    u.seg_off = seg_off;
    NmsArgs na = nms_args(h, p);
    na.H = H;
    na.W = W;

    // 1. peak counts, then the peak tables sized by the largest part
    SPG_CUDA(h, cudaMemsetAsync(ws.status, 0, sizeof(uint32_t), st));
    u.ws = ws;
    if ((rc = launch(h, kStageNms, "ub_peaks_kernel<count>", ub_peaks_kernel<false>, K, kUbPeakThreads, 0, st, u, na))) return rc;
    std::vector<int32_t> counts((size_t)K);
    SPG_CUDA(h, cudaMemcpyAsync(counts.data(), ws.peak_count, sizeof(int32_t) * K, cudaMemcpyDeviceToHost, st));
    SPG_CUDA(h, cudaStreamSynchronize(st));
    const int P = std::max(1, *std::max_element(counts.begin(), counts.end()));
    if (P > kUbMaxPeaks) return fail(h, SPG_E_INVALID, "a part has %d peaks; the unbounded tier holds at most %d per part", P, kUbMaxPeaks);
    ws.capP = P;
    if ((rc = carve(h, h->ub_peaks, [&](Carver &c) {
             ws.peak_x = c.take<double>((size_t)K * P);
             ws.peak_y = c.take<double>((size_t)K * P);
             ws.peak_score = c.take<float>((size_t)K * P);
             ws.peak_anchor = c.take<uint32_t>((size_t)K * P);
             ws.conn_ij = c.take<uint32_t>((size_t)L * P);
             ws.conn_score = c.take<double>((size_t)L * P);
             ws.conn_norm = c.take<double>((size_t)L * P);
             u.row_count = c.take<int32_t>((size_t)L * P);
             u.row_off = c.take<int64_t>((size_t)L * P);
             u.used = c.take<unsigned char>((size_t)L * 2 * P);
         })))
        return rc;
    u.ws = ws;
    na.ws = ws;
    if ((rc = launch(h, kStageNms, "ub_peaks_kernel<write>", ub_peaks_kernel<true>, K, kUbPeakThreads, 0, st, u, na))) return rc;

    // 2. candidates per pair row, their offsets in generation order, then the candidates themselves
    ScoreArgs sa = score_args(h, p);
    sa.H = H;
    sa.W = W;
    sa.image_extent = im->image_extent;
    sa.ws = ws;
    const dim3 sgrid((unsigned)L, (unsigned)((P + kUbScoreThreads - 1) / kUbScoreThreads));
    SPG_CUDA(h, cudaMemsetAsync(u.row_count, 0, sizeof(int32_t) * (size_t)L * P, st));
    if ((rc = launch(h, kStageScore, "ub_score_kernel<count>", kUbScoreKernels[dtype][0], sgrid, kUbScoreThreads, 0, st, u, sa)))
        return rc;
    std::vector<int32_t> row_count((size_t)L * P);
    SPG_CUDA(h, cudaMemcpyAsync(row_count.data(), u.row_count, sizeof(int32_t) * row_count.size(), cudaMemcpyDeviceToHost, st));
    SPG_CUDA(h, cudaStreamSynchronize(st));
    std::vector<int64_t> row_off(row_count.size()), segs((size_t)L + 1);
    int64_t n_cand = 0;
    for (int k = 0; k < L; k++) {
        segs[k] = n_cand;
        for (int i = 0; i < P; i++) {
            row_off[(size_t)k * P + i] = n_cand;
            n_cand += row_count[(size_t)k * P + i];
        }
    }
    segs[L] = n_cand;
    if (n_cand > 0x7fffffffLL) return fail(h, SPG_E_INVALID, "%lld candidates; the unbounded tier sorts at most 2^31 - 1", (long long)n_cand);
    SPG_CUDA(h, cudaMemcpyAsync(const_cast<int64_t *>(u.row_off), row_off.data(), sizeof(int64_t) * row_off.size(), cudaMemcpyHostToDevice, st));
    SPG_CUDA(h, cudaMemcpyAsync(seg_off, segs.data(), sizeof(int64_t) * segs.size(), cudaMemcpyHostToDevice, st));
    size_t sort_bytes = 0;
    SPG_CUDA(h, cub::DeviceSegmentedRadixSort::SortPairsDescending(
                    nullptr, sort_bytes, (const unsigned long long *)nullptr, (unsigned long long *)nullptr, (const uint32_t *)nullptr,
                    (uint32_t *)nullptr, (int)n_cand, L, seg_off, seg_off + 1, 0, 64, st));
    void *sort_tmp = nullptr;
    uint32_t *sorted = nullptr;
    if ((rc = carve(h, h->ub_cands, [&](Carver &c) {
             ws.cand_prio = c.take<double>((size_t)n_cand);
             ws.cand_score = c.take<double>((size_t)n_cand);
             ws.cand_ij = c.take<uint32_t>((size_t)n_cand);
             ws.cand_key = c.take<unsigned long long>((size_t)n_cand);
             u.cand_key_out = c.take<unsigned long long>((size_t)n_cand);
             u.cand_idx = c.take<uint32_t>((size_t)n_cand);
             sorted = c.take<uint32_t>((size_t)n_cand);
             sort_tmp = c.take<unsigned char>(sort_bytes);
         })))
        return rc;
    u.sorted = sorted;
    u.ws = ws;
    if ((rc = launch(h, kStageScore, "ub_score_kernel<write>", kUbScoreKernels[dtype][1], sgrid, kUbScoreThreads, 0, st, u, sa)))
        return rc;

    // 3. each limb's candidates by priority (stable: ties stay in generation order), then the greedy matching
    if (n_cand > 0)
        SPG_CUDA(h, cub::DeviceSegmentedRadixSort::SortPairsDescending(sort_tmp, sort_bytes, ws.cand_key, u.cand_key_out, u.cand_idx, sorted,
                                                                       (int)n_cand, L, seg_off, seg_off + 1, 0, 64, st));
    SPG_CUDA(h, cudaMemsetAsync(u.used, 0, (size_t)L * 2 * P, st));
    if ((rc = launch(h, kStageMatch, "ub_match_kernel", ub_match_kernel, 1, kMaxLimbs, 0, st, u))) return rc;

    // 4. the person table, one row per accepted connection, and the assembly
    std::vector<int32_t> conn_count((size_t)L);
    SPG_CUDA(h, cudaMemcpyAsync(conn_count.data(), ws.conn_count, sizeof(int32_t) * L, cudaMemcpyDeviceToHost, st));
    SPG_CUDA(h, cudaStreamSynchronize(st));
    int64_t n_conn = 0;
    for (int k = 0; k < L; k++) n_conn += std::max(conn_count[k], 0);
    if (n_conn > kUbMaxRows) return fail(h, SPG_E_INVALID, "%lld connections; the unbounded tier's person table holds at most %d rows",
                                         (long long)n_conn, kUbMaxRows);
    const int R = std::max(1, (int)n_conn);
    ws.capR = R;
    PersonTable &t = u.table;
    t.K = K;
    t.capP = P;
    t.capR = R;
    if ((rc = carve(h, h->ub_people, [&](Carver &c) {
             ws.subset = c.take<double>((size_t)R * (K + 2) * 2);
             ws.people_xy = c.take<double>((size_t)R * std::max(J, 1) * 2);
             ws.people_score = c.take<double>((size_t)R);
             t.row = c.take<RowRec>((size_t)R);
             t.slot = c.take<SlotRec>((size_t)K * R);
             t.pscore = c.take<double>((size_t)R);
             t.ps = c.take<float>((size_t)K * P);
             t.postA = c.take<int>((size_t)R);
             t.postB = c.take<int>((size_t)R);
             t.off = c.take<int>((size_t)K + 1);
             t.owner = c.take<short>((size_t)K * P);
         })))
        return rc;
    t.px = ws.peak_x;
    t.py = ws.peak_y;
    u.ws = ws;
    AssembleArgs aa = assemble_args(h, 0, 1, p);
    aa.wire_flag = nullptr;  // the tier writes no wire record and consumes no armed signal
    aa.done_counter = nullptr;
    aa.ws = ws;
    if ((rc = launch(h, kStageAssemble, "ub_assemble_kernel", ub_assemble_kernel, 1, kUbAssembleThreads, 0, st, u, aa))) return rc;
    h->ub_ws = ws;
    h->ub_valid = true;
    return SPG_OK;
}

int spg_download_unbounded(spg_handle *h, spg_unbounded_sizes *sizes, int32_t *peak_count, double *x, double *y, float *score,
                           uint32_t *anchor, int32_t *conn_count, int32_t *cand_count, uint32_t *ij, double *conn_score,
                           double *conn_norm, double *subset, double *people_xy, double *people_score, void *stream) {
    if (!h || !sizes) return SPG_E_INVALID;
    if (!h->ub_valid) return fail(h, SPG_E_STATE, "no spg_group_unbounded call has succeeded on this handle");
    DeviceGuard guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Workspace &ws = h->ub_ws;
    const size_t KP = (size_t)ws.K * ws.capP, LP = (size_t)ws.L * ws.capP;
    int32_t n_persons = 0;
    uint32_t status = 0;
    SPG_CUDA(h, cudaMemcpyAsync(&n_persons, ws.n_persons, sizeof n_persons, cudaMemcpyDeviceToHost, st));
    SPG_CUDA(h, cudaMemcpyAsync(&status, ws.status, sizeof status, cudaMemcpyDeviceToHost, st));
    SPG_D2H(peak_count, ws.peak_count, ws.K);
    SPG_D2H(x, ws.peak_x, KP);
    SPG_D2H(y, ws.peak_y, KP);
    SPG_D2H(score, ws.peak_score, KP);
    SPG_D2H(anchor, ws.peak_anchor, KP);
    SPG_D2H(conn_count, ws.conn_count, ws.L);
    SPG_D2H(cand_count, ws.cand_count, ws.L);
    SPG_D2H(ij, ws.conn_ij, LP);
    SPG_D2H(conn_score, ws.conn_score, LP);
    SPG_D2H(conn_norm, ws.conn_norm, LP);
    SPG_D2H(subset, ws.subset, (size_t)ws.capR * (ws.K + 2) * 2);
    SPG_D2H(people_xy, ws.people_xy, (size_t)ws.capR * ws.J * 2);
    SPG_D2H(people_score, ws.people_score, (size_t)ws.capR);
    SPG_CUDA(h, cudaStreamSynchronize(st));
    sizes->cap_peaks = ws.capP;
    sizes->cap_rows = ws.capR;
    sizes->n_persons = n_persons;
    sizes->status = status;
    return SPG_OK;
}

}  // extern "C"
