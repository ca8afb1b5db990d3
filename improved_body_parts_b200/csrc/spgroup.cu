// spgroup.cu -- C ABI (include/spgroup.h) over the sm_90a grouping kernels.
//
// Host-side runtime of the path: handle/workspace management, launch configuration, the chunked
// host-buffer pipeline (H2D copy of chunk c+1 overlapped with the kernels of chunk c on two streams) and
// the state transfer used by the stage-wise drop-in functions.  No torch, no CPU implementation: if the
// device or a launch fails the call fails.
#include "../../include/spgroup.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "assemble.cuh"
#include "common.cuh"
#include "group_unbounded.cuh"
#include "limb_match.cuh"
#include "limb_score.cuh"
#include "limb_score_persist.cuh"
#include "loss.cuh"
#include "match_assemble.cuh"
#include "nms_peaks.cuh"
#include "nms_peaks_persist.cuh"
#include "nms_peaks_banded.cuh"
#include "postnet.cuh"
#include "prenet.cuh"
#include "targets.cuh"

using namespace spg;

static_assert(sizeof(spg_params) == sizeof(spg::Params), "spg_params layout");

static thread_local std::string g_create_error;

// the stage numbers of spg_stage_kernel (include/spgroup.h)
enum : int { kStageNms, kStageScore, kStageMatch, kStageAssemble, kStagePostnet, kStagePrenet, kStageTargets, kStageLoss, kStageCount };

// device scratch that grows on demand (grow) and lives until spg_destroy
struct Scratch {
    void *p = nullptr;
    size_t bytes = 0;
};

struct spg_handle {
    spg_config cfg{};
    int device = 0;
    int sm_count = 0;
    size_t smem_optin = 0;
    Workspace ws{};
    std::vector<void *> allocs;
    Scratch in_heat, in_paf;  // staging for spg_group_host
    unsigned int *done_counter = nullptr;          // "last CTA done" counter of the in-kernel wire signal
    unsigned int *score_queue = nullptr;           // 2 x 2 words: item queues of limb_score_persist_kernel (launch_score)
    unsigned long long *armed_flag = nullptr;      // spg_arm_wire_signal: consumed by the next assemble launch
    unsigned long long armed_value = 0;
    Scratch heat_acc;  // postnet: float64 accumulator of the keypoint maps over the scale loop
    Scratch pre_grid;  // prenet: the padded uint8 images of a launch's rotated members
    Scratch loss_partial;  // spg_loss_forward: the ticket (first 256 bytes), then the float64 partial sums of the CTAs
    // the capacity-free tier (spg_group_unbounded): fixed-size words, tables sized by the peak counts, the candidate list
    // with the sort's scratch, the person table and outputs; `ub_ws` describes the last call's results
    Scratch ub_small, ub_peaks, ub_cands, ub_people;
    Workspace ub_ws{};
    bool ub_valid = false;
    cudaStream_t streams[2] = {nullptr, nullptr};
    int64_t launches = 0;
    const char *stage_kernel[kStageCount] = {"", "", "", "", "", "", "", ""};
    // tuning / A-B switches, read from the environment ONCE in spg_create (never per launch); none changes a result
    int persist = 1;      // persistent warp-specialised nms_peaks / limb_score when they apply (SPG_PERSIST=0 turns them off)
    int screen = 1;       // limb_score phase A on (SPG_NO_SCREEN=1 turns it off: every pair is evaluated exactly)
    int exact_warps = 14; // scorer warps of the persistent limb_score (SPG_EXACT_WARPS; DESIGN.md §8 has the sweep)
    int ma_warps = kMAMatchWarps;  // matcher warps of the fused kernel (SPG_MA_WARPS, tuning)
    int fuse_ma = 1;      // whole-path calls run the fused match+assemble kernel (SPG_FUSE_MA=0: the two kernels back to back)
    int cand_dtype = SPG_F32;  // dtype of the planes the current candidates were scored on
    int stage = 0;  // 0 none, 1 peaks, 2 candidates, 3 connections, 4 people
    std::string err;
};

namespace {

int fail(spg_handle *h, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (h) h->err = buf; else g_create_error = buf;
    return code;
}

#define SPG_CUDA(h, call)                                                                              \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) return fail((h), SPG_E_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_)); \
    } while (0)

// a workspace array, zero-filled: the downloads copy whole capacity-sized arrays, so the slots no stage has written yet
// (past a count, or before the first call) hold zeros rather than whatever the memory held before
template <typename T>
int dalloc(spg_handle *h, T **p, size_t count) {
    void *q = nullptr;
    const size_t bytes = std::max<size_t>(count, 1) * sizeof(T);
    SPG_CUDA(h, cudaMalloc(&q, bytes));
    h->allocs.push_back(q);
    *p = static_cast<T *>(q);
    SPG_CUDA(h, cudaMemset(q, 0, bytes));
    return SPG_OK;
}

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
    }
    ~DeviceGuard() {
        int cur = -1;
        cudaGetDevice(&cur);
        if (prev >= 0 && cur != prev) cudaSetDevice(prev);
    }
};

int grow(spg_handle *h, Scratch &s, size_t bytes) {
    if (s.bytes >= bytes) return SPG_OK;
    if (s.p) cudaFree(s.p);
    s.p = nullptr;
    s.bytes = 0;
    SPG_CUDA(h, cudaMalloc(&s.p, bytes));
    s.bytes = bytes;
    return SPG_OK;
}

// Every kernel launch on a handle goes through here: it raises the kernel's dynamic shared memory limit to `smem`,
// launches, records `name` as the kernel of `stage` (spg_stage_kernel), counts the launch (spg_launch_count) and turns
// a launch error into the call's error.
template <typename... P, typename... A>
int launch(spg_handle *h, int stage, const char *name, void (*kern)(P...), dim3 grid, int block, size_t smem, cudaStream_t st,
           const A &...args) {
    if (smem > 0) SPG_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, block, smem, st>>>(args...);
    h->stage_kernel[stage] = name;
    h->launches++;
    SPG_CUDA(h, cudaGetLastError());
    return SPG_OK;
}

// Every ragged launch's table boundaries: given each member's CTA count, consecutive ranges of at most `capacity`
// members (the kernel's table) and at most 2^31 - 1 CTAs (grid.x), and each member's first CTA inside its range.  Fails
// only when one member alone has more CTAs than grid.x holds; it is named as `what` and ids[i] (nullptr: its position).
struct RaggedRange {
    size_t begin, end;  // members [begin, end)
    unsigned ctas;      // grid.x
};
int deal_ragged(spg_handle *h, const std::vector<long long> &ctas, size_t capacity, const char *what, const int *ids,
                std::vector<RaggedRange> &ranges, std::vector<int> &first_cta) {
    ranges.clear();
    first_cta.assign(ctas.size(), 0);
    long long total = 0;
    for (size_t i = 0; i < ctas.size(); i++) {
        if (ctas[i] > 0x7fffffffLL)
            return fail(h, SPG_E_INVALID, "%s %d: its %lld CTAs are above grid.x's 2^31 - 1", what, ids ? ids[i] : (int)i, ctas[i]);
        if (ranges.empty() || ranges.back().end - ranges.back().begin == capacity || total + ctas[i] > 0x7fffffffLL) {
            ranges.push_back(RaggedRange{i, i, 0});
            total = 0;
        }
        first_cta[i] = (int)total;
        total += ctas[i];
        ranges.back().end = i + 1;
        ranges.back().ctas = (unsigned)total;
    }
    return SPG_OK;
}

// range g of the members into the table r, each at its first CTA
template <class Table, class M>
void fill_table(Table &r, const std::vector<M> &ms, const std::vector<int> &first_cta, const RaggedRange &g) {
    r.n = (int)(g.end - g.begin);
    for (int k = 0; k < r.n; k++) {
        r.img[k] = ms[g.begin + k];
        r.img[k].first_cta = first_cta[g.begin + k];
    }
}

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

int check_batch(spg_handle *h, int n) {
    if (n < 0 || n > h->cfg.max_batch) return fail(h, SPG_E_INVALID, "n_images %d outside [0, max_batch=%d]", n, h->cfg.max_batch);
    return SPG_OK;
}

int check_dims(spg_handle *h, int n, int H, int W) {
    int rc;
    if ((rc = check_batch(h, n))) return rc;
    if (H < 2 || W < 2 || H > h->cfg.max_h || W > h->cfg.max_w || H > 32767 || W > 32767)
        return fail(h, SPG_E_INVALID, "map %dx%d outside [2, %dx%d]", H, W, h->cfg.max_h, h->cfg.max_w);
    return SPG_OK;
}

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

// `image` >= 0 names the image of a ragged call in the error
int plan_nms(spg_handle *h, const float *heat, int64_t img_stride, int64_t chan_stride, int H, int W, bool persistent, int image,
             NmsPlan *pl) {
    const int capP = h->ws.capP;
    *pl = NmsPlan{};
    pl->use_bulk = (W % 4 == 0) && (img_stride % 4 == 0) && (chan_stride % 4 == 0) && ((reinterpret_cast<uintptr_t>(heat) & 15) == 0);
    const bool persist = persistent && h->persist && pl->use_bulk;
    if (persist && nms_persist_smem_bytes(H, W, capP) <= h->smem_optin && (size_t)H * W / 4 < 65536 &&
        (size_t)H * W * sizeof(float) < (1u << 20) &&
        ((size_t)H * W / 4 + kNmsPScanners - 1) / kNmsPScanners <= (size_t)32 * kNmsPMaxIter) {
        // one resident CTA per SM: loader, 28 scanners, 3 finishers over a ring of 3 plane slots
        pl->kind = NmsPlan::kPersist;
        pl->smem = nms_persist_smem_bytes(H, W, capP);
        return SPG_OK;
    }
    if (persist) pl->bg = nms_banding(H, W, capP, h->smem_optin - 1024);
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
    if (pl->smem <= h->smem_optin) return SPG_OK;
    if (image < 0)
        return fail(h, SPG_E_INVALID, "map width %d needs %zu B of shared memory per band (limit %zu)", W, pl->smem, h->smem_optin);
    return fail(h, SPG_E_INVALID, "image %d: map width %d needs %zu B of shared memory per band (limit %zu)", image, W, pl->smem,
                h->smem_optin);
}

struct ScorePlan {
    enum { kSampled, kStaged, kPersist } kind;  // kSampled and kStaged index the pairs of ScoreKernels
    size_t smem;
};

ScorePlan plan_score(const spg_handle *h, const ScoreKernels &k, const void *paf, int64_t img_stride, int64_t chan_stride, int H,
                     int W, bool persistent) {
    const int capP = h->ws.capP;
    const size_t plane_bytes = (size_t)H * W * k.esz;
    const bool aligned = (plane_bytes % 16 == 0) && ((img_stride * k.esz) % 16 == 0) && ((chan_stride * k.esz) % 16 == 0) &&
                         ((reinterpret_cast<uintptr_t>(paf) & 15) == 0) && plane_bytes < (1u << 20);
    if (persistent && h->persist && k.persist && aligned && capP <= kPersistMaxCapP && persist_smem_bytes(plane_bytes, capP) <= h->smem_optin)
        return {ScorePlan::kPersist, persist_smem_bytes(plane_bytes, capP)};  // one resident CTA per SM walking a ring of 3 plane slots (loader / screeners / scorers)
    const size_t staged = score_smem_bytes(plane_bytes, capP);
    if (aligned && staged <= h->smem_optin) return {ScorePlan::kStaged, staged};
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
    if ((rc = plan_nms(h, heat, img_stride, chan_stride, H, W, true, -1, &pl))) return rc;
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
    if (smem > h->smem_optin) return fail(h, SPG_E_INVALID, "capacities need %zu B of shared memory in assemble (limit %zu)", smem, h->smem_optin);
    return launch(h, kStageAssemble, "assemble_kernel", assemble_kernel, n, kAssembleThreads, smem, st, a);
}

int launch_match_assemble(spg_handle *h, int base, int n, const spg_params *p, cudaStream_t st) {
    if (n == 0) return SPG_OK;
    AssembleArgs a = assemble_args(h, base, n, p);
    a.use_bulk = ((size_t)h->ws.K * h->ws.capP * sizeof(float)) % 16 == 0;  // bulk copies move multiples of 16 bytes
    const size_t smem = match_assemble_smem_bytes(h->ws.K, h->ws.L, h->ws.capP, h->ws.capR, h->ma_warps);
    if (smem > h->smem_optin) {  // very large capacities: the two stand-alone kernels need less shared memory
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

__global__ void wire_signal_kernel(unsigned long long *word, unsigned long long value) {
    __threadfence_system();  // everything earlier on the stream has completed; order it before the flag for every observer
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(word), "l"(value) : "memory");
}

struct WireWords {
    unsigned long long *p[32];
    int n;
};
__global__ void wire_signal_many_kernel(WireWords w, unsigned long long value) {
    __threadfence_system();
    if ((int)threadIdx.x < w.n) asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(w.p[threadIdx.x]), "l"(value) : "memory");
}

__global__ void wire_wait_kernel(const unsigned long long *word, unsigned long long value) {
    unsigned long long v;
    do {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(word) : "memory");
        if (v < value) __nanosleep(500);
    } while (v < value);
}

}  // namespace

extern "C" {

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

int spg_abi_version(void) { return SPG_ABI_VERSION; }

const char *spg_last_error(const spg_handle *h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int spg_create(const spg_config *cfg, spg_handle **out) {
    if (!cfg || !out) return fail(nullptr, SPG_E_INVALID, "cfg/out is NULL");
    *out = nullptr;
    if (cfg->abi_version != SPG_ABI_VERSION) return fail(nullptr, SPG_E_INVALID, "ABI version %d != %d", cfg->abi_version, SPG_ABI_VERSION);
    if (cfg->n_parts < 1 || cfg->n_parts > kMaxParts || cfg->n_limbs < 1 || cfg->n_limbs > kMaxLimbs || !cfg->limbs)
        return fail(nullptr, SPG_E_INVALID, "n_parts in [1,%d], n_limbs in [1,%d], limbs non-NULL required", kMaxParts, kMaxLimbs);
    if (cfg->n_out_joints < 0 || cfg->n_out_joints > kMaxOutJoints || (cfg->n_out_joints && !cfg->out_from_part))
        return fail(nullptr, SPG_E_INVALID, "n_out_joints in [0,%d]", kMaxOutJoints);
    if (cfg->max_peaks_per_part < 1 || cfg->max_peaks_per_part > kMaxCapPeaks)
        return fail(nullptr, SPG_E_INVALID, "max_peaks_per_part in [1,%d]", kMaxCapPeaks);
    if (cfg->max_person_rows < 1 || cfg->max_person_rows > kMaxCapRows)
        return fail(nullptr, SPG_E_INVALID, "max_person_rows in [1,%d]", kMaxCapRows);
    if (cfg->max_cands_per_limb < 1 || cfg->max_batch < 1 || cfg->max_h < 2 || cfg->max_w < 2)
        return fail(nullptr, SPG_E_INVALID, "max_cands_per_limb, max_batch >= 1 and max_h, max_w >= 2 required");
    for (int k = 0; k < cfg->n_limbs * 2; k++)
        if (cfg->limbs[k] < 0 || cfg->limbs[k] >= cfg->n_parts) return fail(nullptr, SPG_E_INVALID, "limb table entry %d out of range", k);
    for (int g = 0; g < cfg->n_out_joints; g++)
        if (cfg->out_from_part[g] < 0 || cfg->out_from_part[g] >= cfg->n_parts) return fail(nullptr, SPG_E_INVALID, "out_from_part[%d] out of range", g);

    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(nullptr, SPG_E_NO_DEVICE, "no CUDA device (this library has no CPU path)");
    if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, SPG_E_INVALID, "device %d outside [0,%d)", cfg->device, ndev);
    cudaDeviceProp prop{};
    if (cudaGetDeviceProperties(&prop, cfg->device) != cudaSuccess) return fail(nullptr, SPG_E_CUDA, "cudaGetDeviceProperties failed");
    if (prop.major != 9 || prop.minor != 0) return fail(nullptr, SPG_E_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major, prop.minor);

    spg_handle *h = new (std::nothrow) spg_handle();
    if (!h) return fail(nullptr, SPG_E_INVALID, "out of host memory");
    h->cfg = *cfg;
    h->cfg.limbs = nullptr;
    h->cfg.out_from_part = nullptr;
    h->device = cfg->device;
    h->sm_count = prop.multiProcessorCount;
    h->smem_optin = prop.sharedMemPerBlockOptin;
    if (const char *e = getenv("SPG_NO_SCREEN")) h->screen = !(e[0] == '1');
    if (const char *e = getenv("SPG_PERSIST")) h->persist = !(e[0] == '0');  // 0: per-item kernels only (A/B tests)
    if (const char *e = getenv("SPG_MA_WARPS")) h->ma_warps = std::max(1, std::min(15, atoi(e)));
    if (const char *e = getenv("SPG_FUSE_MA")) h->fuse_ma = !(e[0] == '0');
    if (const char *e = getenv("SPG_EXACT_WARPS")) h->exact_warps = std::max(1, std::min(30, atoi(e)));  // the kernel keeps >= 1 screener
    DeviceGuard guard(h->device);

    const size_t N = cfg->max_batch, K = cfg->n_parts, L = cfg->n_limbs, J = cfg->n_out_joints;
    const size_t cP = cfg->max_peaks_per_part, cC = cfg->max_cands_per_limb, cR = cfg->max_person_rows;
    Workspace &ws = h->ws;
    ws.K = (int)K; ws.L = (int)L; ws.J = (int)J; ws.capP = (int)cP; ws.capC = (int)cC; ws.capR = (int)cR; ws.max_batch = (int)N;
    int rc = SPG_OK;
    auto A = [&](int r) { if (rc == SPG_OK) rc = r; };
    A(dalloc(h, &ws.peak_x, N * K * cP));
    A(dalloc(h, &ws.peak_y, N * K * cP));
    A(dalloc(h, &ws.peak_score, N * K * cP));
    A(dalloc(h, &ws.peak_anchor, N * K * cP));
    A(dalloc(h, &ws.peak_count, N * K));
    A(dalloc(h, &ws.cand_prio, N * L * cC));
    A(dalloc(h, &ws.cand_score, N * L * cC));
    A(dalloc(h, &ws.cand_ij, N * L * cC));
    A(dalloc(h, &ws.cand_key, N * L * cC));
    A(dalloc(h, &ws.cand_count, N * L));
    A(dalloc(h, &ws.surv_count, N * L));
    A(dalloc(h, &ws.conn_ij, N * L * cP));
    A(dalloc(h, &ws.conn_score, N * L * cP));
    A(dalloc(h, &ws.conn_norm, N * L * cP));
    A(dalloc(h, &ws.conn_count, N * L));
    A(dalloc(h, &ws.subset, N * cR * (K + 2) * 2));
    A(dalloc(h, &ws.n_persons, N));
    A(dalloc(h, &ws.people_xy, N * cR * std::max<size_t>(J, 1) * 2));
    A(dalloc(h, &ws.people_score, N * cR));
    A(dalloc(h, &ws.status, N));
    A(dalloc(h, &h->score_queue, 4));
    for (size_t i = 0; i < L * 2; i++) ws.limbs[i] = (int16_t)cfg->limbs[i];
    for (size_t g = 0; g < J; g++) ws.out_from_part[g] = (int16_t)cfg->out_from_part[g];
    // every array starts zeroed (dalloc): no status, peaks, candidates or connections until a stage writes them, and
    // score_queue's item queues at 0
    for (int s = 0; s < 2 && rc == SPG_OK; s++)
        if (cudaStreamCreateWithFlags(&h->streams[s], cudaStreamNonBlocking) != cudaSuccess) rc = SPG_E_CUDA;
    if (rc != SPG_OK) {
        g_create_error = h->err.empty() ? "device allocation failed" : h->err;
        spg_destroy(h);
        return rc;
    }
    *out = h;
    return SPG_OK;
}

void spg_destroy(spg_handle *h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    cudaDeviceSynchronize();
    for (void *p : h->allocs) cudaFree(p);
    for (Scratch *s : {&h->in_heat, &h->in_paf, &h->heat_acc, &h->pre_grid, &h->loss_partial, &h->ub_small, &h->ub_peaks, &h->ub_cands, &h->ub_people})
        if (s->p) cudaFree(s->p);
    if (h->done_counter) cudaFree(h->done_counter);
    for (auto &s : h->streams)
        if (s) cudaStreamDestroy(s);
    delete h;
}

int spg_get_device_view(const spg_handle *h, spg_device_view *v) {
    if (!h || !v) return SPG_E_INVALID;
    const Workspace &ws = h->ws;
    v->max_batch = ws.max_batch; v->n_parts = ws.K; v->n_limbs = ws.L; v->n_out_joints = ws.J;
    v->cap_peaks = ws.capP; v->cap_cands = ws.capC; v->cap_rows = ws.capR;
    v->peak_x = ws.peak_x; v->peak_y = ws.peak_y; v->peak_score = ws.peak_score; v->peak_anchor = ws.peak_anchor;
    v->peak_count = ws.peak_count;
    v->conn_ij = ws.conn_ij; v->conn_score = ws.conn_score; v->conn_norm = ws.conn_norm; v->conn_count = ws.conn_count;
    v->cand_count = ws.cand_count;
    v->surv_count = ws.surv_count;
    v->subset = ws.subset; v->n_persons = ws.n_persons; v->people_xy = ws.people_xy; v->people_score = ws.people_score;
    v->status = ws.status;
    return SPG_OK;
}

// ---- wire records + peer memory + stream-ordered signalling ------------------------------------------------------
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

int spg_wire_create(int32_t device, uint64_t bytes, void **dev_ptr, unsigned char ipc_handle[64]) {
    if (!dev_ptr || !ipc_handle || bytes == 0) return SPG_E_INVALID;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    DeviceGuard guard(device);
    void *p = nullptr;
    // a dedicated cudaMalloc allocation: an IPC handle exports the whole allocation it points into
    if (cudaMalloc(&p, bytes) != cudaSuccess) return fail(nullptr, SPG_E_CUDA, "cudaMalloc of %llu wire bytes failed", (unsigned long long)bytes);
    cudaIpcMemHandle_t hd;
    if (cudaMemset(p, 0, bytes) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess || cudaIpcGetMemHandle(&hd, p) != cudaSuccess) {
        const char *why = cudaGetErrorString(cudaGetLastError());
        cudaFree(p);
        return fail(nullptr, SPG_E_CUDA, "exporting the wire buffer failed: %s", why);
    }
    memcpy(ipc_handle, &hd, 64);
    *dev_ptr = p;
    return SPG_OK;
}

int spg_wire_open(int32_t device, const unsigned char ipc_handle[64], void **peer_ptr) {
    if (!peer_ptr || !ipc_handle) return SPG_E_INVALID;
    DeviceGuard guard(device);
    cudaIpcMemHandle_t hd;
    memcpy(&hd, ipc_handle, 64);
    void *p = nullptr;
    const cudaError_t e = cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(nullptr, SPG_E_CUDA, "cudaIpcOpenMemHandle failed: %s (no peer access between the two GPUs?)", cudaGetErrorString(e));
    }
    *peer_ptr = p;
    return SPG_OK;
}

int spg_wire_close(void *peer_ptr) { return (!peer_ptr || cudaIpcCloseMemHandle(peer_ptr) == cudaSuccess) ? SPG_OK : SPG_E_CUDA; }

int spg_wire_destroy(int32_t device, void *dev_ptr) {
    if (!dev_ptr) return SPG_OK;
    DeviceGuard guard(device);
    cudaDeviceSynchronize();
    return cudaFree(dev_ptr) == cudaSuccess ? SPG_OK : SPG_E_CUDA;
}

int spg_wire_signal(int32_t device, uint64_t *word_dev, uint64_t value, void *stream) {
    if (!word_dev) return SPG_E_INVALID;
    DeviceGuard guard(device);
    wire_signal_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<unsigned long long *>(word_dev), value);
    return cudaGetLastError() == cudaSuccess ? SPG_OK : fail(nullptr, SPG_E_CUDA, "wire_signal launch failed");
}

int spg_wire_signal_many(int32_t device, uint64_t *const *words_dev, int32_t n_words, uint64_t value, void *stream) {
    if (!words_dev || n_words < 1 || n_words > 32) return SPG_E_INVALID;
    DeviceGuard guard(device);
    WireWords w{};
    w.n = n_words;
    for (int i = 0; i < n_words; i++) {
        if (!words_dev[i]) return SPG_E_INVALID;
        w.p[i] = reinterpret_cast<unsigned long long *>(words_dev[i]);
    }
    wire_signal_many_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(w, value);
    return cudaGetLastError() == cudaSuccess ? SPG_OK : fail(nullptr, SPG_E_CUDA, "wire_signal_many launch failed");
}

int spg_wire_wait(int32_t device, const uint64_t *word_dev, uint64_t value, void *stream) {
    if (!word_dev) return SPG_E_INVALID;
    DeviceGuard guard(device);
    // cuStreamWaitValue64 through the runtime's driver entry-point lookup (no link-time dependency on libcuda)
    typedef int (*wait_fn_t)(cudaStream_t, unsigned long long, unsigned long long, unsigned int);
    static wait_fn_t wait_fn = nullptr;
    static bool looked = false;
    if (!looked) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuStreamWaitValue64", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            wait_fn = reinterpret_cast<wait_fn_t>(fn);
        cudaGetLastError();
        looked = true;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (wait_fn && wait_fn(st, (unsigned long long)reinterpret_cast<uintptr_t>(word_dev), value, 0u /* CU_STREAM_WAIT_VALUE_GEQ */) == 0) return SPG_OK;
    // no stream memory operations on this driver: a one-thread polling kernel (sleeps between polls)
    wire_wait_kernel<<<1, 1, 0, st>>>(reinterpret_cast<const unsigned long long *>(word_dev), value);
    return cudaGetLastError() == cudaSuccess ? SPG_OK : fail(nullptr, SPG_E_CUDA, "wire_wait launch failed");
}

int64_t spg_launch_count(const spg_handle *h) { return h ? h->launches : 0; }

const char *spg_stage_kernel(const spg_handle *h, int32_t stage) { return (h && stage >= 0 && stage < kStageCount) ? h->stage_kernel[stage] : ""; }

// ---- post-network stage ------------------------------------------------------------------------
int spg_postnet(spg_handle *h, const spg_postnet_desc *d, int32_t n, int32_t H, int32_t W, float *heat_out, void *paf_out,
                int32_t paf_dtype, void *stream) {
    return spg_postnet_rotated(h, d, nullptr, n, H, W, heat_out, paf_out, paf_dtype, stream);
}

// warpAffine's inversion of its matrix (imgproc/src/imgwarp.cpp), in its operation order (this file's host code is built
// without FMA contraction): the kernel then repeats its fixed-point coordinates bit for bit
static void invert_affine(const double *M, double *m) {
    for (int i = 0; i < 6; i++) m[i] = M[i];
    double D = m[0] * m[4] - m[1] * m[3];
    D = D != 0 ? 1.0 / D : 0.0;
    const double A11 = m[4] * D, A22 = m[0] * D;
    m[0] = A11; m[1] *= -D; m[3] *= -D; m[4] = A22;
    const double b1 = -m[0] * m[2] - m[1] * m[5], b2 = -m[3] * m[2] - m[4] * m[5];
    m[2] = b1; m[5] = b2;
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
        if ((rc = grow(h, h->heat_acc, (size_t)h->cfg.max_batch * ws.K * H * W * sizeof(double)))) return rc;
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
        if ((rc = grow(h, h->heat_acc, acc_total * sizeof(double)))) return rc;
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
    if ((rc = grow(h, h->pre_grid, grid_need))) return rc;
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

// ---- training samples --------------------------------------------------------------------------
namespace {

// the parameters every sample of a call shares, checked and resolved
int targets_common(spg_handle *h, const spg_target_params *p, TgtCommon &c) {
    if (!p) return fail(h, SPG_E_INVALID, "params is NULL");
    if (p->stride < 1 || p->out_h < 1 || p->out_w < 1 || p->out_h > 32767 || p->out_w > 32767)
        return fail(h, SPG_E_INVALID, "stride %d or output %dx%d outside [1, 32767]", p->stride, p->out_h, p->out_w);
    if (p->out_h % p->stride || p->out_w % p->stride)
        return fail(h, SPG_E_INVALID, "stride %d does not divide the output %dx%d", p->stride, p->out_h, p->out_w);
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
    smem = loss_smem_bytes(p->width);
    if (smem > h->smem_optin)
        return fail(h, SPG_E_INVALID, "targets: map width %d needs %zu B of shared memory (limit %zu)", p->width, smem, h->smem_optin);
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
    // CUDA torch divides by a host scalar b as a multiply by 1.0f / (float)b
    a.inv_batch = 1.0f / (float)p->batch_divisor;
    a.inv_sw = 1.0f / (float)p->scale_weight_sum;
    a.inv_nw = 1.0f / (float)p->nstack_weight_sum;
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

int spg_loss_forward(spg_handle *h, const spg_loss_params *params, const float *mask_miss, const float *labels,
                     const spg_loss_pred *preds, int32_t pred_dtype, float *stack_sums, float *loss, void *stream) {
    if (!h) return SPG_E_INVALID;
    const LossKernels *kern;
    LossArgs a;
    long long ctas;
    size_t smem;
    int rc;
    if ((rc = loss_setup(h, params, mask_miss, labels, preds, pred_dtype, false, kern, a, ctas, smem))) return rc;
    if (!stack_sums || !loss) return fail(h, SPG_E_INVALID, "stack_sums or loss is NULL");
    DeviceGuard guard(h->device);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t need = 256 + sizeof(double) * kLossScales * a.nstack * (size_t)ctas;
    const bool fresh = h->loss_partial.bytes < need;
    if ((rc = grow(h, h->loss_partial, need))) return rc;
    if (fresh) SPG_CUDA(h, cudaMemsetAsync(h->loss_partial.p, 0, 256, st));  // the ticket starts at 0; each launch leaves it so
    a.ticket = static_cast<unsigned int *>(h->loss_partial.p);
    a.partial = reinterpret_cast<double *>(static_cast<unsigned char *>(h->loss_partial.p) + 256);
    a.sums = stack_sums;
    a.loss = loss;
    return launch(h, kStageLoss, kern->fwd_name, kern->fwd, dim3((unsigned)ctas), kLossThreads, smem, st, a);
}

int spg_loss_backward(spg_handle *h, const spg_loss_params *params, const float *mask_miss, const float *labels,
                      const spg_loss_pred *preds, int32_t pred_dtype, const float *grad_output, void *stream) {
    if (!h) return SPG_E_INVALID;
    const LossKernels *kern;
    LossArgs a;
    long long ctas;
    size_t smem;
    int rc;
    if ((rc = loss_setup(h, params, mask_miss, labels, preds, pred_dtype, true, kern, a, ctas, smem))) return rc;
    if (!grad_output) return fail(h, SPG_E_INVALID, "grad_output is NULL");
    a.grad_output = grad_output;
    DeviceGuard guard(h->device);
    return launch(h, kStageLoss, kern->bwd_name, kern->bwd, dim3((unsigned)ctas), kLossThreads, smem, static_cast<cudaStream_t>(stream), a);
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
    // validate every image before the first launch
    std::vector<int> order((size_t)n);
    NmsPlan np;
    for (int i = 0; i < n; i++) {
        const spg_image_maps &im = images[i];
        if (!im.heat || !im.paf) return fail(h, SPG_E_INVALID, "image %d: heat/paf is NULL", i);
        if (im.height < 2 || im.width < 2 || im.height > max_h || im.width > max_w)
            return fail(h, SPG_E_INVALID, "image %d: map %dx%d outside [2, %dx%d]", i, im.height, im.width, max_h, max_w);
        if ((rc = plan_nms(h, im.heat, 0, im.heat_chan_stride, im.height, im.width, false, i, &np))) return rc;
        order[i] = i;
    }
    if (score_smem_bytes(0, ws.capP) > h->smem_optin) return fail(h, SPG_E_INVALID, "capacities need too much shared memory in limb scoring");
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
        plan_nms(h, im.heat, 0, im.heat_chan_stride, H, W, false, i, &np);  // succeeded in the validation above
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
    DeviceGuard guard(h->device);
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

int spg_host_alloc(void **ptr, uint64_t bytes) {
    if (!ptr) return SPG_E_INVALID;
    return cudaMallocHost(ptr, bytes) == cudaSuccess ? SPG_OK : SPG_E_CUDA;
}
int spg_host_free(void *ptr) { return cudaFreeHost(ptr) == cudaSuccess ? SPG_OK : SPG_E_CUDA; }

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
namespace {

// Lays arrays out in one Scratch, each 256-byte aligned: a pass with base == nullptr measures, a pass with the grown
// buffer hands out the pointers.
struct Carver {
    unsigned char *base = nullptr;
    size_t bytes = 0;
    template <typename T>
    T *take(size_t count) {
        const size_t o = (bytes + 255) & ~(size_t)255;
        bytes = o + std::max<size_t>(count, 1) * sizeof(T);
        return base ? reinterpret_cast<T *>(base + o) : nullptr;
    }
};

template <typename F>
int carve(spg_handle *h, Scratch &s, F &&layout) {
    Carver m;
    layout(m);
    int rc;
    if ((rc = grow(h, s, m.bytes))) return rc;
    Carver c;
    c.base = static_cast<unsigned char *>(s.p);
    layout(c);
    return SPG_OK;
}

// [dtype][write]: the scoring kernel for the plane's storage / arithmetic types (kScoreKernels' dtype order)
void (*const kUbScoreKernels[3][2])(UbArgs, ScoreArgs) = {
    {ub_score_kernel<float, float, false>, ub_score_kernel<float, float, true>},
    {ub_score_kernel<double, double, false>, ub_score_kernel<double, double, true>},
    {ub_score_kernel<float, double, false>, ub_score_kernel<float, double, true>},
};

}  // namespace

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
