// spgroup.cu -- C ABI (include/spgroup.h) over the sm_90a kernels: the handle's lifecycle, its errors and counters, the
// host runtime every stage shares (runtime.cuh declares it), and the wire's handle-less entry points.
//
// Each stage is a translation unit of its own, its kernels with its host code, so that each CUDA module holds one
// stage's kernels and an edit to one stage cannot change another's code: group.cu (the grouping pass and its
// capacity-free tier), postnet.cu (the post- and pre-network stages), train.cu (training samples and loss), cocoeval.cu,
// jpeg.cu with jpeg_frame.cu, yuv.cu and track.cu.  No torch, no CPU implementation: if the device or a launch fails the call
// fails.
#include "runtime.cuh"

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

using namespace spg;

static_assert(sizeof(spg_params) == sizeof(spg::Params), "spg_params layout");

static thread_local std::string g_create_error;

namespace spg {

int fail(spg_handle *h, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (h) h->err = buf; else g_create_error = buf;
    return code;
}

int grow(spg_handle *h, Scratch &s, size_t bytes) {
    if (s.bytes >= bytes) return SPG_OK;
    if (s.p) cudaFree(s.p);
    s.p = nullptr;
    s.bytes = 0;
    SPG_CUDA(h, cudaMalloc(&s.p, bytes));
    s.bytes = bytes;
    return SPG_OK;
}

int stream_capturing(spg_handle *h, cudaStream_t st, bool *capturing) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    SPG_CUDA(h, cudaStreamIsCapturing(st, &cs));
    *capturing = cs == cudaStreamCaptureStatusActive;
    return SPG_OK;
}

int grow_on(spg_handle *h, Scratch &s, size_t bytes, cudaStream_t st, const char *what) {
    if (s.bytes >= bytes) return SPG_OK;
    bool capturing = false;
    int rc;
    if ((rc = stream_capturing(h, st, &capturing))) return rc;
    if (capturing)
        return fail(h, SPG_E_CAPTURE, "%s need %zu B of scratch, %zu B are reserved, and the stream is capturing a graph: reserve "
                    "the frame first (spg_reserve_frame)", what, bytes, s.bytes);
    return grow(h, s, bytes);
}

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

void invert_affine(const double *M, double *m) {
    for (int i = 0; i < 6; i++) m[i] = M[i];
    double D = m[0] * m[4] - m[1] * m[3];
    D = D != 0 ? 1.0 / D : 0.0;
    const double A11 = m[4] * D, A22 = m[0] * D;
    m[0] = A11; m[1] *= -D; m[3] *= -D; m[4] = A22;
    const double b1 = -m[0] * m[2] - m[1] * m[5], b2 = -m[3] * m[2] - m[4] * m[5];
    m[2] = b1; m[5] = b2;
}

}  // namespace spg

namespace {

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
    if (rc == SPG_OK) rc = check_score_room(h);
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
    for (Scratch *s : {&h->in_heat, &h->in_paf, &h->heat_acc, &h->pre_grid, &h->coco_sort, &h->coco_acc, &h->jpeg, &h->ub_small, &h->ub_peaks, &h->ub_cands, &h->ub_people})
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

// ---- the wire's peer memory and stream-ordered signalling: no handle ----------------------------------------------
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

int spg_host_alloc(void **ptr, uint64_t bytes) {
    if (!ptr) return SPG_E_INVALID;
    return cudaMallocHost(ptr, bytes) == cudaSuccess ? SPG_OK : SPG_E_CUDA;
}
int spg_host_free(void *ptr) { return cudaFreeHost(ptr) == cudaSuccess ? SPG_OK : SPG_E_CUDA; }

}  // extern "C"
