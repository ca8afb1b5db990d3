// track.cu -- spg_track_frames and its kernel, track_kernel (track.cuh describes it), and spg_smooth_frames and its
// kernel, smooth_kernel (smooth.cuh), which reads the ids tracking wrote.
#include "runtime.cuh"

#include "smooth.cuh"
#include "track.cuh"

#include <climits>
#include <cmath>

namespace spg {

// cocoeval.py's kpt_oks_sigmas before its division by 10 (COCO joint order)
__constant__ double kTrackSigma10[kTrackJoints] = {.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87,
                                                   .87, .89, .89};
// a wire record row: 17 x (x, y), the score, the presence mask (8-byte words)
constexpr int kRowWords = 2 * kTrackJoints + 2;

// (a, ia) comes before (b, ib) in the matching order: the higher OKS first, then the lower index (a track's id, a
// person's row)
__device__ __forceinline__ bool track_before(double a, long long ia, double b, long long ib) {
    return a > b || (a == b && ia < ib);
}

// the warp's first (v, i) in the matching order; i < 0: none
__device__ __forceinline__ void warp_first(double &v, long long &i, int &at) {
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o);
        const long long oi = __shfl_xor_sync(0xffffffffu, i, o);
        const int oa = __shfl_xor_sync(0xffffffffu, at, o);
        if (oa >= 0 && (at < 0 || track_before(ov, oi, v, i))) v = ov, i = oi, at = oa;
    }
}

__global__ void __launch_bounds__(kTrackThreads, 1)
track_kernel(const __grid_constant__ TrackRagged r, spg_track_table *tables, int n_tables, double thr, int max_age, int rows) {
    extern __shared__ double oks[];  // [slot][person row], row stride kTrackSlots
    __shared__ long long s_id[kTrackSlots], s_next;
    __shared__ int s_age[kTrackSlots], s_live[kTrackSlots], s_cnt[kTrackSlots];
    __shared__ unsigned s_tmask[kTrackSlots];
    __shared__ double s_area[kTrackSlots], s_var[kTrackJoints];
    __shared__ int s_row_of[kTrackSlots], s_slot_of[kTrackSlots];    // the matching: slot -> row, row -> slot, or -1
    __shared__ int s_best_row[kTrackSlots], s_best_slot[kTrackSlots];  // a round's best free partner, or -1
    constexpr int kWarps = kTrackThreads / 32;
    const int k = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int s = *r.img[k].stream;
    if (s < 0 || s >= n_tables) {  // skipped: no table changes, the persons get -1
        const int np = min(max(*reinterpret_cast<const int *>(r.img[k].record), 0), rows);
        for (int p = tid; p < np; p += kTrackThreads) r.img[k].ids[p] = -1;
        return;
    }
    for (int j = 0; j < k; j++)
        if (*r.img[j].stream == s) return;  // the stream's frames run in the CTA of its first frame
    spg_track_table *tb = tables + s;
    if (tid < kTrackSlots) {
        s_id[tid] = tb->tracks[tid].id;
        s_age[tid] = tb->tracks[tid].age;
        s_live[tid] = tb->tracks[tid].live != 0;
    }
    if (tid < kTrackJoints) {  // cocoeval's (sigmas * 2) ** 2 with sigmas = kpt_oks_sigmas / 10.0
        const double sg = kTrackSigma10[tid] / 10.0;
        s_var[tid] = (sg * 2.0) * (sg * 2.0);
    }
    if (tid == 0) s_next = tb->next_id;
    __syncthreads();
    for (int j = k; j < r.n; j++) {
        if (*r.img[j].stream != s) continue;
        const TrackFrame &f = r.img[j];
        const int np = min(max(*reinterpret_cast<const int *>(f.record), 0), rows);
        const unsigned status = *reinterpret_cast<const unsigned *>(f.record + 4);
        const double *row0 = reinterpret_cast<const double *>(f.record + 8);
        const bool observed = status == 0 && (!f.jpeg_status || *f.jpeg_status == SPG_JPEG_OK);
        if (!observed) {  // step 4 alone
            for (int p = tid; p < np; p += kTrackThreads) f.ids[p] = -1;
            if (tid < kTrackSlots && s_live[tid] && ++s_age[tid] > max_age) s_live[tid] = 0;
            __syncthreads();
            continue;
        }
        // 1. each live track's joints T, its area and |T|, then the OKS matrix
        if (tid < kTrackSlots) {
            s_row_of[tid] = s_slot_of[tid] = -1;
            if (s_live[tid]) {
                const spg_track &t = tb->tracks[tid];
                unsigned m = 0;
                int c = 0;
                double x0 = 0, x1 = 0, y0 = 0, y1 = 0;
                for (int g = 0; g < kTrackJoints; g++) {
                    const double x = t.xy[g][0], y = t.xy[g][1];
                    if (!((t.present >> g) & 1) || !isfinite(x) || !isfinite(y)) continue;
                    if (c == 0) x0 = x1 = x, y0 = y1 = y;
                    x0 = fmin(x0, x), x1 = fmax(x1, x), y0 = fmin(y0, y), y1 = fmax(y1, y);
                    m |= 1u << g;
                    c++;
                }
                const double a = (x1 - x0) * (y1 - y0);
                s_tmask[tid] = m;
                s_cnt[tid] = c;
                s_area[tid] = a > 1.0 ? a : 1.0;
            }
        }
        __syncthreads();
        for (int q = tid; q < kTrackSlots * np; q += kTrackThreads) {
            const int t = q / np, p = q - t * np;
            if (!s_live[t]) continue;
            const spg_track &tr = tb->tracks[t];
            const double *pr = row0 + (size_t)p * kRowWords;
            const unsigned long long pm = reinterpret_cast<const unsigned long long *>(pr)[kRowWords - 1];
            const unsigned tm = s_tmask[t];
            const double area = s_area[t];
            double sum = 0.0;
            for (int g = 0; g < kTrackJoints; g++) {
                const double px = pr[2 * g], py = pr[2 * g + 1];
                if (!((tm >> g) & 1) || !((pm >> g) & 1) || !isfinite(px) || !isfinite(py)) continue;
                const double dx = px - tr.xy[g][0], dy = py - tr.xy[g][1];
                const double e = (dx * dx + dy * dy) / s_var[g] / area / 2.0;
                sum += exp(-e);
            }
            const double o = s_cnt[t] ? sum / (double)s_cnt[t] : 0.0;
            oks[t * kTrackSlots + p] = o;
            if (f.oks) f.oks[(size_t)t * rows + p] = o;
        }
        __syncthreads();
        // 2. rounds of locally dominant pairs: a pair that is the first free pair of its track and of its person in the
        // strict matching order is the pair the sorted greedy takes next among those two, so the rounds give its result
        for (;;) {
            for (int t = warp; t < kTrackSlots; t += kWarps) {
                double v = 0.0;
                long long i = -1;
                int at = -1;
                if (s_live[t] && s_row_of[t] < 0)
                    for (int p = lane; p < np; p += 32) {
                        const double o = oks[t * kTrackSlots + p];
                        if (s_slot_of[p] < 0 && o >= thr && (at < 0 || track_before(o, p, v, i))) v = o, i = p, at = p;
                    }
                warp_first(v, i, at);
                if (lane == 0) s_best_row[t] = at;
            }
            for (int p = warp; p < np; p += kWarps) {
                double v = 0.0;
                long long i = -1;
                int at = -1;
                if (s_slot_of[p] < 0)
                    for (int t = lane; t < kTrackSlots; t += 32) {
                        if (!s_live[t] || s_row_of[t] >= 0) continue;
                        const double o = oks[t * kTrackSlots + p];
                        if (o >= thr && (at < 0 || track_before(o, s_id[t], v, i))) v = o, i = s_id[t], at = t;
                    }
                warp_first(v, i, at);
                if (lane == 0) s_best_slot[p] = at;
            }
            __syncthreads();
            int taken = 0;
            if (tid < kTrackSlots) {
                const int p = s_best_row[tid];
                if (p >= 0 && s_best_slot[p] == tid) {
                    s_row_of[tid] = p;
                    s_slot_of[p] = tid;
                    taken = 1;
                }
            }
            if (!__syncthreads_or(taken)) break;
        }
        // 3. matched tracks take their person's pose and id; 4. the others age
        if (tid < kTrackSlots && s_live[tid]) {
            const int p = s_row_of[tid];
            if (p >= 0) {
                s_age[tid] = 0;
                f.ids[p] = s_id[tid];
            } else if (++s_age[tid] > max_age) {
                s_live[tid] = 0;
            }
        }
        for (int q = tid; q < kTrackSlots * (kRowWords - 1); q += kTrackThreads) {
            const int t = q / (kRowWords - 1), w = q - t * (kRowWords - 1);
            const int p = s_row_of[t];
            if (p < 0) continue;
            const double *pr = row0 + (size_t)p * kRowWords;
            if (w < 2 * kTrackJoints) tb->tracks[t].xy[w >> 1][w & 1] = pr[w];
            else tb->tracks[t].present = reinterpret_cast<const unsigned long long *>(pr)[kRowWords - 1];
        }
        __syncthreads();
        // 5. unmatched persons in row order: a new track in the lowest free slot, else in place of the largest age
        if (warp == 0) {
            for (int p = 0; p < np; p++) {
                if (s_slot_of[p] >= 0) continue;
                int slot = -1;
                for (int b = 0; b < kTrackSlots && slot < 0; b += 32) {
                    const unsigned open = __ballot_sync(0xffffffffu, !s_live[b + lane]);
                    if (open) slot = b + __ffs(open) - 1;
                }
                if (slot < 0) {  // a full table: the largest age first, then the smallest id, as the matching order
                    double v = 0.0;
                    long long i = -1;
                    int at = -1;
                    for (int t = lane; t < kTrackSlots; t += 32)
                        if (at < 0 || track_before((double)s_age[t], s_id[t], v, i)) v = (double)s_age[t], i = s_id[t], at = t;
                    warp_first(v, i, at);
                    slot = at;
                }
                const double *pr = row0 + (size_t)p * kRowWords;
                for (int w = lane; w < 2 * kTrackJoints; w += 32) tb->tracks[slot].xy[w >> 1][w & 1] = pr[w];
                if (lane == 0) {
                    tb->tracks[slot].present = reinterpret_cast<const unsigned long long *>(pr)[kRowWords - 1];
                    s_id[slot] = s_next;
                    s_age[slot] = 0;
                    s_live[slot] = 1;
                    f.ids[p] = s_next++;
                }
                __syncwarp();
            }
        }
        __syncthreads();
    }
    if (tid < kTrackSlots) {
        tb->tracks[tid].id = s_id[tid];
        tb->tracks[tid].age = s_age[tid];
        tb->tracks[tid].live = s_live[tid];
    }
    if (tid == 0) tb->next_id = s_next;
}

// the double nearest 2 pi
constexpr double kTwoPi = 6.283185307179586;

__global__ void __launch_bounds__(kSmoothThreads, 1)
smooth_kernel(const __grid_constant__ SmoothRagged r, spg_smooth_table *tables, int n_tables, double min_cutoff, double beta,
              double d_cutoff, int rows) {
    extern __shared__ double s_scale[];  // [rows]; then s_slot [rows] and s_used [rows]
    int *s_slot = reinterpret_cast<int *>(s_scale + rows);  // per row: its slot, -1 raw, -2 a claim to make
    unsigned *s_used = reinterpret_cast<unsigned *>(s_slot + rows);  // per row: its used joints
    __shared__ long long s_id[kSmoothSlots], s_last[kSmoothSlots];
    __shared__ int s_live[kSmoothSlots], s_owner[kSmoothSlots];
    __shared__ unsigned s_mask[kSmoothSlots];
    constexpr int kWarps = kSmoothThreads / 32;
    constexpr double kInf = __builtin_huge_val();
    const int k = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int s = *r.img[k].stream;
    if (s < 0 || s >= n_tables) {  // skipped: no table changes, the rows are passed through raw
        const SmoothFrame &f = r.img[k];
        const int np = min(max(*reinterpret_cast<const int *>(f.record), 0), rows);
        const double *row0 = reinterpret_cast<const double *>(f.record + 8);
        for (int q = tid; q < np * 2 * kSmoothJoints; q += kSmoothThreads) {
            const int p = q / (2 * kSmoothJoints);
            f.xy[q] = row0[(size_t)p * kRowWords + q - p * 2 * kSmoothJoints];
        }
        return;
    }
    for (int j = 0; j < k; j++)
        if (*r.img[j].stream == s) return;  // the stream's frames run in the CTA of its first frame
    spg_smooth_table *tb = tables + s;
    if (tid < kSmoothSlots) {
        s_id[tid] = tb->slots[tid].id;
        s_last[tid] = tb->slots[tid].last;
        s_live[tid] = tb->slots[tid].live != 0;
        s_mask[tid] = tb->slots[tid].mask;
    }
    long long tick = tb->clock;
    for (int j = k; j < r.n; j++) {
        if (*r.img[j].stream != s) continue;
        const SmoothFrame &f = r.img[j];
        const int np = min(max(*reinterpret_cast<const int *>(f.record), 0), rows);
        const double *row0 = reinterpret_cast<const double *>(f.record + 8);
        const double t = *f.time;
        tick++;  // 1. the clock advances
        if (tid < kSmoothSlots) s_owner[tid] = INT_MAX;
        __syncthreads();
        // 2. per person (one warp each): its used joints, its scale and the live slot holding its id
        for (int p = warp; p < np; p += kWarps) {
            const double *pr = row0 + (size_t)p * kRowWords;
            const unsigned long long pm = reinterpret_cast<const unsigned long long *>(pr)[kRowWords - 1];
            double x = 0.0, y = 0.0;
            if (lane < kSmoothJoints) x = pr[2 * lane], y = pr[2 * lane + 1];
            const bool used = lane < kSmoothJoints && ((pm >> lane) & 1) && isfinite(x) && isfinite(y);
            const unsigned um = __ballot_sync(0xffffffffu, used);
            double x0 = used ? x : kInf, x1 = used ? x : -kInf, y0 = used ? y : kInf, y1 = used ? y : -kInf;
            for (int o = 16; o > 0; o >>= 1) {
                x0 = fmin(x0, __shfl_xor_sync(0xffffffffu, x0, o));
                x1 = fmax(x1, __shfl_xor_sync(0xffffffffu, x1, o));
                y0 = fmin(y0, __shfl_xor_sync(0xffffffffu, y0, o));
                y1 = fmax(y1, __shfl_xor_sync(0xffffffffu, y1, o));
            }
            double sc = 1.0;
            if (um) {
                sc = ((x1 - x0) + (y1 - y0)) / 2.0;
                sc = sc > 1.0 ? sc : 1.0;
            }
            const long long pid = f.ids[p];
            int slot = -1;
            if (pid >= 0) {
                slot = -2;
                for (int b = 0; b < kSmoothSlots; b += 32) {
                    const unsigned m = __ballot_sync(0xffffffffu, s_live[b + lane] && s_id[b + lane] == pid);
                    if (m) {
                        slot = b + __ffs(m) - 1;
                        break;
                    }
                }
            }
            if (lane == 0) {
                s_scale[p] = sc;
                s_slot[p] = slot;
                s_used[p] = um;
                if (slot >= 0) atomicMin(&s_owner[slot], p);
            }
        }
        __syncthreads();
        // a repeated id: the slot belongs to its first row, the others are passed through raw; 4. used slots' last
        for (int p = tid; p < np; p += kSmoothThreads) {
            const int slot = s_slot[p];
            if (slot < 0) continue;
            if (s_owner[slot] != p) s_slot[p] = -1;
            else s_last[slot] = tick;
        }
        __syncthreads();
        // 3. in row order, each person without a slot claims one: the lowest free slot, else the least recently used
        // slot this frame has not used (ties: the lowest index), reset
        if (warp == 0) {
            for (int b = 0; b < np; b += 32) {
                unsigned need = __ballot_sync(0xffffffffu, b + lane < np && s_slot[b + lane] == -2);
                while (need) {
                    const int p = b + __ffs(need) - 1;
                    need &= need - 1;
                    const long long pid = f.ids[p];
                    int slot = -1;
                    bool taken = false;  // an earlier row of this frame claimed a slot for the same id
                    for (int c = 0; c < kSmoothSlots && !taken; c += 32)
                        taken = __ballot_sync(0xffffffffu, s_live[c + lane] && s_id[c + lane] == pid) != 0;
                    for (int c = 0; c < kSmoothSlots && !taken && slot < 0; c += 32) {
                        const unsigned open = __ballot_sync(0xffffffffu, !s_live[c + lane]);
                        if (open) slot = c + __ffs(open) - 1;
                    }
                    if (!taken && slot < 0) {
                        long long v = LLONG_MAX;
                        int at = -1;
                        for (int c = lane; c < kSmoothSlots; c += 32)
                            if (s_last[c] < tick && (at < 0 || s_last[c] < v)) v = s_last[c], at = c;
                        for (int o = 16; o > 0; o >>= 1) {
                            const long long ov = __shfl_xor_sync(0xffffffffu, v, o);
                            const int oa = __shfl_xor_sync(0xffffffffu, at, o);
                            if (oa >= 0 && (at < 0 || ov < v || (ov == v && oa < at))) v = ov, at = oa;
                        }
                        slot = at;
                    }
                    if (slot >= 0) {
                        double *st = &tb->slots[slot].joint[0][0];
                        for (int w = lane; w < 5 * kSmoothJoints; w += 32) st[w] = 0.0;
                        if (lane == 0) {
                            s_live[slot] = 1;
                            s_id[slot] = pid;
                            s_last[slot] = tick;
                            s_mask[slot] = 0;
                        }
                    }
                    if (lane == 0) s_slot[p] = slot;
                    __syncwarp();
                }
            }
        }
        __syncthreads();
        // 5. the (person, joint) pairs: the filter on each used joint of a person with a slot, every other joint raw
        for (int q = tid; q < np * kSmoothJoints; q += kSmoothThreads) {
            const int p = q / kSmoothJoints, g = q - p * kSmoothJoints;
            const double *pr = row0 + (size_t)p * kRowWords;
            double x = pr[2 * g], y = pr[2 * g + 1];
            const int slot = s_slot[p];
            if (slot >= 0 && ((s_used[p] >> g) & 1)) {
                double *st = tb->slots[slot].joint[g];
                const double dt = t - st[4];
                double xh = x, yh = y, dxh = 0.0, dyh = 0.0;
                if (((s_mask[slot] >> g) & 1) && dt > 0.0 && isfinite(dt)) {
                    const double sc = s_scale[p];
                    const double vx = (x - st[0]) / dt / sc, vy = (y - st[1]) / dt / sc;
                    const double ad = 1.0 / (1.0 + 1.0 / (kTwoPi * d_cutoff * dt));
                    dxh = ad * vx + (1.0 - ad) * st[2];
                    dyh = ad * vy + (1.0 - ad) * st[3];
                    const double fc = min_cutoff + beta * sqrt(dxh * dxh + dyh * dyh);
                    const double a = 1.0 / (1.0 + 1.0 / (kTwoPi * fc * dt));
                    xh = a * x + (1.0 - a) * st[0];
                    yh = a * y + (1.0 - a) * st[1];
                }
                st[0] = xh, st[1] = yh, st[2] = dxh, st[3] = dyh, st[4] = t;
                x = xh, y = yh;
            }
            f.xy[2 * q] = x;
            f.xy[2 * q + 1] = y;
        }
        __syncthreads();
        for (int p = tid; p < np; p += kSmoothThreads)  // one row per slot: the rows' used joints now have state
            if (s_slot[p] >= 0) s_mask[s_slot[p]] |= s_used[p];
        __syncthreads();
    }
    if (tid < kSmoothSlots) {
        tb->slots[tid].id = s_id[tid];
        tb->slots[tid].last = s_last[tid];
        tb->slots[tid].live = s_live[tid];
        tb->slots[tid].mask = s_mask[tid];
    }
    if (tid == 0) tb->clock = tick;
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_track_frames(spg_handle *h, const spg_track_frame *frames, int32_t n, spg_track_table *tables, int32_t n_tables,
                     double oks_threshold, int32_t max_age, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (n < 0 || (n > 0 && !frames)) return fail(h, SPG_E_INVALID, "frames is NULL or n negative");
    if (n > 0 && (n_tables < 1 || !tables)) return fail(h, SPG_E_INVALID, "tables is NULL or n_tables below 1");
    if ((reinterpret_cast<uintptr_t>(tables) & 7) != 0) return fail(h, SPG_E_INVALID, "tables must be 8-byte aligned");
    if (!std::isfinite(oks_threshold)) return fail(h, SPG_E_INVALID, "oks_threshold must be finite");
    if (max_age < 0) return fail(h, SPG_E_INVALID, "max_age %d is negative", max_age);
    if (h->ws.J != kTrackJoints) return fail(h, SPG_E_INVALID, "tracking needs 17 output joints (the handle has %d)", h->ws.J);
    std::vector<TrackFrame> ms((size_t)n);
    for (int i = 0; i < n; i++) {  // validate every frame before the first launch
        const spg_track_frame &s = frames[i];
        if (!s.record || !s.stream || !s.ids) return fail(h, SPG_E_INVALID, "frame %d: record, stream or ids is NULL", i);
        if ((reinterpret_cast<uintptr_t>(s.record) & 7) || (reinterpret_cast<uintptr_t>(s.ids) & 7) ||
            (reinterpret_cast<uintptr_t>(s.oks) & 7) || (reinterpret_cast<uintptr_t>(s.stream) & 3) ||
            (reinterpret_cast<uintptr_t>(s.jpeg_status) & 3))
            return fail(h, SPG_E_INVALID, "frame %d: record, ids and oks must be 8-byte aligned, stream and jpeg_status 4-byte", i);
        ms[i] = TrackFrame{static_cast<const unsigned char *>(s.record), s.stream, s.jpeg_status,
                           reinterpret_cast<long long *>(s.ids), s.oks, 0};
    }
    if (ms.empty()) return SPG_OK;
    if (kTrackSmem > smem_room(h, track_kernel))
        return fail(h, SPG_E_INVALID, "the tracking kernel's %zu B of shared memory exceed the device's room", kTrackSmem);
    std::vector<long long> ctas((size_t)n, 1);
    std::vector<RaggedRange> ranges;
    std::vector<int> first;
    int rc;
    if ((rc = deal_ragged(h, ctas, kTrackTableMax, "frame", nullptr, ranges, first))) return rc;
    const int rows = h->ws.wire_rows > 0 ? h->ws.wire_rows : h->ws.capR;
    DeviceGuard guard(h->device);
    TrackRagged table{};
    for (const RaggedRange &g : ranges) {
        fill_table(table, ms, first, g);
        if ((rc = launch(h, kStageTrack, "track_kernel", track_kernel, dim3(g.ctas), kTrackThreads, kTrackSmem,
                         static_cast<cudaStream_t>(stream), table, tables, n_tables, oks_threshold, max_age, rows)))
            return rc;
    }
    return SPG_OK;
}

int spg_smooth_frames(spg_handle *h, const spg_smooth_frame *frames, int32_t n, spg_smooth_table *tables, int32_t n_tables,
                      double min_cutoff, double beta, double d_cutoff, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (n < 0 || (n > 0 && !frames)) return fail(h, SPG_E_INVALID, "frames is NULL or n negative");
    if (n > 0 && (n_tables < 1 || !tables)) return fail(h, SPG_E_INVALID, "tables is NULL or n_tables below 1");
    if ((reinterpret_cast<uintptr_t>(tables) & 7) != 0) return fail(h, SPG_E_INVALID, "tables must be 8-byte aligned");
    if (!std::isfinite(min_cutoff) || !(min_cutoff > 0.0)) return fail(h, SPG_E_INVALID, "min_cutoff %g must be finite and above 0", min_cutoff);
    if (!std::isfinite(d_cutoff) || !(d_cutoff > 0.0)) return fail(h, SPG_E_INVALID, "d_cutoff %g must be finite and above 0", d_cutoff);
    if (!std::isfinite(beta) || !(beta >= 0.0)) return fail(h, SPG_E_INVALID, "beta %g must be finite and at least 0", beta);
    if (h->ws.J != kSmoothJoints) return fail(h, SPG_E_INVALID, "smoothing needs 17 output joints (the handle has %d)", h->ws.J);
    std::vector<SmoothFrame> ms((size_t)n);
    for (int i = 0; i < n; i++) {  // validate every frame before the first launch
        const spg_smooth_frame &s = frames[i];
        if (!s.record || !s.stream || !s.ids || !s.time || !s.xy)
            return fail(h, SPG_E_INVALID, "frame %d: record, stream, ids, time or xy is NULL", i);
        if ((reinterpret_cast<uintptr_t>(s.record) & 7) || (reinterpret_cast<uintptr_t>(s.ids) & 7) ||
            (reinterpret_cast<uintptr_t>(s.time) & 7) || (reinterpret_cast<uintptr_t>(s.xy) & 7) ||
            (reinterpret_cast<uintptr_t>(s.stream) & 3))
            return fail(h, SPG_E_INVALID, "frame %d: record, ids, time and xy must be 8-byte aligned, stream 4-byte", i);
        ms[i] = SmoothFrame{static_cast<const unsigned char *>(s.record), s.stream, reinterpret_cast<const long long *>(s.ids),
                            s.time, s.xy, 0};
    }
    if (ms.empty()) return SPG_OK;
    const int rows = h->ws.wire_rows > 0 ? h->ws.wire_rows : h->ws.capR;
    const size_t smem = (size_t)rows * kSmoothRowBytes;
    if (smem > smem_room(h, smooth_kernel))
        return fail(h, SPG_E_INVALID, "the smoothing kernel's %zu B of shared memory for %d rows exceed the device's room", smem, rows);
    std::vector<long long> ctas((size_t)n, 1);
    std::vector<RaggedRange> ranges;
    std::vector<int> first;
    int rc;
    if ((rc = deal_ragged(h, ctas, kSmoothTableMax, "frame", nullptr, ranges, first))) return rc;
    DeviceGuard guard(h->device);
    SmoothRagged table{};
    for (const RaggedRange &g : ranges) {
        fill_table(table, ms, first, g);
        if ((rc = launch(h, kStageSmooth, "smooth_kernel", smooth_kernel, dim3(g.ctas), kSmoothThreads, smem,
                         static_cast<cudaStream_t>(stream), table, tables, n_tables, min_cutoff, beta, d_cutoff, rows)))
            return rc;
    }
    return SPG_OK;
}

}  // extern "C"
