// limb_match.cuh -- K2b: greedy per-limb-type bipartite assignment.
//
// Replaces the matching half of find_connections (/root/reference/evaluate.py:259-274): a stable
// descending sort by priority followed by a sequential scan that accepts a candidate iff neither of its
// end points is used, stopping at min(nA, nB) connections.
//
// Sequential greedy over a strict total order is the same as repeatedly taking the best remaining
// candidate whose end points are both free.  One WARP per (image, limb) does exactly that: each lane
// holds a strided slice of the survivors in registers as a sortable key
//     (order-preserving bits of the priority, ~((i << 16) | j))
// whose lexicographic maximum is the reference's next pick -- priority descending, ties in (i-major,
// j-minor) generation order, which is what Python's stable sorted(..., reverse=True) yields (:259).
// For f32 planes the priority is an f32 value and the whole key is ONE 64-bit word written by the scoring
// kernel: a round is a lane-local max, two REDUX.MAX warp reductions (hi word, then lo word among the
// ties), and a strike of every candidate sharing an end point with the winner (two 16-bit compares each;
// no "used" masks).  f64 planes use a three-word key (f64 priority + tie-break) the same way.  Rows come out in acceptance order, which find_people depends on.  No shared memory,
// no block barrier.  Limbs with more than 256 survivors take a slower generic path.
#pragma once

#include "common.cuh"

namespace spg {

struct MatchArgs {
    int n_images, image_base, keys_valid;
    Workspace ws;
};

constexpr int kMatchThreads = 128;
constexpr int kMatchRegF64 = 16;    // f64-priority path: (key, tie) pairs cached per lane (x32 lanes = 512 per limb, as the f32 path)
constexpr int kMatchRegCands = 16;  // survivor keys cached per lane (x32 lanes = 512 per limb)

__device__ __forceinline__ bool key_better(double pa, int ia, double pb, int ib) {
    return pa > pb || (pa == pb && ia < ib);
}

// order-preserving map f64 -> u64 (larger double <=> larger integer); -0.0 < +0.0 is harmless here
__device__ __forceinline__ unsigned long long ordered_bits(double v) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}

// Greedy rounds over <= 32*NS survivors held in registers (f32 planes: one-word keys).  Specialised on the
// number of register slots so that limbs with few survivors do not pay for eight.  The accepted row's (i, j)
// and score are stored by the lane that owns the winner; limb lengths are filled in afterwards in parallel.
template <int NS>
__device__ __forceinline__ int match_rounds_keys(uint32_t *o_ij, double *o_norm, const unsigned long long (&key8)[kMatchRegCands],
                                                 int nC, int lim, int lane) {
    unsigned long long key[NS];  // 0 = dead / absent
#pragma unroll
    for (int r = 0; r < NS; r++) key[r] = (lane + 32 * r < nC) ? key8[r] : 0ull;  // loaded speculatively, before nC was known
    int m = 0;
    while (m < lim) {
        unsigned long long best = key[0];
#pragma unroll
        for (int r = 1; r < NS; r++) best = max(best, key[r]);
        const uint32_t hi = (uint32_t)(best >> 32), lo = (uint32_t)best;
        const uint32_t mhi = __reduce_max_sync(0xffffffffu, hi);
        if (mhi == 0u) break;  // nothing alive (a real priority never has an all-zero hi word)
        const uint32_t mlo = __reduce_max_sync(0xffffffffu, hi == mhi ? lo : 0u);
        const uint32_t wij = ~mlo;  // winner's (i << 16) | j; (i, j) pairs are unique, so exactly one lane owns it
        if (hi == mhi && lo == mlo) {
            int wr = 0;
#pragma unroll
            for (int r = 1; r < NS; r++)
                if (key[r] == best) wr = r;
            o_ij[m] = wij;  // row [idA, idB, score, i, j, norm] (evaluate.py:267); score and norm follow below
            reinterpret_cast<int *>(o_norm + m)[0] = lane + 32 * wr;  // candidate index, replaced by the norm
        }
        // strike everything that shares an end point with the winner (including the winner itself)
#pragma unroll
        for (int r = 0; r < NS; r++) {
            const uint32_t x = ~(uint32_t)key[r] ^ wij;
            if ((x & 0xffff0000u) == 0u || (x & 0x0000ffffu) == 0u) key[r] = 0ull;
        }
        m++;
    }
    return m;
}

// The same rounds for f64 priorities (f64 planes, or f32 planes evaluated in f64): the key is the order-preserving 64-bit
// image of the priority plus the 32-bit tie-break, three REDUX per round.
template <int NS>
__device__ __forceinline__ int match_rounds_f64(const Workspace &ws, size_t cbase, uint32_t *o_ij, double *o_norm, int nC, int lim, int lane) {
    unsigned long long r_key[NS];  // ordered priority bits; 0 = dead / absent
    uint32_t r_tie[NS];            // ~((i << 16) | j): larger = earlier in generation order
#pragma unroll
    for (int r = 0; r < NS; r++) {
        const int cidx = lane + 32 * r;
        const bool ok = cidx < nC;
        r_key[r] = ok ? ordered_bits(ws.cand_prio[cbase + cidx]) : 0ull;
        r_tie[r] = ok ? ~ws.cand_ij[cbase + cidx] : 0u;
    }
    int m = 0;
    while (m < lim) {
        unsigned long long bk = 0ull;
        uint32_t bt = 0u;
        int br = -1;
#pragma unroll
        for (int r = 0; r < NS; r++) {
            const bool better = r_key[r] > bk || (r_key[r] == bk && r_key[r] != 0ull && r_tie[r] > bt);
            if (better) { bk = r_key[r]; bt = r_tie[r]; br = r; }
        }
        const uint32_t hi = (uint32_t)(bk >> 32), lo = (uint32_t)bk;
        const uint32_t mhi = __reduce_max_sync(0xffffffffu, hi);
        if (mhi == 0u) break;
        const uint32_t mlo = __reduce_max_sync(0xffffffffu, hi == mhi ? lo : 0u);
        const bool tied = (hi == mhi) && (lo == mlo);
        const uint32_t mt = __reduce_max_sync(0xffffffffu, tied ? bt : 0u);
        const uint32_t wij = ~mt;
        if (tied && bt == mt) {
            o_ij[m] = wij;
            reinterpret_cast<int *>(o_norm + m)[0] = lane + 32 * br;  // candidate index, replaced by the norm afterwards
        }
#pragma unroll
        for (int r = 0; r < NS; r++) {
            const uint32_t x = ~r_tie[r] ^ wij;
            if ((x & 0xffff0000u) == 0u || (x & 0x0000ffffu) == 0u) r_key[r] = 0ull;
        }
        m++;
    }
    return m;
}

// The greedy matching of ONE (image, limb) by one warp.  Rows go to o_ij / o_score / o_norm (global memory in the
// stand-alone kernel, shared memory in the fused match+assemble kernel); returns the number of connections, -1 for
// special_k (evaluate.py:272-274).
__device__ __forceinline__ int match_limb(const Workspace &ws, int n, int k, int lane, bool keys_valid, uint32_t *o_ij,
                                          double *o_score, double *o_norm) {
    const size_t slot = (size_t)n * ws.L + k;
    const size_t cbase = slot * ws.capC;
    const int pa = ws.limbs[2 * k], pb = ws.limbs[2 * k + 1];
    // One round trip to L2 instead of three: the survivor keys/scores are fetched speculatively (any slot below capC
    // is valid memory; slots >= nC are masked later) together with the three counters they would otherwise wait for.
    unsigned long long key8[kMatchRegCands];
#pragma unroll
    for (int r = 0; r < kMatchRegCands; r++) {
        const int cidx = lane + 32 * r;
        key8[r] = (keys_valid && cidx < ws.capC) ? ws.cand_key[cbase + cidx] : 0ull;
    }
    const int nC = ws.cand_count[slot];
    const int cntA = ws.peak_count[(size_t)n * ws.K + pa], cntB = ws.peak_count[(size_t)n * ws.K + pb];
    if (nC < 0) return -1;  // special_k
    const int nA = min(cntA, ws.capP);
    const int nB = min(cntB, ws.capP);
    const int lim = min(nA, nB);
    const size_t baseA = ((size_t)n * ws.K + pa) * ws.capP, baseB = ((size_t)n * ws.K + pb) * ws.capP;

    // the rest of row c [idA, idB, score, i, j, norm] (evaluate.py:267) once o_ij[c] holds (i, j): the score of candidate
    // cidx and the limb length (the reference's `norm`, :225)
    auto fill_row = [&](int c, int cidx) {
        const uint32_t ij = o_ij[c];
        const int i = (int)(ij >> 16), j = (int)(ij & 0xffff);
        const double vx = __dsub_rn(ws.peak_x[baseB + j], ws.peak_x[baseA + i]);
        const double vy = __dsub_rn(ws.peak_y[baseB + j], ws.peak_y[baseA + i]);
        o_score[c] = ws.cand_score[cbase + cidx];
        o_norm[c] = __dsqrt_rn(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)));
    };

    int m = 0;
    const int nslots = (nC + 31) >> 5;
    if (keys_valid && nC <= 32 * kMatchRegCands) {
        // ---- fast path, f32 planes: one 64-bit key per survivor, all in registers -----------------------
        switch (nslots) {
            case 0: break;
            case 1: m = match_rounds_keys<1>(o_ij, o_norm, key8, nC, lim, lane); break;
            case 2: m = match_rounds_keys<2>(o_ij, o_norm, key8, nC, lim, lane); break;
            case 3: m = match_rounds_keys<3>(o_ij, o_norm, key8, nC, lim, lane); break;
            case 4: m = match_rounds_keys<4>(o_ij, o_norm, key8, nC, lim, lane); break;
            case 5: m = match_rounds_keys<5>(o_ij, o_norm, key8, nC, lim, lane); break;
            case 6: m = match_rounds_keys<6>(o_ij, o_norm, key8, nC, lim, lane); break;
            case 7: m = match_rounds_keys<7>(o_ij, o_norm, key8, nC, lim, lane); break;
            case 8: m = match_rounds_keys<8>(o_ij, o_norm, key8, nC, lim, lane); break;
            case 9: case 10: m = match_rounds_keys<10>(o_ij, o_norm, key8, nC, lim, lane); break;
            case 11: case 12: m = match_rounds_keys<12>(o_ij, o_norm, key8, nC, lim, lane); break;
            default: m = match_rounds_keys<16>(o_ij, o_norm, key8, nC, lim, lane); break;
        }
        __syncwarp();  // the rows were written by different lanes of this warp; the rounds left row c's candidate index in o_norm[c]
        for (int c = lane; c < m; c += 32) fill_row(c, reinterpret_cast<const int *>(o_norm + c)[0]);  // in parallel
    } else if (nC <= 32 * kMatchRegF64) {
        // ---- register path, f64 priorities: (ordered f64 priority bits, tie-break), specialised on the slot count -----
        switch (nslots) {
            case 0: break;
            case 1: m = match_rounds_f64<1>(ws, cbase, o_ij, o_norm, nC, lim, lane); break;
            case 2: m = match_rounds_f64<2>(ws, cbase, o_ij, o_norm, nC, lim, lane); break;
            case 3: m = match_rounds_f64<3>(ws, cbase, o_ij, o_norm, nC, lim, lane); break;
            case 4: m = match_rounds_f64<4>(ws, cbase, o_ij, o_norm, nC, lim, lane); break;
            case 5: case 6: m = match_rounds_f64<6>(ws, cbase, o_ij, o_norm, nC, lim, lane); break;
            case 7: case 8: m = match_rounds_f64<8>(ws, cbase, o_ij, o_norm, nC, lim, lane); break;
            case 9: case 10: case 11: case 12: m = match_rounds_f64<12>(ws, cbase, o_ij, o_norm, nC, lim, lane); break;
            default: m = match_rounds_f64<kMatchRegF64>(ws, cbase, o_ij, o_norm, nC, lim, lane); break;
        }
        __syncwarp();  // as in the f32 path
        for (int c = lane; c < m; c += 32) fill_row(c, reinterpret_cast<const int *>(o_norm + c)[0]);
    } else {
        // ---- generic path: re-read the list from L2 every round, 128-bit used masks -------------------
        unsigned long long uA0 = 0, uA1 = 0, uB0 = 0, uB1 = 0;
        auto used = [&](uint32_t ij) {
            const int i = ij >> 16, j = ij & 0xffff;
            const unsigned long long ma = (i < 64 ? uA0 : uA1) >> (i & 63);
            const unsigned long long mb = (j < 64 ? uB0 : uB1) >> (j & 63);
            return ((ma | mb) & 1ull) != 0;
        };
        while (m < lim) {
            double bp = 0.0;
            int bi = 0x7fffffff, bidx = -1;
            for (int cidx = lane; cidx < nC; cidx += 32) {
                const uint32_t ij = ws.cand_ij[cbase + cidx];
                if (used(ij)) continue;
                const double pr = ws.cand_prio[cbase + cidx];
                const int p = (int)(ij >> 16) * nB + (int)(ij & 0xffff);
                if (bidx < 0 || key_better(pr, p, bp, bi)) { bp = pr; bi = p; bidx = cidx; }
            }
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) {
                const double op = __shfl_xor_sync(0xffffffffu, bp, s);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, s);
                const int oidx = __shfl_xor_sync(0xffffffffu, bidx, s);
                if (oidx >= 0 && (bidx < 0 || key_better(op, oi, bp, bi))) { bp = op; bi = oi; bidx = oidx; }
            }
            if (bidx < 0) break;  // no candidate with both end points free
            const int i = bi / nB, j = bi - i * nB;
            if (i < 64) uA0 |= 1ull << i; else uA1 |= 1ull << (i - 64);
            if (j < 64) uB0 |= 1ull << j; else uB1 |= 1ull << (j - 64);
            if (lane == 0) {
                o_ij[m] = ((uint32_t)i << 16) | (uint32_t)j;
                fill_row(m, bidx);
            }
            m++;
        }
    }
    return m;
}

// ---------------------------------------------------------------------------------------------------------------
// The same matching in PARALLEL rounds (the fused match+assemble kernel's matchers).
//
// Sequential greedy over a strict total order accepts exactly the candidates that are "locally dominant" once every
// better candidate sharing an end point with them has been decided -- so it can run in rounds: every live candidate
// posts its key on its two end points (shared-memory atomicMax), the candidates that hold the maximum on BOTH end points
// are accepted together, everything sharing an end point with an accepted candidate dies, repeat.  A crowded limb
// (30 x 30 peaks, ~80 candidates) needs 2-3 rounds instead of 30 strictly serial ones.  Which rows come out is the
// same set; the ORDER find_people consumes them in (acceptance order = key descending, evaluate.py:259-268) is restored by
// ranking the accepted keys.  The reference's stop at min(nA, nB) rows (:268) never cuts anything off: accepted rows use
// distinct end points, so the count cannot exceed it, and once it is reached no candidate with two free end points is left.
//
// A key is two 32-bit words (priority bits, ~ij); the maximum is taken word by word: first the priority word, then --
// among the candidates that tie on it -- the tie-break word.
constexpr int kMatchLdSlots = 8;  // candidates per lane of the parallel form (x32 = 256 per limb; more: sequential rounds)

__host__ __device__ inline size_t match_scratch_bytes(int capP) {  // per matcher warp
    return (((size_t)capP * (sizeof(unsigned long long) + 4 * sizeof(uint2) + sizeof(int) + 2)) + 15) & ~(size_t)15;
}

struct MatchScratch {
    unsigned long long *acc_key;  // [capP] accepted keys, unordered
    uint2 *best;                  // [2 sets][2 sides][capP] (priority word, tie-break word) maxima; the sets alternate by round
    int *acc_cidx;                // [capP] candidate index of each accepted key
    unsigned char *used;          // [2 sides][capP]
};
__device__ __forceinline__ MatchScratch make_match_scratch(unsigned char *base, int capP) {
    MatchScratch s;
    s.acc_key = reinterpret_cast<unsigned long long *>(base);
    s.best = reinterpret_cast<uint2 *>(s.acc_key + capP);
    s.acc_cidx = reinterpret_cast<int *>(s.best + 4 * (size_t)capP);
    s.used = reinterpret_cast<unsigned char *>(s.acc_cidx + capP);
    return s;
}

template <int NS>
__device__ __forceinline__ int match_rounds_ld(const MatchScratch &sc, int capP, const unsigned long long (&key8)[kMatchRegCands], int nC,
                                               int lane, int tr, const double *score_base) {
    (void)tr;
    int tr_round = 0;
    (void)tr_round;
    for (int e = lane; e < 2 * capP; e += 32) {  // set 0 of the maxima, the used flags
        sc.best[e] = make_uint2(0u, 0u);
        sc.used[e] = 0;
    }
    uint32_t alive = 0u;
#pragma unroll
    for (int r = 0; r < NS; r++) alive |= (lane + 32 * r < nC) ? (1u << r) : 0u;
    __syncwarp();
    const uint32_t lt = (1u << lane) - 1u;
    int m = 0, cur = 0;
    SPG_TR(tr + 0, alive);
    for (;;) {
        uint2 *bA = sc.best + (size_t)(2 * cur) * capP, *bB = bA + capP;
        uint2 *zA = sc.best + (size_t)(2 * (cur ^ 1)) * capP, *zB = zA + capP;
        // (a) candidates whose end point was taken last round die; the others post their priority word and clear the
        //     entries of the other set for the next round
#pragma unroll
        for (int r = 0; r < NS; r++) {
            if ((alive >> r) & 1u) {
                const uint32_t ij = ~(uint32_t)key8[r];
                const int i = (int)(ij >> 16), j = (int)(ij & 0xffffu);
                if (sc.used[i] | sc.used[capP + j]) {
                    alive &= ~(1u << r);
                } else {
                    const uint32_t hi = (uint32_t)(key8[r] >> 32);
                    atomicMax(&bA[i].x, hi);
                    atomicMax(&bB[j].x, hi);
                    zA[i] = make_uint2(0u, 0u);
                    zB[j] = make_uint2(0u, 0u);
                }
            }
        }
        if (!__any_sync(0xffffffffu, alive != 0u)) break;
        __syncwarp();
        // (b) among the holders of an end point's best priority word: the tie-break word
        uint32_t topA = 0u, topB = 0u;
#pragma unroll
        for (int r = 0; r < NS; r++) {
            if ((alive >> r) & 1u) {
                const uint32_t lo = (uint32_t)key8[r], hi = (uint32_t)(key8[r] >> 32);
                const uint32_t ij = ~lo;
                const int i = (int)(ij >> 16), j = (int)(ij & 0xffffu);
                if (bA[i].x == hi) { topA |= 1u << r; atomicMax(&bA[i].y, lo); }
                if (bB[j].x == hi) { topB |= 1u << r; atomicMax(&bB[j].y, lo); }
            }
        }
        __syncwarp();
        // (c) best on both end points: accepted
#pragma unroll
        for (int r = 0; r < NS; r++) {
            bool dom = false;
            const uint32_t lo = (uint32_t)key8[r];
            const uint32_t ij = ~lo;
            const int i = (int)(ij >> 16), j = (int)(ij & 0xffffu);
            if ((alive & topA & topB) >> r & 1u) dom = bA[i].y == lo && bB[j].y == lo;
            const uint32_t bm = __ballot_sync(0xffffffffu, dom);
            if (dom) {
                const int pos = m + __popc(bm & lt);
                sc.acc_key[pos] = key8[r];
                sc.acc_cidx[pos] = lane + 32 * r;
                asm volatile("prefetch.global.L1 [%0];" ::"l"(score_base + lane + 32 * r));  // read when the rows are written out
                sc.used[i] = 1;
                sc.used[capP + j] = 1;
                alive &= ~(1u << r);
            }
            m += __popc(bm);
        }
        __syncwarp();
        cur ^= 1;
        if (tr_round < 4) SPG_TR(tr + 1 + tr_round, m);
        tr_round++;
    }
    __syncwarp();
    SPG_TRV(tr + 7, tr_round * 1024 + nC);
    return m;
}

// One (image, limb) by one warp of the fused kernel: rows to o_ij / o_score / o_norm in acceptance order.  (ax, ay, bx, by)
// are the refined coordinates of the limb's two peak lists (the kernel's shared-memory copy).  Limbs the parallel form
// does not cover (f64 priorities, more than 32 * kMatchLdSlots candidates) take the sequential rounds of match_limb.
__device__ __forceinline__ int match_limb_ld(const Workspace &ws, int n, int k, int lane, bool keys_valid, uint32_t *o_ij, double *o_score,
                                             double *o_norm, const double *ax, const double *ay, const double *bx, const double *by,
                                             unsigned char *scratch, uint64_t *coords_bar) {
    if (!keys_valid) return match_limb(ws, n, k, lane, keys_valid, o_ij, o_score, o_norm);
    const size_t slot = (size_t)n * ws.L + k;
    const size_t cbase = slot * ws.capC;
    unsigned long long key8[kMatchRegCands];
#pragma unroll
    for (int r = 0; r < kMatchLdSlots; r++) {  // speculative, as in match_limb: one round trip to L2
        const int cidx = lane + 32 * r;
        key8[r] = cidx < ws.capC ? ws.cand_key[cbase + cidx] : 0ull;
    }
#pragma unroll
    for (int r = kMatchLdSlots; r < kMatchRegCands; r++) key8[r] = 0ull;
    const int nC = ws.cand_count[slot];
    if (nC < 0) return -1;  // special_k
    SPG_TR(16 + 4 * k + 1, nC + (int)(key8[0] & 1ull));
    if (nC > 32 * kMatchLdSlots) return match_limb(ws, n, k, lane, keys_valid, o_ij, o_score, o_norm);
    const MatchScratch sc = make_match_scratch(scratch, ws.capP);
    const int nslots = (nC + 31) >> 5;
    int m = 0;
    switch (nslots) {
        case 0: break;
        case 1: m = match_rounds_ld<1>(sc, ws.capP, key8, nC, lane, 400 + 8 * k, ws.cand_score + cbase); break;
        case 2: m = match_rounds_ld<2>(sc, ws.capP, key8, nC, lane, 400 + 8 * k, ws.cand_score + cbase); break;
        case 3: m = match_rounds_ld<3>(sc, ws.capP, key8, nC, lane, 400 + 8 * k, ws.cand_score + cbase); break;
        case 4: m = match_rounds_ld<4>(sc, ws.capP, key8, nC, lane, 400 + 8 * k, ws.cand_score + cbase); break;
        case 5: case 6: m = match_rounds_ld<6>(sc, ws.capP, key8, nC, lane, 400 + 8 * k, ws.cand_score + cbase); break;
        default: m = match_rounds_ld<kMatchLdSlots>(sc, ws.capP, key8, nC, lane, 400 + 8 * k, ws.cand_score + cbase); break;
    }
    SPG_TR(400 + 8 * k + 5, m);
    if (coords_bar) mbar_wait(coords_bar, 0);  // the staged coordinates (a bulk copy issued at kernel start) have landed
    // acceptance order = key descending: a row's position is the number of accepted keys above its own
    for (int e = lane; e < m; e += 32) {
        const unsigned long long ke = sc.acc_key[e];
        const double score = ws.cand_score[cbase + sc.acc_cidx[e]];  // in flight during the ranking
        int rank = 0;
        for (int f = 0; f < m; f++) rank += sc.acc_key[f] > ke ? 1 : 0;
        const uint32_t ij = ~(uint32_t)ke;
        const int i = (int)(ij >> 16), j = (int)(ij & 0xffffu);
        const double vx = __dsub_rn(bx[j], ax[i]), vy = __dsub_rn(by[j], ay[i]);
        o_ij[rank] = ij;
        o_score[rank] = score;
        o_norm[rank] = __dsqrt_rn(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)));
    }
    __syncwarp();
    SPG_TR(400 + 8 * k + 6, m);
    return m;
}

__global__ void __launch_bounds__(kMatchThreads) limb_match_kernel(MatchArgs a) {
    const Workspace &ws = a.ws;
    const int lane = threadIdx.x & 31;
    const int w = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
    if (w >= a.n_images * ws.L) return;
    const int k = w % ws.L;
    const int n = a.image_base + w / ws.L;
    const size_t slot = (size_t)n * ws.L + k;
    const size_t obase = slot * ws.capP;
    const int m = match_limb(ws, n, k, lane, a.keys_valid != 0, ws.conn_ij + obase, ws.conn_score + obase, ws.conn_norm + obase);
    if (lane == 0) ws.conn_count[slot] = m;
}

}  // namespace spg
