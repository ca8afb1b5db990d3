// match_assemble.cuh -- K2b + K3 fused: greedy matching (evaluate.py:259-274) and person assembly
// (evaluate.py:279-498 + the process() tail :523-543 + the wire record) of one image in ONE CTA.
//
// Back to back, limb_match (7 680 independent one-warp chains) and assemble (256 one-warp chains of 30 limbs) are both
// latency-bound and use a small fraction of the machine; the second cannot start before the first has finished
// every limb of every image.  Inside one CTA per image the dependency is per limb: warps 1..7 match the image's
// limbs (limb k by warp 1 + k % 7, so limb k is ready long before the assembler needs it) and write each limb's
// rows into the assembler's SHARED-MEMORY tables; warp 0 assembles, acquiring a per-limb flag just before it consumes
// the limb.  The connection tables never make a round trip through L2 on the critical path (they are still stored to
// global memory for the stage-wise API), one launch and one dependent wave disappear, and the assembly of limb 0
// starts as soon as the first matcher is done.  Same device functions as the two stand-alone kernels: same results.
#pragma once

#include "assemble.cuh"
#include "limb_match.cuh"

namespace spg {

constexpr int kMAThreads = 32 * (1 + kMAMatchWarps);
constexpr int kMAMaxThreads = 512;

// connection tables + person table + staged coordinates + one scratch area per matcher warp
inline size_t match_assemble_smem_bytes(int K, int L, int capP, int capR, int n_match) {
    return assemble_conn_bytes(L, capP) + assemble_smem_bytes(K, capP, capR) + 2 * (size_t)K * capP * sizeof(double) +
           (size_t)n_match * match_scratch_bytes(capP);
}

__global__ void __launch_bounds__(kMAMaxThreads) match_assemble_kernel(AssembleArgs a, int keys_valid) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ int s_ready[kMaxLimbs];
    __shared__ AsmResult s_res;
    __shared__ int s_out;
    __shared__ uint64_t s_bar;  // the staged peak arrays have landed (bulk copies)
    const Workspace &ws = a.ws;
    if ((int)blockIdx.x >= a.n_images) return;
    const int n = a.image_base + blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = ws.K, L = ws.L, capP = ws.capP, capR = ws.capR;
    SPG_TR(warp == 0 ? 0 : 2 + warp, 0);
    // tables laid out as the stand-alone assembler expects them
    const size_t LC = (size_t)L * capP;
    double *s_cs = reinterpret_cast<double *>(smem_raw);
    double *s_cn = s_cs + LC;
    uint32_t *s_cij = reinterpret_cast<uint32_t *>(s_cn + LC);
    int *s_cc = reinterpret_cast<int *>(s_cij + LC);
    unsigned char *table_base = smem_raw + assemble_conn_bytes(L, capP);
    PersonTable t = make_person_table(table_base, K, capP, capR);
    double *s_xy = reinterpret_cast<double *>(table_base + assemble_smem_bytes(K, capP, capR));
    t.px = s_xy;
    t.py = s_xy + (size_t)K * capP;
    const int n_match = (int)blockDim.x / 32 - 1;
    if (tid < L) s_ready[tid] = 0;
    const bool bulk = a.use_bulk != 0;
    if (tid == 0 && bulk) {
        mbar_init(&s_bar, 1);
        fence_mbar_init();
    }
    __syncthreads();
    if (tid == 0 && bulk) {  // the image's peak scores and refined coordinates: three bulk copies, nobody waits for them yet
        const size_t KP = (size_t)K * capP, g = (size_t)n * KP;
        mbar_expect_tx(&s_bar, (uint32_t)(KP * (sizeof(float) + 2 * sizeof(double))));
        bulk_g2s(t.ps, ws.peak_score + g, (uint32_t)(KP * sizeof(float)), &s_bar);
        bulk_g2s(s_xy, ws.peak_x + g, (uint32_t)(KP * sizeof(double)), &s_bar);
        bulk_g2s(s_xy + KP, ws.peak_y + g, (uint32_t)(KP * sizeof(double)), &s_bar);
    }
    if (warp == 0) {
        // ---- assembler: stamps, owner map, offsets; the peak scores come by bulk copy (or from the matchers, with limb 0's flag)
        SPG_TR(1, 0);
        init_person_rows(t, ws, n, lane);
        __syncwarp();
        if (bulk) mbar_wait(&s_bar, 0);
        const AsmResult res = assemble_limbs<true>(a, t, s_cs, s_cn, s_cij, s_cc, lane, s_ready);
        if (lane == 0) s_res = res;
    } else {
        // ---- matchers: stage the image's peak scores and refined coordinates (every matcher needs its limbs' coordinates
        // for the limb lengths, the assembler the scores, the output phase the coordinates) unless the bulk copies do; then the limbs, strided
        if (!bulk) {
            stage_peaks(t, ws, n, tid - 32, 32 * n_match, s_xy);
            asm volatile("bar.sync 1, %0;" ::"r"(32 * n_match) : "memory");
        }
        unsigned char *scratch = reinterpret_cast<unsigned char *>(s_xy + 2 * (size_t)K * capP) + (size_t)(warp - 1) * match_scratch_bytes(capP);
        for (int k = warp - 1; k < L; k += n_match) {
            uint32_t *o_ij = s_cij + (size_t)k * capP;
            double *o_sc = s_cs + (size_t)k * capP, *o_nm = s_cn + (size_t)k * capP;
            const int pa = ws.limbs[2 * k], pb = ws.limbs[2 * k + 1];
            SPG_TR(16 + 4 * k, 0);
            const int m = match_limb_ld(ws, n, k, lane, keys_valid != 0, o_ij, o_sc, o_nm, t.px + pa * capP, t.py + pa * capP, t.px + pb * capP,
                                        t.py + pb * capP, scratch, bulk ? &s_bar : nullptr);
            __syncwarp();
            SPG_TR(16 + 4 * k + 2, m);
            if (lane == 0) {
                s_cc[k] = m;
                asm volatile("st.release.cta.shared.s32 [%0], %1;" ::"r"(smem_u32(s_ready + k)), "r"(1) : "memory");
            }
            SPG_TR(16 + 4 * k + 3, 0);
            // the stage-wise API (spg_download_connections, spg_assemble) reads the tables from global memory
            const size_t obase = ((size_t)n * L + k) * capP;
            for (int c = lane; c < m; c += 32) {
                ws.conn_ij[obase + c] = o_ij[c];
                ws.conn_score[obase + c] = o_sc[c];
                ws.conn_norm[obase + c] = o_nm[c];
            }
            if (lane == 0) ws.conn_count[(size_t)n * L + k] = m;
        }
    }
    __syncthreads();
    if (bulk) mbar_wait(&s_bar, 0);  // (every thread observes the copies itself)
    // ---- prune + outputs + wire record by the whole CTA (the connection tables are dead: staging space)
    emit_people(a, t, reinterpret_cast<double *>(smem_raw), assemble_conn_bytes(L, capP), &s_out, n, blockIdx.x, s_res, tid, (int)blockDim.x);
}

}  // namespace spg
