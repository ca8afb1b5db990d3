// jpeg_kernels.cuh -- the JPEG decoder's device code (jpeg.cuh describes the kernels), compiled twice:
//
//   jpeg.cu        the kernels of spg_jpeg_decode_ragged: each member's segment, length and chunk and subsequence counts
//                  are in its __grid_constant__ table entry.
//   jpeg_frame.cu  the frame form's count to write kernels (spg_jpeg_decode_frame, a call that can be recorded into a
//                  CUDA graph): the table entry holds capacities, and the frame's segment and length are read from its
//                  device record when the kernel runs.  The DC, IDCT and colour kernels read neither; the frame form
//                  uses the ragged ones.
//
// The including unit defines what differs: JPEG_KERNEL(name) the kernel's name, JPEG_MEMBER(r) the CTA's member,
// JPEG_FRAME_EXIT(past) a return for the CTAs past the frame's work (nothing in the ragged form), JPEG_INTERVAL_END(m)
// the bound of an interval's end in the unstuffed stream, and JPEG_FRAME_FORM to leave out the ragged-only kernels.
// Expanded in jpeg.cu, the source is token for token the ragged kernels' own, so their code does not depend on the frame
// form (a kernel added to jpeg.cu's module changed how nvcc compiled jpeg_color_kernel).
#pragma once

#include "jpeg.cuh"

namespace spg {

__device__ __forceinline__ void jpeg_flag(const JpegMember &m, int code) { atomicCAS(m.status, 0, code); }

// ---- unstuffing ------------------------------------------------------------------------------------------------------
// Byte i of a segment that the parser accepted: a data byte unless it is 0xFF followed by anything but 0x00 (a fill byte
// or the first byte of a marker) or follows a 0xFF (stuffing, or a marker's second byte).
__device__ __forceinline__ unsigned jpeg_byte(const JpegMember &m, long long i) { return i >= 0 && i < m.seg_len ? __ldg(m.seg + i) : 0u; }
__device__ __forceinline__ bool jpeg_kept(const JpegMember &m, long long i) {
    const unsigned b = jpeg_byte(m, i);
    if (i > 0 && jpeg_byte(m, i - 1) == 0xFF) return false;
    return b != 0xFF || (i + 1 < m.seg_len && jpeg_byte(m, i + 1) == 0x00);
}
__device__ __forceinline__ bool jpeg_rst(const JpegMember &m, long long i) {
    const unsigned b = jpeg_byte(m, i);
    return i > 0 && i < m.seg_len && b >= 0xD0 && b <= 0xD7 && jpeg_byte(m, i - 1) == 0xFF;
}

// thread's 16 bytes of chunk `c`: kept bytes and restart markers
__device__ __forceinline__ void jpeg_thread_counts(const JpegMember &m, int c, int *kept, int *rst) {
    const long long i0 = (long long)c * kJpegChunk + threadIdx.x * 16;
    int k = 0, r = 0;
    for (int t = 0; t < 16; t++) {
        k += jpeg_kept(m, i0 + t) && i0 + t < m.seg_len;
        r += jpeg_rst(m, i0 + t);
    }
    *kept = k;
    *rst = r;
}

// block-wide sum of two ints (blockDim.x == kJpegPackThreads)
__device__ __forceinline__ int2 jpeg_block_sum2(int a, int b) {
    __shared__ int2 part[kJpegPackThreads / 32];
    for (int o = 16; o; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = make_int2(a, b);
    __syncthreads();
    int2 s = make_int2(0, 0);
    for (int w = 0; w < kJpegPackThreads / 32; w++) {
        s.x += part[w].x;
        s.y += part[w].y;
    }
    return s;
}

__global__ void __launch_bounds__(kJpegPackThreads) JPEG_KERNEL(jpeg_count)(const __grid_constant__ JpegRagged r) {
    const JpegMember &m = JPEG_MEMBER(r);
    const int c = (int)blockIdx.x - m.first_cta;
    JPEG_FRAME_EXIT(c >= m.n_chunks)
    if (c == 0 && threadIdx.x == 0) *m.status = kJpegStOk;
    int k, rs;
    jpeg_thread_counts(m, c, &k, &rs);
    const int2 s = jpeg_block_sum2(k, rs);
    if (threadIdx.x == 0) {
        m.chunk_counts[2 * c] = s.x;
        m.chunk_counts[2 * c + 1] = s.y;
    }
}

// One CTA per image: the chunks' (kept bytes, restart markers) counts turned in place into exclusive prefix sums, a
// block scan over chunks of kJpegPackThreads with a carry, so that each pack CTA reads its offsets in one load.
__global__ void __launch_bounds__(kJpegPackThreads) JPEG_KERNEL(jpeg_prefix)(const __grid_constant__ JpegRagged r) {
    __shared__ int2 warp_tot[kJpegPackThreads / 32];
    const JpegMember &m = JPEG_MEMBER(r);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int ck = 0, cr = 0;  // carry: the totals of the chunks before this round
    for (int c0 = 0; c0 < m.n_chunks; c0 += kJpegPackThreads) {
        const int c = c0 + threadIdx.x;
        const int k = c < m.n_chunks ? m.chunk_counts[2 * c] : 0, rs = c < m.n_chunks ? m.chunk_counts[2 * c + 1] : 0;
        int ik = k, ir = rs;
        for (int o = 1; o < 32; o <<= 1) {
            const int a = __shfl_up_sync(0xffffffffu, ik, o), b = __shfl_up_sync(0xffffffffu, ir, o);
            if (lane >= o) {
                ik += a;
                ir += b;
            }
        }
        if (lane == 31) warp_tot[warp] = make_int2(ik, ir);
        __syncthreads();
        int ok = ck + ik - k, orr = cr + ir - rs, tk = 0, tr = 0;
        for (int w = 0; w < kJpegPackThreads / 32; w++) {
            if (w < warp) {
                ok += warp_tot[w].x;
                orr += warp_tot[w].y;
            }
            tk += warp_tot[w].x;
            tr += warp_tot[w].y;
        }
        if (c < m.n_chunks) {
            m.chunk_counts[2 * c] = ok;
            m.chunk_counts[2 * c + 1] = orr;
        }
        ck += tk;
        cr += tr;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kJpegPackThreads) JPEG_KERNEL(jpeg_pack)(const __grid_constant__ JpegRagged r) {
    const JpegMember &m = JPEG_MEMBER(r);
    const int c = (int)blockIdx.x - m.first_cta;
    JPEG_FRAME_EXIT(c >= m.n_chunks)
    // the kept bytes and markers of the image's earlier chunks (jpeg_prefix_kernel)
    const int2 before = make_int2(m.chunk_counts[2 * c], m.chunk_counts[2 * c + 1]);
    int k, rs;
    jpeg_thread_counts(m, c, &k, &rs);
    // exclusive scan of (k, rs) over the CTA's threads
    __shared__ int2 warp_tot[kJpegPackThreads / 32];
    int ik = k, ir = rs;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int o = 1; o < 32; o <<= 1) {
        const int a = __shfl_up_sync(0xffffffffu, ik, o), b = __shfl_up_sync(0xffffffffu, ir, o);
        if (lane >= o) {
            ik += a;
            ir += b;
        }
    }
    if (lane == 31) warp_tot[warp] = make_int2(ik, ir);
    __syncthreads();
    int ok = before.x + ik - k, orr = before.y + ir - rs;
    for (int w = 0; w < warp; w++) {
        ok += warp_tot[w].x;
        orr += warp_tot[w].y;
    }
    const long long i0 = (long long)c * kJpegChunk + threadIdx.x * 16;
    for (int t = 0; t < 16; t++) {
        const long long i = i0 + t;
        if (i >= m.seg_len) break;
        if (jpeg_kept(m, i)) m.packed[ok++] = (unsigned char)jpeg_byte(m, i);
        if (jpeg_rst(m, i)) {
            if (orr + 1 < m.n_intervals) m.starts[orr + 1] = ok;
            orr++;
        }
    }
    if (c == m.n_chunks - 1 && threadIdx.x == kJpegPackThreads - 1) {
        m.starts[0] = 0;
        m.starts[m.n_intervals] = ok;  // the last thread holds the stream's length
        if (orr != m.n_intervals - 1) jpeg_flag(m, kJpegStCorrupt);
    }
}

// ---- Huffman decoding ------------------------------------------------------------------------------------------------
// The image's six tables (DC of components 0..2, then AC) in shared memory.
struct JpegTables {
    uint16_t lookup[6][512];
    int maxcode[6][18];
    int valoff[6][18];
    unsigned char sym[6][256];
};

__device__ __forceinline__ void jpeg_load_tables(JpegTables &t, const spg_jpeg_record *rec) {
    for (int i = threadIdx.x; i < 6 * 512; i += blockDim.x) {
        const spg_jpeg_huff &hf = i < 3 * 512 ? rec->dc[i / 512] : rec->ac[i / 512 - 3];
        t.lookup[i / 512][i % 512] = hf.lookup[i % 512];
    }
    for (int i = threadIdx.x; i < 6 * 18; i += blockDim.x) {
        const spg_jpeg_huff &hf = i < 3 * 18 ? rec->dc[i / 18] : rec->ac[i / 18 - 3];
        t.maxcode[i / 18][i % 18] = hf.maxcode[i % 18];
        t.valoff[i / 18][i % 18] = hf.valoff[i % 18];
    }
    for (int i = threadIdx.x; i < 6 * 256; i += blockDim.x) {
        const spg_jpeg_huff &hf = i < 3 * 256 ? rec->dc[i / 256] : rec->ac[i / 256 - 3];
        t.sym[i / 256][i % 256] = hf.symbols[i % 256];
    }
}

// MSB-first bit reader over [0, nbits) of a byte stream; past the end it reads zeros, as libjpeg inserts them.
struct JpegBits {
    const unsigned char *buf;
    int nbytes;
    long long pos;       // bits consumed
    unsigned long long cache;
    int cbits;           // valid bits at the top of cache
    int next;            // next byte to load
    __device__ __forceinline__ void seek(long long p) {
        pos = p;
        next = (int)(p >> 3);
        cache = 0;
        cbits = 0;
        fill();
        const int drop = (int)(p & 7);
        cache <<= drop;
        cbits -= drop;
    }
    __device__ __forceinline__ void fill() {
        while (cbits <= 56) {
            const unsigned long long b = next < nbytes ? (unsigned long long)__ldg(buf + next) : 0ull;
            cache |= b << (56 - cbits);
            cbits += 8;
            next++;
        }
    }
    __device__ __forceinline__ unsigned peek16() { return (unsigned)(cache >> 48); }
    __device__ __forceinline__ void skip(int n) {
        cache <<= n;
        cbits -= n;
        pos += n;
    }
    __device__ __forceinline__ int get(int n) {  // n in 1..16
        const int v = (int)(cache >> (64 - n));
        skip(n);
        return v;
    }
};

// One symbol of table t; -1 for a code that is not in the table.
__device__ __forceinline__ int jpeg_huff(const JpegTables &T, int t, JpegBits &b) {
    b.fill();
    const unsigned w = b.peek16();
    const unsigned e = T.lookup[t][w >> 7];
    if (e) {
        const int len = (int)(e >> 8);
        if (len < 1 || len > 9) return -1;  // not a table spg_jpeg_parse builds; every symbol must consume bits
        b.skip(len);
        return (int)(e & 0xFF);
    }
    for (int l = 10; l <= 16; l++) {
        const int code = (int)(w >> (16 - l));
        if (code <= T.maxcode[t][l]) {
            const int idx = code + T.valoff[t][l];
            if (idx < 0 || idx > 255) return -1;
            b.skip(l);
            return T.sym[t][idx];
        }
    }
    return -1;
}

__device__ __forceinline__ int jpeg_extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

__constant__ unsigned char kJpegZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                              12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                              35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                              58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// component of block u of an MCU
__device__ __forceinline__ int jpeg_comp(const JpegMember &m, int u) {
    const int y = m.hs * m.vs;
    return u < y ? 0 : u - y + 1;
}

// One symbol from state (b.pos, u, k): a DC symbol and its bits (k == 0) or an AC run/size symbol and its bits.  blk is
// the index of the block in progress (k > 0) or of the next one (k == 0); with WRITE the coefficient goes to coef[blk]
// unless blk >= stop_blk.  *started counts DC symbols.  Returns false for a code not in the table or a coefficient
// index past 63 (u, k unchanged then).
template <bool WRITE>
__device__ __forceinline__ bool jpeg_symbol(const JpegMember &m, const JpegTables &T, JpegBits &b, int &u, int &k,
                                            long long &blk, long long stop_blk, int *started) {
    const int c = jpeg_comp(m, u);
    if (k == 0) {
        const int s = jpeg_huff(T, c, b);
        if (s < 0 || s > 15) return false;
        int diff = 0;
        if (s) {
            b.fill();
            diff = jpeg_extend(b.get(s), s);
        }
        if (WRITE && blk < stop_blk) m.coef[blk * 64] = (short)diff;
        ++*started;
        k = 1;
    } else {
        const int rs = jpeg_huff(T, 3 + c, b);
        if (rs < 0) return false;
        const int run = rs >> 4, s = rs & 15;
        int nk;
        if (s) {
            nk = k + run;
            if (nk > 63) return false;
            b.fill();
            const int v = jpeg_extend(b.get(s), s);
            if (WRITE && blk < stop_blk) m.coef[blk * 64 + kJpegZigzag[nk]] = (short)v;
            nk++;
        } else if (run == 15) {
            nk = k + 16;
            if (nk > 64) return false;
        } else {
            nk = 64;
        }
        k = nk;
    }
    if (k == 64) {
        k = 0;
        u = u + 1 == m.bpm ? 0 : u + 1;
        blk++;
    }
    return true;
}

// Decode from state (b.pos, u, k) at a symbol boundary until the position reaches `end` (at a symbol boundary), or
// block index `blk` reaches `stop_blk` at a block boundary.  A bad symbol returns false -- or, for a speculative decode
// (RECOVER), which in a well-formed stream meets one only while it is misaligned, restarts one bit further on at block 0,
// coefficient 0: a rule that depends on the state alone, so that the decode still meets the true chain of states
// (without it a third of the speculative decodes of a 640 x 480 file stop before they synchronise; DESIGN.md §3).
template <bool WRITE, bool RECOVER = false>
__device__ bool jpeg_decode(const JpegMember &m, const JpegTables &T, JpegBits &b, int &u, int &k, long long end,
                            long long &blk, long long stop_blk, int *started) {
    while (b.pos < end && !(k == 0 && blk >= stop_blk)) {
        const long long at = b.pos;
        if (!jpeg_symbol<WRITE>(m, T, b, u, k, blk, stop_blk, started)) {
            if (!RECOVER) return false;
            b.seek(at + 1);
            u = 0;
            k = 0;
        }
    }
    return true;
}

// a packed-stream reader of image m over [0, nbits)
__device__ __forceinline__ JpegBits jpeg_reader(const JpegMember &m, int first_byte, int nbytes) {
    JpegBits b;
    b.buf = m.packed + first_byte;
    b.nbytes = nbytes;
    return b;
}

// Images with restart intervals: thread = interval.
__global__ void __launch_bounds__(kJpegThreads) JPEG_KERNEL(jpeg_interval)(const __grid_constant__ JpegRagged r) {
    __shared__ JpegTables T;
    const JpegMember &m = JPEG_MEMBER(r);
    jpeg_load_tables(T, m.rec);
    __syncthreads();
    const int i = ((int)blockIdx.x - m.first_cta) * kJpegThreads + threadIdx.x;
    if (i >= m.n_intervals) return;
    const int s0 = m.starts[i], s1 = m.starts[i + 1];
    if (s0 < 0 || s1 < s0 || s1 > JPEG_INTERVAL_END(m)) {
        jpeg_flag(m, kJpegStCorrupt);
        return;
    }
    const long long mcus = (long long)m.mcus_x * m.mcus_y;
    const long long first = (long long)i * m.restart * m.bpm;
    const long long last = min((long long)(i + 1) * m.restart, mcus) * m.bpm;
    JpegBits b = jpeg_reader(m, s0, s1 - s0);
    b.seek(0);
    int u = 0, k = 0, started = 0;
    long long blk = first;
    const long long nbits = 8ll * (s1 - s0);
    // decode until the interval's last block is complete; running past its bits reads zeros and is caught below
    const bool ok = jpeg_decode<true>(m, T, b, u, k, nbits + 64 * 32, blk, last, &started);
    if (!ok || blk < last || b.pos > nbits) jpeg_flag(m, kJpegStCorrupt);
}

__device__ __forceinline__ long long jpeg_sub_end(const JpegMember &m, int j, int nbits) {
    return min((long long)(j + 1) * kJpegSubBits, (long long)nbits);
}

// Decode subsequence j from entry (pos, uk) to its exit (speculatively: bad symbols are stepped over); returns the exit
// and the number of DC symbols decoded.
__device__ __forceinline__ void jpeg_speculate(const JpegMember &m, const JpegTables &T, int nbytes, int j, int pos, int uk,
                                               int *exit_pos, int *exit_uk, int *n) {
    *n = 0;
    JpegBits b = jpeg_reader(m, 0, nbytes);
    b.seek(pos);
    int u = uk >> 8, k = uk & 0xFF;
    long long blk = 0;
    jpeg_decode<false, true>(m, T, b, u, k, jpeg_sub_end(m, j, nbytes * 8), blk, 0x7fffffffffffll, n);
    *exit_pos = (int)b.pos;
    *exit_uk = (u << 8) | k;
}

// Images without restart intervals, pass 1: every subsequence from a guessed entry, then rounds inside the CTA.
__global__ void __launch_bounds__(kJpegSubThreads) JPEG_KERNEL(jpeg_sync)(const __grid_constant__ JpegRagged r) {
    __shared__ JpegTables T;
    __shared__ int xp[kJpegSubThreads], xuk[kJpegSubThreads];
    const JpegMember &m = JPEG_MEMBER(r);
    JPEG_FRAME_EXIT(((int)blockIdx.x - m.first_cta) * kJpegSubThreads >= m.n_subs)
    jpeg_load_tables(T, m.rec);
    __syncthreads();
    const int nbytes = m.starts[1], nbits = 8 * nbytes;
    const int j = ((int)blockIdx.x - m.first_cta) * kJpegSubThreads + threadIdx.x;
    const bool live = j < m.n_subs && (long long)j * kJpegSubBits < nbits;
    int ep = live ? j * kJpegSubBits : 0, euk = 0, op = 0, ouk = 0, n = 0;
    if (live) jpeg_speculate(m, T, nbytes, j, ep, euk, &op, &ouk, &n);
    xp[threadIdx.x] = op;
    xuk[threadIdx.x] = ouk;
    __syncthreads();
    // round: take the predecessor's exit; re-decode if it differs from the entry used.  At most one round per thread of
    // the CTA: the first subsequence's entry never changes, so round t fixes the first t + 1 for good.
    for (int round = 0; round < kJpegSubThreads; round++) {
        int changed = 0;
        int np = 0, nuk = 0;
        if (live && threadIdx.x > 0) {
            np = xp[threadIdx.x - 1];
            nuk = xuk[threadIdx.x - 1];
        }
        __syncthreads();
        if (live && threadIdx.x > 0 && (np != ep || nuk != euk)) {
            ep = np;
            euk = nuk;
            int p2, uk2;
            jpeg_speculate(m, T, nbytes, j, ep, euk, &p2, &uk2, &n);
            if (p2 != op || uk2 != ouk) changed = 1;
            op = p2;
            ouk = uk2;
            xp[threadIdx.x] = op;
            xuk[threadIdx.x] = ouk;
        }
        if (!__syncthreads_or(changed)) break;
    }
    if (j < m.n_subs) m.subs[j] = JpegSub{ep, euk, op, ouk, live ? n : 0, 0};
}

// Pass 2, one CTA per image: carry the true state across the CTA boundaries of pass 1, then scan the DC counts.  A thread
// per boundary re-decodes from the previous range's last exit until an exit stops changing, all boundaries at once; a
// boundary whose walk changed its range's last exit makes another round (the first range is exact, so round t settles
// range t at the latest).
__global__ void __launch_bounds__(kJpegThreads) JPEG_KERNEL(jpeg_fixup)(const __grid_constant__ JpegRagged r) {
    __shared__ JpegTables T;
    __shared__ int warp_tot[kJpegThreads / 32];
    const JpegMember &m = JPEG_MEMBER(r);
    jpeg_load_tables(T, m.rec);
    __syncthreads();
    const int nbytes = m.starts[1], nbits = 8 * nbytes;
    const int live = min(m.n_subs, (nbits + kJpegSubBits - 1) / kJpegSubBits);
    if (threadIdx.x == 0 && live == 0 && m.total_blocks > 0) jpeg_flag(m, kJpegStCorrupt);
    const int ranges = (live + kJpegSubThreads - 1) / kJpegSubThreads;
    for (int round = 0; round < ranges; round++) {
        int changed = 0;
        for (int g = threadIdx.x + 1; g < ranges; g += kJpegThreads) {
            const int j0 = g * kJpegSubThreads, j1 = min(j0 + kJpegSubThreads, live);
            int ep = m.subs[j0 - 1].exit_pos, euk = m.subs[j0 - 1].exit_uk;
            for (int j = j0; j < j1; j++) {
                const JpegSub s = m.subs[j];
                if (s.entry_pos == ep && s.entry_uk == euk) break;
                int op, ouk, n;
                jpeg_speculate(m, T, nbytes, j, ep, euk, &op, &ouk, &n);
                m.subs[j] = JpegSub{ep, euk, op, ouk, n, 0};
                if (op == s.exit_pos && ouk == s.exit_uk) break;
                ep = op;
                euk = ouk;
                if (j == j1 - 1) changed = 1;  // the next range's entry moved
            }
        }
        __threadfence_block();
        if (!__syncthreads_or(changed)) break;
    }
    __syncthreads();
    // exclusive scan of n over the live subsequences
    int carry = 0;
    for (int j0 = 0; j0 < live; j0 += kJpegThreads) {
        const int j = j0 + threadIdx.x;
        const int v = j < live ? m.subs[j].n : 0;
        int incl = v;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int o = 1; o < 32; o <<= 1) {
            const int a = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += a;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        int off = carry;
        int tot = 0;
        for (int w = 0; w < kJpegThreads / 32; w++) {
            if (w < warp) off += warp_tot[w];
            tot += warp_tot[w];
        }
        if (j < live) m.subs[j].base = off + incl - v;
        carry += tot;
        __syncthreads();
    }
}

// Pass 3: every subsequence from its true entry, writing its coefficients.
__global__ void __launch_bounds__(kJpegSubThreads) JPEG_KERNEL(jpeg_write)(const __grid_constant__ JpegRagged r) {
    __shared__ JpegTables T;
    const JpegMember &m = JPEG_MEMBER(r);
    JPEG_FRAME_EXIT(((int)blockIdx.x - m.first_cta) * kJpegSubThreads >= m.n_subs)
    jpeg_load_tables(T, m.rec);
    __syncthreads();
    const int nbytes = m.starts[1], nbits = 8 * nbytes;
    const int j = ((int)blockIdx.x - m.first_cta) * kJpegSubThreads + threadIdx.x;
    const int live = min(m.n_subs, (nbits + kJpegSubBits - 1) / kJpegSubBits);
    if (j >= live) return;
    const JpegSub s = m.subs[j];
    const long long total = m.total_blocks;
    long long blk = s.base - ((s.entry_uk & 0xFF) ? 1 : 0);
    const bool last = j == live - 1;
    if (blk >= total) return;  // past the image's last block: data libjpeg never reads
    if (blk < 0 || (int)(blk % m.bpm) != (s.entry_uk >> 8)) {  // the chain does not add up to the MCU structure
        jpeg_flag(m, kJpegStCorrupt);
        return;
    }
    JpegBits b = jpeg_reader(m, 0, nbytes);
    b.seek(s.entry_pos);
    int u = s.entry_uk >> 8, k = s.entry_uk & 0xFF, started = 0;
    // the last subsequence runs on until the last block is complete (zeros past the end are caught below)
    const long long end = last ? (long long)nbits + 64 * 32 : jpeg_sub_end(m, j, nbits);
    const bool ok = jpeg_decode<true>(m, T, b, u, k, end, blk, total, &started);
    if (!ok && (blk < total)) jpeg_flag(m, kJpegStCorrupt);
    if (last && (blk < total || b.pos > nbits)) jpeg_flag(m, kJpegStCorrupt);
}

// ---- DC prediction ---------------------------------------------------------------------------------------------------
// CTA (image, component): the component's blocks in scan order, DC = running sum of the differences (int, as libjpeg's
// predictor), reset at every restart interval, stored as a 16-bit coefficient.
#ifndef JPEG_FRAME_FORM
__global__ void __launch_bounds__(kJpegThreads) jpeg_dc_kernel(const __grid_constant__ JpegRagged r) {
    __shared__ int warp_v[kJpegThreads / 32], warp_f[kJpegThreads / 32];
    const JpegMember &m = ragged_member(r, (int)blockIdx.x);
    const int comp = (int)blockIdx.x - m.first_cta;
    const int per = comp == 0 ? m.hs * m.vs : 1;
    const int u0 = comp == 0 ? 0 : m.hs * m.vs + comp - 1;
    const long long mcus = (long long)m.mcus_x * m.mcus_y;
    const long long nb = mcus * per;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int carry = 0;
    for (long long i0 = 0; i0 < nb; i0 += kJpegThreads) {
        const long long i = i0 + threadIdx.x;
        int v = 0, f = 0;
        long long g = 0;
        if (i < nb) {
            const long long mcu = i / per;
            const int t = (int)(i % per);
            g = mcu * m.bpm + u0 + t;
            v = m.coef[g * 64];
            f = t == 0 && (m.restart ? mcu % m.restart == 0 : mcu == 0);
        }
        // segmented inclusive scan: (v, f) o (v', f') = (f' ? v' : v + v', f | f')
        for (int o = 1; o < 32; o <<= 1) {
            const int pv = __shfl_up_sync(0xffffffffu, v, o), pf = __shfl_up_sync(0xffffffffu, f, o);
            if (lane >= o && !f) v = (int)((unsigned)v + (unsigned)pv);
            if (lane >= o) f |= pf;
        }
        if (lane == 31) {
            warp_v[warp] = v;
            warp_f[warp] = f;
        }
        __syncthreads();
        int pv = carry, pf = 0;  // the prefix before this warp
        for (int w = 0; w < warp; w++) {
            pv = warp_f[w] ? warp_v[w] : (int)((unsigned)pv + (unsigned)warp_v[w]);
            pf |= warp_f[w];
        }
        if (!f) v = (int)((unsigned)v + (unsigned)pv);
        if (i < nb) m.coef[g * 64] = (short)v;
        // the carry into the next chunk: the last thread's value
        __syncthreads();
        if (threadIdx.x == kJpegThreads - 1) warp_v[0] = v;
        __syncthreads();
        carry = warp_v[0];
        __syncthreads();
    }
}
#endif

// ---- dequantisation + islow IDCT ---------------------------------------------------------------------------------------
constexpr int kF0298 = 2446, kF0390 = 3196, kF0541 = 4433, kF0765 = 6270, kF0899 = 7373, kF1175 = 9633, kF1501 = 12299,
              kF1847 = 15137, kF1961 = 16069, kF2053 = 16819, kF2562 = 20995, kF3072 = 25172;

// one 8-point pass (libjpeg's jidctint.c, in 64-bit as its JLONG); outputs descaled by `shift`
__device__ __forceinline__ void jpeg_idct8(const long long *d, long long *o, int shift) {
    long long z1 = (d[2] + d[6]) * kF0541;
    const long long tmp2 = z1 + d[6] * -kF1847, tmp3 = z1 + d[2] * kF0765;
    const long long tmp0 = (d[0] + d[4]) * 8192, tmp1 = (d[0] - d[4]) * 8192;
    const long long t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
    long long a0 = d[7], a1 = d[5], a2 = d[3], a3 = d[1];
    z1 = a0 + a3;
    long long z2 = a1 + a2, z3 = a0 + a2, z4 = a1 + a3;
    const long long z5 = (z3 + z4) * kF1175;
    a0 *= kF0298;
    a1 *= kF2053;
    a2 *= kF3072;
    a3 *= kF1501;
    z1 *= -kF0899;
    z2 *= -kF2562;
    z3 *= -kF1961;
    z4 *= -kF0390;
    z3 += z5;
    z4 += z5;
    a0 += z1 + z3;
    a1 += z2 + z4;
    a2 += z2 + z3;
    a3 += z1 + z4;
    const long long rnd = 1ll << (shift - 1);
    o[0] = (t10 + a3 + rnd) >> shift;
    o[7] = (t10 - a3 + rnd) >> shift;
    o[1] = (t11 + a2 + rnd) >> shift;
    o[6] = (t11 - a2 + rnd) >> shift;
    o[2] = (t12 + a1 + rnd) >> shift;
    o[5] = (t12 - a1 + rnd) >> shift;
    o[3] = (t13 + a0 + rnd) >> shift;
    o[4] = (t13 - a0 + rnd) >> shift;
}

// libjpeg's post-IDCT range limit of an output x (before the +128 level shift)
__device__ __forceinline__ unsigned jpeg_range_limit(long long x) {
    const int i = (int)(x & 1023);
    return i < 128 ? i + 128 : i < 512 ? 255 : i < 896 ? 0 : i - 896;
}

#ifndef JPEG_FRAME_FORM
__global__ void __launch_bounds__(kJpegThreads) jpeg_idct_kernel(const __grid_constant__ JpegRagged r) {
    __shared__ int q[3][64];
    const JpegMember &m = ragged_member(r, (int)blockIdx.x);
    for (int i = threadIdx.x; i < 192; i += kJpegThreads) q[i / 64][i % 64] = m.rec->quant[i / 64][i % 64];
    __syncthreads();
    const long long g = (long long)((int)blockIdx.x - m.first_cta) * kJpegThreads + threadIdx.x;
    if (g >= m.total_blocks) return;
    const long long mcu = g / m.bpm;
    const int u = (int)(g % m.bpm), c = jpeg_comp(m, u);
    const int my = (int)(mcu / m.mcus_x), mx = (int)(mcu % m.mcus_x);
    int by, bx;
    if (c == 0) {
        by = my * m.vs + u / m.hs;
        bx = mx * m.hs + u % m.hs;
    } else {
        by = my;
        bx = mx;
    }
    int pk[32];  // the block's 64 coefficients, two per int (little-endian: the even index in the low half)
    const int4 *src = reinterpret_cast<const int4 *>(m.coef + g * 64);
#pragma unroll
    for (int v = 0; v < 8; v++) {
        const int4 w = src[v];
        pk[4 * v] = w.x;
        pk[4 * v + 1] = w.y;
        pk[4 * v + 2] = w.z;
        pk[4 * v + 3] = w.w;
    }
    bool inside = true;
    int ws[64];  // libjpeg's int workspace
    long long col[8], res[8];
    // pass 1: columns, from the dequantised coefficients (DEQUANTIZE is an int product)
#pragma unroll
    for (int cc = 0; cc < 8; cc++) {
#pragma unroll
        for (int rr = 0; rr < 8; rr++) {
            const int w = pk[(8 * rr + cc) >> 1];
            const int coefv = (cc & 1) ? (short)((unsigned)w >> 16) : (short)(w & 0xFFFF);
            col[rr] = (long long)coefv * q[c][8 * rr + cc];
            inside &= col[rr] >= -16383 && col[rr] <= 16383;
        }
        jpeg_idct8(col, res, 11);
#pragma unroll
        for (int rr = 0; rr < 8; rr++) {
            ws[8 * rr + cc] = (int)res[rr];
            inside &= res[rr] >= -8191 && res[rr] <= 8191;
        }
    }
    unsigned char *dst = m.plane[c] + (long long)by * 8 * m.plane_w[c] + bx * 8;
#pragma unroll
    for (int rr = 0; rr < 8; rr++) {
#pragma unroll
        for (int cc = 0; cc < 8; cc++) col[cc] = ws[8 * rr + cc];
        jpeg_idct8(col, res, 18);
        unsigned lo = 0, hi = 0;
#pragma unroll
        for (int cc = 0; cc < 8; cc++) {
            inside &= res[cc] >= -512 && res[cc] <= 511;
            const unsigned v = jpeg_range_limit(res[cc]);
            if (cc < 4) lo |= v << (8 * cc);
            else hi |= v << (8 * (cc - 4));
        }
        *reinterpret_cast<uint2 *>(dst + (long long)rr * m.plane_w[c]) = make_uint2(lo, hi);
    }
    if (!inside) jpeg_flag(m, kJpegStRange);
}
#endif

// ---- upsampling, colour, orientation ---------------------------------------------------------------------------------
__device__ __forceinline__ int jpeg_px(const JpegMember &m, int c, int y, int x) {
    return m.plane[c][(long long)y * m.plane_w[c] + x];
}

// chroma plane c at frame pixel (y, x): libjpeg's upsampler for the image's sampling (fancy h2v1 / h2v2 when the
// downsampled width exceeds 2, box replication otherwise; fancy h1v2 always), edges replicated
__device__ __forceinline__ int jpeg_chroma(const JpegMember &m, int c, int y, int x) {
    const int dh = (m.frame_h + m.vs - 1) / m.vs, dw = (m.frame_w + m.hs - 1) / m.hs;
    if (m.hs == 1 && m.vs == 1) return jpeg_px(m, c, y, x);
    if (m.vs == 1) {  // h2v1
        const int j = x >> 1;
        if (dw <= 2) return jpeg_px(m, c, y, j);
        if (x == 0) return jpeg_px(m, c, y, 0);
        if (x == 2 * dw - 1) return jpeg_px(m, c, y, dw - 1);
        const int t = 3 * jpeg_px(m, c, y, j);
        return x & 1 ? (t + jpeg_px(m, c, y, j + 1) + 2) >> 2 : (t + jpeg_px(m, c, y, j - 1) + 1) >> 2;
    }
    const int i = y >> 1, odd = y & 1;
    const int nb = odd ? min(i + 1, dh - 1) : max(i - 1, 0);
    if (m.hs == 1) return (3 * jpeg_px(m, c, i, x) + jpeg_px(m, c, nb, x) + (odd ? 2 : 1)) >> 2;  // h1v2
    const int j = x >> 1;  // h2v2
    if (dw <= 2) return jpeg_px(m, c, i, j);
    auto cs = [&](int jj) { return 3 * jpeg_px(m, c, i, jj) + jpeg_px(m, c, nb, jj); };
    if (x == 0) return (4 * cs(0) + 8) >> 4;
    if (x == 2 * dw - 1) return (4 * cs(dw - 1) + 7) >> 4;
    return x & 1 ? (3 * cs(j) + cs(j + 1) + 7) >> 4 : (3 * cs(j) + cs(j - 1) + 8) >> 4;
}

__device__ __forceinline__ unsigned jpeg_clamp(int v) { return (unsigned)min(max(v, 0), 255); }

#ifndef JPEG_FRAME_FORM
__global__ void __launch_bounds__(kJpegThreads) jpeg_color_kernel(const __grid_constant__ JpegRagged r) {
    const JpegMember &m = ragged_member(r, (int)blockIdx.x);
    const long long p = (long long)((int)blockIdx.x - m.first_cta) * kJpegThreads + threadIdx.x;
    if (p >= (long long)m.out_h * m.out_w) return;
    const int oy = (int)(p / m.out_w), ox = (int)(p % m.out_w);
    // OpenCV's ApplyExifOrientation: transpose for 5..8, then flip horizontally (2, 3, 6, 7) / vertically (3, 4, 7, 8)
    const int o = m.orientation;
    const bool hflip = o == 2 || o == 3 || o == 6 || o == 7, vflip = o == 3 || o == 4 || o == 7 || o == 8;
    const int vy = vflip ? m.out_h - 1 - oy : oy, vx = hflip ? m.out_w - 1 - ox : ox;
    const int fy = o >= 5 ? vx : vy, fx = o >= 5 ? vy : vx;
    const int y = jpeg_px(m, 0, fy, fx);
    unsigned b, g, rr;
    if (m.n_comp == 1) {
        b = g = rr = (unsigned)y;
    } else {
        const int cb = jpeg_chroma(m, 1, fy, fx) - 128, cr = jpeg_chroma(m, 2, fy, fx) - 128;
        // libjpeg's tables: FIX(1.40200), FIX(1.77200), FIX(0.71414), FIX(0.34414) with 16 fraction bits
        rr = jpeg_clamp(y + ((91881 * cr + 32768) >> 16));
        g = jpeg_clamp(y + ((-22554 * cb + 32768 + -46802 * cr) >> 16));
        b = jpeg_clamp(y + ((116130 * cb + 32768) >> 16));
    }
    unsigned char *dst = m.out + p * 3;
    dst[0] = (unsigned char)b;
    dst[1] = (unsigned char)g;
    dst[2] = (unsigned char)rr;
}
#endif

}  // namespace spg
