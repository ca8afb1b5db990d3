// jpeg.cu -- cv2.imread's JPEG decode (jpeg.cuh): the host parser and checks of spg_jpeg_parse, the decode's scratch
// layout and launches, and the ragged form of the kernels (jpeg_kernels.cuh holds their source).  The frame form's count
// to write kernels are compiled in jpeg_frame.cu.
#include "runtime.cuh"

#include <cstdio>
#include <cstring>

#define JPEG_KERNEL(name) name##_kernel
#define JPEG_MEMBER(r) ragged_member(r, (int)blockIdx.x)
#define JPEG_FRAME_EXIT(past)
#define JPEG_INTERVAL_END(m) m.seg_len
#include "jpeg_kernels.cuh"

using namespace spg;

namespace {

// the ragged form's kernels by JpegKernel (the frame form's are kJpegFrameKernels); every kernel's spg_stage_kernel name
void (*const kJpegRaggedKernels[kJpegCountFrame])(JpegRagged) = {jpeg_count_kernel, jpeg_prefix_kernel, jpeg_pack_kernel, jpeg_interval_kernel,
                                                                 jpeg_sync_kernel,  jpeg_fixup_kernel,  jpeg_write_kernel,
                                                                 jpeg_dc_kernel,    jpeg_idct_kernel,   jpeg_color_kernel};
const char *const kJpegKernelName[kJpegKernels] = {"jpeg_count_kernel", "jpeg_prefix_kernel", "jpeg_pack_kernel", "jpeg_interval_kernel",
                                                   "jpeg_sync_kernel", "jpeg_fixup_kernel", "jpeg_write_kernel",
                                                   "jpeg_dc_kernel", "jpeg_idct_kernel", "jpeg_color_kernel",
                                                   "jpeg_count_frame_kernel", "jpeg_prefix_frame_kernel", "jpeg_pack_frame_kernel",
                                                   "jpeg_interval_frame_kernel", "jpeg_sync_frame_kernel",
                                                   "jpeg_fixup_frame_kernel", "jpeg_write_frame_kernel"};

const int kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                         41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                         30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct JpegRefuse {
    int status;
};

// libjpeg's derived decoding table and its checks: at most 256 codes, and one more than the last code of each length
// (up to the longest) must still fit that length -- no code is all ones.  Throws JpegRefuse.
void jpeg_build_huff(const uint8_t bits[17], const uint8_t *symbols, int count, spg_jpeg_huff *t) {
    memset(t, 0, sizeof *t);
    for (int l = 0; l < 18; l++) t->maxcode[l] = -1;
    t->maxcode[17] = 0x7fffffff;
    memcpy(t->symbols, symbols, (size_t)count);
    int longest = 0;
    for (int l = 1; l <= 16; l++)
        if (bits[l]) longest = l;
    int code = 0, p = 0;
    for (int l = 1; l <= longest; l++) {
        if (bits[l]) {
            t->valoff[l] = p - code;
            for (int i = 0; i < bits[l]; i++, code++, p++)
                if (code < (1 << l) && l <= 9) {
                    const int lo = code << (9 - l);
                    for (int e = 0; e < (1 << (9 - l)); e++) t->lookup[lo + e] = (uint16_t)((l << 8) | symbols[p]);
                }
            t->maxcode[l] = code - 1;
        }
        if (code >= (1 << l)) throw JpegRefuse{SPG_JPEG_TABLES};
        code <<= 1;
    }
}

// OpenCV's ExifReader on the first APP1 segment (its data after the length): the TIFF header 6 bytes in, IFD0's first
// orientation entry (the 16-bit value at entry + 8, whatever the entry's type); 1..8 apply, anything else is 1.  A read
// outside the segment, where OpenCV gives up part way, refuses the file.
int jpeg_exif_orientation(const uint8_t *seg, long long len) {
    if (len <= 6) return 1;
    const uint8_t *t = seg + 6;
    const long long n = len - 6;
    if (n < 2) throw JpegRefuse{SPG_JPEG_EXIF};
    bool le;
    if (t[0] == 'I' && t[1] == 'I') le = true;
    else if (t[0] == 'M' && t[1] == 'M') le = false;
    else throw JpegRefuse{SPG_JPEG_EXIF};
    if (n < 8) throw JpegRefuse{SPG_JPEG_EXIF};
    auto u16 = [&](long long o) { return le ? t[o] | t[o + 1] << 8 : t[o] << 8 | t[o + 1]; };
    auto u32 = [&](long long o) {
        return le ? (uint32_t)t[o] | (uint32_t)t[o + 1] << 8 | (uint32_t)t[o + 2] << 16 | (uint32_t)t[o + 3] << 24
                  : (uint32_t)t[o] << 24 | (uint32_t)t[o + 1] << 16 | (uint32_t)t[o + 2] << 8 | (uint32_t)t[o + 3];
    };
    if (u16(2) != 0x2A) return 1;
    const long long off = u32(4);
    if (off + 2 > n) throw JpegRefuse{SPG_JPEG_EXIF};
    const long long entries = u16(off);
    if (off + 2 + 12 * entries > n) throw JpegRefuse{SPG_JPEG_EXIF};
    for (long long e = 0; e < entries; e++) {
        const long long o = off + 2 + 12 * e;
        if (u16(o) == 0x0112) {
            const int v = u16(o + 8);
            return v >= 1 && v <= 8 ? v : 1;
        }
    }
    return 1;
}

// The parse; throws JpegRefuse.  oracle/jpeg_port.py's parse() is the same algorithm.
void jpeg_parse(const uint8_t *d, long long n, spg_jpeg_record *r) {
    auto u16 = [&](long long o) { return d[o] << 8 | d[o + 1]; };
    if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) throw JpegRefuse{SPG_JPEG_NOT_JPEG};
    long long p = 2;
    bool have_qt[4] = {false, false, false, false}, have_ht[2][4] = {{false}};
    uint16_t qt[4][64];
    uint8_t hbits[2][4][17], hsym[2][4][256];
    int hcount[2][4] = {{0}};
    int restart = 0, orientation = 0, nc = 0, fh = 0, fw = 0;
    bool frame = false, jfif = false, adobe = false;
    int adobe_transform = -1;
    int cid[3], ch[3], cv[3], ctq[3];
    const uint8_t *seg = nullptr;
    long long len = 0;
    for (;;) {
        if (p >= n) throw JpegRefuse{SPG_JPEG_TRUNCATED};
        if (d[p] != 0xFF) throw JpegRefuse{SPG_JPEG_MALFORMED};
        while (p < n && d[p] == 0xFF) p++;
        if (p >= n) throw JpegRefuse{SPG_JPEG_TRUNCATED};
        const int m = d[p++];
        if (m == 0xD8 || m == 0xD9 || m == 0x01 || (m >= 0xD0 && m <= 0xD7)) throw JpegRefuse{SPG_JPEG_MALFORMED};
        if (p + 2 > n) throw JpegRefuse{SPG_JPEG_TRUNCATED};
        const long long length = u16(p);
        if (length < 2) throw JpegRefuse{SPG_JPEG_MALFORMED};
        if (p + length > n) throw JpegRefuse{SPG_JPEG_TRUNCATED};
        seg = d + p + 2;
        len = length - 2;
        p += length;
        if (m == 0xC0 || m == 0xC1) {
            if (frame) throw JpegRefuse{SPG_JPEG_MALFORMED};
            if (len < 6) throw JpegRefuse{SPG_JPEG_MALFORMED};
            if (seg[0] != 8) throw JpegRefuse{SPG_JPEG_PRECISION};
            fh = seg[1] << 8 | seg[2];
            fw = seg[3] << 8 | seg[4];
            nc = seg[5];
            if (fh == 0 || fw == 0) throw JpegRefuse{SPG_JPEG_MALFORMED};
            if (nc != 1 && nc != 3) throw JpegRefuse{SPG_JPEG_COLOR};
            if (len != 6 + 3 * nc) throw JpegRefuse{SPG_JPEG_MALFORMED};
            for (int c = 0; c < nc; c++) {
                cid[c] = seg[6 + 3 * c];
                ch[c] = seg[7 + 3 * c] >> 4;
                cv[c] = seg[7 + 3 * c] & 15;
                ctq[c] = seg[8 + 3 * c];
                if (ch[c] < 1 || ch[c] > 4 || cv[c] < 1 || cv[c] > 4 || ctq[c] > 3) throw JpegRefuse{SPG_JPEG_MALFORMED};
                for (int e = 0; e < c; e++)
                    if (cid[e] == cid[c]) throw JpegRefuse{SPG_JPEG_MALFORMED};
            }
            frame = true;
        } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8) {
            throw JpegRefuse{SPG_JPEG_PROCESS};  // SOF2/3/5-7/9-11/13-15 and DAC
        } else if (m == 0xC4) {
            long long o = 0;
            while (o < len) {
                if (o + 17 > len) throw JpegRefuse{SPG_JPEG_MALFORMED};
                const int tc = seg[o] >> 4, th = seg[o] & 15;
                int count = 0;
                for (int l = 1; l <= 16; l++) count += seg[o + l];
                if (tc > 1 || th > 3 || count > 256) throw JpegRefuse{SPG_JPEG_TABLES};
                if (o + 17 + count > len) throw JpegRefuse{SPG_JPEG_MALFORMED};
                hbits[tc][th][0] = 0;
                memcpy(&hbits[tc][th][1], seg + o + 1, 16);
                memcpy(hsym[tc][th], seg + o + 17, (size_t)count);
                hcount[tc][th] = count;
                have_ht[tc][th] = true;
                o += 17 + count;
            }
        } else if (m == 0xDB) {
            long long o = 0;
            while (o < len) {
                const int pq = seg[o] >> 4, tq = seg[o] & 15;
                if (tq > 3 || pq > 1) throw JpegRefuse{SPG_JPEG_TABLES};
                const int size = pq ? 128 : 64;
                if (o + 1 + size > len) throw JpegRefuse{SPG_JPEG_MALFORMED};
                for (int k = 0; k < 64; k++)
                    qt[tq][kZigzag[k]] = (uint16_t)(pq ? seg[o + 1 + 2 * k] << 8 | seg[o + 2 + 2 * k] : seg[o + 1 + k]);
                have_qt[tq] = true;
                o += 1 + size;
            }
        } else if (m == 0xDD) {
            if (len != 2) throw JpegRefuse{SPG_JPEG_MALFORMED};
            restart = seg[0] << 8 | seg[1];
        } else if (m == 0xE0) {
            if (len >= 14 && !memcmp(seg, "JFIF\0", 5)) jfif = true;
        } else if (m == 0xE1) {
            if (!orientation) orientation = jpeg_exif_orientation(seg, len);
        } else if (m == 0xEE) {
            if (len >= 12 && !memcmp(seg, "Adobe", 5)) {
                adobe = true;
                adobe_transform = seg[11];
            }
        } else if (m == 0xDA) {
            break;
        } else if (!((m >= 0xE0 && m <= 0xEF) || m == 0xFE)) {
            throw JpegRefuse{SPG_JPEG_MALFORMED};
        }
    }
    // SOS
    if (!frame) throw JpegRefuse{SPG_JPEG_MALFORMED};
    const int ns = len ? seg[0] : 0;
    if (ns == 0 || len != 4 + 2 * ns) throw JpegRefuse{SPG_JPEG_MALFORMED};
    if (ns != nc) throw JpegRefuse{SPG_JPEG_SCAN};
    int td[3], ta[3];
    for (int c = 0; c < ns; c++) {
        if (seg[1 + 2 * c] != cid[c]) throw JpegRefuse{SPG_JPEG_SCAN};
        td[c] = seg[2 + 2 * c] >> 4;
        ta[c] = seg[2 + 2 * c] & 15;
    }
    if (seg[1 + 2 * ns] != 0 || seg[2 + 2 * ns] != 63 || seg[3 + 2 * ns] != 0) throw JpegRefuse{SPG_JPEG_SCAN};
    int hs = 1, vs = 1;
    if (nc == 3) {
        const bool rgb = jfif ? false : adobe ? adobe_transform == 0 : (cid[0] == 82 && cid[1] == 71 && cid[2] == 66);
        if (rgb || (adobe && !jfif && adobe_transform != 1)) throw JpegRefuse{SPG_JPEG_COLOR};
        hs = ch[0];
        vs = cv[0];
        if (hs > 2 || vs > 2 || ch[1] != 1 || cv[1] != 1 || ch[2] != 1 || cv[2] != 1) throw JpegRefuse{SPG_JPEG_SAMPLING};
    }
    for (int c = 0; c < nc; c++) {
        if (!have_qt[ctq[c]]) throw JpegRefuse{SPG_JPEG_TABLES};
        memcpy(r->quant[c], qt[ctq[c]], sizeof r->quant[c]);
        if (td[c] > 3 || ta[c] > 3 || !have_ht[0][td[c]] || !have_ht[1][ta[c]]) throw JpegRefuse{SPG_JPEG_TABLES};
        for (int i = 0; i < hcount[0][td[c]]; i++)
            if (hsym[0][td[c]][i] > 15) throw JpegRefuse{SPG_JPEG_TABLES};
        jpeg_build_huff(hbits[0][td[c]], hsym[0][td[c]], hcount[0][td[c]], &r->dc[c]);
        jpeg_build_huff(hbits[1][ta[c]], hsym[1][ta[c]], hcount[1][ta[c]], &r->ac[c]);
    }
    for (int c = nc; c < 3; c++) {
        memcpy(r->quant[c], r->quant[0], sizeof r->quant[c]);
        r->dc[c] = r->dc[0];
        r->ac[c] = r->ac[0];
    }
    const long long mcus_x = (fw + 8 * hs - 1) / (8 * hs), mcus_y = (fh + 8 * vs - 1) / (8 * vs);
    const long long n_intervals = restart ? (mcus_x * mcus_y + restart - 1) / restart : 1;
    // the entropy-coded data: up to EOI, with RST0..7 in order between the intervals and no other marker
    const long long start = p;
    long long q = start, end = -1, found = 0;
    int expect = 0;
    while (end < 0) {
        const uint8_t *f = static_cast<const uint8_t *>(q < n ? memchr(d + q, 0xFF, (size_t)(n - q)) : nullptr);
        if (!f) throw JpegRefuse{SPG_JPEG_TRUNCATED};
        q = f - d;
        long long t = q + 1;
        while (t < n && d[t] == 0xFF) t++;
        if (t >= n) throw JpegRefuse{SPG_JPEG_TRUNCATED};
        const int mk = d[t];
        if (mk == 0x00) {
            // fill bytes before a stuffed 0xFF: libjpeg-turbo ends the data at the first FF FF, the unstuffing would not
            if (t > q + 1) throw JpegRefuse{SPG_JPEG_MALFORMED};
            q = t + 1;
        } else if (mk >= 0xD0 && mk <= 0xD7) {
            if (!restart || mk != 0xD0 + expect || found + 1 >= n_intervals) throw JpegRefuse{SPG_JPEG_MALFORMED};
            expect = (expect + 1) & 7;
            found++;
            q = t + 1;
        } else if (mk == 0xD9) {
            end = q;
        } else {
            throw JpegRefuse{SPG_JPEG_SCAN};
        }
    }
    if (found != n_intervals - 1) throw JpegRefuse{SPG_JPEG_MALFORMED};
    r->orientation = orientation ? orientation : 1;
    r->frame_height = fh;
    r->frame_width = fw;
    r->height = r->orientation >= 5 ? fw : fh;
    r->width = r->orientation >= 5 ? fh : fw;
    r->n_components = nc;
    r->h_samp = hs;
    r->v_samp = vs;
    r->mcus_x = (int32_t)mcus_x;
    r->mcus_y = (int32_t)mcus_y;
    r->blocks_per_mcu = hs * vs + (nc == 3 ? 2 : 0);
    r->restart_interval = restart;
    r->n_intervals = (int32_t)n_intervals;
    r->scan_offset = start;
    r->scan_length = end - start;
}

// the largest entropy-coded segment a decode takes: bit positions are int
constexpr long long kJpegMaxSegment = (1ll << 28) - 1;

// A record's checks before any launch: the fields the kernels size their work by (`what` names it in the message).
int jpeg_check(spg_handle *h, const spg_jpeg_record &r, const char *what) {
    if (r.status != SPG_JPEG_OK) return fail(h, SPG_E_INVALID, "%s: status %d is not SPG_JPEG_OK", what, r.status);
    if (!r.data || !r.out || !r.decode_status) return fail(h, SPG_E_INVALID, "%s: data, out or decode_status is NULL", what);
    const bool grey = r.n_components == 1;
    if (!(grey || r.n_components == 3) || r.h_samp < 1 || r.h_samp > 2 || r.v_samp < 1 || r.v_samp > 2 ||
        (grey && (r.h_samp != 1 || r.v_samp != 1)) || r.blocks_per_mcu != r.h_samp * r.v_samp + (grey ? 0 : 2))
        return fail(h, SPG_E_INVALID, "%s: components or sampling", what);
    if (r.frame_height < 1 || r.frame_width < 1 || r.orientation < 1 || r.orientation > 8 ||
        r.mcus_x != (r.frame_width + 8 * r.h_samp - 1) / (8 * r.h_samp) ||
        r.mcus_y != (r.frame_height + 8 * r.v_samp - 1) / (8 * r.v_samp) ||
        r.height != (r.orientation >= 5 ? r.frame_width : r.frame_height) ||
        r.width != (r.orientation >= 5 ? r.frame_height : r.frame_width))
        return fail(h, SPG_E_INVALID, "%s: geometry", what);
    const long long mcus = (long long)r.mcus_x * r.mcus_y;
    if (r.restart_interval < 0 || r.n_intervals != (r.restart_interval ? (mcus + r.restart_interval - 1) / r.restart_interval : 1))
        return fail(h, SPG_E_INVALID, "%s: restart interval", what);
    if (r.scan_offset < 0 || r.scan_length < 0 || r.scan_length > kJpegMaxSegment)
        return fail(h, SPG_E_INVALID, "%s: scan length %lld outside [0, 2^28)", what, (long long)r.scan_length);
    if (mcus * r.blocks_per_mcu > 0x7fffffffLL) return fail(h, SPG_E_INVALID, "%s: more than 2^31 - 1 blocks", what);
    return SPG_OK;
}

// One image's member and its arrays in the decode's scratch, for `scan_bytes` of entropy-coded data: its chunk counts,
// interval starts, subsequence states, unstuffed stream and component planes (rec and coef are the caller's).
JpegMember jpeg_member(Carver &c, const spg_jpeg_record &r, long long scan_bytes) {
    JpegMember m{};
    m.seg = r.data + r.scan_offset;
    m.seg_len = (int)scan_bytes;
    m.n_chunks = (int)std::max<long long>(1, (scan_bytes + kJpegChunk - 1) / kJpegChunk);
    m.chunk_counts = c.take<int>(2 * (size_t)m.n_chunks);
    m.starts = c.take<int>((size_t)r.n_intervals + 1);
    m.n_subs = r.restart_interval ? 0 : (int)std::max<long long>(1, (8 * scan_bytes + kJpegSubBits - 1) / kJpegSubBits);
    m.subs = c.take<JpegSub>((size_t)m.n_subs);
    m.packed = c.take<unsigned char>((size_t)scan_bytes);
    m.frame_h = r.frame_height;
    m.frame_w = r.frame_width;
    m.out_h = r.height;
    m.out_w = r.width;
    m.orientation = r.orientation;
    m.n_comp = r.n_components;
    m.hs = r.h_samp;
    m.vs = r.v_samp;
    m.mcus_x = r.mcus_x;
    m.mcus_y = r.mcus_y;
    m.bpm = r.blocks_per_mcu;
    m.restart = r.restart_interval;
    m.n_intervals = r.n_intervals;
    m.total_blocks = r.mcus_x * r.mcus_y * r.blocks_per_mcu;
    m.out = r.out;
    m.status = r.decode_status;
    for (int k = 0; k < r.n_components; k++) {
        const int hk = k == 0 ? r.h_samp : 1, vk = k == 0 ? r.v_samp : 1;
        m.plane_w[k] = r.mcus_x * hk * 8;
        m.plane[k] = c.take<unsigned char>((size_t)m.plane_w[k] * r.mcus_y * vk * 8);
    }
    return m;
}

// spg_jpeg_reserve_frames / spg_jpeg_decode_frames' arguments
int jpeg_check_frames(spg_handle *h, const spg_jpeg_record *formats, const int64_t *capacities, int32_t n) {
    if (n < 1 || !formats || !capacities) return fail(h, SPG_E_INVALID, "formats or capacities is NULL or n %d below 1", n);
    for (int i = 0; i < n; i++) {
        char what[32];
        snprintf(what, sizeof what, "format %d", i);
        if (capacities[i] < 1 || capacities[i] > kJpegMaxSegment)
            return fail(h, SPG_E_INVALID, "%s: capacity %lld outside [1, 2^28)", what, (long long)capacities[i]);
        int rc;
        if ((rc = jpeg_check(h, formats[i], what))) return rc;
    }
    return SPG_OK;
}

// the frame form's scratch: each member for its capacity, then every member's coefficients back to back (one memset);
// *coef_count is their total
void jpeg_frames_layout(Carver &c, const spg_jpeg_record *formats, const int64_t *capacities, int n, JpegMember *ms,
                        size_t *coef_count) {
    *coef_count = 0;
    for (int i = 0; i < n; i++) {
        ms[i] = jpeg_member(c, formats[i], capacities[i]);
        *coef_count += (size_t)ms[i].total_blocks * 64;
    }
    short *coef = c.take<short>(*coef_count);
    for (int i = 0; i < n; i++) {
        ms[i].coef = coef;
        if (coef) coef += (size_t)ms[i].total_blocks * 64;
    }
}

// One ragged launch of JPEG kernel k over the members `sel` selects, each taking ctas_of(m) CTAs.
template <class Ctas, class Sel>
int jpeg_run(spg_handle *h, JpegKernel k, const std::vector<JpegMember> &ms, Ctas &&ctas_of, Sel &&sel, cudaStream_t st) {
    std::vector<JpegMember> sub;
    std::vector<long long> ctas;
    for (const JpegMember &m : ms)
        if (sel(m)) {
            sub.push_back(m);
            ctas.push_back(ctas_of(m));
        }
    if (sub.empty()) return SPG_OK;
    void (*const kern)(JpegRagged) = k < kJpegCountFrame ? kJpegRaggedKernels[k] : kJpegFrameKernels[k - kJpegCountFrame];
    std::vector<RaggedRange> ranges;
    std::vector<int> first;
    int rc;
    if ((rc = deal_ragged(h, ctas, kJpegTableMax, "image", nullptr, ranges, first))) return rc;
    JpegRagged table{};
    for (const RaggedRange &g : ranges) {
        fill_table(table, sub, first, g);
        if ((rc = launch(h, kStageJpeg, kJpegKernelName[k], kern, dim3(g.ctas), kJpegBlock[k], 0, st, table))) return rc;
    }
    return SPG_OK;
}

// Every launch of a decode, in order: the count to write kernels of the ragged form, or of the frame form (`frame`), then
// the DC, IDCT and colour kernels.  Interval members and subsequence members go in one call.
int jpeg_decode_launches(spg_handle *h, const std::vector<JpegMember> &ms, bool frame, cudaStream_t st) {
    const int f = frame ? kJpegCountFrame - kJpegCount : 0;
    auto run = [&](int k, auto &&ctas_of, auto &&sel) { return jpeg_run(h, (JpegKernel)k, ms, ctas_of, sel, st); };
    auto all = [](const JpegMember &) { return true; };
    auto with_rst = [](const JpegMember &m) { return m.restart > 0; };
    auto without_rst = [](const JpegMember &m) { return m.restart == 0; };
    auto chunks = [](const JpegMember &m) { return (long long)m.n_chunks; };
    auto subs = [](const JpegMember &m) { return (long long)(m.n_subs + kJpegSubThreads - 1) / kJpegSubThreads; };
    auto one = [](const JpegMember &) { return 1ll; };
    int rc;
    if ((rc = run(kJpegCount + f, chunks, all)) || (rc = run(kJpegPrefix + f, one, all)) || (rc = run(kJpegPack + f, chunks, all)) ||
        (rc = run(kJpegInterval + f, [](const JpegMember &m) { return (long long)(m.n_intervals + kJpegThreads - 1) / kJpegThreads; },
                  with_rst)) ||
        (rc = run(kJpegSync + f, subs, without_rst)) || (rc = run(kJpegFixup + f, one, without_rst)) ||
        (rc = run(kJpegWrite + f, subs, without_rst)) ||
        (rc = run(kJpegDc, [](const JpegMember &m) { return (long long)m.n_comp; }, all)) ||
        (rc = run(kJpegIdct, [](const JpegMember &m) { return ((long long)m.total_blocks + kJpegThreads - 1) / kJpegThreads; }, all)) ||
        (rc = run(kJpegColor, [](const JpegMember &m) { return ((long long)m.out_h * m.out_w + kJpegThreads - 1) / kJpegThreads; }, all)))
        return rc;
    return SPG_OK;
}

}  // namespace

extern "C" {

int spg_jpeg_parse(const uint8_t *data, int64_t size, spg_jpeg_record *record) {
    if (!record || size < 0 || (size > 0 && !data)) return SPG_E_INVALID;
    memset(record, 0, sizeof *record);
    try {
        jpeg_parse(data, size, record);
        record->status = SPG_JPEG_OK;
    } catch (const JpegRefuse &e) {
        memset(record, 0, sizeof *record);
        record->status = e.status;
    }
    return SPG_OK;
}

int spg_jpeg_decode_ragged(spg_handle *h, const spg_jpeg_record *records, int32_t n, void *stream) {
    if (!h) return SPG_E_INVALID;
    if (n < 0 || (n > 0 && !records)) return fail(h, SPG_E_INVALID, "records is NULL or n negative");
    if (n == 0) return SPG_OK;
    // every record validated before the first launch: the fields the kernels size their work by
    for (int i = 0; i < n; i++) {
        char what[32];
        snprintf(what, sizeof what, "record %d", i);
        int rc;
        if ((rc = jpeg_check(h, records[i], what))) return rc;
    }
    DeviceGuard guard(h->device);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    // one scratch: records, then per image its counts, interval starts, subsequence states, stream, coefficients, planes
    std::vector<JpegMember> ms((size_t)n);
    spg_jpeg_record *recs = nullptr;
    short *coef_base = nullptr;
    size_t coef_count = 0;
    int rc = carve(h, h->jpeg, [&](Carver &c) {
        recs = c.take<spg_jpeg_record>((size_t)n);
        coef_count = 0;
        for (int i = 0; i < n; i++) {
            ms[i] = jpeg_member(c, records[i], records[i].scan_length);
            ms[i].rec = recs + i;
            coef_count += (size_t)ms[i].total_blocks * 64;
        }
        coef_base = c.take<short>(coef_count);
        size_t o = 0;
        for (JpegMember &m : ms) {
            m.coef = coef_base ? coef_base + o : nullptr;
            o += (size_t)m.total_blocks * 64;
        }
    });
    if (rc) return rc;
    SPG_CUDA(h, cudaMemcpyAsync(recs, records, sizeof(spg_jpeg_record) * n, cudaMemcpyHostToDevice, st));
    SPG_CUDA(h, cudaMemsetAsync(coef_base, 0, coef_count * sizeof(short), st));
    return jpeg_decode_launches(h, ms, false, st);
}

int spg_jpeg_reserve_frames(spg_handle *h, const spg_jpeg_record *formats, const int64_t *capacities, int32_t n,
                            int32_t *moved) {
    if (!h) return SPG_E_INVALID;
    if (moved) *moved = 0;
    int rc;
    if ((rc = jpeg_check_frames(h, formats, capacities, n))) return rc;
    Carver c;
    std::vector<JpegMember> ms((size_t)n);
    size_t coef_count;
    jpeg_frames_layout(c, formats, capacities, n, ms.data(), &coef_count);
    if (moved) *moved = c.bytes > h->jpeg.bytes;  // set before a failed growth too
    DeviceGuard guard(h->device);
    return grow(h, h->jpeg, c.bytes);
}

int spg_jpeg_reserve_frame(spg_handle *h, const spg_jpeg_record *format, int64_t max_scan_bytes, int32_t *moved) {
    return spg_jpeg_reserve_frames(h, format, &max_scan_bytes, 1, moved);
}

int spg_jpeg_decode_frames(spg_handle *h, const spg_jpeg_record *device_records, const spg_jpeg_record *formats,
                           const int64_t *capacities, int32_t n, void *stream) {
    if (!h) return SPG_E_INVALID;
    int rc;
    if ((rc = jpeg_check_frames(h, formats, capacities, n))) return rc;
    if (!device_records) return fail(h, SPG_E_INVALID, "device_records is NULL");
    DeviceGuard guard(h->device);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::vector<JpegMember> ms((size_t)n);
    size_t coef_count = 0;
    if ((rc = carve(h, h->jpeg, [&](Carver &c) { jpeg_frames_layout(c, formats, capacities, n, ms.data(), &coef_count); }, st,
                    "the JPEG frame decode's unstuffed streams, coefficients and planes")))
        return rc;
    for (int i = 0; i < n; i++) ms[i].rec = device_records + i;
    SPG_CUDA(h, cudaMemsetAsync(ms[0].coef, 0, coef_count * sizeof(short), st));
    // the grids cover each member's capacity (its seg_len, n_chunks and n_subs); the kernels read the frame's own length,
    // and a member's CTAs past it return at once
    return jpeg_decode_launches(h, ms, true, st);
}

int spg_jpeg_decode_frame(spg_handle *h, const spg_jpeg_record *device_record, const spg_jpeg_record *format,
                          int64_t max_scan_bytes, void *stream) {
    return spg_jpeg_decode_frames(h, device_record, format, &max_scan_bytes, 1, stream);
}

}  // extern "C"
