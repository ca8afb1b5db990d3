/*
 * spg_oracle.c -- CPU restatement of SimplePose's keypoint-grouping hot path.
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load this library; the
 * product path (improved_body_parts_b200/) never does and fails loudly without
 * its CUDA library.
 *
 * It restates, in plain C and in the reference's arithmetic (same precision,
 * same operation order, no FMA contraction -- build with -ffp-contract=off):
 *
 *   spgo_find_peaks        evaluate.py:169-203  + utils/util.py:177-183 (3x3 NMS)
 *                                               + utils/util.py:186-211 (centroid refine)
 *   spgo_find_connections  evaluate.py:206-276
 *   spgo_find_people       evaluate.py:279-498
 *   spgo_to_coco           evaluate.py:523-543  (person -> 17 COCO joints + score)
 *
 * (paths relative to /root/reference).  Parity is PINNED: the reference ships
 * no tests or golden vectors, so tests/golden/ holds fixtures produced by
 * executing the reference's own functions unmodified in the build container
 * (tests/golden/make_golden.py); tests/test_oracle.py checks this restatement
 * against them bit-for-bit, floats included.
 *
 * Arithmetic facts this file relies on (all probed against numpy 2.3.5 /
 * torch 2.11 in the build container, see DESIGN.md "numerics"):
 *   - util.keypoint_heatmap_nms: reflect-pad-1 + 3x3 max == window clipped to
 *     the image; `heat >= thre` is an f32 compare against (float)thre.
 *   - refine_centroid: both the f32 `score_box.sum()` of the strided 5x5 view
 *     and the f64 `(score_box * grid).sum()` reduce a 25-element buffer with
 *     numpy's 8-accumulator pairwise order; mean = f32 sum / f32(25).
 *   - find_connections with an f32 plane: sequential f32 sum (Python sum()),
 *     f32 divide, `+ min(0.5*h/norm - 1, 0)` rounds the f64 term to f32 first
 *     (NEP 50 weak scalars), `> thre2` is an f32 compare against (float)thre2.
 *     With an f64 plane everything is f64.
 *   - np.linspace: y_t = fl(fl(t*step) + start), step = fl(delta/div), last
 *     sample forced to `stop`; n == 1 -> [start].  round() is half-to-even.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#if defined(_OPENMP)
#include <omp.h>
#endif

#define SPGO_ERR_CAPACITY (-1)   /* an output capacity was exceeded                      */
#define SPGO_ERR_INDEX    (-2)   /* the reference would raise IndexError (sample index)  */
#define SPGO_ERR_ASSERT   (-3)   /* the reference would raise in find_people :437-439    */
#define SPGO_ERR_NONFINITE (-4)  /* a pair's length is not finite: round() raises at :226  */
#define SPGO_ERR_NAN_PRIORITY (-5) /* a NaN priority among >= 2 candidates: the order sorted() gives at :259 is not reproduced */

typedef struct spgo_params {
    double thre1, thre2, connect_ration, len_rate, connection_tole, min_mean_score;
    int32_t mid_num, offset_radius, remove_recon, min_parts;
    int32_t crit1_strict, refresh_len_check; /* demo_image.py:288 (`>`), :414-415 (length check in the same-B refresh); 0 = evaluate.py */
} spgo_params;

/* Branch counters (tests only): which rarely-taken reference branches an input set reached. */
enum { COV_NORM0, COV_SPECIAL, COV_MIDNUM1, COV_CAND, COV_ACCEPT, COV_ASSIGN, COV_REPLACE, COV_REPLACE_LEN_REJECT,
       COV_KEEP_OLD, COV_REFRESH, COV_ASSIGN_LEN_REJECT, COV_MERGE, COV_MERGE_REJECT, COV_OVERLAP, COV_RECON_REMOVE,
       COV_NEW_PERSON, COV_PRUNED, COV_THIRD_MATCH, COV_BORDER_PEAK, COV_NEG_WRAP, COV_N };
static int64_t g_cov[COV_N];
static inline void cov(int w) {
#if defined(_OPENMP)
#pragma omp atomic
#endif
    g_cov[w]++;
}
void spgo_cov_reset(void) { memset(g_cov, 0, sizeof g_cov); }
int spgo_cov_read(int64_t *out, int n) { for (int i = 0; i < n && i < COV_N; i++) out[i] = g_cov[i]; return COV_N; }

/* ---- numpy's pairwise summation (umath loops_utils: *_pairwise_sum), n <= 128 blocks ---- */
#define PW_DEF(NAME, T)                                                              \
    static T NAME(const T *a, int n) {                                               \
        if (n < 8) {                                                                 \
            T res = (T)0;                                                            \
            for (int i = 0; i < n; i++) res += a[i];                                 \
            return res;                                                              \
        } else if (n <= 128) {                                                       \
            T r[8];                                                                  \
            int i;                                                                   \
            for (int k = 0; k < 8; k++) r[k] = a[k];                                 \
            for (i = 8; i < n - (n % 8); i += 8)                                     \
                for (int k = 0; k < 8; k++) r[k] += a[i + k];                        \
            T res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7])); \
            for (; i < n; i++) res += a[i];                                          \
            return res;                                                              \
        } else {                                                                     \
            int n2 = n / 2;                                                          \
            n2 -= n2 % 8;                                                            \
            return NAME(a, n2) + NAME(a + n2, n - n2);                               \
        }                                                                            \
    }
PW_DEF(pw_sum_f32, float)
PW_DEF(pw_sum_f64, double)

/* ------------------------------------------------------------------------------------------
 * find_peaks (evaluate.py:169-203).  heat is channel-first: heat[c*cs + y*rs + x].
 * Peaks come out part-major, raster order inside a part (np.nonzero, :193); the global id of a
 * peak is its position in that order (:197-201).  Returns the total number of peaks (> cap means
 * the tail was not stored -> caller treats as SPGO_ERR_CAPACITY).
 * ------------------------------------------------------------------------------------------ */
int spgo_find_peaks(const float *heat, int K, int H, int W, int64_t cs, int64_t rs, const spgo_params *p,
                    int cap, double *px, double *py, float *pscore, int32_t *pxi, int32_t *pyi,
                    uint8_t *pint, int32_t *part_count) {
    const float thr = (float)p->thre1;
    const int R = p->offset_radius, D = 2 * R + 1;
    float *box = (float *)malloc(sizeof(float) * (size_t)D * D);
    double *wr = (double *)malloc(sizeof(double) * (size_t)D * D);
    double *wc = (double *)malloc(sizeof(double) * (size_t)D * D);
    int total = 0;
    for (int c = 0; c < K; c++) {
        const float *m = heat + (int64_t)c * cs;
        int n_c = 0;
        for (int y = 0; y < H; y++) {
            for (int x = 0; x < W; x++) {
                const float v = m[(int64_t)y * rs + x];
                /* util.py:182: keep = (hmax == heat) * (heat >= thre); np.nonzero(heat*keep) at :193.  A non-finite
                 * pixel is always a peak (NaN*0, inf*0, -inf*0 are NaN); a finite one needs keep = 1 and v != 0, and
                 * keep = 1 needs v >= thre and no neighbour greater or NaN (torch's max-pool propagates NaN). */
                int is_max = 1;
                if (isfinite(v) && (!(v >= thr) || v == 0.0f)) continue;
                for (int dy = -1; dy <= 1 && is_max && isfinite(v); dy++) {
                    const int yy = y + dy;
                    if (yy < 0 || yy >= H) continue;
                    for (int dx = -1; dx <= 1; dx++) {
                        const int xx = x + dx;
                        if (xx < 0 || xx >= W) continue;
                        if (!(m[(int64_t)yy * rs + xx] <= v)) { is_max = 0; break; }
                    }
                }
                if (!is_max) continue;
                if (total < cap) {
                    pxi[total] = x;
                    pyi[total] = y;
                    /* util.py:201-202: box leaves the image -> integer anchor + raw value */
                    if (y + R + 1 > H || y - R < 0 || x + R + 1 > W || x - R < 0) {
                        px[total] = (double)x;
                        py[total] = (double)y;
                        pscore[total] = v;
                        pint[total] = 1;
                        cov(COV_BORDER_PEAK);
                    } else {
                        /* util.py:204-211.  np.mgrid[-R:R+1,-R:R+1]: first grid varies along ROWS, and it is
                         * the one added to x (axes swapped relative to intent; kept). */
                        int n = 0;
                        for (int r = -R; r <= R; r++)
                            for (int q = -R; q <= R; q++) {
                                const float b = m[(int64_t)(y + r) * rs + (x + q)];
                                box[n] = b;
                                wr[n] = (double)b * (double)r;
                                wc[n] = (double)b * (double)q;
                                n++;
                            }
                        const float s32 = pw_sum_f32(box, n);
                        const double off_x = pw_sum_f64(wr, n) / (double)s32;
                        const double off_y = pw_sum_f64(wc, n) / (double)s32;
                        px[total] = (double)x + off_x;
                        py[total] = (double)y + off_y;
                        pscore[total] = s32 / (float)n; /* score_box.mean() in f32 */
                        pint[total] = 0;
                    }
                }
                total++;
                n_c++;
            }
        }
        part_count[c] = n_c;
    }
    free(box);
    free(wr);
    free(wc);
    return total;
}

/* ---- candidates of one limb ---- */
typedef struct cand {
    int32_t i, j;
    double score; /* f32 value widened exactly when the plane is f32 */
    double norm;
    double prio;  /* idem */
} cand;

/* stable merge sort, descending priority: Python sorted(key=prio, reverse=True) keeps equal keys in
 * generation order (evaluate.py:259) */
static void sort_cands(cand *a, cand *tmp, int n) {
    for (int w = 1; w < n; w *= 2) {
        for (int lo = 0; lo < n; lo += 2 * w) {
            int mid = lo + w < n ? lo + w : n, hi = lo + 2 * w < n ? lo + 2 * w : n;
            int l = lo, r = mid, o = lo;
            while (l < mid && r < hi) tmp[o++] = (a[r].prio > a[l].prio) ? a[r++] : a[l++];
            while (l < mid) tmp[o++] = a[l++];
            while (r < hi) tmp[o++] = a[r++];
        }
        memcpy(a, tmp, sizeof(cand) * (size_t)n);
    }
}

/* Python-style index: negatives wrap once, anything else out of range is an IndexError */
static inline int py_index(long v, int n, int *err) {
    if (v < 0) { v += n; cov(COV_NEG_WRAP); }
    if (v < 0 || v >= n) { *err = 1; return 0; }
    return (int)v;
}

/* ------------------------------------------------------------------------------------------
 * find_connections (evaluate.py:206-276).  paf[k*cs + y*rs + x], f32 or f64 plane.
 * peaks are the flat part-major arrays of spgo_find_peaks; part_count[K].
 * Output per limb k: conn_count[k] = -1 for special_k (:272-274), else the number of accepted rows;
 * row r: conn_ij[(k*cap+r)*2 + {0,1}] = (i, j) indices inside candA / candB, conn_score, conn_norm.
 * cand_count[k] (optional) = number of candidates that passed both criteria (:252).
 * ------------------------------------------------------------------------------------------ */
int spgo_find_connections(const double *px, const double *py, const float *pscore, const int32_t *part_count,
                          int K, const void *paf, int paf_is_f64, int L, const int32_t *limbs, int H, int W,
                          int64_t cs, int64_t rs, double image_extent, const spgo_params *p, int cap,
                          int32_t *conn_ij, double *conn_score, double *conn_norm, int32_t *conn_count,
                          int32_t *cand_count) {
    int *off = (int *)malloc(sizeof(int) * (size_t)(K + 1));
    off[0] = 0;
    for (int c = 0; c < K; c++) off[c + 1] = off[c] + part_count[c];
    int max_n = 0;
    for (int c = 0; c < K; c++) if (part_count[c] > max_n) max_n = part_count[c];
    cand *cands = (cand *)malloc(sizeof(cand) * ((size_t)max_n * max_n + 1));
    cand *tmp = (cand *)malloc(sizeof(cand) * ((size_t)max_n * max_n + 1));
    uint8_t *usedA = (uint8_t *)malloc((size_t)max_n + 1), *usedB = (uint8_t *)malloc((size_t)max_n + 1);
    const float thre2_f = (float)p->thre2;
    int rc = 0;

    for (int k = 0; k < L && rc == 0; k++) {
        const int a = limbs[2 * k], b = limbs[2 * k + 1];
        const int nA = part_count[a], nB = part_count[b];
        if (cand_count) cand_count[k] = 0;
        if (nA == 0 || nB == 0) { conn_count[k] = -1; cov(COV_SPECIAL); continue; }
        const float *plane32 = paf_is_f64 ? NULL : (const float *)paf + (int64_t)k * cs;
        const double *plane64 = paf_is_f64 ? (const double *)paf + (int64_t)k * cs : NULL;
        int nc = 0;
        for (int i = 0; i < nA; i++) {
            const double ax = px[off[a] + i], ay = py[off[a] + i];
            for (int j = 0; j < nB; j++) {
                const double bx = px[off[b] + j], by = py[off[b] + j];
                const double vx = bx - ax, vy = by - ay;           /* :224 */
                const double norm = sqrt(vx * vx + vy * vy);       /* :225 */
                if (!isfinite(norm)) { rc = SPGO_ERR_NONFINITE; break; } /* int(round(norm + 1)) raises at :226 */
                if (norm == 0.0) { cov(COV_NORM0); continue; }      /* :228-230 */
                long mn = (long)rint(norm + 1.0);                   /* :226 round() half-even */
                if (mn > p->mid_num) mn = p->mid_num;
                const int n = (int)mn;
                if (n == 1) cov(COV_MIDNUM1);
                /* np.linspace(A, B, n) (:232-233) */
                const double stepx = n > 1 ? vx / (double)(n - 1) : 0.0;
                const double stepy = n > 1 ? vy / (double)(n - 1) : 0.0;
                float sum32 = 0.0f;
                double sum64 = 0.0;
                int above = 0, err = 0;
                for (int t = 0; t < n; t++) {
                    double sx, sy;
                    if (t == n - 1 && n > 1) { sx = bx; sy = by; }
                    else { sx = (double)t * stepx + ax; sy = (double)t * stepy + ay; }
                    const int yi = py_index((long)rint(sy), H, &err);
                    const int xi = py_index((long)rint(sx), W, &err);  /* :235 nearest neighbour */
                    if (err) break;
                    if (paf_is_f64) {
                        const double v = plane64[(int64_t)yi * rs + xi];
                        sum64 += v;
                        above += v > p->thre2;
                    } else {
                        const float v = plane32[(int64_t)yi * rs + xi];
                        sum32 += v;                                 /* Python sum() over np.float32 */
                        above += v > thre2_f;
                    }
                }
                if (err) { rc = SPGO_ERR_INDEX; break; }
                /* :241 -- `image_width` is the image HEIGHT at the call site (:510) */
                double prior = 0.5 * image_extent / norm - 1.0;
                const int prior_neg = prior < 0.0;
                double score, prio;
                if (paf_is_f64) {
                    score = sum64 / (double)n + (prior_neg ? prior : 0.0);
                    prio = (0.5 * score + (double)(0.25f * pscore[off[a] + i])) + (double)(0.25f * pscore[off[b] + j]);
                } else {
                    float s = sum32 / (float)n;
                    s = s + (prior_neg ? (float)prior : 0.0f);
                    score = (double)s;
                    const float pr = (0.5f * s + 0.25f * pscore[off[a] + i]) + 0.25f * pscore[off[b] + j];
                    prio = (double)pr;
                }
                const int crit1 = p->crit1_strict ? (double)above > p->connect_ration * (double)n   /* demo_image.py:288 */
                                                  : (double)above >= p->connect_ration * (double)n; /* :246 */
                const int crit2 = score > 0.0;                                      /* :251 */
                if (crit1 && crit2) {
                    cands[nc].i = i; cands[nc].j = j; cands[nc].score = score; cands[nc].norm = norm;
                    cands[nc].prio = prio;
                    nc++;
                    cov(COV_CAND);
                }
            }
            if (rc) break;
        }
        if (rc) break;
        if (cand_count) cand_count[k] = nc;
        for (int c = 0; c < nc && nc > 1; c++)
            if (isnan(cands[c].prio)) rc = SPGO_ERR_NAN_PRIORITY;
        if (rc) break;
        sort_cands(cands, tmp, nc);
        memset(usedA, 0, (size_t)nA);
        memset(usedB, 0, (size_t)nB);
        const int lim = nA < nB ? nA : nB;
        int m = 0;
        for (int c = 0; c < nc; c++) {                              /* :263-270 */
            if (usedA[cands[c].i] || usedB[cands[c].j]) continue;
            if (m >= cap) { rc = SPGO_ERR_CAPACITY; break; }
            usedA[cands[c].i] = 1; usedB[cands[c].j] = 1;
            conn_ij[((int64_t)k * cap + m) * 2 + 0] = cands[c].i;
            conn_ij[((int64_t)k * cap + m) * 2 + 1] = cands[c].j;
            conn_score[(int64_t)k * cap + m] = cands[c].score;
            conn_norm[(int64_t)k * cap + m] = cands[c].norm;
            m++;
            cov(COV_ACCEPT);
            if (m >= lim) break;
        }
        conn_count[k] = m;
    }
    free(off); free(cands); free(tmp); free(usedA); free(usedB);
    return rc;
}

/* ------------------------------------------------------------------------------------------
 * find_people (evaluate.py:279-498).
 * subset rows are [K+2][2] doubles: slot c = (peak id | -1, connection score | -1),
 * row K = (total score, -1), row K+1 = (part count, longest limb).
 * Returns the number of persons left after the prune (:491-496), or a negative error.
 * ------------------------------------------------------------------------------------------ */
#define SUB(j, c, f) subset[((int64_t)(j) * RS + (c)) * 2 + (f)]
int spgo_find_people(const float *pscore, const int32_t *part_count, int K, int L, const int32_t *limbs,
                     int cap, const int32_t *conn_ij, const double *conn_score, const double *conn_norm,
                     const int32_t *conn_count, const spgo_params *p, int cap_rows, double *subset) {
    const int RS = K + 2;
    int *off = (int *)malloc(sizeof(int) * (size_t)(K + 1));
    off[0] = 0;
    for (int c = 0; c < K; c++) off[c + 1] = off[c] + part_count[c];
    int n = 0, rc = 0;
    for (int k = 0; k < L && rc == 0; k++) {
        if (conn_count[k] < 0) continue;                                 /* :290 special_k */
        const int A = limbs[2 * k], B = limbs[2 * k + 1];
        for (int r = 0; r < conn_count[k]; r++) {
            const int idA = off[A] + conn_ij[((int64_t)k * cap + r) * 2 + 0];
            const int idB = off[B] + conn_ij[((int64_t)k * cap + r) * 2 + 1];
            const double s = conn_score[(int64_t)k * cap + r];
            const double len = conn_norm[(int64_t)k * cap + r];
            int found = 0, idx[2] = {-1, -1};
            for (int j = 0; j < n; j++)                                  /* :304-318 */
                if ((int)SUB(j, A, 0) == idA || (int)SUB(j, B, 0) == idB) {
                    if (found >= 2) { cov(COV_THIRD_MATCH); continue; }  /* :314-316 */
                    idx[found++] = j;
                }
            if (found == 1) {                                            /* :320-383, always slot B */
                const int j = idx[0];
                if ((int)SUB(j, B, 0) == -1 && p->len_rate * SUB(j, K + 1, 1) > len) {
                    cov(COV_ASSIGN);
                    SUB(j, B, 0) = (double)idB;
                    SUB(j, B, 1) = s;
                    SUB(j, K + 1, 0) += 1.0;
                    SUB(j, K, 0) += (double)pscore[idB] + s;
                    SUB(j, K + 1, 1) = len > SUB(j, K + 1, 1) ? len : SUB(j, K + 1, 1);
                } else if ((int)SUB(j, B, 0) != idB) {
                    if (SUB(j, B, 1) >= s) {
                        /* existing connection is at least as confident: keep it */
                        if ((int)SUB(j, B, 0) == -1) cov(COV_ASSIGN_LEN_REJECT); else cov(COV_KEEP_OLD);
                    } else {
                        if (p->len_rate * SUB(j, K + 1, 1) <= len) {
                            cov((int)SUB(j, B, 0) == -1 ? COV_ASSIGN_LEN_REJECT : COV_REPLACE_LEN_REJECT);
                            continue;
                        }
                        cov(COV_REPLACE);
                        int old = (int)SUB(j, B, 0);
                        if (old < 0) old += off[K];                       /* candidate[-1] wraps in numpy */
                        SUB(j, K, 0) -= (double)pscore[old] + SUB(j, B, 1);
                        SUB(j, B, 0) = (double)idB;
                        SUB(j, B, 1) = s;
                        SUB(j, K, 0) += (double)pscore[idB] + s;
                        SUB(j, K + 1, 1) = len > SUB(j, K + 1, 1) ? len : SUB(j, K + 1, 1);
                    }
                } else if (SUB(j, B, 1) <= s) {                          /* same B, refresh (:368-380) */
                    if (p->refresh_len_check && p->len_rate * SUB(j, K + 1, 1) <= len) continue; /* demo_image.py:414-415 */
                    cov(COV_REFRESH);
                    SUB(j, K, 0) -= (double)pscore[idB] + SUB(j, B, 1);
                    SUB(j, B, 0) = (double)idB;
                    SUB(j, B, 1) = s;
                    SUB(j, K, 0) += (double)pscore[idB] + s;
                    SUB(j, K + 1, 1) = len > SUB(j, K + 1, 1) ? len : SUB(j, K + 1, 1);
                }
            } else if (found == 2) {                                     /* :385-460 */
                const int j1 = idx[0], j2 = idx[1];
                int overlap = 0;
                for (int c = 0; c < K; c++) overlap += (SUB(j1, c, 0) >= 0) && (SUB(j2, c, 0) >= 0);
                if (!overlap) {
                    double m1 = INFINITY, m2 = INFINITY;
                    for (int c = 0; c < K; c++) {
                        if (SUB(j1, c, 0) >= 0 && SUB(j1, c, 1) < m1) m1 = SUB(j1, c, 1);
                        if (SUB(j2, c, 0) >= 0 && SUB(j2, c, 1) < m2) m2 = SUB(j2, c, 1);
                    }
                    const double tol = m1 < m2 ? m1 : m2;
                    if (s < p->connection_tole * tol || p->len_rate * SUB(j1, K + 1, 1) <= len) {
                        cov(COV_MERGE_REJECT);
                        continue;
                    }
                    cov(COV_MERGE);
                    for (int c = 0; c < K; c++) {                        /* :415 the "+1" merge */
                        SUB(j1, c, 0) += SUB(j2, c, 0) + 1.0;
                        SUB(j1, c, 1) += SUB(j2, c, 1) + 1.0;
                    }
                    SUB(j1, K, 0) += SUB(j2, K, 0);                      /* :419 */
                    SUB(j1, K + 1, 0) += SUB(j2, K + 1, 0);
                    SUB(j1, K, 0) += s;                                  /* :421 */
                    SUB(j1, K + 1, 1) = len > SUB(j1, K + 1, 1) ? len : SUB(j1, K + 1, 1);
                    memmove(&SUB(j2, 0, 0), &SUB(j2 + 1, 0, 0), sizeof(double) * 2 * RS * (size_t)(n - j2 - 1));
                    n--;                                                 /* :424 np.delete */
                } else {
                    /* :429-460; only remove_recon > 0 has side effects */
                    cov(COV_OVERLAP);
                    int in_j1 = 0, c1 = -1, c2 = -1, n1 = 0, n2 = 0;
                    for (int c = 0; c < K; c++) in_j1 |= (SUB(j1, c, 0) == (double)idA);
                    const double k1 = in_j1 ? (double)idA : (double)idB, k2 = in_j1 ? (double)idB : (double)idA;
                    for (int c = 0; c < K; c++) {
                        if (SUB(j1, c, 0) == k1) { c1 = c; n1++; }
                        if (SUB(j2, c, 0) == k2) { c2 = c; n2++; }
                    }
                    if (n1 != 1 || n2 != 1 || c1 == c2) { rc = SPGO_ERR_ASSERT; break; }
                    if (s < SUB(j1, c1, 1) && s < SUB(j2, c2, 1)) continue;
                    int small_j = j1, remove_c = c1;
                    if (SUB(j1, c1, 1) > SUB(j2, c2, 1)) { small_j = j2; remove_c = c2; }
                    if (p->remove_recon > 0) {
                        cov(COV_RECON_REMOVE);
                        SUB(small_j, K, 0) -= (double)pscore[(int)SUB(small_j, remove_c, 0)] + SUB(small_j, remove_c, 1);
                        SUB(small_j, remove_c, 0) = -1.0;
                        SUB(small_j, remove_c, 1) = -1.0;
                        SUB(small_j, K + 1, 0) -= 1.0;
                    }
                }
            } else {                                                     /* :473-488 new person */
                if (n >= cap_rows) { rc = SPGO_ERR_CAPACITY; break; }
                cov(COV_NEW_PERSON);
                for (int c = 0; c < RS; c++) { SUB(n, c, 0) = -1.0; SUB(n, c, 1) = -1.0; }
                SUB(n, A, 0) = (double)idA; SUB(n, A, 1) = s;
                SUB(n, B, 0) = (double)idB; SUB(n, B, 1) = s;
                SUB(n, K + 1, 0) = 2.0;
                SUB(n, K + 1, 1) = len;
                SUB(n, K, 0) = (0.0 + (double)pscore[idA] + (double)pscore[idB]) + s; /* builtin sum(), :484 */
                n++;
            }
        }
    }
    free(off);
    if (rc) return rc;
    int m = 0;                                                           /* :491-496 */
    for (int j = 0; j < n; j++) {
        if (SUB(j, K + 1, 0) < (double)p->min_parts || SUB(j, K, 0) / SUB(j, K + 1, 0) < p->min_mean_score) {
            cov(COV_PRUNED);
            continue;
        }
        if (m != j) memcpy(&SUB(m, 0, 0), &SUB(j, 0, 0), sizeof(double) * 2 * RS);
        m++;
    }
    return m;
}
#undef SUB

/* ------------------------------------------------------------------------------------------
 * process() tail (evaluate.py:523-543): ids -> coordinates, (0,0) for missing joints, re-ordered
 * to COCO joints by coco_from_part[n_out] (the inverse of dt_gt_mapping, config/config.py:117-118);
 * person score = 1 - 1/total (:541).
 * ------------------------------------------------------------------------------------------ */
void spgo_to_coco(const double *subset, int n_persons, int K, const double *px, const double *py,
                  const int32_t *coco_from_part, int n_out, double *kp_xy, double *person_score) {
    const int RS = K + 2;
    for (int j = 0; j < n_persons; j++) {
        for (int g = 0; g < n_out; g++) {
            const int id = (int)subset[((int64_t)j * RS + coco_from_part[g]) * 2];
            kp_xy[((int64_t)j * n_out + g) * 2 + 0] = id < 0 ? 0.0 : px[id];
            kp_xy[((int64_t)j * n_out + g) * 2 + 1] = id < 0 ? 0.0 : py[id];
        }
        person_score[j] = 1.0 - 1.0 / subset[((int64_t)j * RS + K) * 2];
    }
}

/* ------------------------------------------------------------------------------------------
 * Whole path for a batch (the window evaluate.py:507-513 times), images in parallel over OpenMP
 * threads when n_threads > 1.  Outputs use fixed capacities per image; status[n] is 0 or an error.
 * Any of the intermediate output pointers except the workspaces it needs may NOT be NULL -- this
 * is the checker, it always materialises everything.
 * ------------------------------------------------------------------------------------------ */
int spgo_group_batch(const float *heat, const void *paf, int paf_is_f64, int N, int K, int L,
                     const int32_t *limbs, int H, int W, double image_extent, const spgo_params *p,
                     int cap_peaks, int cap_conn, int cap_rows, int n_threads,
                     double *px, double *py, float *pscore, int32_t *pxi, int32_t *pyi, uint8_t *pint,
                     int32_t *part_count, int32_t *conn_ij, double *conn_score, double *conn_norm,
                     int32_t *conn_count, int32_t *cand_count, double *subset, int32_t *n_persons,
                     int32_t *status) {
    const int64_t plane = (int64_t)H * W;
    const int RS = K + 2;
    int bad = 0;
#if defined(_OPENMP)
    if (n_threads < 1) n_threads = 1;
#pragma omp parallel for schedule(dynamic, 1) num_threads(n_threads) reduction(+ : bad)
#endif
    for (int n = 0; n < N; n++) {
        const float *h = heat + (int64_t)n * K * plane;
        const void *f = paf_is_f64 ? (const void *)((const double *)paf + (int64_t)n * L * plane)
                                   : (const void *)((const float *)paf + (int64_t)n * L * plane);
        double *x = px + (int64_t)n * cap_peaks, *y = py + (int64_t)n * cap_peaks;
        float *sc = pscore + (int64_t)n * cap_peaks;
        int32_t *pc = part_count + (int64_t)n * K;
        int32_t *cij = conn_ij + (int64_t)n * L * cap_conn * 2;
        double *cs_ = conn_score + (int64_t)n * L * cap_conn, *cn = conn_norm + (int64_t)n * L * cap_conn;
        int32_t *cc = conn_count + (int64_t)n * L;
        int st = 0;
        n_persons[n] = 0;
        int tot = spgo_find_peaks(h, K, H, W, plane, W, p, cap_peaks, x, y, sc, pxi + (int64_t)n * cap_peaks,
                                  pyi + (int64_t)n * cap_peaks, pint + (int64_t)n * cap_peaks, pc);
        if (tot > cap_peaks) st = SPGO_ERR_CAPACITY;
        if (!st)
            st = spgo_find_connections(x, y, sc, pc, K, f, paf_is_f64, L, limbs, H, W, plane, W, image_extent, p,
                                       cap_conn, cij, cs_, cn, cc, cand_count ? cand_count + (int64_t)n * L : NULL);
        if (!st) {
            int m = spgo_find_people(sc, pc, K, L, limbs, cap_conn, cij, cs_, cn, cc, p, cap_rows,
                                     subset + (int64_t)n * cap_rows * RS * 2);
            if (m < 0) st = m; else n_persons[n] = m;
        }
        status[n] = st;
        bad += st != 0;
    }
    return bad;
}

int spgo_max_threads(void) {
#if defined(_OPENMP)
    return omp_get_max_threads();
#else
    return 1;
#endif
}
