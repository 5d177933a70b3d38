/* oracle/ps_oracle.c -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * CPU restatement of the PocketSphinx acoustic-scoring + Viterbi hot path; see ps_oracle.h.
 * Citations are to /root/reference (cmusphinx/pocketsphinx 5.1.1 @ 511126b), default float
 * build.  Compile with -ffp-contract=off: the reference accumulates the Gaussian exponent
 * with separate subtract / multiply / multiply / subtract roundings (ptm_mgau.c:64-69).
 */
#include "ps_oracle.h"

#include <limits.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ------------------------------------------------------------------------------------ */
/* helpers                                                                               */

/* (int32)d with the clamp both tied back-ends apply first (ptm_mgau.c:129-132,219-222;
 * s2_semi_mgau.c:97-100,143-146). */
static int32_t
f2i_clamped(float d)
{
    if (d < (float)INT32_MIN)
        return INT32_MIN;
    return (int32_t)d;
}

/* fast_logmath_add on negated logs (tied_mgau_common.h:111-127). */
static int
logadd8(const uint8_t *tab, int mlx, int mly)
{
    int d, r;
    if (mlx > mly) { d = mlx - mly; r = mly; }
    else { d = mly - mlx; r = mlx; }
    /* mixw + ascr can reach 255 + 96, so d can exceed the reference's 256-entry table
     * (logmath.c:116-120), where the reference reads past its allocation.  The table is
     * identically 0 from entry ~30 on; continue it with zeros. */
    return r - (d < 256 ? tab[d] : 0);
}

static size_t
gau_offset(const pso_model_t *m, int cb, int f)
{
    /* start of (cb, f) inside mean/var: [n_mgau][n_feat][n_density][featlen[f]] */
    size_t sum = 0, off = 0;
    int i;
    for (i = 0; i < m->n_feat; ++i) sum += m->featlen[i];
    for (i = 0; i < f; ++i) off += m->featlen[i];
    return ((size_t)cb * sum + off) * m->n_density;
}

/* Full (no early exit) log-density of one codeword: det - sum_j ((x_j - mu_j)^2 * v_j), each
 * product and difference rounded separately, dimensions in ascending order.  The chunked
 * order of ptm_mgau.c:107-128 (ceplen%4 leading dims, then groups of four MAP then REDUCE)
 * performs the same operations on d in the same order. */
static float
gau_full(const float *mean, const float *var, float det, const float *x, int len)
{
    float d = det;
    int j;
    for (j = 0; j < len; ++j) {
        float diff = x[j] - mean[j];
        float sq = diff * diff;
        float c = sq * var[j];
        d = d - c;
    }
    return d;
}

/* ---- fixed point (-DFIXED_POINT build, SURVEY A.1.11) --------------------------------- */
/* MFCCMUL = FIXMUL (fe/fixpoint.h:98-100): the 64-bit product shifted right by the radix (12),
 * truncated to 32 bits. */
static int32_t
fx_mul(int32_t a, int32_t b)
{
    return (int32_t)(uint32_t)(((int64_t)a * (int64_t)b) >> 12);
}

/* GMMSUB (tied_mgau_common.h:62-66) is written ((a)-(b) > a) ? INT_MIN : (a)-(b) on signed ints;
 * gcc folds the overflow test to (b < 0) at every optimisation level, which is what the
 * reference's own build computes: (b < 0) ? INT_MIN : wrap32(a - b). */
static int32_t
fx_gmmsub(int32_t a, int32_t b)
{
    return b < 0 ? INT32_MIN : (int32_t)((uint32_t)a - (uint32_t)b);
}

/* ------------------------------------------------------------------------------------ */
/* state                                                                                 */

pso_gmm_t *
pso_gmm_new(const pso_model_t *m, int32_t n_hist)
{
    pso_gmm_t *g = calloc(1, sizeof(*g));
    int i;
    g->m = m;
    g->n_hist = n_hist < 1 ? 1 : n_hist;
    for (i = 0; i < m->n_feat; ++i) g->sumlen += m->featlen[i];
    if (m->kind == PSO_KIND_PTM) {
        g->hist = calloc((size_t)g->n_hist * m->n_mgau * m->n_feat * m->topn, sizeof(pso_topn_t));
        g->cb_active = calloc((size_t)g->n_hist * m->n_mgau, 1);
    }
    else if (m->kind == PSO_KIND_SEMI) {
        g->hist = calloc((size_t)g->n_hist * m->n_feat * m->topn, sizeof(pso_topn_t));
        g->hist_n = calloc((size_t)g->n_hist * m->n_feat, 1);
    }
    else {
        g->ms_dist = calloc((size_t)m->n_mgau * m->n_feat * m->topn, sizeof(pso_topn_t));
    }
    pso_gmm_reset(g);
    return g;
}

void
pso_gmm_free(pso_gmm_t *g)
{
    if (!g) return;
    free(g->hist); free(g->cb_active); free(g->hist_n); free(g->ms_dist);
    free(g);
}

/* ptm_mgau_reset_fast_hist (ptm_mgau.c:777-803); s2_semi_mgau_init (s2_semi_mgau.c:1319-1327):
 * codewords 0..N-1 with WORST_DIST, every codebook active. */
void
pso_gmm_reset(pso_gmm_t *g)
{
    const pso_model_t *m = g->m;
    size_t n, i;
    g->frame_idx = 0;
    if (m->kind == PSO_KIND_PTM) {
        n = (size_t)g->n_hist * m->n_mgau * m->n_feat;
        for (i = 0; i < n * m->topn; ++i) {
            g->hist[i].cw = (int32_t)(i % m->topn);
            g->hist[i].score = PSO_WORST_DIST;
        }
        memset(g->cb_active, 1, (size_t)g->n_hist * m->n_mgau);
    }
    else if (m->kind == PSO_KIND_SEMI) {
        n = (size_t)g->n_hist * m->n_feat;
        for (i = 0; i < n * m->topn; ++i) {
            g->hist[i].cw = (int32_t)(i % m->topn);
            g->hist[i].score = PSO_WORST_DIST;
        }
        memset(g->hist_n, 0, n);
    }
}

/* ------------------------------------------------------------------------------------ */
/* tied back-ends: re-score last frame's list, then scan the codebook                    */

/* eval_topn (ptm_mgau.c:88-136, s2_semi_mgau.c:70-109): re-score the N listed codewords
 * for this frame; stable insertion sort, descending, strict '>' (ptm_mgau.c:72-85). */
static void
rescore_topn(const pso_model_t *m, pso_topn_t *topn, int cb, int f, const float *x)
{
    int len = m->featlen[f], i, j;
    size_t base = gau_offset(m, cb, f);
    const float *det = m->det + ((size_t)cb * m->n_feat + f) * m->n_density;

    for (i = 0; i < m->topn; ++i) {
        int32_t cw = topn[i].cw;
        pso_topn_t v;
        float d = gau_full(m->mean + base + (size_t)cw * len, m->var + base + (size_t)cw * len,
                           det[cw], x, len);
        v.cw = cw;
        v.score = f2i_clamped(d);
        for (j = i - 1; j >= 0 && v.score > topn[j].score; --j)
            topn[j + 1] = topn[j];
        topn[j + 1] = v;
    }
}

/* eval_topn in the fixed-point build (ptm_mgau.c:88-136): no early exit, every step through
 * GMMSUB. */
static void
rescore_topn_fx(const pso_model_t *m, pso_topn_t *topn, int cb, int f, const int32_t *x)
{
    int len = m->featlen[f], i, j;
    size_t base = gau_offset(m, cb, f);
    const int32_t *det = (const int32_t *)m->det + ((size_t)cb * m->n_feat + f) * m->n_density;
    const int32_t *mean0 = (const int32_t *)m->mean + base, *var0 = (const int32_t *)m->var + base;

    for (i = 0; i < m->topn; ++i) {
        int32_t cw = topn[i].cw, d = det[cw];
        const int32_t *mean = mean0 + (size_t)cw * len, *var = var0 + (size_t)cw * len;
        pso_topn_t v;
        for (j = 0; j < len; ++j) {
            int32_t diff = (int32_t)((uint32_t)x[j] - (uint32_t)mean[j]);
            d = fx_gmmsub(d, fx_mul(fx_mul(diff, diff), var[j]));
        }
        v.cw = cw;
        v.score = d;                     /* already an int; the INT_MIN clamp (:129-132) is a no-op */
        for (j = i - 1; j >= 0 && v.score > topn[j].score; --j)
            topn[j + 1] = topn[j];
        topn[j + 1] = v;
    }
}

/* insertion_sort_cb (ptm_mgau.c:140-149) / the tail of eval_cb (s2_semi_mgau.c:156-161):
 * drop the worst entry, shift down every entry whose score is <= intd. */
static void
insert_cw(pso_topn_t *topn, int n, int32_t cw, int32_t intd)
{
    int k = n - 1;
    while (k > 0 && intd >= topn[k - 1].score) {
        topn[k] = topn[k - 1];
        --k;
    }
    topn[k].cw = cw;
    topn[k].score = intd;
}

static int
listed(const pso_topn_t *topn, int n, int32_t cw)
{
    int i;
    for (i = 0; i < n; ++i)
        if (topn[i].cw == cw) return 1;
    return 0;
}

/* eval_cb, PTM flavour (ptm_mgau.c:152-226): early exit tested in float against
 * (float)worst->score before the leading ceplen%4 dims one at a time, then before each group
 * of four, and once more after the last dimension. */
static void
scan_cb_ptm(const pso_model_t *m, pso_topn_t *topn, int cb, int f, const float *x)
{
    int len = m->featlen[f], n = m->topn, cw;
    size_t base = gau_offset(m, cb, f);
    const float *det = m->det + ((size_t)cb * m->n_feat + f) * m->n_density;

    for (cw = 0; cw < m->n_density; ++cw) {
        const float *mean = m->mean + base + (size_t)cw * len;
        const float *var = m->var + base + (size_t)cw * len;
        float d = det[cw];
        float thresh = (float)topn[n - 1].score;
        int j = 0, k;

        while (j < len % 4 && d >= thresh) {
            float diff = x[j] - mean[j];
            float sq = diff * diff;
            d = d - sq * var[j];
            ++j;
        }
        while (j < len && d >= thresh) {
            float c[4];
            for (k = 0; k < 4; ++k) {
                float diff = x[j + k] - mean[j + k];
                float sq = diff * diff;
                c[k] = sq * var[j + k];
            }
            for (k = 0; k < 4; ++k)
                d = d - c[k];
            j += 4;
        }
        if (j < len) continue;          /* knocked out early */
        if (d < thresh) continue;
        if (listed(topn, n, cw)) continue;
        insert_cw(topn, n, cw, f2i_clamped(d));
    }
}

/* eval_cb in the fixed-point build: the same loop structure with int arithmetic.  The early exits
 * are NOT result-neutral here (a wrapped subtraction can climb back above the threshold), so the
 * loop is restated literally: tests before the leading ceplen%4 dimensions one at a time, then
 * before every group of four. */
static void
scan_cb_ptm_fx(const pso_model_t *m, pso_topn_t *topn, int cb, int f, const int32_t *x)
{
    int len = m->featlen[f], n = m->topn, cw;
    size_t base = gau_offset(m, cb, f);
    const int32_t *det = (const int32_t *)m->det + ((size_t)cb * m->n_feat + f) * m->n_density;
    const int32_t *mean0 = (const int32_t *)m->mean + base, *var0 = (const int32_t *)m->var + base;

    for (cw = 0; cw < m->n_density; ++cw) {
        const int32_t *mean = mean0 + (size_t)cw * len, *var = var0 + (size_t)cw * len;
        int32_t d = det[cw], thresh = topn[n - 1].score;
        int j = 0, k;

        while (j < len % 4 && d >= thresh) {
            int32_t diff = (int32_t)((uint32_t)x[j] - (uint32_t)mean[j]);
            d = fx_gmmsub(d, fx_mul(fx_mul(diff, diff), var[j]));
            ++j;
        }
        while (j < len && d >= thresh) {
            int32_t c[4];
            for (k = 0; k < 4; ++k) {
                int32_t diff = (int32_t)((uint32_t)x[j + k] - (uint32_t)mean[j + k]);
                c[k] = fx_mul(fx_mul(diff, diff), var[j + k]);
            }
            for (k = 0; k < 4; ++k)
                d = fx_gmmsub(d, c[k]);
            j += 4;
        }
        if (j < len) continue;
        if (d < thresh) continue;
        if (listed(topn, n, cw)) continue;
        insert_cw(topn, n, cw, d);
    }
}

/* eval_cb, semi-continuous flavour (s2_semi_mgau.c:112-170): the per-dimension test compares
 * float d with the int worst score (promoted to float); after a complete pass the test is on
 * the truncated int. */
static void
scan_cb_semi(const pso_model_t *m, pso_topn_t *topn, int f, const float *x)
{
    int len = m->featlen[f], n = m->topn, cw;
    size_t base = gau_offset(m, 0, f);
    const float *det = m->det + (size_t)f * m->n_density;

    for (cw = 0; cw < m->n_density; ++cw) {
        const float *mean = m->mean + base + (size_t)cw * len;
        const float *var = m->var + base + (size_t)cw * len;
        float d = det[cw];
        int32_t di;
        int j;

        for (j = 0; j < len && d >= (float)topn[n - 1].score; ++j) {
            float diff = x[j] - mean[j];
            float sq = diff * diff;
            d = d - sq * var[j];
        }
        if (j < len) continue;
        di = f2i_clamped(d);
        if (di < topn[n - 1].score) continue;
        if (listed(topn, n, cw)) continue;
        insert_cw(topn, n, cw, di);
    }
}

/* eval_cb, semi-continuous flavour in the fixed-point build (s2_semi_mgau.c:112-170): the test
 * before every dimension and the final test compare ints. */
static void
scan_cb_semi_fx(const pso_model_t *m, pso_topn_t *topn, int f, const int32_t *x)
{
    int len = m->featlen[f], n = m->topn, cw;
    size_t base = gau_offset(m, 0, f);
    const int32_t *det = (const int32_t *)m->det + (size_t)f * m->n_density;
    const int32_t *mean0 = (const int32_t *)m->mean + base, *var0 = (const int32_t *)m->var + base;

    for (cw = 0; cw < m->n_density; ++cw) {
        const int32_t *mean = mean0 + (size_t)cw * len, *var = var0 + (size_t)cw * len;
        int32_t d = det[cw];
        int j;
        for (j = 0; j < len && d >= topn[n - 1].score; ++j) {
            int32_t diff = (int32_t)((uint32_t)x[j] - (uint32_t)mean[j]);
            d = fx_gmmsub(d, fx_mul(fx_mul(diff, diff), var[j]));
        }
        if (j < len) continue;
        if (d < topn[n - 1].score) continue;
        if (listed(topn, n, cw)) continue;
        insert_cw(topn, n, cw, d);
    }
}

/* ------------------------------------------------------------------------------------ */
/* PTM                                                                                   */

/* ptm_mgau_codebook_norm (ptm_mgau.c:266-295): per stream, max over active codebooks of
 * (best score >> 10); every listed score becomes min(96, -((score >> 10) - norm)). */
static void
ptm_norm(const pso_model_t *m, pso_topn_t *slot, const uint8_t *active)
{
    int f, cb, k;
    for (f = 0; f < m->n_feat; ++f) {
        int32_t norm = PSO_WORST_SCORE;
        for (cb = 0; cb < m->n_mgau; ++cb) {
            int32_t top;
            if (!active[cb]) continue;
            top = slot[((size_t)cb * m->n_feat + f) * m->topn].score >> PSO_SENSCR_SHIFT;
            if (norm < top) norm = top;
        }
        for (cb = 0; cb < m->n_mgau; ++cb) {
            pso_topn_t *t = slot + ((size_t)cb * m->n_feat + f) * m->topn;
            if (!active[cb]) continue;
            for (k = 0; k < m->topn; ++k) {
                int32_t s = t[k].score >> PSO_SENSCR_SHIFT;
                s = -(s - norm);
                if (s > PSO_MAX_NEG_ASCR) s = PSO_MAX_NEG_ASCR;
                t[k].score = s;
            }
        }
    }
}

/* ptm_mgau_senone_eval (ptm_mgau.c:327-403). */
static void
ptm_senones(const pso_model_t *m, pso_topn_t *slot, const uint8_t *active, int16_t *senscr,
            const uint8_t *list, int32_t n_list, int compall)
{
    int32_t i, last = 0, best = 0x7fffffff;
    size_t row = m->mixw_4bit ? (size_t)(m->n_sen + 1) / 2 : (size_t)m->n_sen;

    memset(senscr, 0, (size_t)m->n_sen * sizeof(*senscr));
    if (compall) n_list = m->n_sen;
    for (i = 0; i < n_list; ++i) {
        int32_t sen = compall ? i : list[i] + last;
        int cb, f, j, ascore = 0;
        last = sen;
        cb = m->sen2cb[sen];
        if (!active[cb]) {
            /* senones of a pruned codebook see every density at the floor (:353-364) */
            for (f = 0; f < m->n_feat; ++f)
                for (j = 0; j < m->topn; ++j)
                    slot[((size_t)cb * m->n_feat + f) * m->topn + j].score = PSO_MAX_NEG_ASCR;
        }
        for (f = 0; f < m->n_feat; ++f) {
            const pso_topn_t *t = slot + ((size_t)cb * m->n_feat + f) * m->topn;
            int fden = 0;
            for (j = 0; j < m->topn; ++j) {
                const uint8_t *r = m->mixw + ((size_t)f * m->n_density + t[j].cw) * row;
                int w;
                if (m->mixw_4bit) {
                    int b = r[sen / 2];
                    /* NB the reference tests the low bit of the *byte*, not of sen (:376-377) */
                    b = (b & 1) ? b >> 4 : b & 0x0f;
                    w = m->mixw_cb[b];
                }
                else
                    w = r[sen];
                fden = j == 0 ? w + t[j].score : logadd8(m->logadd8, fden, w + t[j].score);
            }
            ascore += fden;
        }
        if (ascore < best) best = ascore;
        senscr[sen] = (int16_t)ascore;
    }
    for (i = 0; i < m->n_sen; ++i)
        senscr[i] = (int16_t)(senscr[i] - best);
}

/* ptm_mgau_frame_eval (ptm_mgau.c:409-454). */
static int
ptm_frame_eval(pso_gmm_t *g, int16_t *senscr, const uint8_t *list, int32_t n_list,
               const float *feat, int32_t frame, int32_t compall)
{
    const pso_model_t *m = g->m;
    size_t per = (size_t)m->n_mgau * m->n_feat * m->topn;
    int idx = frame % g->n_hist;
    pso_topn_t *slot = g->hist + per * idx;
    uint8_t *active = g->cb_active + (size_t)idx * m->n_mgau;
    int cb, f, off;

    if (frame >= g->frame_idx) {
        int prev = idx == 0 ? g->n_hist - 1 : idx - 1;
        int32_t i, last = 0;
        if (prev != idx)
            memcpy(slot, g->hist + per * prev, per * sizeof(*slot));
        /* ptm_mgau_calc_cb_active (:298-321) */
        if (compall)
            memset(active, 1, m->n_mgau);
        else {
            memset(active, 0, m->n_mgau);
            for (i = 0; i < n_list; ++i) {
                int32_t sen = list[i] + last;
                active[m->sen2cb[sen]] = 1;
                last = sen;
            }
        }
        /* ptm_mgau_codebook_eval (:232-254) */
        for (cb = 0; cb < m->n_mgau; ++cb)
            for (f = 0, off = 0; f < m->n_feat; off += m->featlen[f], ++f)
                if (m->fixed_point)
                    rescore_topn_fx(m, slot + ((size_t)cb * m->n_feat + f) * m->topn, cb, f, (const int32_t *)feat + off);
                else
                    rescore_topn(m, slot + ((size_t)cb * m->n_feat + f) * m->topn, cb, f, feat + off);
        if (frame % m->ds_ratio == 0)
            for (cb = 0; cb < m->n_mgau; ++cb) {
                if (!active[cb]) continue;
                for (f = 0, off = 0; f < m->n_feat; off += m->featlen[f], ++f)
                    if (m->fixed_point)
                        scan_cb_ptm_fx(m, slot + ((size_t)cb * m->n_feat + f) * m->topn, cb, f, (const int32_t *)feat + off);
                    else
                        scan_cb_ptm(m, slot + ((size_t)cb * m->n_feat + f) * m->topn, cb, f, feat + off);
            }
        if (g->raw)
            memcpy(g->raw, slot, per * sizeof(*slot));
        ptm_norm(m, slot, active);
    }
    ptm_senones(m, slot, active, senscr, list, n_list, compall);
    return 0;
}

/* ------------------------------------------------------------------------------------ */
/* semi-continuous                                                                       */

/* mgau_norm (s2_semi_mgau.c:186-203): returns how many entries survive topn_beam. */
static int
semi_norm(const pso_model_t *m, pso_topn_t *t, int f)
{
    int32_t norm = t[0].score >> PSO_SENSCR_SHIFT;
    int beam = m->topn_beam ? m->topn_beam[f] : 0;
    int j;
    for (j = 0; j < m->topn; ++j) {
        t[j].score = -((t[j].score >> PSO_SENSCR_SHIFT) - norm);
        if (t[j].score > PSO_MAX_NEG_ASCR) t[j].score = PSO_MAX_NEG_ASCR;
        if (beam && t[j].score > beam) break;
    }
    return j;
}

static int
nib(const uint8_t *row, int sen)
{
    return (sen & 1) ? row[sen / 2] >> 4 : row[sen / 2] & 0x0f;
}

/* get_scores_{8b,4b}_feat{_N,_any,_all} (s2_semi_mgau.c:206-831), one stream.  All 8-bit
 * variants compute the same int expression.  4-bit: the unrolled N=1..6 active-list variants
 * pre-add mixw_cb + score into uint8 (wraps mod 256, :453-463); _any and _all use int;
 * _all stops at n_sen & ~1 (:809). */
static void
semi_senones(const pso_model_t *m, const pso_topn_t *t, int f, int topn, int16_t *senscr,
             const uint8_t *list, int32_t n_list, int compall)
{
    size_t row = m->mixw_4bit ? (size_t)(m->n_sen + 1) / 2 : (size_t)m->n_sen;
    const uint8_t *base = m->mixw + (size_t)f * m->n_density * row;
    int wrap8 = m->mixw_4bit && !compall && topn >= 1 && topn <= 6;
    int32_t n = compall ? (m->mixw_4bit ? (m->n_sen & ~1) : m->n_sen) : n_list;
    int32_t i, last = 0;
    int k;

    for (i = 0; i < n; ++i) {
        int32_t sen = compall ? i : list[i] + last;
        int tmp = 0;
        last = sen;
        for (k = 0; k == 0 || k < topn; ++k) {
            const uint8_t *r = base + (size_t)t[k].cw * row;
            int w = m->mixw_4bit ? m->mixw_cb[nib(r, sen)] : r[sen];
            int v = w + t[k].score;
            if (wrap8) v &= 0xff;
            tmp = k == 0 ? v : logadd8(m->logadd8, tmp, v);
        }
        senscr[sen] = (int16_t)(senscr[sen] + tmp);
    }
}

/* s2_semi_mgau_frame_eval (s2_semi_mgau.c:837-883). */
static int
semi_frame_eval(pso_gmm_t *g, int16_t *senscr, const uint8_t *list, int32_t n_list,
                const float *feat, int32_t frame, int32_t compall)
{
    const pso_model_t *m = g->m;
    size_t per = (size_t)m->n_feat * m->topn;
    int idx = frame % g->n_hist, f, off = 0;
    pso_topn_t *slot = g->hist + per * idx;

    memset(senscr, 0, (size_t)m->n_sen * sizeof(*senscr));
    for (f = 0; f < m->n_feat; off += m->featlen[f], ++f) {
        pso_topn_t *t = slot + (size_t)f * m->topn;
        if (frame >= g->frame_idx) {
            int prev = idx == 0 ? g->n_hist - 1 : idx - 1;
            if (prev != idx)
                memcpy(t, g->hist + per * prev + (size_t)f * m->topn, m->topn * sizeof(*t));
            /* mgau_dist (:172-183) */
            if (m->fixed_point) {
                rescore_topn_fx(m, t, 0, f, (const int32_t *)feat + off);
                if (frame % m->ds_ratio == 0)
                    scan_cb_semi_fx(m, t, f, (const int32_t *)feat + off);
            }
            else {
                rescore_topn(m, t, 0, f, feat + off);
                if (frame % m->ds_ratio == 0)
                    scan_cb_semi(m, t, f, feat + off);
            }
            g->hist_n[(size_t)idx * m->n_feat + f] = (uint8_t)semi_norm(m, t, f);
        }
        semi_senones(m, t, f, g->hist_n[(size_t)idx * m->n_feat + f], senscr, list, n_list, compall);
    }
    return 0;
}

/* ------------------------------------------------------------------------------------ */
/* ms (continuous / generic multi-stream)                                                */

typedef struct { int32_t id; float dist; } ms_dist_t;

/* compute_dist / compute_dist_all (ms_gauden.c:378-489). */
static void
ms_compute_dist(const pso_model_t *m, ms_dist_t *out, int cb, int f, const float *x)
{
    int len = m->featlen[f], n = m->topn, d, i, j;
    size_t base = gau_offset(m, cb, f);
    const float *det = m->det + ((size_t)cb * m->n_feat + f) * m->n_density;

    if (n >= m->n_density) {
        for (d = 0; d < m->n_density; ++d) {
            out[d].dist = gau_full(m->mean + base + (size_t)d * len, m->var + base + (size_t)d * len,
                                   det[d], x, len);
            out[d].id = d;
        }
        return;
    }
    for (i = 0; i < n; ++i) {
        out[i].dist = (float)PSO_WORST_DIST;
        out[i].id = 0;   /* ckd_calloc'ed, and never read before being overwritten... */
    }
    for (d = 0; d < m->n_density; ++d) {
        const float *mean = m->mean + base + (size_t)d * len;
        const float *var = m->var + base + (size_t)d * len;
        float dv = det[d];
        for (i = 0; i < len && dv >= out[n - 1].dist; ++i) {
            float diff = x[i] - mean[i];
            dv -= diff * diff * var[i];
        }
        if (i < len || dv < out[n - 1].dist) continue;
        for (i = 0; i < n && dv < out[i].dist; ++i) ;
        for (j = n - 1; j > i; --j) out[j] = out[j - 1];
        out[i].dist = dv;
        out[i].id = d;
    }
}

/* logmath_add with a shifted table (logmath.c:402-446). */
static int
logadd_wide(const pso_model_t *m, int x, int y)
{
    int d, r;
    if (x <= m->logadd_ms_zero) return y;
    if (y <= m->logadd_ms_zero) return x;
    if (x > y) { d = x - y; r = x; }
    else { d = y - x; r = y; }
    if (d < 0) return r;
    if (d >= m->logadd_ms_size) return r;
    return r + (int)m->logadd_ms[d];
}

/* senone_eval (ms_senone.c:358-407). */
static int32_t
ms_senone(const pso_model_t *m, int id, const ms_dist_t *dist /* [n_feat][topn] */)
{
    int32_t scr = 0;
    int f, t, n = m->topn < m->n_density ? m->topn : m->n_density;
    for (f = 0; f < m->n_feat; ++f) {
        const ms_dist_t *fd = dist + (size_t)f * m->topn;
        int32_t fscr = 0;
        for (t = 0; t < n; ++t) {
            int32_t fden, w, fw;
            if (fd[t].dist < (float)INT32_MIN)
                fden = INT32_MIN >> PSO_SENSCR_SHIFT;
            else
                fden = ((int32_t)fd[t].dist + ((1 << PSO_SENSCR_SHIFT) - 1)) >> PSO_SENSCR_SHIFT;
            w = m->pdf_transposed
                ? m->mixw[((size_t)f * m->n_density + fd[t].id) * m->n_sen + id]
                : m->mixw[((size_t)id * m->n_feat + f) * m->n_density + fd[t].id];
            fw = fden - w;
            fscr = t == 0 ? fw : logadd_wide(m, fscr, fw);
        }
        scr -= fscr;
    }
    scr /= m->aw;
    if (scr > 32767) scr = 32767;
    if (scr < -32768) scr = -32768;
    return scr;
}

/* ms_cont_mgau_frame_eval (ms_mgau.c:192-282). */
static int
ms_frame_eval(pso_gmm_t *g, int16_t *senscr, const uint8_t *list, int32_t n_list,
              const float *feat, int32_t compall)
{
    const pso_model_t *m = g->m;
    ms_dist_t *dist = (ms_dist_t *)g->ms_dist;
    size_t per = (size_t)m->n_feat * m->topn;
    uint8_t *active = calloc(m->n_mgau, 1);
    int32_t i, last, best = INT32_MAX;
    int cb, f, off;

    if (compall)
        memset(active, 1, m->n_mgau);
    else
        for (i = 0, last = 0; i < n_list; ++i) {
            last += list[i];
            active[m->sen2cb[last]] = 1;
        }
    for (cb = 0; cb < m->n_mgau; ++cb) {
        if (!active[cb]) continue;
        for (f = 0, off = 0; f < m->n_feat; off += m->featlen[f], ++f)
            ms_compute_dist(m, dist + per * cb + (size_t)f * m->topn, cb, f, feat + off);
    }
    free(active);
    if (compall) n_list = m->n_sen;
    for (i = 0, last = 0; i < n_list; ++i) {
        int32_t s = compall ? i : last + list[i];
        last = s;
        senscr[s] = (int16_t)ms_senone(m, s, dist + per * m->sen2cb[s]);
        if (best > senscr[s]) best = senscr[s];
    }
    for (i = 0, last = 0; i < n_list; ++i) {
        int32_t s = compall ? i : last + list[i];
        int32_t bs;
        last = s;
        bs = senscr[s] - best;
        if (bs > 32767) bs = 32767;
        if (bs < -32768) bs = -32768;
        senscr[s] = (int16_t)bs;
    }
    return 0;
}

/* ------------------------------------------------------------------------------------ */

int
pso_frame_eval(pso_gmm_t *g, int16_t *senscr, const uint8_t *senone_active,
               int32_t n_senone_active, const float *feat, int32_t frame, int32_t compallsen)
{
    switch (g->m->kind) {
    case PSO_KIND_PTM:
        return ptm_frame_eval(g, senscr, senone_active, n_senone_active, feat, frame, compallsen);
    case PSO_KIND_SEMI:
        return semi_frame_eval(g, senscr, senone_active, n_senone_active, feat, frame, compallsen);
    default:
        return ms_frame_eval(g, senscr, senone_active, n_senone_active, feat, compallsen);
    }
}

int
pso_score_utt(const pso_model_t *m, const float *feats, int32_t T, int16_t *senscr,
              int32_t *topn_out, int32_t *raw_out)
{
    pso_gmm_t *g = pso_gmm_new(m, 2);
    size_t per_ptm = (size_t)m->n_mgau * m->n_feat * m->topn;
    int32_t t;
    for (t = 0; t < T; ++t) {
        g->raw = raw_out && m->kind == PSO_KIND_PTM ? (pso_topn_t *)raw_out + (size_t)t * per_ptm : NULL;
        pso_frame_eval(g, senscr + (size_t)t * m->n_sen, NULL, 0, feats + (size_t)t * g->sumlen, t, 1);
        g->frame_idx = t + 1;       /* acmod_advance (acmod.c:868-877) */
        if (topn_out && m->kind != PSO_KIND_MS) {
            size_t per = (size_t)(m->kind == PSO_KIND_PTM ? m->n_mgau : 1) * m->n_feat * m->topn;
            memcpy(topn_out + (size_t)t * per * 2, g->hist + per * (t % g->n_hist), per * sizeof(pso_topn_t));
        }
    }
    pso_gmm_free(g);
    return 0;
}

/* acmod_flags2list (acmod.c:1224-1275): ascending senone ids as uint8 deltas from the
 * previous listed id (first from 0); a gap above 255 is bridged by 255-steps, which makes the
 * intermediate senones part of the list. */
int32_t
pso_flags2list(const uint8_t *flags, int32_t n_sen, uint8_t *list)
{
    int32_t s, last = 0, n = 0;
    for (s = 0; s < n_sen; ++s) {
        int32_t delta;
        if (!flags[s]) continue;
        delta = s - last;
        while (delta > 255) {
            list[n++] = 255;
            delta -= 255;
        }
        list[n++] = (uint8_t)delta;
        last = s;
    }
    return n;
}

double
pso_time_score_utt(const pso_model_t *m, const float *feats, int32_t T, int32_t reps)
{
    int16_t *scr = malloc((size_t)T * m->n_sen * sizeof(*scr));
    struct timespec a, b;
    int r;
    pso_score_utt(m, feats, T < 16 ? T : 16, scr, NULL, NULL);
    clock_gettime(CLOCK_MONOTONIC, &a);
    for (r = 0; r < reps; ++r)
        pso_score_utt(m, feats, T, scr, NULL, NULL);
    clock_gettime(CLOCK_MONOTONIC, &b);
    free(scr);
    return (b.tv_sec - a.tv_sec) + 1e-9 * (b.tv_nsec - a.tv_nsec);
}

/* ------------------------------------------------------------------------------------ */
/* HMM                                                                                   */

void
pso_hmm_clear_scores(pso_hmm_t *h)        /* hmm.c:167-178 */
{
    int i;
    for (i = 0; i < h->n_emit_state; ++i) h->score[i] = PSO_WORST_SCORE;
    h->out_score = PSO_WORST_SCORE;
    h->bestscore = PSO_WORST_SCORE;
}

void
pso_hmm_clear(pso_hmm_t *h)               /* hmm.c:180-196 */
{
    int i;
    for (i = 0; i < h->n_emit_state; ++i) {
        h->score[i] = PSO_WORST_SCORE;
        h->history[i] = -1;
    }
    h->out_score = PSO_WORST_SCORE;
    h->out_history = -1;
    h->bestscore = PSO_WORST_SCORE;
    h->frame = -1;
}

void
pso_hmm_init(const pso_hmmctx_t *c, pso_hmm_t *h, int mpx, int ssid, int tmatid)  /* hmm.c:85-105 */
{
    int i;
    h->ctx = NULL;
    h->mpx = (uint8_t)mpx;
    h->n_emit_state = (uint8_t)c->n_emit_state;
    if (mpx) {
        h->ssid = PSO_BAD_SSID;
        h->senid[0] = (uint16_t)ssid;
        for (i = 1; i < c->n_emit_state; ++i) h->senid[i] = PSO_BAD_SSID;
    }
    else {
        h->ssid = (uint16_t)ssid;
        for (i = 0; i < c->n_emit_state; ++i)
            h->senid[i] = c->sseq[(size_t)ssid * c->n_emit_state + i];
    }
    h->tmatid = (int16_t)tmatid;
    pso_hmm_clear(h);
}

void
pso_hmm_enter(pso_hmm_t *h, int32_t score, int32_t histid, int frame)   /* hmm.c:198-204 */
{
    h->score[0] = score;
    h->history[0] = histid;
    h->frame = frame;
}

void
pso_hmm_normalize(pso_hmm_t *h, int32_t bestscr)                        /* hmm.c:206-216 */
{
    int i;
    for (i = 0; i < h->n_emit_state; ++i)
        if (h->score[i] > PSO_WORST_SCORE) h->score[i] -= bestscr;
    if (h->out_score > PSO_WORST_SCORE) h->out_score -= bestscr;
}

/* Three-way max with the reference's tie order (e.g. hmm.c:257-271): returns which
 * candidate wins: 0 = self loop t0, 1 = from the state below t1, 2 = skip t2. */
static int
pick3(int32_t t0, int32_t t1, int32_t t2, int32_t *out)
{
    if (t0 > t1) {
        if (t2 > t0) { *out = t2; return 2; }
        *out = t0; return 0;
    }
    if (t2 > t1) { *out = t2; return 2; }
    *out = t1; return 1;
}

#define FLOOR(s) do { if ((s) < PSO_WORST_SCORE) (s) = PSO_WORST_SCORE; } while (0)
#define RAISE(b, s) do { if ((s) > (b)) (b) = (s); } while (0)

/* hmm_vit_eval_5st_lr / _3st_lr share this shape (hmm.c:223-353, 530-607); they differ in
 * which blocks are guarded and in the 3-state skip-arc handling, so they stay separate. */
static int32_t
vit_5st(const pso_hmmctx_t *c, pso_hmm_t *h)
{
    const uint8_t *tp = c->tp + (size_t)h->tmatid * 30;
    const int16_t *sen = c->senscore;
#define TP(i, j) (-(int32_t)tp[(i) * 6 + (j)])
#define OBS(i) (-(int32_t)sen[h->senid[i]])
    int32_t s0, s1, s2, s3, s4, s5, t0, t1, t2, best = PSO_WORST_SCORE;

    s4 = h->score[4] + OBS(4);
    s3 = h->score[3] + OBS(3);
    if (s3 > PSO_WORST_SCORE) {                       /* exit state (:237-250) */
        t1 = s4 + TP(4, 5);
        t2 = s3 + TP(3, 5);
        if (t1 > t2) { s5 = t1; h->out_history = h->history[4]; }
        else { s5 = t2; h->out_history = h->history[3]; }
        FLOOR(s5);
        h->out_score = s5;
        best = s5;
    }
    s2 = h->score[2] + OBS(2);
    if (s2 > PSO_WORST_SCORE) {                       /* state 4 (:254-276) */
        int w = pick3(s4 + TP(4, 4), s3 + TP(3, 4), s2 + TP(2, 4), &s4);
        if (w == 2) h->history[4] = h->history[2];
        else if (w == 1) h->history[4] = h->history[3];
        FLOOR(s4); RAISE(best, s4);
        h->score[4] = s4;
    }
    s1 = h->score[1] + OBS(1);
    if (s1 > PSO_WORST_SCORE) {                       /* state 3 (:280-302) */
        int w = pick3(s3 + TP(3, 3), s2 + TP(2, 3), s1 + TP(1, 3), &s3);
        if (w == 2) h->history[3] = h->history[1];
        else if (w == 1) h->history[3] = h->history[2];
        FLOOR(s3); RAISE(best, s3);
        h->score[3] = s3;
    }
    s0 = h->score[0] + OBS(0);
    {                                                 /* state 2 (:306-326) */
        int w = pick3(s2 + TP(2, 2), s1 + TP(1, 2), s0 + TP(0, 2), &s2);
        if (w == 2) h->history[2] = h->history[0];
        else if (w == 1) h->history[2] = h->history[1];
        FLOOR(s2); RAISE(best, s2);
        h->score[2] = s2;
    }
    t0 = s1 + TP(1, 1);                               /* state 1 (:329-340) */
    t1 = s0 + TP(0, 1);
    if (t0 > t1) s1 = t0;
    else { s1 = t1; h->history[1] = h->history[0]; }
    FLOOR(s1); RAISE(best, s1);
    h->score[1] = s1;
    s0 = s0 + TP(0, 0);                               /* state 0 (:342-346) */
    FLOOR(s0); RAISE(best, s0);
    h->score[0] = s0;
    h->bestscore = best;
    return best;
#undef TP
#undef OBS
}

static int32_t
vit_3st(const pso_hmmctx_t *c, pso_hmm_t *h)
{
    const uint8_t *tp = c->tp + (size_t)h->tmatid * 12;
    const int16_t *sen = c->senscore;
#define TP(i, j) (-(int32_t)tp[(i) * 4 + (j)])
#define OBS(i) (-(int32_t)sen[h->senid[i]])
    int32_t s0, s1, s2, s3, t0, t1, t2, best = PSO_WORST_SCORE;

    s2 = h->score[2] + OBS(2);
    s1 = h->score[1] + OBS(1);
    s0 = h->score[0] + OBS(0);
    t2 = INT32_MIN;          /* only overwritten when a skip arc exists (:543, SURVEY A.1.5) */
    if (s1 > PSO_WORST_SCORE) {                       /* exit state (:546-559) */
        t1 = s2 + TP(2, 3);
        if (TP(1, 3) > PSO_TMAT_WORST_SCORE) t2 = s1 + TP(1, 3);
        if (t1 > t2) { s3 = t1; h->out_history = h->history[2]; }
        else { s3 = t2; h->out_history = h->history[1]; }
        FLOOR(s3);
        h->out_score = s3;
        best = s3;
    }
    t0 = s2 + TP(2, 2);                               /* state 2 (:562-583); stale t2 reused */
    t1 = s1 + TP(1, 2);
    if (TP(0, 2) > PSO_TMAT_WORST_SCORE) t2 = s0 + TP(0, 2);
    {
        int w = pick3(t0, t1, t2, &s2);
        if (w == 2) h->history[2] = h->history[0];
        else if (w == 1) h->history[2] = h->history[1];
    }
    FLOOR(s2); RAISE(best, s2);
    h->score[2] = s2;
    t0 = s1 + TP(1, 1);                               /* state 1 (:586-596) */
    t1 = s0 + TP(0, 1);
    if (t0 > t1) s1 = t0;
    else { s1 = t1; h->history[1] = h->history[0]; }
    FLOOR(s1); RAISE(best, s1);
    h->score[1] = s1;
    s0 = s0 + TP(0, 0);                               /* state 0 (:599-602) */
    FLOOR(s0); RAISE(best, s0);
    h->score[0] = s0;
    h->bestscore = best;
    return best;
#undef TP
#undef OBS
}

/* Multiplexed variants: senid[] holds per-state senone-sequence ids which travel with the
 * winning predecessor (hmm.c:356-525, 610-706). */
#define MPX_OBS(st) (-(int32_t)sen[c->sseq[(size_t)h->senid[st] * c->n_emit_state + (st)]])

static int32_t
vit_5st_mpx(const pso_hmmctx_t *c, pso_hmm_t *h)
{
    const uint8_t *tp = c->tp + (size_t)h->tmatid * 30;
    const int16_t *sen = c->senscore;
    uint16_t *ssid = h->senid;
#define TP(i, j) (-(int32_t)tp[(i) * 6 + (j)])
    int32_t s0, s1, s2, s3, s4, s5, t0, t1, t2, best;
    int w;

    if (ssid[4] == PSO_BAD_SSID) s4 = t1 = PSO_WORST_SCORE;
    else { s4 = h->score[4] + MPX_OBS(4); t1 = s4 + TP(4, 5); }
    if (ssid[3] == PSO_BAD_SSID) s3 = t2 = PSO_WORST_SCORE;
    else { s3 = h->score[3] + MPX_OBS(3); t2 = s3 + TP(3, 5); }
    if (t1 > t2) { s5 = t1; h->out_history = h->history[4]; }
    else { s5 = t2; h->out_history = h->history[3]; }
    FLOOR(s5);
    h->out_score = s5;
    best = s5;

    if (ssid[2] == PSO_BAD_SSID) s2 = t2 = PSO_WORST_SCORE;
    else { s2 = h->score[2] + MPX_OBS(2); t2 = s2 + TP(2, 4); }
    t0 = t1 = PSO_WORST_SCORE;
    if (s4 != PSO_WORST_SCORE) t0 = s4 + TP(4, 4);
    if (s3 != PSO_WORST_SCORE) t1 = s3 + TP(3, 4);
    w = pick3(t0, t1, t2, &s4);
    if (w == 2) { h->history[4] = h->history[2]; ssid[4] = ssid[2]; }
    else if (w == 1) { h->history[4] = h->history[3]; ssid[4] = ssid[3]; }
    FLOOR(s4); RAISE(best, s4);
    h->score[4] = s4;

    if (ssid[1] == PSO_BAD_SSID) s1 = t2 = PSO_WORST_SCORE;
    else { s1 = h->score[1] + MPX_OBS(1); t2 = s1 + TP(1, 3); }
    t0 = t1 = PSO_WORST_SCORE;
    if (s3 != PSO_WORST_SCORE) t0 = s3 + TP(3, 3);
    if (s2 != PSO_WORST_SCORE) t1 = s2 + TP(2, 3);
    w = pick3(t0, t1, t2, &s3);
    if (w == 2) { h->history[3] = h->history[1]; ssid[3] = ssid[1]; }
    else if (w == 1) { h->history[3] = h->history[2]; ssid[3] = ssid[2]; }
    FLOOR(s3); RAISE(best, s3);
    h->score[3] = s3;

    s0 = h->score[0] + MPX_OBS(0);
    t0 = t1 = PSO_WORST_SCORE;
    if (s2 != PSO_WORST_SCORE) t0 = s2 + TP(2, 2);
    if (s1 != PSO_WORST_SCORE) t1 = s1 + TP(1, 2);
    t2 = s0 + TP(0, 2);
    w = pick3(t0, t1, t2, &s2);
    if (w == 2) { h->history[2] = h->history[0]; ssid[2] = ssid[0]; }
    else if (w == 1) { h->history[2] = h->history[1]; ssid[2] = ssid[1]; }
    FLOOR(s2); RAISE(best, s2);
    h->score[2] = s2;

    t0 = PSO_WORST_SCORE;
    if (s1 != PSO_WORST_SCORE) t0 = s1 + TP(1, 1);
    t1 = s0 + TP(0, 1);
    if (t0 > t1) s1 = t0;
    else { s1 = t1; h->history[1] = h->history[0]; ssid[1] = ssid[0]; }
    FLOOR(s1); RAISE(best, s1);
    h->score[1] = s1;

    s0 += TP(0, 0);
    FLOOR(s0); RAISE(best, s0);
    h->score[0] = s0;
    h->bestscore = best;
    return best;
#undef TP
}

static int32_t
vit_3st_mpx(const pso_hmmctx_t *c, pso_hmm_t *h)
{
    const uint8_t *tp = c->tp + (size_t)h->tmatid * 12;
    const int16_t *sen = c->senscore;
    uint16_t *ssid = h->senid;
#define TP(i, j) (-(int32_t)tp[(i) * 4 + (j)])
    int32_t s0, s1, s2, s3, t0, t1, t2, best;
    int w;

    t2 = INT32_MIN;
    if (ssid[2] == PSO_BAD_SSID) s2 = t1 = PSO_WORST_SCORE;
    else { s2 = h->score[2] + MPX_OBS(2); t1 = s2 + TP(2, 3); }
    if (ssid[1] == PSO_BAD_SSID) s1 = t2 = PSO_WORST_SCORE;
    else {
        s1 = h->score[1] + MPX_OBS(1);
        if (TP(1, 3) > PSO_TMAT_WORST_SCORE) t2 = s1 + TP(1, 3);
    }
    if (t1 > t2) { s3 = t1; h->out_history = h->history[2]; }
    else { s3 = t2; h->out_history = h->history[1]; }
    FLOOR(s3);
    h->out_score = s3;
    best = s3;

    s0 = h->score[0] + MPX_OBS(0);
    t0 = t1 = PSO_WORST_SCORE;
    if (s2 != PSO_WORST_SCORE) t0 = s2 + TP(2, 2);
    if (s1 != PSO_WORST_SCORE) t1 = s1 + TP(1, 2);
    if (TP(0, 2) > PSO_TMAT_WORST_SCORE) t2 = s0 + TP(0, 2);
    w = pick3(t0, t1, t2, &s2);
    if (w == 2) { h->history[2] = h->history[0]; ssid[2] = ssid[0]; }
    else if (w == 1) { h->history[2] = h->history[1]; ssid[2] = ssid[1]; }
    FLOOR(s2); RAISE(best, s2);
    h->score[2] = s2;

    t0 = PSO_WORST_SCORE;
    if (s1 != PSO_WORST_SCORE) t0 = s1 + TP(1, 1);
    t1 = s0 + TP(0, 1);
    if (t0 > t1) s1 = t0;
    else { s1 = t1; h->history[1] = h->history[0]; ssid[1] = ssid[0]; }
    FLOOR(s1); RAISE(best, s1);
    h->score[1] = s1;

    s0 += TP(0, 0);
    FLOOR(s0); RAISE(best, s0);
    h->score[0] = s0;
    h->bestscore = best;
    return best;
#undef TP
}

/* hmm_vit_eval_anytopo (hmm.c:709-784), any n_emit_state <= 5, mpx or not. */
static int32_t
vit_any(const pso_hmmctx_t *c, pso_hmm_t *h)
{
    int n = h->n_emit_state, to, from, bestfrom;
    const uint8_t *tp = c->tp + (size_t)h->tmatid * n * (n + 1);
    int32_t st[PSO_MAX_NSTATE], scr, nscr, best;
#define TP(i, j) (-(int32_t)tp[(i) * (n + 1) + (j)])

    for (from = 0; from < n; ++from) {
        /* hmm_senscr (hmm.h:207-209) with hmm_senid (hmm.h:199-205) */
        uint16_t sid;
        int32_t o;
        if (h->mpx)
            sid = h->senid[from] == PSO_BAD_SSID ? PSO_BAD_SSID
                : c->sseq[(size_t)h->senid[from] * c->n_emit_state + from];
        else
            sid = h->senid[from];
        o = sid == PSO_BAD_SSID ? PSO_WORST_SCORE : -(int32_t)c->senscore[sid];
        st[from] = h->score[from] + o;
        if (from > 0 && st[from] < PSO_WORST_SCORE) st[from] = PSO_WORST_SCORE;
    }
    to = n;
    scr = PSO_WORST_SCORE;
    bestfrom = -1;
    for (from = to - 1; from >= 0; --from)
        if (TP(from, to) > PSO_TMAT_WORST_SCORE && (nscr = st[from] + TP(from, to)) > scr) {
            scr = nscr;
            bestfrom = from;
        }
    h->out_score = scr;
    if (bestfrom >= 0) h->out_history = h->history[bestfrom];
    best = scr;
    for (to = n - 1; to >= 0; --to) {
        scr = TP(to, to) > PSO_TMAT_WORST_SCORE ? st[to] + TP(to, to) : PSO_WORST_SCORE;
        bestfrom = -1;
        for (from = to - 1; from >= 0; --from)
            if (TP(from, to) > PSO_TMAT_WORST_SCORE && (nscr = st[from] + TP(from, to)) > scr) {
                scr = nscr;
                bestfrom = from;
            }
        h->score[to] = scr;
        if (bestfrom >= 0) {
            h->history[to] = h->history[bestfrom];
            if (h->mpx) h->senid[to] = h->senid[bestfrom];
        }
        if (best < scr) best = scr;
    }
    h->bestscore = best;
    return best;
#undef TP
}

int32_t
pso_hmm_vit_eval(const pso_hmmctx_t *c, pso_hmm_t *h)      /* dispatcher: hmm.c:786-805 */
{
    if (h->mpx) {
        if (h->n_emit_state == 5) return vit_5st_mpx(c, h);
        if (h->n_emit_state == 3) return vit_3st_mpx(c, h);
        return vit_any(c, h);
    }
    if (h->n_emit_state == 5) return vit_5st(c, h);
    if (h->n_emit_state == 3) return vit_3st(c, h);
    return vit_any(c, h);
}

int32_t
pso_hmm_vit_eval_batch(const pso_hmmctx_t *c, pso_hmm_t *h, int32_t n)
{
    int32_t best = PSO_WORST_SCORE, i;
    for (i = 0; i < n; ++i) {
        int32_t s = pso_hmm_vit_eval(c, &h[i]);
        if (s > best) best = s;
    }
    return best;
}

/* ------------------------------------------------------------------------------------ */
/* phone loop (phone_loop_search.c)                                                      */

pso_phoneloop_t *
pso_phoneloop_new(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq,
                  int32_t n_phones, const int32_t *ssid, const int32_t *tmatid,
                  int32_t window, int32_t beam, int32_t pbeam, int32_t pip, double penalty_weight)
{
    pso_phoneloop_t *p = calloc(1, sizeof(*p));
    int i;
    p->ctx.n_emit_state = n_emit_state;
    p->ctx.tp = tp;
    p->ctx.sseq = sseq;
    p->n_phones = n_phones;
    p->window = window;
    p->beam = beam; p->pbeam = pbeam; p->pip = pip;
    p->penalty_weight = penalty_weight;
    p->hmms = calloc(n_phones, sizeof(*p->hmms));
    p->pen_buf = calloc((size_t)window * n_phones, sizeof(int32_t));
    p->penalties = calloc(n_phones, sizeof(int32_t));
    for (i = 0; i < n_phones; ++i)                    /* :98-103 */
        pso_hmm_init(&p->ctx, &p->hmms[i], 0, ssid[i], tmatid[i]);
    return p;
}

void
pso_phoneloop_free(pso_phoneloop_t *p)
{
    if (!p) return;
    free(p->hmms); free(p->pen_buf); free(p->penalties); free(p);
}

void
pso_phoneloop_start(pso_phoneloop_t *p)               /* :155-175 */
{
    int i;
    for (i = 0; i < p->n_phones; ++i) {
        pso_hmm_clear(&p->hmms[i]);
        pso_hmm_enter(&p->hmms[i], 0, -1, 0);
    }
    memset(p->penalties, 0, p->n_phones * sizeof(int32_t));
    memset(p->pen_buf, 0, (size_t)p->window * p->n_phones * sizeof(int32_t));
    p->best_score = 0;
    p->pen_buf_ptr = 0;
    p->n_renorm = 0;
}

void
pso_phoneloop_step(pso_phoneloop_t *p, const int16_t *senscr, int32_t frame_idx)   /* :301-337 */
{
    int32_t bs = PSO_WORST_SCORE, thresh, nf = frame_idx + 1;
    int i, j, itr;

    /* renormalize_hmms (:177-191) */
    if (p->best_score + 2 * p->beam < PSO_WORST_SCORE) {
        for (i = 0; i < p->n_phones; ++i)
            pso_hmm_normalize(&p->hmms[i], p->best_score);
        p->n_renorm++;
    }
    /* evaluate_hmms (:193-214) */
    p->ctx.senscore = senscr;
    for (i = 0; i < p->n_phones; ++i) {
        int32_t s;
        if (p->hmms[i].frame < frame_idx) continue;
        s = pso_hmm_vit_eval(&p->ctx, &p->hmms[i]);
        if (s > bs) bs = s;
    }
    p->best_score = bs;
    /* store_scores (:216-239) */
    for (i = 0; i < p->n_phones; ++i)
        p->pen_buf[(size_t)p->pen_buf_ptr * p->n_phones + i] =
            (int32_t)((p->hmms[i].bestscore - p->best_score) * p->penalty_weight);
    p->pen_buf_ptr = (p->pen_buf_ptr + 1) % p->window;
    for (i = 0; i < p->n_phones; ++i) {
        p->penalties[i] = PSO_WORST_SCORE;
        for (j = 0, itr = p->pen_buf_ptr + 1; j < p->window; ++j, ++itr) {
            itr = itr % p->window;
            if (p->pen_buf[(size_t)itr * p->n_phones + i] > p->penalties[i])
                p->penalties[i] = p->pen_buf[(size_t)itr * p->n_phones + i];
        }
    }
    /* prune_hmms (:241-261) */
    thresh = p->best_score + p->beam;
    for (i = 0; i < p->n_phones; ++i) {
        pso_hmm_t *h = &p->hmms[i];
        if (h->frame < frame_idx) continue;
        if (h->bestscore > thresh) h->frame = nf;
        else pso_hmm_clear_scores(h);
    }
    /* phone_transition (:263-299) */
    thresh = p->best_score + p->pbeam;
    for (i = 0; i < p->n_phones; ++i) {
        pso_hmm_t *h = &p->hmms[i];
        int32_t ns;
        if (h->frame != nf) continue;
        ns = h->out_score + p->pip;
        if (ns > thresh)
            for (j = 0; j < p->n_phones; ++j) {
                pso_hmm_t *nh = &p->hmms[j];
                if (nh->frame < frame_idx || ns > nh->score[0])
                    pso_hmm_enter(nh, ns, h->out_history, nf);
            }
    }
}

void
pso_phoneloop_run(pso_phoneloop_t *p, const int16_t *senscr, int32_t n_sen, int32_t T,
                  pso_hmm_t *hmm_out, int32_t *best_out, int32_t *pen_out)
{
    int32_t t;
    pso_phoneloop_start(p);
    for (t = 0; t < T; ++t) {
        pso_phoneloop_step(p, senscr + (size_t)t * n_sen, t);
        if (hmm_out) memcpy(hmm_out + (size_t)t * p->n_phones, p->hmms, p->n_phones * sizeof(pso_hmm_t));
        if (best_out) best_out[t] = p->best_score;
        if (pen_out) memcpy(pen_out + (size_t)t * p->n_phones, p->penalties, p->n_phones * sizeof(int32_t));
    }
}

/* ---------------------------------------------------------------------------------------
 * Forced alignment: state_align_search.c restated (start :43-53, renormalize :55-62,
 * evaluate_hmms :64-86, prune_hmms :88-107, phone_transition :109-136, record_transitions
 * :153-182, step :184-219, finish :221-279).  One utterance; phones given as (ssid, tmatid),
 * constraints sf/ef per phone (NULL = always active: 0 / INT_MAX).  Outputs per emitting state
 * of every phone (state index = phone * n_emit + j): start, duration, score, all -1 where the
 * reference's backtrace never visits the state.  Returns 0, -1 ("Failed to reach final state"),
 * or -2 - frame ("Alignment failed in frame"). */
int32_t
pso_align_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, int32_t n_phones,
              const int32_t *ssid, const int32_t *tmatid, const int32_t *sf, const int32_t *ef,
              const int16_t *senscr, int32_t n_sen, int32_t T,
              int32_t *st_start, int32_t *st_dur, int32_t *st_score)
{
    pso_hmmctx_t ctx;
    pso_hmm_t *hmms = calloc(n_phones, sizeof(*hmms));
    const int32_t n_st = n_phones * n_emit_state;
    int32_t *tok_id = malloc((size_t)(T > 0 ? T : 1) * n_st * sizeof(int32_t));
    int32_t *tok_sc = malloc((size_t)(T > 0 ? T : 1) * n_st * sizeof(int32_t));
    int32_t best_score = 0, frame = 0, rc = 0;
    int i, j, f;

    memset(&ctx, 0, sizeof(ctx));
    ctx.n_emit_state = n_emit_state; ctx.tp = tp; ctx.sseq = sseq;
    for (i = 0; i < n_phones; ++i)
        pso_hmm_init(&ctx, &hmms[i], 0, ssid[i], tmatid[i]);
    for (i = 0; i < n_st; ++i) st_start[i] = st_dur[i] = st_score[i] = -1;
    pso_hmm_enter(&hmms[0], 0, 0, 0);                                    /* start */
    for (f = 0; f < T; ++f) {
        const int nf = f + 1;
        int32_t bs = PSO_WORST_SCORE;
        ctx.senscore = senscr + (size_t)f * n_sen;
        if (best_score - 0x300000 < PSO_WORST_SCORE)                      /* step :199-203 */
            for (i = 0; i < n_phones; ++i) pso_hmm_normalize(&hmms[i], best_score);
        for (i = 0; i < n_phones; ++i) {                                  /* evaluate_hmms */
            int32_t score;
            if (hmms[i].frame < f) continue;
            score = pso_hmm_vit_eval(&ctx, &hmms[i]);
            if (score > bs) bs = score;
        }
        best_score = bs;
        for (i = 0; i < n_phones; ++i) {                                  /* prune_hmms */
            if (hmms[i].frame < f) continue;
            if (nf > (ef ? ef[i] : INT32_MAX)) continue;
            hmms[i].frame = nf;
        }
        for (i = 0; i < n_phones - 1; ++i) {                              /* phone_transition */
            pso_hmm_t *h = &hmms[i], *nh = &hmms[i + 1];
            int32_t newphone_score;
            if (h->frame != nf) continue;
            if (nf < (sf ? sf[i + 1] : 0)) continue;
            newphone_score = h->out_score;
            if (nh->frame < f || newphone_score > nh->score[0])
                pso_hmm_enter(nh, newphone_score, h->out_history, nf);
        }
        for (i = 0; i < n_st; ++i) {                                      /* record_transitions */
            tok_id[(size_t)f * n_st + i] = -1;
            tok_sc[(size_t)f * n_st + i] = -1;
        }
        for (i = 0; i < n_phones; ++i) {
            if (hmms[i].frame < f) continue;
            for (j = 0; j < n_emit_state; ++j) {
                const int s = i * n_emit_state + j;
                tok_id[(size_t)f * n_st + s] = hmms[i].history[j];
                tok_sc[(size_t)f * n_st + s] = hmms[i].score[j];
                hmms[i].history[j] = s;
            }
        }
        frame = f;
    }
    /* finish: backtrace */
    {
        int32_t last_id, last_sc, cur_id, cur_sc, last_frame, cur_frame;
        last_id = cur_id = hmms[n_phones - 1].out_history;
        last_sc = hmms[n_phones - 1].out_score;
        if (last_id == -1 || T == 0) { rc = -1; goto done; }
        last_frame = frame + 1;
        for (cur_frame = frame - 1; cur_frame >= 0; --cur_frame) {
            const int32_t prev = cur_id;
            cur_id = tok_id[(size_t)cur_frame * n_st + prev];
            cur_sc = tok_sc[(size_t)cur_frame * n_st + prev];
            if (cur_id == -1) { rc = -2 - cur_frame; goto done; }
            if (cur_id != last_id) {
                st_start[last_id] = cur_frame + 1;
                st_dur[last_id] = last_frame - st_start[last_id];
                st_score[last_id] = last_sc - cur_sc;
                last_id = cur_id; last_sc = cur_sc;
                last_frame = cur_frame + 1;
            }
        }
        st_start[0] = 0;                              /* "Update alignment entry for initial state" */
        st_dur[0] = last_frame;
        st_score[0] = 0;                              /* the reference leaves the entry's initial 0 */
    }
done:
    free(hmms); free(tok_id); free(tok_sc);
    return rc;
}

/* ---------------------------------------------------------------------------------------
 * Keyword spotting: kws_search.c restated (start :577-597, step :599-628 = hmm_eval :194-229,
 * hmm_prune :234-251, trans :256-348).  One utterance.  Phone loop of n_pl phones, n_kp keyphrases
 * whose HMM chains are concatenated (kp_off).  Every detection the reference would hand to
 * kws_detections_add is appended to hits as (frame, keyphrase, sf, prob, ascr), in its order
 * (frame-major, keyphrases in list order); returns their number (at most cap are stored). */
#define PSO_KWS_MAX 1500
int32_t
pso_kws_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq,
            int32_t n_pl, const int32_t *pl_ssid, const int32_t *pl_tmat,
            int32_t n_kp, const int32_t *kp_off, const int32_t *kp_thresh,
            const int32_t *kp_ssid, const int32_t *kp_tmat, int32_t beam, int32_t plp,
            const int16_t *senscr, int32_t n_sen, int32_t T, int32_t *hits, int32_t cap)
{
    pso_hmmctx_t ctx;
    const int32_t n_k = kp_off[n_kp];
    pso_hmm_t *pl = calloc(n_pl > 0 ? n_pl : 1, sizeof(*pl)), *kh = calloc(n_k > 0 ? n_k : 1, sizeof(*kh));
    int32_t n_hits = 0, frame, i, k;

    memset(&ctx, 0, sizeof(ctx));
    ctx.n_emit_state = n_emit_state; ctx.tp = tp; ctx.sseq = sseq;
    for (i = 0; i < n_pl; ++i) pso_hmm_init(&ctx, &pl[i], 0, pl_ssid[i], pl_tmat[i]);
    for (i = 0; i < n_k; ++i) pso_hmm_init(&ctx, &kh[i], 0, kp_ssid[i], kp_tmat[i]);
    for (i = 0; i < n_pl; ++i) { pso_hmm_clear(&pl[i]); pso_hmm_enter(&pl[i], 0, -1, 0); }   /* start */
    for (frame = 0; frame < T; ++frame) {
        int32_t bestscore = PSO_WORST_SCORE, thresh, best_out = PSO_WORST_SCORE;
        pso_hmm_t *plb = NULL;
        ctx.senscore = senscr + (size_t)frame * n_sen;
        for (i = 0; i < n_pl; ++i) {                                      /* hmm_eval */
            int32_t sc = pso_hmm_vit_eval(&ctx, &pl[i]);
            if (sc > bestscore) bestscore = sc;
        }
        for (i = 0; i < n_k; ++i)
            if (kh[i].frame > 0) {
                int32_t sc = pso_hmm_vit_eval(&ctx, &kh[i]);
                if (sc > bestscore) bestscore = sc;
            }
        thresh = bestscore + beam;                                        /* hmm_prune */
        for (i = 0; i < n_k; ++i)
            if (kh[i].frame > 0 && kh[i].bestscore < thresh) pso_hmm_clear(&kh[i]);
        for (i = 0; i < n_pl; ++i)                                        /* trans */
            if (pl[i].out_score > best_out) { best_out = pl[i].out_score; plb = &pl[i]; }
        if (!plb) continue;
        for (k = 0; k < n_kp; ++k) {
            pso_hmm_t *last;
            if (kp_off[k + 1] - kp_off[k] < 1) continue;
            last = &kh[kp_off[k + 1] - 1];
            if (last->frame > 0 && plb->out_score > PSO_WORST_SCORE
                && last->out_score - plb->out_score >= kp_thresh[k]) {
                if (n_hits < cap) {
                    int32_t *h = hits + (size_t)n_hits * 5;
                    h[0] = frame; h[1] = k; h[2] = last->out_history;
                    h[3] = last->out_score - plb->out_score - PSO_KWS_MAX; h[4] = last->out_score;
                }
                ++n_hits;
            }
        }
        for (i = 0; i < n_pl; ++i)
            if (plb->out_score + plp > pl[i].score[0])
                pso_hmm_enter(&pl[i], plb->out_score + plp, plb->out_history, frame + 1);
        for (k = 0; k < n_kp; ++k) {
            const int32_t o = kp_off[k], n = kp_off[k + 1] - kp_off[k];
            if (n < 1) continue;
            for (i = n - 1; i > 0; --i) {
                pso_hmm_t *pred = &kh[o + i - 1], *h = &kh[o + i];
                if (pred->frame > 0)
                    if (!(h->frame > 0) || pred->out_score > h->score[0])
                        pso_hmm_enter(h, pred->out_score, pred->out_history, frame + 1);
            }
            if (plb->out_score > kh[o].score[0])
                pso_hmm_enter(&kh[o], plb->out_score, frame, frame + 1);
        }
    }
    free(pl); free(kh);
    return n_hits;
}

/* ---------------------------------------------------------------------------------------
 * Phone decoding: allphone_search.c without a phone LM restated (start :640-677, step :700-722 =
 * phmm_eval_all :349-378, phmm_exit :380-456, phmm_trans :458-524).  One utterance.  The graph is
 * n_nodes PHMMs (ssid, tmatid) in the reference's walk order with successor lists in CSR form.
 * Every history entry is returned as a row (ef, node, hist, score); returns their number (at most
 * cap are stored). */
int32_t
pso_allphone_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, int32_t n_nodes,
                 const int32_t *ssid, const int32_t *tmatid, const int32_t *succ_off, const int32_t *succ,
                 int32_t start, int32_t beam, int32_t pbeam, int32_t inspen,
                 const int16_t *senscr, int32_t n_sen, int32_t T, int32_t *hist, int32_t cap)
{
    pso_hmmctx_t ctx;
    pso_hmm_t *h = calloc(n_nodes > 0 ? n_nodes : 1, sizeof(*h));
    int32_t n_hist = 0, frame, i, l;
    /* history scores are needed by phmm_trans even past cap: keep a private copy */
    int32_t hcap = 1024, *hscore = malloc(hcap * sizeof(int32_t)), *hnode = malloc(hcap * sizeof(int32_t));

    memset(&ctx, 0, sizeof(ctx));
    ctx.n_emit_state = n_emit_state; ctx.tp = tp; ctx.sseq = sseq;
    for (i = 0; i < n_nodes; ++i) { pso_hmm_init(&ctx, &h[i], 0, ssid[i], tmatid[i]); pso_hmm_clear(&h[i]); }
    pso_hmm_enter(&h[start], 0, 0, 0);
    for (frame = 0; frame < T; ++frame) {
        const int32_t nf = frame + 1, first = n_hist;
        int32_t best = PSO_WORST_SCORE, th, k;
        ctx.senscore = senscr + (size_t)frame * n_sen;
        for (i = 0; i < n_nodes; ++i)                                    /* phmm_eval_all */
            if (h[i].frame == frame) {
                int32_t sc = pso_hmm_vit_eval(&ctx, &h[i]);
                if (sc > best) best = sc;
            }
        th = best + pbeam;                                               /* phmm_exit */
        for (i = 0; i < n_nodes; ++i)
            if (h[i].frame == frame) {
                if (h[i].bestscore >= th) {
                    if (n_hist == hcap) {
                        hcap *= 2;
                        hscore = realloc(hscore, hcap * sizeof(int32_t));
                        hnode = realloc(hnode, hcap * sizeof(int32_t));
                    }
                    hscore[n_hist] = h[i].out_score; hnode[n_hist] = i;
                    if (n_hist < cap) {
                        int32_t *r = hist + (size_t)n_hist * 4;
                        r[0] = frame; r[1] = i; r[2] = h[i].out_history; r[3] = h[i].out_score;
                    }
                    ++n_hist;
                    h[i].frame = nf;
                }
                else pso_hmm_clear(&h[i]);
            }
        for (k = first; k < n_hist; ++k) {                               /* phmm_trans */
            const int32_t from = hnode[k];
            for (l = succ_off[from]; l < succ_off[from + 1]; ++l) {
                pso_hmm_t *to = &h[succ[l]];
                const int32_t newscore = hscore[k] + inspen;
                if (newscore > best + beam && newscore > to->score[0])
                    pso_hmm_enter(to, newscore, k, nf);
            }
        }
    }
    free(h); free(hscore); free(hnode);
    return n_hist;
}

/* ---------------------------------------------------------------------------------------
 * DESIGN EXPERIMENT (not a restatement of the reference): does a codeword filter that is looser
 * than the scan's own running threshold change the final PTM top-N list?  For every frame and
 * (codebook, stream) the exact list is computed as usual (rescore_topn + scan_cb_ptm).  Next to
 * it, the same seeds are re-scored and only the codewords with  d >= F  are scanned, in order and
 * with the exact tests, where F = (worst re-scored score of a DIFFERENT, stale set of four
 * codewords: the exact list of `lag` frames ago, or codewords 0..3) - 1.  F is a lower bound of
 * the final worst score but, unlike the scan's threshold, it can lie ABOVE the threshold the
 * reference applies early in the scan, so codewords the reference inserts transiently are skipped.
 * stats: [0] lists compared, [1] lists that differ, [2] codewords skipped by the filter that the
 * exact scan inserted (transients), [3] scanned candidates, [4] all codewords. */
int32_t
pso_filter_experiment(const pso_model_t *m, const float *feats, int32_t T, int32_t lag, int64_t *stats)
{
    const int K = m->n_mgau * m->n_feat, n = m->topn;
    pso_topn_t *cur = calloc((size_t)K * n, sizeof(*cur));
    pso_topn_t *ring = calloc((size_t)(lag + 1) * K * n, sizeof(*ring));
    pso_topn_t filt[16], stale[16];
    float *dist = malloc((size_t)m->n_density * sizeof(float));
    int32_t t, cb, f, i, cw, sumlen = 0;

    if (m->kind != PSO_KIND_PTM || n > 16) return -1;
    for (f = 0; f < m->n_feat; ++f) sumlen += m->featlen[f];
    for (i = 0; i < K * n; ++i) { cur[i].cw = i % n; cur[i].score = INT32_MIN; }
    for (i = 0; i < (lag + 1) * K * n; ++i) { ring[i].cw = i % n; ring[i].score = INT32_MIN; }
    memset(stats, 0, 5 * sizeof(*stats));
    for (t = 0; t < T; ++t) {
        const float *z = feats + (size_t)t * sumlen;
        int off = 0;
        for (f = 0; f < m->n_feat; ++f) {
            for (cb = 0; cb < m->n_mgau; ++cb) {
                pso_topn_t *L = cur + ((size_t)cb * m->n_feat + f) * n;
                const pso_topn_t *old = ring + ((size_t)((t + 1) % (lag + 1)) * K + (size_t)cb * m->n_feat + f) * n;
                const int len = m->featlen[f];
                const size_t base = gau_offset(m, cb, f);
                const float *det = m->det + ((size_t)cb * m->n_feat + f) * m->n_density;
                const float *x = z + off;
                int32_t F;
                pso_topn_t before[16];
                memcpy(filt, L, n * sizeof(*L));                 /* same seeds */
                memcpy(before, L, n * sizeof(*L));
                for (cw = 0; cw < m->n_density; ++cw)
                    dist[cw] = gau_full(m->mean + base + (size_t)cw * len, m->var + base + (size_t)cw * len, det[cw], x, len);
                /* exact */
                rescore_topn(m, L, cb, f, x);
                {
                    pso_topn_t seeded[16];
                    memcpy(seeded, L, n * sizeof(*L));
                    scan_cb_ptm(m, L, cb, f, x);
                    /* filter bound from the stale set */
                    memcpy(stale, old, n * sizeof(*old));
                    rescore_topn(m, stale, cb, f, x);
                    F = stale[n - 1].score == INT32_MIN ? INT32_MIN : stale[n - 1].score - 1;
                    /* filtered replay */
                    rescore_topn(m, filt, cb, f, x);
                    for (cw = 0; cw < m->n_density; ++cw) {
                        const float d = dist[cw];
                        ++stats[4];
                        if (d < (float)F) {
                            /* would the exact scan have inserted it at its turn?  (diagnostic) */
                            continue;
                        }
                        ++stats[3];
                        if (d < (float)filt[n - 1].score) continue;
                        if (listed(filt, n, cw)) continue;
                        insert_cw(filt, n, cw, f2i_clamped(d));
                    }
                    (void)seeded; (void)before;
                }
                ++stats[0];
                if (memcmp(filt, L, n * sizeof(*L)) != 0) ++stats[1];
                memcpy(ring + ((size_t)(t % (lag + 1)) * K + (size_t)cb * m->n_feat + f) * n, L, n * sizeof(*L));
            }
            off += m->featlen[f];
        }
    }
    free(cur); free(ring); free(dist);
    return 0;
}

/* allphone_search.c WITH a phone LM (phmm_exit :416-441, phmm_trans :497-513): same search as
 * pso_allphone_run, but every transition carries its own LM score.  bg [n_ci][n_ci] and
 * tg [n_ci][n_ci][n_ci] are the LM scores >> SENSCR_SHIFT tabulated with the reference's argument
 * positions; node_ci maps nodes to CI phones.  History rows get a fifth column, tscore, computed
 * the way phmm_exit does -- including its reading the SAME history entry for "pred" and
 * "pred_pred" (:417-423), so the trigram it scores is (pred, pred, p). */
int32_t
pso_allphone_lm_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, int32_t n_nodes,
                    const int32_t *ssid, const int32_t *tmatid, const int32_t *succ_off, const int32_t *succ,
                    int32_t start, int32_t beam, int32_t pbeam, int32_t n_ci, const int32_t *node_ci,
                    const int32_t *bg, const int32_t *tg,
                    const int16_t *senscr, int32_t n_sen, int32_t T, int32_t *hist, int32_t cap)
{
    pso_hmmctx_t ctx;
    pso_hmm_t *h = calloc(n_nodes > 0 ? n_nodes : 1, sizeof(*h));
    int32_t n_hist = 0, frame, i, l;
    int32_t hcap = 1024;
    int32_t *hscore = malloc(hcap * sizeof(int32_t)), *hnode = malloc(hcap * sizeof(int32_t)), *hhist = malloc(hcap * sizeof(int32_t));

    memset(&ctx, 0, sizeof(ctx));
    ctx.n_emit_state = n_emit_state; ctx.tp = tp; ctx.sseq = sseq;
    for (i = 0; i < n_nodes; ++i) { pso_hmm_init(&ctx, &h[i], 0, ssid[i], tmatid[i]); pso_hmm_clear(&h[i]); }
    pso_hmm_enter(&h[start], 0, 0, 0);
    for (frame = 0; frame < T; ++frame) {
        const int32_t nf = frame + 1, first = n_hist;
        int32_t best = PSO_WORST_SCORE, th, k;
        ctx.senscore = senscr + (size_t)frame * n_sen;
        for (i = 0; i < n_nodes; ++i)
            if (h[i].frame == frame) {
                int32_t sc = pso_hmm_vit_eval(&ctx, &h[i]);
                if (sc > best) best = sc;
            }
        th = best + pbeam;
        for (i = 0; i < n_nodes; ++i)
            if (h[i].frame == frame) {
                if (h[i].bestscore >= th) {
                    int32_t tscore = 0;
                    const int32_t hh = h[i].out_history;
                    if (n_hist == hcap) {
                        hcap *= 2;
                        hscore = realloc(hscore, hcap * sizeof(int32_t));
                        hnode = realloc(hnode, hcap * sizeof(int32_t));
                        hhist = realloc(hhist, hcap * sizeof(int32_t));
                    }
                    if (hh > 0) {
                        const int32_t pc = node_ci[hnode[hh]];
                        if (hhist[hh] > 0) tscore = tg[((size_t)pc * n_ci + pc) * n_ci + node_ci[i]];   /* pred_pred == pred */
                        else tscore = bg[(size_t)pc * n_ci + node_ci[i]];
                    }
                    hscore[n_hist] = h[i].out_score; hnode[n_hist] = i; hhist[n_hist] = hh;
                    if (n_hist < cap) {
                        int32_t *r = hist + (size_t)n_hist * 5;
                        r[0] = frame; r[1] = i; r[2] = hh; r[3] = h[i].out_score; r[4] = tscore;
                    }
                    ++n_hist;
                    h[i].frame = nf;
                }
                else pso_hmm_clear(&h[i]);
            }
        for (k = first; k < n_hist; ++k) {
            const int32_t from = hnode[k], fc = node_ci[from];
            for (l = succ_off[from]; l < succ_off[from + 1]; ++l) {
                pso_hmm_t *to = &h[succ[l]];
                const int32_t tc = node_ci[succ[l]];
                int32_t tscore, newscore;
                if (hhist[k] > 0) tscore = tg[((size_t)node_ci[hnode[hhist[k]]] * n_ci + fc) * n_ci + tc];
                else tscore = bg[(size_t)fc * n_ci + tc];
                newscore = hscore[k] + tscore;
                if (newscore > best + beam && newscore > to->score[0])
                    pso_hmm_enter(to, newscore, k, nf);
            }
        }
    }
    free(h); free(hscore); free(hnode); free(hhist);
    return n_hist;
}

/* ---------------------------------------------------------------------------------------
 * Grammar decoding: fsg_search.c + fsg_history.c restated for one utterance, all senones computed.
 * Inputs are the reference's own lextree flattened by oracle/ref_driver.c:refdrv_fsg
 * (pnodes [n][16] = ssid, tmatid, next, sibling, logs2prob, ci_ext, ppos, leaf, ctxt.bv[8];
 * links [n][5] = from, to, wid, logs2prob, all-right-contexts flag; null arcs per state in
 * fsg_model_arcs order).  Output: the history table rows (link, frame, score, pred, lc, rc.bv[8])
 * in table order; returns their number (at most cap rows are stored).
 *   start       fsg_search.c:770-817      step          :683-761
 *   hmm_eval    :335-407 (incl. the maxhmmpf beam narrowing)
 *   prune_prop  :516-560  pnode_trans :410-441  pnode_exit :444-507
 *   null_prop   :566-614  word_trans  :621-680
 *   history     fsg_history.c:132-213 (entry_add, right-context subtraction), :220-240 (end_frame)
 * The active lists are glists built by PREPENDING (glist_add_ptr); an array filled in order of
 * insertion and walked backwards visits the same sequence. */
typedef struct { int32_t link, frame, score, pred, lc; uint32_t rc[8]; } fsg_hent_t;
typedef struct fsg_fent_s { fsg_hent_t e; struct fsg_fent_s *next; } fsg_fent_t;
typedef struct {
    fsg_hent_t *ent; int32_t n, cap;
    fsg_fent_t **frame_entries;         /* [n_state * n_ci] */
    int32_t n_state, n_ci;
    const int32_t *links;
} fsg_hist_t;

static void
fsg_hist_append(fsg_hist_t *h, const fsg_hent_t *e)
{
    if (h->n == h->cap) { h->cap = h->cap ? h->cap * 2 : 1024; h->ent = realloc(h->ent, h->cap * sizeof(*h->ent)); }
    h->ent[h->n++] = *e;
}

static uint32_t
fsg_ctxt_sub(uint32_t *src, const uint32_t *sub)        /* fsg_lextree.c:333-341 */
{
    uint32_t res = 0; int i;
    for (i = 0; i < 8; ++i) res |= (src[i] = ~sub[i] & src[i]);
    return res;
}

static void
fsg_hist_add(fsg_hist_t *h, int32_t link, int32_t frame, int32_t score, int32_t pred, int32_t lc, const uint32_t *rc_in)
{
    fsg_hent_t ne;
    fsg_fent_t **slot, *gn, *prev = NULL, *nn;
    ne.link = link; ne.frame = frame; ne.score = score; ne.pred = pred; ne.lc = lc;
    memcpy(ne.rc, rc_in, sizeof(ne.rc));
    if (frame < 0) { fsg_hist_append(h, &ne); return; }
    slot = &h->frame_entries[(size_t)h->links[link * 5 + 1] * h->n_ci + lc];
    for (gn = *slot; gn; gn = gn->next) {
        if (score > gn->e.score) break;
        if (fsg_ctxt_sub(ne.rc, gn->e.rc) == 0) return;
        prev = gn;
    }
    nn = malloc(sizeof(*nn));
    nn->e = ne;
    if (!prev) { nn->next = *slot; *slot = nn; }
    else { nn->next = prev->next; prev->next = nn; }
    prev = nn;
    while (gn) {
        if (fsg_ctxt_sub(gn->e.rc, ne.rc) == 0) { prev->next = gn->next; free(gn); gn = prev->next; }
        else { prev = gn; gn = gn->next; }
    }
}

static void
fsg_hist_end_frame(fsg_hist_t *h)
{
    int32_t i;
    for (i = 0; i < h->n_state * h->n_ci; ++i) {
        fsg_fent_t *gn = h->frame_entries[i], *nx;
        for (; gn; gn = nx) { nx = gn->next; fsg_hist_append(h, &gn->e); free(gn); }
        h->frame_entries[i] = NULL;
    }
}

int32_t
pso_fsg_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq,
            int32_t n_pnode, const int32_t *pn, int32_t n_state, const int32_t *roots,
            int32_t n_link, const int32_t *links, const int32_t *nulloff, const int32_t *nullarc,
            int32_t n_ci, int32_t silcipid, int32_t start_state,
            int32_t beam_orig, int32_t pbeam_orig, int32_t wbeam_orig, int32_t maxhmmpf,
            const int16_t *senscr, int32_t n_sen, int32_t T, int32_t *hist_out, int32_t cap)
{
    pso_hmmctx_t ctx;
    pso_hmm_t *hmm = calloc(n_pnode > 0 ? n_pnode : 1, sizeof(*hmm));
    int32_t *act = malloc((size_t)(n_pnode + 1) * sizeof(int32_t)), *nxt = malloc((size_t)(n_pnode + 1) * sizeof(int32_t));
    int32_t n_act = 0, n_nxt = 0, frame, i, k, bestscore, bpidx_start, beam, pbeam, wbeam, pass;
    float beam_factor = 1.0f;
    fsg_hist_t H;
    uint32_t all[8];
    (void)n_link;

    memset(&ctx, 0, sizeof(ctx));
    ctx.n_emit_state = n_emit_state; ctx.tp = tp; ctx.sseq = sseq;
    for (i = 0; i < n_pnode; ++i) { pso_hmm_init(&ctx, &hmm[i], 0, pn[i * 16], pn[i * 16 + 1]); pso_hmm_clear(&hmm[i]); }
    memset(&H, 0, sizeof(H));
    H.n_state = n_state; H.n_ci = n_ci; H.links = links;
    H.frame_entries = calloc((size_t)n_state * n_ci, sizeof(*H.frame_entries));
    memset(all, 0xff, sizeof(all));
    beam = beam_orig; pbeam = pbeam_orig; wbeam = wbeam_orig;

    /* fsg_search_start: dummy entry, then the null/word transitions of the step with frame = -1 */
    frame = -1; bestscore = 0; bpidx_start = 0;
    fsg_hist_add(&H, -1, -1, 0, -1, silcipid, all);
    for (pass = 0;; ++pass) {
        int32_t n_entries, bp, th;
        if (frame >= 0) {
            ctx.senscore = senscr + (size_t)frame * n_sen;
            bpidx_start = H.n;
            /* hmm_eval */
            bestscore = PSO_WORST_SCORE;
            for (k = n_act - 1; k >= 0; --k) {
                int32_t sc = pso_hmm_vit_eval(&ctx, &hmm[act[k]]);
                if (sc > bestscore) bestscore = sc;
            }
            if (maxhmmpf != -1 && n_act > maxhmmpf) {
                if (beam_factor > 0.1) {
                    beam_factor *= 0.9f;
                    beam = (int32_t)(beam_orig * beam_factor);
                    pbeam = (int32_t)(pbeam_orig * beam_factor);
                    wbeam = (int32_t)(wbeam_orig * beam_factor);
                }
            }
            else { beam_factor = 1.0f; beam = beam_orig; pbeam = pbeam_orig; wbeam = wbeam_orig; }
            /* prune_prop */
            {
                const int32_t thresh = bestscore + beam, pth = bestscore + pbeam, wth = bestscore + wbeam, nf = frame + 1;
                for (k = n_act - 1; k >= 0; --k) {
                    const int32_t p = act[k];
                    const int32_t *r = pn + (size_t)p * 16;
                    pso_hmm_t *h = &hmm[p];
                    if (h->bestscore < thresh) continue;
                    if (h->frame == frame) { h->frame = nf; nxt[n_nxt++] = p; }
                    if (!r[7]) {
                        if (h->out_score >= pth) {                              /* pnode_trans */
                            int32_t c;
                            for (c = r[2]; c >= 0; c = pn[(size_t)c * 16 + 3]) {
                                const int32_t ns = h->out_score + pn[(size_t)c * 16 + 4];
                                if (ns > thresh && ns > hmm[c].score[0]) {
                                    if (hmm[c].frame < nf) nxt[n_nxt++] = c;
                                    pso_hmm_enter(&hmm[c], ns, h->out_history, nf);
                                }
                            }
                        }
                    }
                    else if (h->out_score >= wth) {                             /* pnode_exit */
                        const int32_t l = r[2];
                        fsg_hist_add(&H, l, frame, h->out_score, h->out_history, r[5],
                                     links[l * 5 + 4] ? all : (const uint32_t *)(r + 8));
                    }
                }
            }
            fsg_hist_end_frame(&H);
        }
        /* null_prop */
        th = bestscore + wbeam;
        n_entries = H.n;
        for (bp = bpidx_start; bp < n_entries; ++bp) {
            const int32_t s = H.ent[bp].link >= 0 ? links[H.ent[bp].link * 5 + 1] : start_state;
            for (k = nulloff[s]; k < nulloff[s + 1]; ++k) {
                const int32_t l = nullarc[k];
                const int32_t ns = H.ent[bp].score + (links[l * 5 + 3] >> 10);
                if (ns >= th) {
                    fsg_hent_t src = H.ent[bp];          /* by value: the table may be reallocated */
                    fsg_hist_add(&H, l, src.frame, ns, bp, src.lc, src.rc);
                }
            }
        }
        if (frame >= 0) fsg_hist_end_frame(&H);
        /* word_trans */
        n_entries = H.n;
        th = bestscore + beam;
        for (bp = bpidx_start; bp < n_entries; ++bp) {
            const fsg_hent_t *e = &H.ent[bp];
            const int32_t d = e->link >= 0 ? links[e->link * 5 + 1] : start_state, lc = e->lc, nf = frame + 1;
            int32_t root;
            for (root = roots[d]; root >= 0; root = pn[(size_t)root * 16 + 3]) {
                const int32_t *r = pn + (size_t)root * 16;
                const int32_t rc = r[5];
                if ((((const uint32_t *)(r + 8))[lc >> 5] & (1u << (lc & 31))) && (e->rc[rc >> 5] & (1u << (rc & 31)))) {
                    const int32_t ns = e->score + r[4];
                    if (ns > th && ns > hmm[root].score[0]) {
                        if (hmm[root].frame < nf) nxt[n_nxt++] = root;
                        pso_hmm_enter(&hmm[root], ns, bp, nf);
                    }
                }
            }
        }
        /* deactivate what did not survive, swap lists */
        if (frame >= 0)
            for (k = n_act - 1; k >= 0; --k)
                if (hmm[act[k]].frame == frame) pso_hmm_clear(&hmm[act[k]]);
        { int32_t *t = act; act = nxt; nxt = t; n_act = n_nxt; n_nxt = 0; }
        ++frame;
        if (frame >= T) break;
    }
    for (i = 0; i < H.n && i < cap; ++i) {
        int32_t *r = hist_out + (size_t)i * 13;
        r[0] = H.ent[i].link; r[1] = H.ent[i].frame; r[2] = H.ent[i].score; r[3] = H.ent[i].pred; r[4] = H.ent[i].lc;
        memcpy(r + 5, H.ent[i].rc, 32);
    }
    i = H.n;
    free(H.ent); free(H.frame_entries); free(hmm); free(act); free(nxt);
    return i;
}

/* ---------------------------------------------------------------------------------------
 * Trigram score from the LM as sorted arrays (integration/ps_search_cuda.c:cuda_ngram_export_lm):
 * ngram_tg_score(lmset, w, h1, h2) >> SENSCR_SHIFT restated -- ngram_model_set_score
 * (ngram_model_set.c:685-732, one model) -> ngram_ng_score (ngram_model.c:388-417) ->
 * ngram_model_trie_score (ngram_model_trie.c:716-742: history cut at the first missing word, float
 * score truncated to int32, then weight_score = (int32)(score * lw + log_wip)) -> lm_trie_score
 * (lm_trie.c:653-825: full history = cached backoffs + lm_trie_hist_score, shorter =
 * lm_trie_nobo_score).  w, h1, h2 are DICTIONARY word ids (h = -1: none). */
typedef struct {
    int32_t order, V, n2, n3, log_wip, log_zero, n_words, max_vocab2, max_vocab3;
    float lw;
    const int32_t *widmap, *uni_next, *bg_word, *bg_next, *tg_word;
    const float *uni_prob, *uni_bo, *bg_prob, *bg_bo, *tg_prob;
} lmarr_t;

static void
lmarr_bind(lmarr_t *L, const int32_t *a)
{
    L->order = a[0]; L->V = a[1]; L->n2 = a[2]; L->n3 = a[3]; memcpy(&L->lw, &a[4], 4);
    L->log_wip = a[5]; L->log_zero = a[6]; L->n_words = a[7]; L->max_vocab2 = a[8]; L->max_vocab3 = a[9];
    a += 10;
    L->widmap = a; a += L->n_words;
    L->uni_prob = (const float *)a; a += L->V;  L->uni_bo = (const float *)a; a += L->V;  L->uni_next = a; a += L->V + 1;
    L->bg_word = a; a += L->n2;  L->bg_prob = (const float *)a; a += L->n2;  L->bg_bo = (const float *)a; a += L->n2;
    L->bg_next = a; a += L->n2 + 1;  L->tg_word = a; a += L->n3;  L->tg_prob = (const float *)a;
}

/* uniform_find (lm_trie.c:556-592) as it stands: interpolation search between (begin - 1, value 0) and
 * (end, value max_vocab) in uint32 arithmetic.  On a sorted range it finds exactly the entries that
 * exist; shipped models contain ranges that are not sorted, where what it finds is a property of this
 * very procedure -- so no other search will do. */
static int32_t
lmarr_find(const int32_t *words, int32_t begin, int32_t end, int32_t key_, uint32_t max_vocab)
{
    uint32_t before_it = (uint32_t)begin - 1u, before_v = 0, after_it = (uint32_t)end, after_v = max_vocab, key = (uint32_t)key_;
    if (key > after_v) return -1;
    while (after_it - before_it > 1) {
        const uint32_t off = key - before_v, range = after_v - before_v, width = after_it - before_it - 1;
        const uint32_t pivot = before_it + (1u + (uint32_t)(size_t)((uint32_t)(off * width) / (range + 1)));
        const uint32_t mid = (uint32_t)words[pivot];
        if (mid < key) { before_it = pivot; before_v = mid; }
        else if (mid > key) { after_it = pivot; after_v = mid; }
        else return (int32_t)pivot;
    }
    return -1;
}

static int32_t
lmarr_tg(const lmarr_t *L, int32_t w_dict, int32_t h1_dict, int32_t h2_dict)
{
    const int32_t w = w_dict < 0 ? -1 : L->widmap[w_dict];
    int32_t hist[2], n_hist = 2, i, raw;
    float score;
    hist[0] = h1_dict < 0 ? -1 : L->widmap[h1_dict];
    hist[1] = h2_dict < 0 ? -1 : L->widmap[h2_dict];
    if (w < 0) return L->log_zero;                                          /* ngram_ng_score: OOV */
    if (n_hist > L->order - 1) n_hist = L->order - 1;
    for (i = 0; i < n_hist; ++i) if (hist[i] < 0) { n_hist = i; break; }
    score = L->uni_prob[w];
    if (n_hist > 0) {
        /* bigram (w | h1) */
        const int32_t b = (w < L->V) ? lmarr_find(L->bg_word, L->uni_next[w], L->uni_next[w + 1], hist[0], L->max_vocab2) : -1;
        if (n_hist == L->order - 1 && L->order == 3) {                      /* lm_trie_hist_score with update_backoff's cache */
            float bc0 = L->uni_bo[hist[0]], bc1 = 0.0f;
            const int32_t hb = lmarr_find(L->bg_word, L->uni_next[hist[0]], L->uni_next[hist[0] + 1], hist[1], L->max_vocab2);
            if (hb >= 0) bc1 = L->bg_bo[hb];
            if (b < 0) { score += bc0; score += bc1; }
            else {
                const int32_t t = lmarr_find(L->tg_word, L->bg_next[b], L->bg_next[b + 1], hist[1], L->max_vocab3);
                score = L->bg_prob[b];
                if (t < 0) score = score + bc1;
                else score = L->tg_prob[t];
            }
        }
        else if (n_hist == L->order - 1 && L->order == 2) {                 /* bigram LM: longest_find directly */
            if (b < 0) score = score + L->uni_bo[hist[0]];
            else score = L->bg_prob[b];
        }
        else {                                                              /* lm_trie_nobo_score, one history word of a trigram LM */
            if (b >= 0) score = L->bg_prob[b];
            else score = score + (0.0f + L->uni_bo[hist[0]]);
        }
    }
    raw = (int32_t)score;
    return (int32_t)(raw * L->lw + L->log_wip);
}

/* scores[i] = tg(q[i][0] | q[i][1], q[i][2]) >> SENSCR_SHIFT for n_q queries */
void
pso_lm_scores(const int32_t *lmarr, const int32_t *q, int64_t n_q, int32_t *scores)
{
    lmarr_t L;
    int64_t i;
    lmarr_bind(&L, lmarr);
    for (i = 0; i < n_q; ++i) scores[i] = lmarr_tg(&L, q[i * 3], q[i * 3 + 1], q[i * 3 + 2]) >> 10;
}

/* ---------------------------------------------------------------------------------------
 * N-gram lextree decoding, first pass: ngram_search_fwdtree.c (search step :1454-1496 =
 * evaluate_channels :702, prune_channels :1130 [prune_root_chan :723, prune_nonroot_chan :800,
 * last_phone_transition :885, prune_word_chan :1042], bptable_maxwpf :1188, word_transition :1241,
 * deactivate_channels :1432; start :470) with the backpointer-table side of ngram_search.c
 * (mark_bptable :324, set_real_wid :343, save_bp :378, alloc_all_rc :593, exit_score :655) restated
 * for one utterance, all senones computed; pen [T][n_ci] = the phone-loop look-ahead penalties in
 * force while frame t is searched (pls->penalties, NULL without look-ahead).  `info` and
 * `model` are what oracle/ref_driver.c:refdrv_fwdtree exports (the reference's own lextree,
 * dictionary / dict2pid tables, dense trigram table, parameters).  Output: the backpointer table
 * rows (frame, valid, wid, bp, score, s_idx, real_wid, prev_real_wid, last_phone, last2_phone), the
 * right-context score stack and bp_table_idx; returns the number of entries, *bss_out the stack size. */
typedef struct { int32_t frame, valid, wid, bp, score, s_idx, real_wid, prev_real_wid, last_phone, last2_phone; } ft_bp_t;
typedef struct { int32_t wid, score, bp, next; } ft_cand_t;
typedef struct {
    /* model */
    int32_t n_words, n_root, n_nonroot, n_1ph, n_1ph_lm, n_ci, sil, n_lm;
    int32_t beam, pbeam, wbeam, lpbeam, lponlybeam, maxhmmpf, maxwpf, nwpen, pip, silpen, fillpen;
    int32_t start_wid, finish_wid, silence_wid, filler_start, filler_end;
    const int32_t *roots, *nonroot, *words, *w1ph, *r1ph, *rs_n, *rs_ssid, *rs_cimap, *ldiph, *lm, *ci_tmat;
    const int32_t *inlm, *pron_off, *pron_ci, *pron_ssid;
    const lmarr_t *lma;               /* NULL: dense table */
    int32_t fwdflatbeam, fwdflatwbeam, min_ef_width, max_sf_win;
    float lwf;
    pso_hmmctx_t ctx;
    /* channels */
    pso_hmm_t *rh, *nh, *h1;          /* root, non-root, single-phone words */
    pso_hmm_t **wc;                   /* [n_words] right-context fan-out of multi-phone words, by rc id */
    uint8_t **wc_alloc;
    int32_t *w2h1;                    /* word -> index of its permanent channel, or -1 */
    /* search state */
    int32_t *acl[2], n_acl[2], *awl[2], n_awl[2];
    uint8_t *word_active;
    int32_t *word_lat_idx, *lt_sf, *lt_dscr, *lt_bp;
    ft_cand_t *cand; int32_t n_cand;
    int32_t *csf_ef, *csf_cand;
    int32_t *brc_score, *brc_path, *brc_lc;
    ft_bp_t *bp; int32_t bpidx, bp_cap;
    int32_t *bss; int32_t bss_head, bss_cap;
    int32_t *bp_idx;
    int32_t best_score, last_phone_best_score, dynamic_beam;
    int64_t n_root_eval, n_nonroot_eval;
} ft_t;

#define FT_W(s, w, k) ((s)->words[(size_t)(w) * 8 + (k)])        /* 0 first 1 last 2 last2 3 single 4 filler 5 base 6 homophone 7 lmidx */

static int32_t
ft_nrc(const ft_t *s, int32_t w) { return s->rs_n[(size_t)FT_W(s, w, 1) * s->n_ci + FT_W(s, w, 2)]; }

static int32_t
ft_tg(const ft_t *s, int32_t w, int32_t h1, int32_t h2)
{
    const int32_t n = s->n_lm + 1;
    if (s->lma) return lmarr_tg(s->lma, w, h1, h2) >> 10;
    const int32_t a = FT_W(s, w, 7), b = h1 < 0 ? 0 : FT_W(s, h1, 7) + 1, c = h2 < 0 ? 0 : FT_W(s, h2, 7) + 1;
    return s->lm[((size_t)a * n + b) * n + c];
}

static int32_t
ft_exit_score(const ft_t *s, const ft_bp_t *e, int32_t rcphone)           /* ngram_search.c:655-676 */
{
    if (e->last2_phone == -1) return e->score;
    return s->bss[e->s_idx + s->rs_cimap[((size_t)e->last_phone * s->n_ci + e->last2_phone) * s->n_ci + rcphone]];
}

static void
ft_set_real_wid(ft_t *s, int32_t bp)                                      /* :343-373 */
{
    ft_bp_t *e = &s->bp[bp], *prev = e->bp == -1 ? NULL : &s->bp[e->bp];
    if (FT_W(s, e->wid, 4)) {
        if (prev) { e->real_wid = prev->real_wid; e->prev_real_wid = prev->prev_real_wid; }
        else { e->real_wid = FT_W(s, e->wid, 5); e->prev_real_wid = -1; }
    }
    else {
        e->real_wid = FT_W(s, e->wid, 5);
        e->prev_real_wid = prev ? prev->real_wid : -1;
    }
}

static void
ft_save_bp(ft_t *s, int32_t frame, int32_t w, int32_t score, int32_t path, int32_t rc)   /* :378-497 */
{
    int32_t bp = s->word_lat_idx[w];
    if (bp != -1) {
        ft_bp_t *e = &s->bp[bp];
        if (e->score < score) {
            if (e->bp != path) {
                int32_t a0 = e->bp == -1 ? -1 : s->bp[e->bp].prev_real_wid, a1 = e->bp == -1 ? -1 : s->bp[e->bp].real_wid;
                int32_t b0 = path == -1 ? -1 : s->bp[path].prev_real_wid, b1 = path == -1 ? -1 : s->bp[path].real_wid;
                if (a0 != b0 || a1 != b1) ft_set_real_wid(s, bp);          /* (still on the old path: :436-438) */
                e->bp = path;
            }
            e->score = score;
        }
        if (e->s_idx != -1) s->bss[e->s_idx + rc] = score;
    }
    else {
        ft_bp_t *e;
        int32_t i, rcsize;
        if (s->bpidx >= s->bp_cap) { s->bp_cap *= 2; s->bp = realloc(s->bp, (size_t)s->bp_cap * sizeof(*s->bp)); }
        if (s->bss_head >= s->bss_cap - s->n_ci) { s->bss_cap *= 2; s->bss = realloc(s->bss, (size_t)s->bss_cap * sizeof(*s->bss)); }
        s->word_lat_idx[w] = s->bpidx;
        e = &s->bp[s->bpidx];
        e->wid = w; e->frame = frame; e->bp = path; e->score = score; e->s_idx = s->bss_head; e->valid = 1;
        e->last_phone = FT_W(s, w, 1);
        if (FT_W(s, w, 3)) { e->last2_phone = -1; e->s_idx = -1; rcsize = 0; }
        else { e->last2_phone = FT_W(s, w, 2); rcsize = ft_nrc(s, w); }
        for (i = 0; i < rcsize; ++i) s->bss[s->bss_head + i] = PSO_WORST_SCORE;
        if (rcsize) s->bss[s->bss_head + rc] = score;
        ft_set_real_wid(s, s->bpidx);
        s->bpidx++;
        s->bss_head += rcsize;
    }
}

static void
ft_alloc_all_rc(ft_t *s, int32_t w)                                        /* :593-639 */
{
    const int32_t n = ft_nrc(s, w), last = FT_W(s, w, 1), last2 = FT_W(s, w, 2);
    int32_t i;
    if (!s->wc[w]) { s->wc[w] = calloc(n > 0 ? n : 1, sizeof(pso_hmm_t)); s->wc_alloc[w] = calloc(n > 0 ? n : 1, 1); }
    for (i = 0; i < n; ++i)
        if (!s->wc_alloc[w][i]) {
            pso_hmm_init(&s->ctx, &s->wc[w][i], 0, s->rs_ssid[((size_t)last * s->n_ci + last2) * s->n_ci + i], s->ci_tmat[last]);
            s->wc_alloc[w][i] = 1;
        }
}

static void
ft_setup(ft_t *s, int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, const int32_t *ci_tmat,
         const int32_t *info, const int32_t *model, int32_t T)
{
    const int32_t *m = model;
    int32_t i, w;
    memset(s, 0, sizeof(*s));
    s->n_words = info[1]; s->n_root = info[2]; s->n_nonroot = info[3]; s->n_1ph = info[4]; s->n_1ph_lm = info[5];
    s->n_ci = info[6]; s->sil = info[7]; s->beam = info[8]; s->pbeam = info[9]; s->wbeam = info[10]; s->lpbeam = info[11];
    s->lponlybeam = info[12]; s->maxhmmpf = info[13]; s->maxwpf = info[14]; s->nwpen = info[15]; s->pip = info[16];
    s->silpen = info[17]; s->fillpen = info[18]; s->start_wid = info[19]; s->finish_wid = info[20]; s->silence_wid = info[21];
    s->filler_start = info[22]; s->filler_end = info[23]; s->n_lm = info[26];
    {
        const size_t nc = (size_t)s->n_ci;
        s->roots = m; m += (size_t)s->n_root * 5;  s->nonroot = m; m += (size_t)s->n_nonroot * 6;
        s->words = m; m += (size_t)s->n_words * 8;  s->w1ph = m; m += s->n_1ph;  s->r1ph = m; m += (size_t)s->n_1ph * 4;
        s->rs_n = m; m += nc * nc;  s->rs_ssid = m; m += nc * nc * nc;  s->rs_cimap = m; m += nc * nc * nc;
        s->ldiph = m; m += nc * nc * nc;  s->lm = m;
    }
    s->ctx.n_emit_state = n_emit_state; s->ctx.tp = tp; s->ctx.sseq = sseq; s->ci_tmat = ci_tmat;
    s->rh = calloc(s->n_root + 1, sizeof(pso_hmm_t)); s->nh = calloc(s->n_nonroot + 1, sizeof(pso_hmm_t));
    s->h1 = calloc(s->n_1ph + 1, sizeof(pso_hmm_t));
    s->wc = calloc(s->n_words, sizeof(*s->wc)); s->wc_alloc = calloc(s->n_words, sizeof(*s->wc_alloc));
    s->w2h1 = malloc(s->n_words * sizeof(int32_t));
    for (w = 0; w < s->n_words; ++w) s->w2h1[w] = -1;
    for (i = 0; i < s->n_root; ++i) pso_hmm_init(&s->ctx, &s->rh[i], 1, 0, s->roots[i * 5 + 4]);
    for (i = 0; i < s->n_nonroot; ++i) pso_hmm_init(&s->ctx, &s->nh[i], 0, s->nonroot[i * 6], s->nonroot[i * 6 + 1]);
    for (i = 0; i < s->n_1ph; ++i) {
        pso_hmm_init(&s->ctx, &s->h1[i], 1, s->r1ph[i * 4 + 2], s->r1ph[i * 4 + 3]);
        s->w2h1[s->w1ph[i]] = i;
    }
    for (i = 0; i < 2; ++i) { s->acl[i] = malloc((s->n_nonroot + 1) * sizeof(int32_t)); s->awl[i] = malloc((s->n_words + 1) * sizeof(int32_t)); }
    s->word_active = calloc(s->n_words, 1);
    s->word_lat_idx = malloc(s->n_words * sizeof(int32_t)); s->lt_sf = malloc(s->n_words * sizeof(int32_t));
    s->lt_dscr = calloc(s->n_words, sizeof(int32_t)); s->lt_bp = calloc(s->n_words, sizeof(int32_t));
    s->cand = malloc((s->n_words + 1) * sizeof(ft_cand_t));
    s->csf_ef = malloc((s->n_words + 1) * sizeof(int32_t)); s->csf_cand = malloc((s->n_words + 1) * sizeof(int32_t));
    s->brc_score = malloc(s->n_ci * sizeof(int32_t)); s->brc_path = calloc(s->n_ci, sizeof(int32_t)); s->brc_lc = calloc(s->n_ci, sizeof(int32_t));
    s->bp_cap = 2048; s->bp = malloc((size_t)s->bp_cap * sizeof(*s->bp));
    s->bss_cap = 16384 + 2 * s->n_ci; s->bss = malloc((size_t)s->bss_cap * sizeof(*s->bss));
    s->bp_idx = malloc(((size_t)T + 2) * sizeof(int32_t));
    s->inlm = m + (size_t)s->n_lm * (s->n_lm + 1) * (s->n_lm + 1);
    s->pron_off = s->inlm + s->n_words;
    s->pron_ci = s->pron_off + s->n_words + 1;
    s->pron_ssid = s->pron_ci + info[33];
    s->fwdflatbeam = info[28]; s->fwdflatwbeam = info[29]; s->min_ef_width = info[30]; s->max_sf_win = info[31];
    memcpy(&s->lwf, &info[32], 4);
}

static void
ft_free(ft_t *s)
{
    int32_t w;
    for (w = 0; w < s->n_words; ++w) { free(s->wc[w]); free(s->wc_alloc[w]); }
    free(s->rh); free(s->nh); free(s->h1); free(s->wc); free(s->wc_alloc); free(s->w2h1);
    free(s->acl[0]); free(s->acl[1]); free(s->awl[0]); free(s->awl[1]); free(s->word_active); free(s->word_lat_idx);
    free(s->lt_sf); free(s->lt_dscr); free(s->lt_bp); free(s->cand); free(s->csf_ef); free(s->csf_cand);
    free(s->brc_score); free(s->brc_path); free(s->brc_lc); free(s->bp); free(s->bss); free(s->bp_idx);
}

int32_t
pso_fwdtree_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, const int32_t *ci_tmat,
                const int32_t *info, const int32_t *model, const int16_t *senscr, int32_t n_sen, int32_t T,
                const int32_t *pen, const int32_t *lmarr, int32_t *bp_out, int32_t bp_cap, int32_t *bss_out, int32_t bss_cap, int32_t *bss_n,
                int32_t *bp_idx_out)
{
    ft_t S, *s = &S;
    lmarr_t LMA;
    int32_t i, w, frame, n_done = 0;
    const int32_t *pl = NULL;
#define FT_PL(ci) (pl ? pl[ci] : 0)      /* phone_loop_search_score, phone_loop_search.h:103 */
    ft_setup(s, n_emit_state, tp, sseq, ci_tmat, info, model, T);
    if (lmarr) { lmarr_bind(&LMA, lmarr); s->lma = &LMA; }
    /* ngram_fwdtree_start :470-520 */
    for (w = 0; w < s->n_words; ++w) { s->word_lat_idx[w] = -1; s->lt_sf[w] = -1; }
    s->best_score = 0;
    pso_hmm_enter(&s->h1[s->w2h1[s->start_wid]], 0, -1, 0);

    for (frame = 0; frame < T; ++frame) {
        const int32_t nf = frame + 1, cur = frame & 1, nxt = nf & 1;
        int32_t bs, k, j, thresh, newphone_thresh, lastphn_thresh;
        s->ctx.senscore = senscr + (size_t)frame * n_sen;
        pl = pen ? pen + (size_t)frame * s->n_ci : NULL;
        s->bp_idx[frame] = s->bpidx;                                       /* mark_bptable */
        if (s->best_score <= PSO_WORST_SCORE) break;
        if (s->best_score + 2 * s->beam < PSO_WORST_SCORE) {               /* renormalize_scores :566-603 */
            const int32_t norm = s->best_score;
            for (i = 0; i < s->n_root; ++i) if (s->rh[i].frame == frame) pso_hmm_normalize(&s->rh[i], norm);
            for (i = 0; i < s->n_acl[cur]; ++i) pso_hmm_normalize(&s->nh[s->acl[cur][i]], norm);
            for (i = 0; i < s->n_awl[cur]; ++i) {
                w = s->awl[cur][i];
                for (j = 0; j < ft_nrc(s, w); ++j) if (s->wc_alloc[w][j]) pso_hmm_normalize(&s->wc[w][j], norm);
            }
            for (i = 0; i < s->n_1ph; ++i) if (s->h1[i].frame == frame) pso_hmm_normalize(&s->h1[i], norm);
        }
        /* evaluate_channels :702-716 */
        bs = PSO_WORST_SCORE;
        for (i = 0; i < s->n_root; ++i)
            if (s->rh[i].frame == frame) { const int32_t sc = pso_hmm_vit_eval(&s->ctx, &s->rh[i]); if (sc > bs) bs = sc; ++s->n_root_eval; }
        s->best_score = bs;
        bs = PSO_WORST_SCORE;
        s->n_nonroot_eval += s->n_acl[cur];
        for (i = 0; i < s->n_acl[cur]; ++i) { const int32_t sc = pso_hmm_vit_eval(&s->ctx, &s->nh[s->acl[cur][i]]); if (sc > bs) bs = sc; }
        if (bs > s->best_score) s->best_score = bs;
        bs = PSO_WORST_SCORE; k = 0; j = 0;
        for (i = 0; i < s->n_awl[cur]; ++i) {
            int32_t r;
            w = s->awl[cur][i];
            s->word_active[w] = 0;
            for (r = 0; r < ft_nrc(s, w); ++r)
                if (s->wc_alloc[w][r]) { const int32_t sc = pso_hmm_vit_eval(&s->ctx, &s->wc[w][r]); if (sc > bs) bs = sc; ++k; }
        }
        for (i = 0; i < s->n_1ph; ++i) {
            int32_t sc;
            if (s->h1[i].frame < frame) continue;
            sc = pso_hmm_vit_eval(&s->ctx, &s->h1[i]);
            if (sc > bs && s->w1ph[i] != s->finish_wid) bs = sc;
            ++j;
        }
        s->n_nonroot_eval += k + j;
        if (bs > s->best_score) s->best_score = bs;
        s->last_phone_best_score = bs;
        /* prune_channels :1130-1180 */
        s->n_cand = 0;
        s->dynamic_beam = s->beam;
        if (s->maxhmmpf != -1 && s->n_root_eval + s->n_nonroot_eval > s->maxhmmpf) {
            int32_t bins[256], bw = -s->beam / 256, nh = 0;
            memset(bins, 0, sizeof(bins));
            for (i = 0; i < s->n_root; ++i) { int32_t b = (s->best_score - s->rh[i].bestscore) / bw; if (b >= 256) b = 255; ++bins[b]; }
            for (i = 0; i < s->n_acl[cur]; ++i) { int32_t b = (s->best_score - s->nh[s->acl[cur][i]].bestscore) / bw; if (b >= 256) b = 255; ++bins[b]; }
            for (i = 0; i < 256; ++i) { nh += bins[i]; if (nh > s->maxhmmpf) break; }
            s->dynamic_beam = -(i * bw);
        }
        thresh = s->best_score + s->dynamic_beam; newphone_thresh = s->best_score + s->pbeam; lastphn_thresh = s->best_score + s->lpbeam;
        /* prune_root_chan :723-794 */
        s->n_acl[nxt] = 0;
        for (i = 0; i < s->n_root; ++i) {
            pso_hmm_t *rh = &s->rh[i];
            int32_t nps, c;
            if (rh->frame < frame) continue;
            if (!(rh->bestscore > thresh)) continue;
            rh->frame = nf;
            nps = rh->out_score + s->pip;
            if (pl || nps > newphone_thresh)
                for (c = s->roots[i * 5 + 3]; c >= 0; c = s->nonroot[c * 6 + 5])
                    if (nps + FT_PL(s->nonroot[c * 6 + 2]) > newphone_thresh && (s->nh[c].frame < frame || nps > s->nh[c].score[0])) {
                        pso_hmm_enter(&s->nh[c], nps, rh->out_history, nf);
                        s->acl[nxt][s->n_acl[nxt]++] = c;
                    }
            if (pl || nps > lastphn_thresh)
                for (w = s->roots[i * 5 + 2]; w >= 0; w = FT_W(s, w, 6)) {
                    ft_cand_t *cp;
                    if (!(nps + FT_PL(FT_W(s, w, 1)) > lastphn_thresh)) continue;
                    cp = &s->cand[s->n_cand++];
                    cp->wid = w; cp->score = nps - s->nwpen; cp->bp = rh->out_history;
                }
        }
        /* prune_nonroot_chan :800-878 */
        for (i = 0; i < s->n_acl[cur]; ++i) {
            const int32_t id = s->acl[cur][i];
            pso_hmm_t *h = &s->nh[id];
            if (h->bestscore > thresh) {
                int32_t nps, c;
                if (h->frame != nf) { h->frame = nf; s->acl[nxt][s->n_acl[nxt]++] = id; }
                nps = h->out_score + s->pip;
                if (pl || nps > newphone_thresh)
                    for (c = s->nonroot[id * 6 + 4]; c >= 0; c = s->nonroot[c * 6 + 5])
                        if (nps + FT_PL(s->nonroot[c * 6 + 2]) > newphone_thresh && (s->nh[c].frame < frame || nps > s->nh[c].score[0])) {
                            if (s->nh[c].frame != nf) s->acl[nxt][s->n_acl[nxt]++] = c;
                            pso_hmm_enter(&s->nh[c], nps, h->out_history, nf);
                        }
                if (pl || nps > lastphn_thresh)
                    for (w = s->nonroot[id * 6 + 3]; w >= 0; w = FT_W(s, w, 6)) {
                        ft_cand_t *cp;
                        if (!(nps + FT_PL(FT_W(s, w, 1)) > lastphn_thresh)) continue;
                        cp = &s->cand[s->n_cand++];
                        cp->wid = w; cp->score = nps - s->nwpen; cp->bp = h->out_history;
                    }
            }
            else if (h->frame != nf) pso_hmm_clear(h);
        }
        /* last_phone_transition :885-1035 */
        {
            int32_t n_csf = 0, bestscore, th;
            s->n_awl[nxt] = 0;
            for (i = 0; i < s->n_cand; ++i) {
                ft_cand_t *cp = &s->cand[i];
                const ft_bp_t *e;
                if (cp->bp == -1) continue;
                e = &s->bp[cp->bp];
                cp->score -= ft_exit_score(s, e, FT_W(s, cp->wid, 0));
                if (s->lt_sf[cp->wid] != e->frame + 1) {
                    for (j = 0; j < n_csf; ++j) if (s->csf_ef[j] == e->frame) break;
                    if (j < n_csf) cp->next = s->csf_cand[j];
                    else { j = n_csf++; cp->next = -1; s->csf_ef[j] = e->frame; }
                    s->csf_cand[j] = i;
                    s->lt_dscr[cp->wid] = PSO_WORST_SCORE;
                    s->lt_sf[cp->wid] = e->frame + 1;
                }
            }
            for (i = 0; i < n_csf; ++i) {
                int32_t bp;
                for (bp = s->bp_idx[s->csf_ef[i]]; bp < s->bp_idx[s->csf_ef[i] + 1]; ++bp) {
                    const ft_bp_t *e = &s->bp[bp];
                    if (!e->valid) continue;
                    for (j = s->csf_cand[i]; j >= 0; j = s->cand[j].next) {
                        const ft_cand_t *cp = &s->cand[j];
                        int32_t dscr = ft_exit_score(s, e, FT_W(s, cp->wid, 0));
                        if (dscr > PSO_WORST_SCORE) dscr += ft_tg(s, FT_W(s, cp->wid, 5), e->real_wid, e->prev_real_wid);
                        if (dscr > s->lt_dscr[cp->wid]) { s->lt_dscr[cp->wid] = dscr; s->lt_bp[cp->wid] = bp; }
                    }
                }
            }
            bestscore = s->last_phone_best_score;
            for (i = 0; i < s->n_cand; ++i) {
                ft_cand_t *cp = &s->cand[i];
                cp->score += s->lt_dscr[cp->wid];
                cp->bp = s->lt_bp[cp->wid];
                if (cp->score > bestscore) bestscore = cp->score;
            }
            s->last_phone_best_score = bestscore;
            th = bestscore + s->lponlybeam;
            for (i = 0; i < s->n_cand; ++i) {
                const ft_cand_t *cp = &s->cand[i];
                int32_t r;
                if (!(cp->score > th)) continue;
                w = cp->wid;
                ft_alloc_all_rc(s, w);
                k = 0;
                for (r = 0; r < ft_nrc(s, w); ++r) {
                    pso_hmm_t *h = &s->wc[w][r];
                    if (h->frame < frame || cp->score > h->score[0]) { pso_hmm_enter(h, cp->score, cp->bp, nf); ++k; }
                }
                if (k > 0) { s->awl[nxt][s->n_awl[nxt]++] = w; s->word_active[w] = 1; }
            }
        }
        /* prune_word_chan :1042-1126 */
        {
            const int32_t newword_thresh = s->last_phone_best_score + s->wbeam, lp_thresh = s->last_phone_best_score + s->lponlybeam;
            for (i = 0; i < s->n_awl[cur]; ++i) {
                int32_t r;
                w = s->awl[cur][i];
                k = 0;
                for (r = 0; r < ft_nrc(s, w); ++r) {
                    pso_hmm_t *h;
                    if (!s->wc_alloc[w][r]) continue;
                    h = &s->wc[w][r];
                    if (h->bestscore > lp_thresh) {
                        h->frame = nf; ++k;
                        if (h->out_score > newword_thresh) ft_save_bp(s, frame, w, h->out_score, h->out_history, r);
                    }
                    else if (h->frame != nf) s->wc_alloc[w][r] = 0;         /* hmm_deinit + listelem_free */
                }
                if (k > 0 && !s->word_active[w]) { s->awl[nxt][s->n_awl[nxt]++] = w; s->word_active[w] = 1; }
            }
            for (i = 0; i < s->n_1ph; ++i) {
                pso_hmm_t *h = &s->h1[i];
                if (h->frame < frame) continue;
                if (h->bestscore > lp_thresh) {
                    h->frame = nf;
                    if (h->out_score > newword_thresh) ft_save_bp(s, frame, s->w1ph[i], h->out_score, h->out_history, 0);
                }
            }
        }
        /* bptable_maxwpf :1188-1238 */
        if (s->maxwpf != -1 && s->maxwpf != s->n_words) {
            int32_t bp, n = 0, bestscr = INT32_MIN, bestbp = -1;
            for (bp = s->bp_idx[frame]; bp < s->bpidx; ++bp)
                if (FT_W(s, s->bp[bp].wid, 4)) {
                    if (s->bp[bp].score > bestscr) { bestscr = s->bp[bp].score; bestbp = bp; }
                    s->bp[bp].valid = 0; ++n;
                }
            if (bestbp >= 0) { s->bp[bestbp].valid = 1; --n; }
            n = (s->bpidx - s->bp_idx[frame]) - n;
            for (; n > s->maxwpf; --n) {
                int32_t worstscr = INT32_MAX, worstbp = -1;
                for (bp = s->bp_idx[frame]; bp < s->bpidx; ++bp)
                    if (s->bp[bp].valid && s->bp[bp].score < worstscr) { worstscr = s->bp[bp].score; worstbp = bp; }
                if (worstbp < 0) break;
                s->bp[worstbp].valid = 0;
            }
        }
        /* word_transition :1241-1430 */
        {
            int32_t bp, rc;
            const int32_t nc = s->n_ci;
            for (i = nc - 1; i >= 0; --i) s->brc_score[i] = PSO_WORST_SCORE;
            k = 0;
            for (bp = s->bp_idx[frame]; bp < s->bpidx; ++bp) {
                const ft_bp_t *e = &s->bp[bp];
                s->word_lat_idx[e->wid] = -1;
                if (e->wid == s->finish_wid) continue;
                ++k;
                if (e->last2_phone == -1) {
                    for (rc = 0; rc < nc; ++rc)
                        if (e->score > s->brc_score[rc]) { s->brc_score[rc] = e->score; s->brc_path[rc] = bp; s->brc_lc[rc] = e->last_phone; }
                }
                else {
                    const int32_t *cimap = s->rs_cimap + ((size_t)e->last_phone * nc + e->last2_phone) * nc;
                    const int32_t *rcss = s->bss + e->s_idx;
                    for (rc = 0; rc < nc; ++rc)
                        if (rcss[cimap[rc]] > s->brc_score[rc]) { s->brc_score[rc] = rcss[cimap[rc]]; s->brc_path[rc] = bp; s->brc_lc[rc] = e->last_phone; }
                }
            }
            if (k > 0) {
                const int32_t th = s->best_score + s->dynamic_beam;
                int32_t newscore;
                for (i = 0; i < s->n_root; ++i) {
                    const int32_t ci = s->roots[i * 5], ci2 = s->roots[i * 5 + 1];
                    newscore = s->brc_score[ci] + s->nwpen + s->pip;
                    if (newscore + FT_PL(ci) > th && (s->rh[i].frame < frame || newscore > s->rh[i].score[0])) {
                        pso_hmm_enter(&s->rh[i], newscore, s->brc_path[ci], nf);
                        s->rh[i].senid[0] = (uint16_t)s->ldiph[((size_t)ci * nc + ci2) * nc + s->brc_lc[ci]];
                    }
                }
                for (i = 0; i < s->n_1ph_lm; ++i) s->lt_dscr[s->w1ph[i]] = INT32_MIN;
                for (bp = s->bp_idx[frame]; bp < s->bpidx; ++bp) {
                    const ft_bp_t *e = &s->bp[bp];
                    if (!e->valid) continue;
                    for (i = 0; i < s->n_1ph_lm; ++i) {
                        w = s->w1ph[i];
                        newscore = ft_exit_score(s, e, FT_W(s, w, 0));
                        if (newscore != PSO_WORST_SCORE) newscore += ft_tg(s, FT_W(s, w, 5), e->real_wid, e->prev_real_wid);
                        if (newscore > s->lt_dscr[w]) { s->lt_dscr[w] = newscore; s->lt_bp[w] = bp; }
                    }
                }
                for (i = 0; i < s->n_1ph_lm; ++i) {
                    pso_hmm_t *h = &s->h1[i];
                    w = s->w1ph[i];
                    if (w == s->start_wid) continue;
                    newscore = (int32_t)((uint32_t)s->lt_dscr[w] + (uint32_t)s->pip);
                    if ((int64_t)newscore + FT_PL(s->r1ph[i * 4]) > th && (h->frame < frame || newscore > h->score[0])) {
                        pso_hmm_enter(h, newscore, s->lt_bp[w], nf);
                        h->senid[0] = (uint16_t)s->ldiph[((size_t)s->r1ph[i * 4] * nc + s->r1ph[i * 4 + 1]) * nc
                                                        + FT_W(s, s->bp[s->lt_bp[w]].wid, 1)];
                    }
                }
                {
                    pso_hmm_t *h = &s->h1[s->w2h1[s->silence_wid]];
                    newscore = s->brc_score[s->sil] + s->silpen + s->pip;
                    if (newscore + FT_PL(s->r1ph[s->w2h1[s->silence_wid] * 4]) > th && (h->frame < frame || newscore > h->score[0])) pso_hmm_enter(h, newscore, s->brc_path[s->sil], nf);
                }
                for (w = s->filler_start; w <= s->filler_end; ++w) {
                    pso_hmm_t *h;
                    if (w == s->silence_wid || w == s->start_wid || s->w2h1[w] < 0) continue;
                    h = &s->h1[s->w2h1[w]];
                    newscore = s->brc_score[s->sil] + s->fillpen + s->pip;
                    if (newscore + FT_PL(s->r1ph[s->w2h1[w] * 4]) > th && (h->frame < frame || newscore > h->score[0])) pso_hmm_enter(h, newscore, s->brc_path[s->sil], nf);
                }
            }
        }
        /* deactivate_channels :1432-1451 */
        for (i = 0; i < s->n_root; ++i) if (s->rh[i].frame == frame) pso_hmm_clear(&s->rh[i]);
        for (i = 0; i < s->n_1ph; ++i) if (s->h1[i].frame == frame) pso_hmm_clear(&s->h1[i]);
        ++n_done;
    }
    s->bp_idx[n_done] = s->bpidx;                                          /* ngram_fwdtree_finish :1507 */
    for (i = 0; i < s->bpidx && i < bp_cap; ++i) memcpy(bp_out + (size_t)i * 10, &s->bp[i], 10 * sizeof(int32_t));
    for (i = 0; i < s->bss_head && i < bss_cap; ++i) bss_out[i] = s->bss[i];
    for (i = 0; i <= n_done; ++i) bp_idx_out[i] = s->bp_idx[i];
    *bss_n = s->bss_head;
    i = s->bpidx;
    ft_free(s);
#undef FT_PL
    return i;
}

/* ---------------------------------------------------------------------------------------
 * N-gram decoding, second pass: ngram_search_fwdflat.c (start :371-414 with
 * build_fwdflat_wordlist :224-300 and build_fwdflat_chan :306-368, search step :813-875 =
 * fwdflat_eval_chan :445, fwdflat_prune_chan :483-607, fwdflat_word_transition :643-782 with
 * get_expand_wordlist :610-640) restated for one utterance (n_bp_in < 0: -fwdtree no, every LM word is in
 * the vocabulary and can follow every exit).  Input: the FIRST pass's backpointer
 * table (bp_in [n_bp_in][10], the utterance vocabulary and the start-frame windows come from it) and
 * the same flattened search as pso_fwdtree_run (exported with fwdflat=yes so that info holds
 * fwdflatbeam / fwdflatwbeam / fwdflatefwid / fwdflatsfwin / the language-weight ratio).
 * ci_ssid[n_ci]: senone sequence of every CI phone (roots start from it).  Output as pso_fwdtree_run. */
typedef struct { int32_t wid, fef, lef, next; } ff_node_t;

int32_t
pso_fwdflat_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, const int32_t *ci_tmat, const int32_t *ci_ssid,
                const int32_t *info, const int32_t *model, const int32_t *bp_in, int32_t n_bp_in,
                const int16_t *senscr, int32_t n_sen, int32_t T, const int32_t *lmarr,
                int32_t *bp_out, int32_t bp_cap, int32_t *bss_out, int32_t bss_cap, int32_t *bss_n, int32_t *bp_idx_out)
{
    ft_t S, *s = &S;
    int32_t i, w, f, frame, n_done = 0, n_node = 0, nwd = 0, all_words = 0;
    ff_node_t *node = malloc(((size_t)(n_bp_in > 0 ? n_bp_in : 0) + 1) * sizeof(*node));
    int32_t *head = malloc(((size_t)T + 1) * sizeof(int32_t));
    int32_t *wordlist, *expand, *n_int;
    uint8_t *expand_flag;
    pso_hmm_t *fr, **fi;
    lmarr_t LMA2;

    ft_setup(s, n_emit_state, tp, sseq, ci_tmat, info, model, T);
    if (lmarr) { lmarr_bind(&LMA2, lmarr); s->lma = &LMA2; }
    wordlist = malloc((s->n_words + 1) * sizeof(int32_t)); expand = malloc((s->n_words + 1) * sizeof(int32_t));
    expand_flag = calloc(s->n_words, 1);
    fr = calloc(s->n_words, sizeof(*fr)); fi = calloc(s->n_words, sizeof(*fi)); n_int = calloc(s->n_words, sizeof(int32_t));
    if (n_bp_in < 0) {                                                     /* no first pass: ngram_fwdflat_expand_all :61-87 */
        for (f = 0; f <= T; ++f) head[f] = -1;
        for (w = 0; w < s->n_words; ++w) if (s->inlm[w]) wordlist[nwd++] = w;
        wordlist[nwd] = -1;
        all_words = 1;
    }
    else {
        /* build_fwdflat_wordlist */
        for (f = 0; f <= T; ++f) head[f] = -1;
        for (i = 0; i < n_bp_in; ++i) {
            const int32_t *b = bp_in + (size_t)i * 10;
            const int32_t sf = b[3] < 0 ? 0 : bp_in[(size_t)b[3] * 10] + 1, ef = b[0], wid = b[2];
            int32_t n;
            if (!s->inlm[wid]) continue;
            for (n = head[sf]; n >= 0 && node[n].wid != wid; n = node[n].next);
            if (n >= 0) node[n].lef = ef;
            else { n = n_node++; node[n].wid = wid; node[n].fef = node[n].lef = ef; node[n].next = head[sf]; head[sf] = n; }
        }
        for (f = 0; f < T; ++f) {
            int32_t prev = -1, n, nx;
            for (n = head[f]; n >= 0; n = nx) {
                nx = node[n].next;
                if (node[n].lef - node[n].fef < s->min_ef_width || (node[n].wid == s->finish_wid && node[n].lef < T - 1)) {
                    if (prev < 0) head[f] = nx; else node[prev].next = nx;
                }
                else prev = n;
            }
        }
        memset(s->word_active, 0, s->n_words);
        for (f = 0; f < T; ++f) {
            int32_t n;
            for (n = head[f]; n >= 0; n = node[n].next)
                if (!s->word_active[node[n].wid]) { s->word_active[node[n].wid] = 1; wordlist[nwd++] = node[n].wid; }
        }
        wordlist[nwd] = -1;
    }
    /* build_fwdflat_chan */
    for (i = 0; i < nwd; ++i) {
        int32_t p, len;
        w = wordlist[i];
        if (FT_W(s, w, 3)) continue;
        len = s->pron_off[w + 1] - s->pron_off[w];
        pso_hmm_init(&s->ctx, &fr[w], 1, ci_ssid[FT_W(s, w, 0)], ci_tmat[FT_W(s, w, 0)]);
        n_int[w] = len - 2;
        fi[w] = calloc(len > 2 ? len - 2 : 1, sizeof(pso_hmm_t));
        for (p = 1; p < len - 1; ++p)
            pso_hmm_init(&s->ctx, &fi[w][p - 1], 0, s->pron_ssid[s->pron_off[w] + p], ci_tmat[s->pron_ci[s->pron_off[w] + p]]);
        ft_alloc_all_rc(s, w);
    }
    /* ngram_fwdflat_start */
    for (w = 0; w < s->n_words; ++w) { s->word_lat_idx[w] = -1; s->lt_sf[w] = -1; }
    for (i = 0; i < s->n_1ph; ++i) pso_hmm_clear(&s->h1[i]);
    pso_hmm_enter(&s->h1[s->w2h1[s->start_wid]], 0, -1, 0);
    s->awl[0][0] = s->start_wid; s->n_awl[0] = 1;
    s->best_score = 0;

#define FF_ROOT(w) (FT_W(s, (w), 3) ? &s->h1[s->w2h1[(w)]] : &fr[(w)])
    for (frame = 0; frame < T; ++frame) {
        const int32_t cf = frame, nf = frame + 1, cur = cf & 1, nxt = nf & 1, nw = s->n_awl[cur], pip = s->pip;
        int32_t thresh, wordthresh, bestscore, k, r;
        s->ctx.senscore = senscr + (size_t)frame * n_sen;
        s->bp_idx[frame] = s->bpidx;
        if (s->best_score <= PSO_WORST_SCORE) break;
        if (s->best_score + 2 * s->beam < PSO_WORST_SCORE) {                /* fwdflat_renormalize_scores :785-810 */
            const int32_t norm = s->best_score;
            for (i = 0; i < nw; ++i) {
                pso_hmm_t *rh;
                w = s->awl[cur][i]; rh = FF_ROOT(w);
                if (rh->frame == cf) pso_hmm_normalize(rh, norm);
                if (FT_W(s, w, 3)) continue;
                for (k = 0; k < n_int[w]; ++k) if (fi[w][k].frame == cf) pso_hmm_normalize(&fi[w][k], norm);
                for (r = 0; r < ft_nrc(s, w); ++r) if (s->wc[w][r].frame == cf) pso_hmm_normalize(&s->wc[w][r], norm);
            }
        }
        /* fwdflat_eval_chan */
        bestscore = PSO_WORST_SCORE;
        for (i = 0; i < nw; ++i) {
            pso_hmm_t *rh;
            w = s->awl[cur][i]; rh = FF_ROOT(w);
            if (rh->frame == cf) { const int32_t sc = pso_hmm_vit_eval(&s->ctx, rh); if (sc > bestscore && w != s->finish_wid) bestscore = sc; }
            if (FT_W(s, w, 3)) continue;
            for (k = 0; k < n_int[w]; ++k)
                if (fi[w][k].frame == cf) { const int32_t sc = pso_hmm_vit_eval(&s->ctx, &fi[w][k]); if (sc > bestscore) bestscore = sc; }
            for (r = 0; r < ft_nrc(s, w); ++r)
                if (s->wc[w][r].frame == cf) { const int32_t sc = pso_hmm_vit_eval(&s->ctx, &s->wc[w][r]); if (sc > bestscore) bestscore = sc; }
        }
        s->best_score = bestscore;
        /* fwdflat_prune_chan */
        memset(s->word_active, 0, s->n_words);
        thresh = s->best_score + s->fwdflatbeam; wordthresh = s->best_score + s->fwdflatwbeam;
        for (i = 0; i < nw; ++i) {
            pso_hmm_t *rh;
            int32_t newscore, nrc, ni;
            w = s->awl[cur][i]; rh = FF_ROOT(w);
            nrc = FT_W(s, w, 3) ? 0 : ft_nrc(s, w); ni = FT_W(s, w, 3) ? 0 : n_int[w];
            if (rh->frame == cf && rh->bestscore > thresh) {
                rh->frame = nf; s->word_active[w] = 1;
                newscore = rh->out_score;
                if (!FT_W(s, w, 3)) {
                    newscore += pip;
                    if (newscore > thresh) {
                        if (ni == 0) {
                            for (r = 0; r < nrc; ++r)
                                if (s->wc[w][r].frame < cf || newscore > s->wc[w][r].score[0]) pso_hmm_enter(&s->wc[w][r], newscore, rh->out_history, nf);
                        }
                        else if (fi[w][0].frame < cf || newscore > fi[w][0].score[0]) pso_hmm_enter(&fi[w][0], newscore, rh->out_history, nf);
                    }
                }
                else if (newscore > wordthresh) ft_save_bp(s, cf, w, newscore, rh->out_history, 0);
            }
            for (k = 0; k < ni; ++k) {
                pso_hmm_t *h = &fi[w][k];
                if (h->frame < cf) continue;
                if (h->bestscore > thresh) {
                    h->frame = nf; s->word_active[w] = 1;
                    newscore = h->out_score + pip;
                    if (newscore > thresh) {
                        if (k == ni - 1) {
                            for (r = 0; r < nrc; ++r)
                                if (s->wc[w][r].frame < cf || newscore > s->wc[w][r].score[0]) pso_hmm_enter(&s->wc[w][r], newscore, h->out_history, nf);
                        }
                        else if (fi[w][k + 1].frame < cf || newscore > fi[w][k + 1].score[0]) pso_hmm_enter(&fi[w][k + 1], newscore, h->out_history, nf);
                    }
                }
                else if (h->frame != nf) pso_hmm_clear_scores(h);
            }
            for (r = 0; r < nrc; ++r) {
                pso_hmm_t *h = &s->wc[w][r];
                if (h->frame < cf) continue;
                if (h->bestscore > thresh) {
                    h->frame = nf; s->word_active[w] = 1;
                    if (h->out_score > wordthresh) ft_save_bp(s, cf, w, h->out_score, h->out_history, r);
                }
                else if (h->frame != nf) pso_hmm_clear_scores(h);
            }
        }
        /* fwdflat_word_transition */
        {
            int32_t best_silrc_score = PSO_WORST_SCORE, best_silrc_bp = 0, b, sf = cf - s->max_sf_win, ef = cf + s->max_sf_win, nexp = 0, newscore;
            if (sf < 0) sf = 0;
            if (ef > T) ef = T;
            memset(expand_flag, 0, s->n_words);
            if (all_words)                                                  /* get_expand_wordlist :615-618: the static list */
                for (i = 0; i < nwd; ++i) expand[nexp++] = wordlist[i];
            for (f = sf; f < ef && !all_words; ++f) {
                int32_t n;
                for (n = head[f]; n >= 0; n = node[n].next)
                    if (!expand_flag[node[n].wid]) { expand[nexp++] = node[n].wid; expand_flag[node[n].wid] = 1; }
            }
            for (b = s->bp_idx[cf]; b < s->bpidx; ++b) {
                const ft_bp_t *e = &s->bp[b];
                const int32_t *cimap = NULL, *rcss = s->bss + e->s_idx;
                int32_t silscore;
                s->word_lat_idx[e->wid] = -1;
                if (e->wid == s->finish_wid) continue;
                if (e->last2_phone != -1) cimap = s->rs_cimap + ((size_t)e->last_phone * s->n_ci + e->last2_phone) * s->n_ci;
                for (i = 0; i < nexp; ++i) {
                    pso_hmm_t *rh;
                    w = expand[i];
                    newscore = cimap ? rcss[cimap[FT_W(s, w, 0)]] : e->score;
                    if (newscore == PSO_WORST_SCORE) continue;
                    newscore = (int32_t)((float)newscore + s->lwf * (float)ft_tg(s, FT_W(s, w, 5), e->real_wid, e->prev_real_wid));
                    newscore += pip;
                    if (!(newscore > thresh)) continue;
                    rh = FF_ROOT(w);
                    if (rh->frame < cf || newscore > rh->score[0]) {
                        const int32_t ci = FT_W(s, w, 0), ci2 = FT_W(s, w, 3) ? s->sil : s->pron_ci[s->pron_off[w] + 1];
                        pso_hmm_enter(rh, newscore, b, nf);
                        rh->senid[0] = (uint16_t)s->ldiph[((size_t)ci * s->n_ci + ci2) * s->n_ci + FT_W(s, e->wid, 1)];
                        s->word_active[w] = 1;
                    }
                }
                silscore = cimap ? rcss[cimap[s->sil]] : e->score;
                if (silscore > best_silrc_score) { best_silrc_score = silscore; best_silrc_bp = b; }
            }
            newscore = best_silrc_score + s->silpen + pip;
            if (newscore > thresh && newscore > PSO_WORST_SCORE) {
                pso_hmm_t *rh = &s->h1[s->w2h1[s->silence_wid]];
                if (rh->frame < cf || newscore > rh->score[0]) { pso_hmm_enter(rh, newscore, best_silrc_bp, nf); s->word_active[s->silence_wid] = 1; }
            }
            newscore = best_silrc_score + s->fillpen + pip;
            if (newscore > thresh && newscore > PSO_WORST_SCORE)
                for (w = s->filler_start; w <= s->filler_end; ++w) {
                    pso_hmm_t *rh;
                    if (w == s->silence_wid || s->w2h1[w] < 0) continue;
                    rh = &s->h1[s->w2h1[w]];
                    if (rh->frame < cf || newscore > rh->score[0]) { pso_hmm_enter(rh, newscore, best_silrc_bp, nf); s->word_active[w] = 1; }
                }
            for (i = 0; i < nw; ++i) {
                pso_hmm_t *rh = FF_ROOT(s->awl[cur][i]);
                if (rh->frame == cf) pso_hmm_clear_scores(rh);
            }
        }
        /* next active word list :852-866 */
        k = 0;
        for (i = 0; i < nwd; ++i) if (s->word_active[wordlist[i]] && wordlist[i] < s->start_wid) s->awl[nxt][k++] = wordlist[i];
        for (w = s->start_wid; w < s->n_words; ++w) if (s->word_active[w]) s->awl[nxt][k++] = w;
        s->n_awl[nxt] = k;
        ++n_done;
    }
#undef FF_ROOT
    s->bp_idx[n_done] = s->bpidx;
    for (i = 0; i < s->bpidx && i < bp_cap; ++i) memcpy(bp_out + (size_t)i * 10, &s->bp[i], 10 * sizeof(int32_t));
    for (i = 0; i < s->bss_head && i < bss_cap; ++i) bss_out[i] = s->bss[i];
    for (i = 0; i <= n_done; ++i) bp_idx_out[i] = s->bp_idx[i];
    *bss_n = s->bss_head;
    i = s->bpidx;
    for (w = 0; w < s->n_words; ++w) free(fi[w]);
    free(fr); free(fi); free(n_int); free(wordlist); free(expand); free(expand_flag); free(node); free(head);
    ft_free(s);
    return i;
}

