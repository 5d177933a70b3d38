/* align_banded.c -- state_align_search.c restated (as oracle/ps_oracle.c: pso_align_run) with the token table kept
 * the way align_kernel keeps it: frame f holds phones lo[f] .. hi[f] only, in a row of (hi[f] - lo[f] + 1) x n_emit
 * tokens.  A token of a phone outside the band is counted in *n_outside instead of stored, and a backtrace read
 * outside it gives id -1.  Built by the tests against libpsoracle.so (its hmm_t functions); TEST INFRASTRUCTURE. */
#include <limits.h>
#include <stdint.h>
#include <stdlib.h>

#include "ps_oracle.h"

/* The band rule of psb_hmm.cu (align_band): lo[f] = the first phone with ef >= f (0 in frame 0), hi[f] = the last
 * phone i with sf[j] <= f + 1 for every 1 <= j <= i, hi[f] = lo[f] - 1 for an empty band.  sf / ef NULL: always
 * active. */
void
emul_align_band(int32_t n_phones, const int32_t *sf, const int32_t *ef, int32_t T, int32_t *lo, int32_t *hi)
{
    int f, l = 0, h = n_phones > 0 ? 0 : -1;
    for (f = 0; f < T; ++f) {
        if (f > 0)
            while (l < n_phones && ef && ef[l] < f) ++l;
        while (h + 1 < n_phones && (!sf || sf[h + 1] <= f + 1)) ++h;
        lo[f] = l;
        hi[f] = h > l - 1 ? h : l - 1;
    }
}

static int64_t
tok_at(const int32_t *lo, const int32_t *hi, const int64_t *row, int32_t n_emit, int f, int s)
{
    const int i = s / n_emit;
    if (i < lo[f] || i > hi[f])
        return -1;
    return row[f] + (s - lo[f] * n_emit);
}

/* Returns 0, -1 ("Failed to reach final state") or -2 - frame ("Alignment failed in frame"), as pso_align_run. */
int32_t
emul_align_run_banded(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, int32_t n_phones,
                      const int32_t *ssid, const int32_t *tmatid, const int32_t *sf, const int32_t *ef,
                      const int16_t *senscr, int32_t n_sen, int32_t T,
                      int32_t *st_start, int32_t *st_dur, int32_t *st_score,
                      const int32_t *lo, const int32_t *hi, int64_t *n_outside)
{
    pso_hmmctx_t ctx;
    pso_hmm_t *hmms = calloc(n_phones > 0 ? n_phones : 1, sizeof(*hmms));
    const int32_t n_st = n_phones * n_emit_state;
    int64_t *row = malloc((size_t)(T > 0 ? T : 1) * sizeof(*row)), n_tok = 0;
    int32_t *tok_id, *tok_sc;
    int32_t best_score = 0, frame = 0, rc = 0;
    int i, j, f;

    for (f = 0; f < T; ++f) {
        row[f] = n_tok;
        n_tok += (int64_t)(hi[f] - lo[f] + 1) * n_emit_state;
    }
    tok_id = malloc((size_t)(n_tok > 0 ? n_tok : 1) * sizeof(int32_t));
    tok_sc = malloc((size_t)(n_tok > 0 ? n_tok : 1) * sizeof(int32_t));
    *n_outside = 0;
    ctx.n_emit_state = n_emit_state; ctx.tp = tp; ctx.sseq = sseq; ctx.senscore = NULL;
    for (i = 0; i < n_phones; ++i)
        pso_hmm_init(&ctx, &hmms[i], 0, ssid[i], tmatid[i]);
    for (i = 0; i < n_st; ++i) st_start[i] = st_dur[i] = st_score[i] = -1;
    if (n_phones == 0) { rc = -1; goto done; }
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
            if (nf > (ef ? ef[i] : INT_MAX)) continue;
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
            const int64_t k = tok_at(lo, hi, row, n_emit_state, f, i);
            if (k >= 0) { tok_id[k] = -1; tok_sc[k] = -1; }
        }
        for (i = 0; i < n_phones; ++i) {
            if (hmms[i].frame < f) continue;
            for (j = 0; j < n_emit_state; ++j) {
                const int s = i * n_emit_state + j;
                const int64_t k = tok_at(lo, hi, row, n_emit_state, f, s);
                if (k >= 0) { tok_id[k] = hmms[i].history[j]; tok_sc[k] = hmms[i].score[j]; }
                else ++*n_outside;
                hmms[i].history[j] = s;
            }
        }
        frame = f;
    }
    {                                                                     /* finish: backtrace */
        int32_t last_id, last_sc, cur_id, cur_sc, last_frame, cur_frame;
        last_id = cur_id = hmms[n_phones - 1].out_history;
        last_sc = hmms[n_phones - 1].out_score;
        if (last_id == -1 || T == 0) { rc = -1; goto done; }
        last_frame = frame + 1;
        for (cur_frame = frame - 1; cur_frame >= 0; --cur_frame) {
            const int64_t k = tok_at(lo, hi, row, n_emit_state, cur_frame, cur_id);
            cur_id = k >= 0 ? tok_id[k] : -1;
            cur_sc = k >= 0 ? tok_sc[k] : -1;
            if (cur_id == -1) { rc = -2 - cur_frame; goto done; }
            if (cur_id != last_id) {
                st_start[last_id] = cur_frame + 1;
                st_dur[last_id] = last_frame - st_start[last_id];
                st_score[last_id] = last_sc - cur_sc;
                last_id = cur_id; last_sc = cur_sc;
                last_frame = cur_frame + 1;
            }
        }
        st_start[0] = 0;
        st_dur[0] = last_frame;
        st_score[0] = 0;
    }
done:
    free(hmms); free(tok_id); free(tok_sc); free(row);
    return rc;
}
