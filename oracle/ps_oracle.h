/* oracle/ps_oracle.h -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * Plain-C CPU restatement of the PocketSphinx hot path (GMM senone evaluation for the
 * ptm / s2_semi / ms back-ends, hmm_vit_eval, and the phone-loop caller), written from the
 * algorithm, each function citing the reference file:line it follows (paths relative to
 * /root/reference).  Default float build (mfcc_t = float32) semantics.
 *
 * Pinned: tests/test_oracle_vs_ref.py compares every function here with the compiled
 * reference (oracle/_ref/libpsref.so) when it is present, and tests/test_oracle_golden.py
 * compares it with committed fixtures (tests/golden/) generated from that reference by
 * oracle/make_golden.py.
 */
#ifndef PS_ORACLE_H
#define PS_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PSO_MAX_FEAT 8
#define PSO_MAX_TOPN 16
#define PSO_MAX_NSTATE 5                       /* hmm.h:159 HMM_MAX_NSTATE */
#define PSO_SENSCR_SHIFT 10                    /* hmm.h:72 */
#define PSO_WORST_SCORE ((int32_t)0xE0000000)  /* hmm.h:83 */
#define PSO_TMAT_WORST_SCORE (-255)            /* hmm.h:89 */
#define PSO_BAD_SSID 0xffff                    /* bin_mdef.h BAD_SSID / BAD_SENID */
#define PSO_MAX_NEG_ASCR 96                    /* tied_mgau_common.h:91 */
#define PSO_WORST_DIST INT32_MIN               /* tied_mgau_common.h:60 */

enum { PSO_KIND_PTM = 0, PSO_KIND_SEMI = 1, PSO_KIND_MS = 2 };

/* Acoustic model, as flat arrays in the reference's in-memory order. */
typedef struct pso_model_s {
    int32_t kind, n_sen, n_mgau, n_feat, n_density, topn;
    int32_t featlen[PSO_MAX_FEAT];
    int32_t ds_ratio;              /* -ds; 1 = every frame */
    int32_t aw;                    /* ms: inverse acoustic weight (-aw) */
    int32_t mixw_4bit;             /* sendump with cluster_bits 4 */
    int32_t pdf_transposed;        /* ms: 1 = pdf[feat][cw][sen] (n_gauden==1), 0 = pdf[sen][feat][cw] */
    int32_t logadd_ms_size, logadd_ms_zero;
    const float *mean;             /* [n_mgau][n_feat][n_density][featlen[f]] */
    const float *var;              /* same; precomputed 1/(2 sigma^2) in log-base units */
    const float *det;              /* [n_mgau][n_feat][n_density] */
    const uint8_t *mixw;           /* ptm/semi: [n_feat][n_density][row]; ms: pdf */
    const uint8_t *mixw_cb;        /* 16 entries when mixw_4bit */
    const int32_t *sen2cb;         /* [n_sen] */
    const uint8_t *logadd8;        /* 256-entry table of logmath_init(base, 10, 1) */
    const uint32_t *logadd_ms;     /* ms: wide table widened to uint32 */
    const uint8_t *topn_beam;      /* semi: [n_feat] or NULL */
    int32_t fixed_point;           /* 1: the -DFIXED_POINT build's arithmetic (PTM only): mean / var /
                                    * det / features are int32 (Q12 means and features), bit-cast into the
                                    * float pointers; see the "fixed point" block of ps_oracle.c */
} pso_model_t;

typedef struct pso_topn_s { int32_t cw, score; } pso_topn_t;

/* Per-decoder GMM state: the top-N history ring (ptm_mgau.h:64-94, s2_semi_mgau.h:79-82). */
typedef struct pso_gmm_s {
    const pso_model_t *m;
    int32_t n_hist;        /* pl_window + 2 */
    int32_t frame_idx;     /* ps_mgau_t.frame_idx (acmod.h:113-116) */
    pso_topn_t *hist;      /* ptm: [n_hist][n_mgau][n_feat][topn]; semi: [n_hist][n_feat][topn] */
    uint8_t *cb_active;    /* ptm: [n_hist][n_mgau] */
    uint8_t *hist_n;       /* semi: [n_hist][n_feat] */
    pso_topn_t *ms_dist;   /* ms scratch: [n_mgau][n_feat][topn], score field holds float bits */
    pso_topn_t *raw;       /* ptm, optional: receives each evaluated frame's lists before ptm_norm */
    int32_t sumlen;
} pso_gmm_t;

pso_gmm_t *pso_gmm_new(const pso_model_t *m, int32_t n_hist);
void pso_gmm_free(pso_gmm_t *g);
void pso_gmm_reset(pso_gmm_t *g);

/* One ps_mgau frame_eval call (acmod.h:101-107).  feat = one row of sumlen floats. */
int pso_frame_eval(pso_gmm_t *g, int16_t *senscr, const uint8_t *senone_active,
                   int32_t n_senone_active, const float *feat, int32_t frame, int32_t compallsen);

/* Fresh state, compallsen, frames 0..T-1, frame_idx advanced like acmod_advance.
 * topn_out optional: ptm [T][n_mgau][n_feat][topn]{cw,score}, semi [T][n_feat][topn].
 * raw_out optional (ptm): the same lists before ptm_norm, with the integer distances that
 * decide their order (what the device's top-N records hold). */
int pso_score_utt(const pso_model_t *m, const float *feats, int32_t T, int16_t *senscr,
                  int32_t *topn_out, int32_t *raw_out);

/* acmod_flags2list (acmod.c:1224-1275): flags[n_sen] bytes -> delta list; returns count. */
int32_t pso_flags2list(const uint8_t *flags, int32_t n_sen, uint8_t *list);

/* ---- HMM ---- */

/* Same 88-byte LP64 layout as the reference's hmm_t (hmm.h:169-182). */
typedef struct pso_hmm_s {
    void *ctx;
    int32_t score[PSO_MAX_NSTATE];
    int32_t history[PSO_MAX_NSTATE];
    int32_t out_score;
    int32_t out_history;
    uint16_t ssid;
    uint16_t senid[PSO_MAX_NSTATE];
    int32_t bestscore;
    int16_t tmatid;
    int32_t frame;
    uint8_t mpx;
    uint8_t n_emit_state;
} pso_hmm_t;

typedef struct pso_hmmctx_s {
    int32_t n_emit_state;
    const uint8_t *tp;        /* [n_tmat][n_emit][n_emit+1] */
    const uint16_t *sseq;     /* [n_sseq][n_emit] */
    const int16_t *senscore;
} pso_hmmctx_t;

void pso_hmm_init(const pso_hmmctx_t *c, pso_hmm_t *h, int mpx, int ssid, int tmatid);
void pso_hmm_clear(pso_hmm_t *h);
void pso_hmm_clear_scores(pso_hmm_t *h);
void pso_hmm_enter(pso_hmm_t *h, int32_t score, int32_t histid, int frame);
void pso_hmm_normalize(pso_hmm_t *h, int32_t bestscr);
int32_t pso_hmm_vit_eval(const pso_hmmctx_t *c, pso_hmm_t *h);
/* loop + max, like evaluate_hmms (phone_loop_search.c:202-221) without the frame test */
int32_t pso_hmm_vit_eval_batch(const pso_hmmctx_t *c, pso_hmm_t *h, int32_t n);

/* ---- phone loop (phone_loop_search.c) ---- */
typedef struct pso_phoneloop_s {
    pso_hmmctx_t ctx;
    int32_t n_phones, window;
    int32_t beam, pbeam, pip;
    double penalty_weight;
    pso_hmm_t *hmms;
    int32_t *pen_buf;      /* [window][n_phones] */
    int32_t *penalties;    /* [n_phones] */
    int32_t pen_buf_ptr;
    int32_t best_score;
    int32_t n_renorm;
} pso_phoneloop_t;

pso_phoneloop_t *pso_phoneloop_new(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq,
                                   int32_t n_phones, const int32_t *ssid, const int32_t *tmatid,
                                   int32_t window, int32_t beam, int32_t pbeam, int32_t pip,
                                   double penalty_weight);
void pso_phoneloop_free(pso_phoneloop_t *p);
void pso_phoneloop_start(pso_phoneloop_t *p);
void pso_phoneloop_step(pso_phoneloop_t *p, const int16_t *senscr, int32_t frame_idx);
/* start + T steps; optional per-frame dumps: hmm_out [T][n_phones] pso_hmm_t, best_out [T],
 * pen_out [T][n_phones]. */
void pso_phoneloop_run(pso_phoneloop_t *p, const int16_t *senscr, int32_t n_sen, int32_t T,
                       pso_hmm_t *hmm_out, int32_t *best_out, int32_t *pen_out);

double pso_time_score_utt(const pso_model_t *m, const float *feats, int32_t T, int32_t reps);

/* ---- forced alignment (state_align_search.c) ---- */
int32_t pso_align_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, int32_t n_phones,
                      const int32_t *ssid, const int32_t *tmatid, const int32_t *sf, const int32_t *ef,
                      const int16_t *senscr, int32_t n_sen, int32_t T,
                      int32_t *st_start, int32_t *st_dur, int32_t *st_score);

/* ---- keyword spotting (kws_search.c) ---- */
int32_t pso_kws_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq,
                    int32_t n_pl, const int32_t *pl_ssid, const int32_t *pl_tmat,
                    int32_t n_kp, const int32_t *kp_off, const int32_t *kp_thresh,
                    const int32_t *kp_ssid, const int32_t *kp_tmat, int32_t beam, int32_t plp,
                    const int16_t *senscr, int32_t n_sen, int32_t T, int32_t *hits, int32_t cap);

/* ---- phone decoding (allphone_search.c, no phone LM) ---- */
int32_t pso_allphone_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, int32_t n_nodes,
                         const int32_t *ssid, const int32_t *tmatid, const int32_t *succ_off, const int32_t *succ,
                         int32_t start, int32_t beam, int32_t pbeam, int32_t inspen,
                         const int16_t *senscr, int32_t n_sen, int32_t T, int32_t *hist, int32_t cap);

int32_t pso_allphone_lm_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, int32_t n_nodes,
                            const int32_t *ssid, const int32_t *tmatid, const int32_t *succ_off, const int32_t *succ,
                            int32_t start, int32_t beam, int32_t pbeam, int32_t n_ci, const int32_t *node_ci,
                            const int32_t *bg, const int32_t *tg,
                            const int16_t *senscr, int32_t n_sen, int32_t T, int32_t *hist, int32_t cap);
/* design experiment for a looser codeword filter (see ps_oracle.c) */
int32_t pso_filter_experiment(const pso_model_t *m, const float *feats, int32_t T, int32_t lag, int64_t *stats);

/* fsg_search.c + fsg_history.c for one utterance (see ps_oracle.c); hist_out [cap][13]. */
int32_t pso_fsg_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq,
                    int32_t n_pnode, const int32_t *pn, int32_t n_state, const int32_t *roots,
                    int32_t n_link, const int32_t *links, const int32_t *nulloff, const int32_t *nullarc,
                    int32_t n_ci, int32_t silcipid, int32_t start_state,
                    int32_t beam_orig, int32_t pbeam_orig, int32_t wbeam_orig, int32_t maxhmmpf,
                    const int16_t *senscr, int32_t n_sen, int32_t T, int32_t *hist_out, int32_t cap);

/* ngram_search_fwdtree.c for one utterance (see ps_oracle.c); info / model as exported by
 * oracle/ref_driver.c:refdrv_fwdtree, ci_tmat[n_ci] = transition matrix of every CI phone. */
int32_t pso_fwdtree_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, const int32_t *ci_tmat,
                        const int32_t *info, const int32_t *model, const int16_t *senscr, int32_t n_sen, int32_t T,
                        const int32_t *pen, const int32_t *lmarr, int32_t *bp_out, int32_t bp_cap, int32_t *bss_out, int32_t bss_cap,
                        int32_t *bss_n, int32_t *bp_idx_out);

/* ngram_search_fwdflat.c for one utterance, from the first pass's backpointer table (see ps_oracle.c). */
int32_t pso_fwdflat_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, const int32_t *ci_tmat,
                        const int32_t *ci_ssid, const int32_t *info, const int32_t *model, const int32_t *bp_in,
                        int32_t n_bp_in, const int16_t *senscr, int32_t n_sen, int32_t T, const int32_t *lmarr,
                        int32_t *bp_out, int32_t bp_cap, int32_t *bss_out, int32_t bss_cap, int32_t *bss_n,
                        int32_t *bp_idx_out);

/* trigram scores from the LM as sorted arrays (see ps_oracle.c) */
void pso_lm_scores(const int32_t *lmarr, const int32_t *q, int64_t n_q, int32_t *scores);

#ifdef __cplusplus
}
#endif
#endif

