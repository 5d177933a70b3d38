/* psb200.h -- C ABI of the H100-native PocketSphinx hot path (libpsb200.so).
 *
 * Plain C, no CUDA or torch types in any signature: a host program (the reference's own C,
 * or anything with an FFI) binds these exactly like the symbols they stand in for.  Every
 * entry point names the reference interface it replaces (paths relative to the
 * cmusphinx/pocketsphinx 5.1.1 tree).  All functions return 0 on success and a negative
 * psb_status_t on failure (the reference's "<0 + E_ERROR, never exit()" convention,
 * include/pocketsphinx/err.h:80-88); psb_last_error() gives the message for the calling
 * thread.  Handles are opaque; one handle may be used from one thread at a time, different
 * handles from different threads (each owns its CUDA stream).
 *
 * Numerics contract: int16 senone scores, int32 path scores, histories and best scores are
 * bit-identical to the reference's default (float) build for the same inputs.
 */
#ifndef PSB200_H
#define PSB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PSB_ABI_VERSION 2

typedef enum psb_status_e {
    PSB_OK = 0,
    PSB_ERR_ARG = -1,        /* bad argument / unsupported shape */
    PSB_ERR_CUDA = -2,       /* CUDA runtime error (message in psb_last_error) */
    PSB_ERR_NOMEM = -3,
    PSB_ERR_STATE = -4       /* call not valid in the handle's current state */
} psb_status_t;

enum { PSB_KIND_PTM = 0, PSB_KIND_SEMI = 1, PSB_KIND_MS = 2 };

#define PSB_MAX_FEAT 8
#define PSB_MAX_TOPN 8
#define PSB_HMM_MAX_NSTATE 5          /* hmm.h:159 */
#define PSB_WORST_SCORE ((int32_t)0xE0000000)   /* hmm.h:83 */

const char *psb_last_error(void);
int psb_abi_version(void);
int psb_device_count(void);

/* ------------------------------------------------------------------------------------ */
/* Acoustic model (replaces what ptm_mgau_init ptm_mgau.c:805, s2_semi_mgau_init
 * s2_semi_mgau.c:1236 and ms_mgau_init ms_mgau.c:80 build in host memory: gauden_t +
 * mixture weights + sen2cb + the 8-bit log-add table).  Arrays are in the reference's
 * in-memory order *after* its loaders ran (gauden_dist_precompute, ms_gauden.c:264-308):
 *   mean, var  float [n_mgau][n_feat][n_density][featlen[f]]
 *   det        float [n_mgau][n_feat][n_density]
 *   mixw       ptm/semi: uint8 [n_feat][n_density][row], row = n_sen or (n_sen+1)/2 (4-bit)
 *              ms:       uint8 pdf[n_sen][n_feat][n_density] (n_mgau > 1)
 *                         or   pdf[n_feat][n_density][n_sen] (n_mgau == 1)  (ms_senone.h:73-80)
 *   mixw_cb    16 bytes or NULL;  sen2cb int32 [n_sen];  logadd8 uint8 [256]
 *   logadd_ms  uint32 [logadd_ms_size] (the shifted logmath table, ms back-end only)
 * Pointers are host pointers unless on_device != 0 (then they are device pointers on
 * `device`, e.g. after an NCCL broadcast of the packed model).                            */
typedef struct psb_model_desc_s {
    int32_t kind, n_sen, n_mgau, n_feat, n_density, topn;
    int32_t featlen[PSB_MAX_FEAT];
    int32_t ds_ratio;           /* -ds   (ptm_mgau.c:242) */
    int32_t aw;                 /* -aw   (ms_senone.c:396) */
    int32_t logadd_ms_size, logadd_ms_zero;
    int32_t on_device;
    const float *mean, *var, *det;
    const uint8_t *mixw, *mixw_cb;
    const int32_t *sen2cb;
    const uint8_t *logadd8;
    const uint32_t *logadd_ms;
    const uint8_t *topn_beam;   /* semi: [n_feat] or NULL (s2_semi_mgau.c:1302-1309) */
    int32_t fixed_point;        /* != 0: the host is a -DFIXED_POINT build (mfcc_t = int32 Q12,
                                 * fe/fixpoint.h:98-100): mean / var / det and every feature value are
                                 * int32 bit patterns carried in the float-typed arrays, and the Gaussian
                                 * arithmetic is FIXMUL / GMMSUB with the early exits of
                                 * ptm_mgau.c:182-206 / s2_semi_mgau.c:137-143 (ptm and semi only) */
} psb_model_desc_t;

typedef struct psb_model_s psb_model_t;

int psb_model_create(const psb_model_desc_t *desc, int device, psb_model_t **out);
void psb_model_free(psb_model_t *m);
/* ps_mgaufuncs_t.transform (acmod.h:108-109; gauden_mllr_transform ms_gauden.c:512):
 * the host applies MLLR and re-precomputes; this re-uploads the Gaussians. */
int psb_model_update_gaussians(psb_model_t *m, const float *mean, const float *var, const float *det);
int psb_model_n_sen(const psb_model_t *m);
int psb_model_device(const psb_model_t *m);

/* ------------------------------------------------------------------------------------ */
/* Per-stream scorer: the drop-in behind ps_mgau_t's vtable (acmod.h:98-125).
 * psb_scorer_frame_eval has the argument meaning of ps_mgaufuncs_t.frame_eval
 * (acmod.h:101-107) as called from acmod_score (acmod.c:1108-1114): host buffers, senscr is
 * int16[n_sen] owned by the caller and fully defined on return, senone_active is the uint8
 * delta list from acmod_flags2list (acmod.c:1224-1275), feat[f] points at stream f of the
 * frame, frame is absolute, past frames (frame < frame_idx, within n_hist) are re-scored from
 * the top-N history ring (ptm_mgau.c:419-451).  frame_idx is ps_mgau_t.frame_idx: the host
 * mirrors acmod_start_utt / acmod_advance / acmod_rewind (acmod.c:419,862,874) through
 * psb_scorer_set_frame_idx.  n_hist = pl_window + 2 (ptm_mgau.c:884).                      */
typedef struct psb_scorer_s psb_scorer_t;

int psb_scorer_create(psb_model_t *m, int32_t n_hist, psb_scorer_t **out);
void psb_scorer_free(psb_scorer_t *s);
int psb_scorer_reset(psb_scorer_t *s);       /* ptm_mgau_reset_fast_hist (ptm_mgau.c:777) */
int psb_scorer_set_frame_idx(psb_scorer_t *s, int32_t frame_idx);
int32_t psb_scorer_get_frame_idx(const psb_scorer_t *s);
int psb_scorer_frame_eval(psb_scorer_t *s, int16_t *senscr, const uint8_t *senone_active,
                          int32_t n_senone_active, const float *const *feat, int32_t frame,
                          int32_t compallsen);

/* ------------------------------------------------------------------------------------ */
/* Batched utterance scoring (the acmod_score loop of SURVEY 8d config 2: all senones,
 * every utterance starting from the post-init top-N state).
 *   feats    float [total_frames][sumlen]   utterance u owns rows utt_off[u]..utt_off[u+1]-1
 *   utt_off  int32 [n_utt + 1]
 *   senscr   int16 [total_frames][n_sen]
 * _host: host buffers; the H2D copy of feats and the D2H copy of senscr are part of the call.
 * _device: device buffers on the model's device (utt_off stays a host array); asynchronous
 * on the batch's stream until psb_batch_sync.                                              */
typedef struct psb_batch_s psb_batch_t;

int psb_batch_create(psb_model_t *m, int32_t max_utts, int64_t max_frames, psb_batch_t **out);
void psb_batch_free(psb_batch_t *b);
int psb_batch_score_host(psb_batch_t *b, const float *feats, const int32_t *utt_off,
                         int32_t n_utt, int16_t *senscr);
int psb_batch_score_device(psb_batch_t *b, const float *d_feats, const int32_t *utt_off,
                           int32_t n_utt, int16_t *d_senscr);
int psb_batch_sync(psb_batch_t *b);
/* device address of the batch's own score matrix after psb_batch_score_device(..., NULL) */
int16_t *psb_batch_senscr_device(psb_batch_t *b);
/* timing of the last score call's kernels on the batch stream (CUDA events), ms:
 * out[0] transpose, out[1] gaussian top-N, out[2] senone eval */
int psb_batch_last_kernel_ms(psb_batch_t *b, float *out3);
/* CUDA-event stopwatch on the batch's stream (the stream every kernel of this batch is
 * launched on): record slot 0/1, then elapsed ms between them (synchronises). */
int psb_batch_event_record(psb_batch_t *b, int slot);
int psb_batch_event_elapsed_ms(psb_batch_t *b, float *ms);
/* debugging: with PSB_TC_CHECK=1 in the environment the tensor-core filter kernels (the default top-N path
 * for 13-dimensional PTM streams; PSB_TOPN_VARIANT=5 selects the scan over time instead) measure, over
 * everything this batch has scored, the largest |filter value - exact distance| / error bound (must stay
 * below 1) and the largest candidate count per (frame, codebook-stream pair); stats4 (may be NULL) = rows seen,
 * rows whose record came from the filter values alone, exact distances computed, rows handed to the tie fix-up. */
int psb_batch_tc_check(psb_batch_t *b, float *ratio, int32_t *max_candidates, int64_t *stats4);
/* debugging (PSB_TC_CHECK=1): which decisions the tensor-core filter took over everything this batch has scored.
 * out[0..n-1] receives the first n of, in order: the four stats4 values; rows with more than 18 candidates
 * (the filter kernel's per-row list capacity); rows where one lane of the filter stored more than 18 column
 * pairs; rows in doubt rescored inside the filter kernel because its work list was full, with a candidate
 * list and over all codewords; rows in doubt whose candidate list the filter's two threads per row both
 * wrote; rows with a candidate list that failed the gap test, the >> 10 agreement test, the sign guard and the
 * saturation guard (one row can fail several); then, without PSB_TC_CHECK too, the last filter launch's tiles per
 * CTA and its CTAs per codebook-stream pair. */
#define PSB_TC_N_COUNTERS 15
int psb_batch_tc_counters(psb_batch_t *b, int64_t *out, int32_t n);
/* debugging/parity: copy the per-frame top-N records of the last call to the host:
 * rec int32 [total_frames][n_mgau*n_feat][4] = {top>>10, cw[4] bytes, e[4] bytes, 0} */
int psb_batch_get_topn(psb_batch_t *b, int32_t *rec, int64_t n_frames);

/* ------------------------------------------------------------------------------------ */
/* HMM evaluation.  psb_hmm_t is the reference's hmm_t byte for byte (hmm.h:169-182, 88 bytes
 * on LP64): the search modules touch its fields directly (hmm.h:185-213), so the layout is
 * ABI.  The ctx pointer is ignored by this library.                                        */
typedef struct psb_hmm_s {
    void *ctx;
    int32_t score[PSB_HMM_MAX_NSTATE];
    int32_t history[PSB_HMM_MAX_NSTATE];
    int32_t out_score;
    int32_t out_history;
    uint16_t ssid;
    uint16_t senid[PSB_HMM_MAX_NSTATE];
    int32_t bestscore;
    int16_t tmatid;
    int32_t frame;
    uint8_t mpx;
    uint8_t n_emit_state;
} psb_hmm_t;

/* hmm_context_init (hmm.h:218-224): tp uint8 [n_tmat][n_emit][n_emit+1] (tmat.h:57-63),
 * sseq uint16 [n_sseq][n_emit] (bin_mdef.h:137). */
typedef struct psb_hmmctx_s psb_hmmctx_t;

int psb_hmmctx_create(int32_t n_emit_state, const uint8_t *tp, int32_t n_tmat,
                      const uint16_t *sseq, int32_t n_sseq, int32_t n_sen, int device,
                      psb_hmmctx_t **out);
void psb_hmmctx_free(psb_hmmctx_t *c);

/* The batched twin of "for each active hmm: hmm_vit_eval(hmm); best = max" as in
 * evaluate_hmms (phone_loop_search.c:202-221), eval_*_chan (ngram_search_fwdtree.c:606-699),
 * fsg_search_hmm_eval (fsg_search.c:336-408): hmms is a host array of n records updated in
 * place; senscr is the frame's host int16[n_sen] (hmm_context_set_senscore); *best gets the
 * max bestscore (PSB_WORST_SCORE when n == 0). */
int psb_hmm_vit_eval_batch(psb_hmmctx_t *c, psb_hmm_t *hmms, int32_t n, const int16_t *senscr,
                           int32_t *best);
/* Same through an array of pointers (the active lists are arrays of chan_t*,
 * ngram_search.h:278; hmm_t is the first member of chan_t / root_chan_t / fsg_pnode_t). */
int psb_hmm_vit_eval_ptrs(psb_hmmctx_t *c, psb_hmm_t *const *hmms, int32_t n,
                          const int16_t *senscr, int32_t *best);

/* Device-resident HMM sets: the instances that evaluate_channels
 * (ngram_search_fwdtree.c:702-715), fsg_search_hmm_eval (fsg_search.c:336-408),
 * kws_search_hmm_eval (kws_search.c:194) and phmm_eval_all (allphone_search.c:349) walk every
 * frame, kept in HBM between frames as a structure of arrays instead of crossing the bus as
 * 88-byte records.  Instances are grouped in n_seg segments (one per utterance / decoder);
 * segment s owns instances [seg_off[s], seg_off[s+1]) and has its own senone-score row and best
 * score per frame. */
typedef struct psb_hmmset_s psb_hmmset_t;
int psb_hmmset_create(psb_hmmctx_t *c, int64_t n_max, int32_t n_seg_max, psb_hmmset_t **out);
void psb_hmmset_free(psb_hmmset_t *s);
/* host hmm_t records -> device SoA (hmm_init / hmm_enter happen on the host), and back */
int psb_hmmset_upload(psb_hmmset_t *s, const psb_hmm_t *hmms, int64_t n, const int64_t *seg_off,
                      int32_t n_seg);
int psb_hmmset_download(psb_hmmset_t *s, psb_hmm_t *hmms);
/* n_frames consecutive frames: in frame t every instance of segment s takes one hmm_vit_eval
 * step (hmm.c:787-805) against the device int16 row  d_senscr[(d_row0[s] + t) * n_sen]  (with
 * d_row0 == NULL: row t * n_seg + s) and d_best[t * n_seg + s] = max bestscore of the segment
 * (PSB_WORST_SCORE if it is empty or finished: d_n_rows[s] <= t, d_n_rows may be NULL).
 * *ms (may be NULL) = device time of the n_frames launches (CUDA events on the set's stream). */
int psb_hmmset_eval_frames_device(psb_hmmset_t *s, const int16_t *d_senscr, const int64_t *d_row0,
                                  const int32_t *d_n_rows, int32_t n_frames, int32_t *d_best,
                                  float *ms);
/* The same n_frames steps fused in ONE launch: every CTA keeps its slice of a segment in registers
 * for the whole run and only the segment's score row of each frame is staged (TMA bulk copy +
 * mbarrier, two frames ahead) -- the evaluate_channels loop (ngram_search_fwdtree.c:702-715) over a
 * fixed active set, where nothing else has to see the state between frames.  Same arguments and
 * bit-identical results (state after the last frame, d_best) as psb_hmmset_eval_frames_device;
 * rows_total = number of rows of the d_senscr matrix (its last row is never over-read).  Sets with
 * multiplexed instances, topologies other than 3 / 5 states or an odd senone count are served by
 * the per-frame launches. */
int psb_hmmset_sweep_device(psb_hmmset_t *s, const int16_t *d_senscr, int64_t rows_total,
                            const int64_t *d_row0, const int32_t *d_n_rows, int32_t n_frames,
                            int32_t *d_best, float *ms);
/* The fused sweep WITH beam pruning between frames -- evaluate_channels (ngram_search_fwdtree.c:702-715) followed by
 * the beam part of prune_channels (:1130-1181: best score, the -maxhmmpf histogram that narrows the beam) and the
 * keep-or-clear decision of prune_nonroot_chan (:811, :823-827, :872-874), without the lexicon tree's transitions: an instance is
 * active in frame frame0 + t iff its frame field equals frame0 + t; active instances take one hmm_vit_eval step; with
 * best = the segment's maximum and n = the number evaluated, dynamic beam = beam, or, when maxhmmpf >= 0 and
 * n > maxhmmpf, -(i * bw) with bw = -beam / 256 and i the first of 256 bins of (best - bestscore) / bw (clipped to 255)
 * at which the running count exceeds maxhmmpf; instances with bestscore > best + dynamic beam move to frame
 * frame0 + t + 1, the others are hmm_clear'ed (hmm.c:181-196: WORST_SCORE, history -1, frame -1) and stay out.
 * d_best[t * n_seg + s] as above; d_n_active[t * n_seg + s] (may be NULL) = instances evaluated.  One thread-block
 * cluster per segment exchanges maxima, counts and histograms through distributed shared memory: a segment may hold
 * at most 16 x 1024 instances; plain (not multiplexed) 3- or 5-state instances, even senone count. */
int psb_hmmset_sweep_beam_device(psb_hmmset_t *s, const int16_t *d_senscr, int64_t rows_total,
                                 const int64_t *d_row0, const int32_t *d_n_rows, int32_t n_frames,
                                 int32_t frame0, int32_t beam, int32_t maxhmmpf, int32_t *d_best,
                                 int32_t *d_n_active, float *ms);
/* With ms == NULL psb_hmmset_sweep_device is asynchronous on the set's stream.
 * psb_hmmset_use_batch_stream: run the set's kernels on batch b's stream, i.e. behind the kernels
 * that write the scores it reads (b == NULL: back to the set's own stream).
 * psb_hmmset_snapshot / _restore: keep / bring back a device copy of the mutable state (scores,
 * histories, exit score / history, best), so that the next batch of utterances starts from the same
 * entered instances without another upload. */
int psb_hmmset_use_batch_stream(psb_hmmset_t *s, psb_batch_t *b);
int psb_hmmset_snapshot(psb_hmmset_t *s);
int psb_hmmset_restore(psb_hmmset_t *s);
/* one frame from host buffers: senscr int16 [n_seg][n_sen], best int32 [n_seg] */
int psb_hmmset_eval_host(psb_hmmset_t *s, const int16_t *senscr, int32_t *best);

/* ------------------------------------------------------------------------------------ */
/* Device-resident phone-loop Viterbi over whole utterances: the frame-synchronous caller
 * of hmm_vit_eval in phone_loop_search.c (start :155, renormalize :177, evaluate_hmms :193,
 * store_scores :216, prune_hmms :241, phone_transition :263, step :301) run for every
 * utterance of a batch, consuming senone scores already on the device.
 * ssid/tmatid: the n_phones HMMs (CI phones for the reference's phone loop).
 * beam/pbeam/pip: already >> SENSCR_SHIFT (phone_loop_search.c:106-108).                  */
typedef struct psb_phoneloop_s psb_phoneloop_t;

int psb_phoneloop_create(psb_hmmctx_t *c, int32_t n_phones, const int32_t *ssid,
                         const int32_t *tmatid, int32_t window, int32_t beam, int32_t pbeam,
                         int32_t pip, double penalty_weight, psb_phoneloop_t **out);
void psb_phoneloop_free(psb_phoneloop_t *p);
/* d_senscr int16 [total_frames][n_sen] on the device; outputs (device, may be NULL):
 *   d_best int32 [total_frames]              best_score after each frame
 *   d_pen  int32 [total_frames][n_phones]    penalties after each frame
 * final HMM states (host, may be NULL): psb_hmm_t [n_utt][n_phones] */
int psb_phoneloop_run_device(psb_phoneloop_t *p, const int16_t *d_senscr, const int32_t *utt_off,
                             int32_t n_utt, int32_t *d_best, int32_t *d_pen, psb_hmm_t *final_hmms,
                             void *stream_of_batch /* psb_batch_t* or NULL */);
/* host-buffer twin (copies in/out inside the call); per-frame HMM dump optional:
 * hmm_trace psb_hmm_t [total_frames][n_phones] */
int psb_phoneloop_run_host(psb_phoneloop_t *p, const int16_t *senscr, const int32_t *utt_off,
                           int32_t n_utt, int32_t *best, int32_t *pen, psb_hmm_t *hmm_trace);

/* ------------------------------------------------------------------------------------ */
/* End-to-end: host features in -> senone scores -> phone-loop Viterbi -> host results out
 * (best[total_frames], pen[total_frames][n_phones]); senscr (host, may be NULL) also
 * returned when wanted.  This is the call bench.py times as "e2e". */
int psb_decode_batch_host(psb_batch_t *b, psb_phoneloop_t *p, const float *feats,
                          const int32_t *utt_off, int32_t n_utt, int32_t *best, int32_t *pen,
                          int16_t *senscr);

/* Device-resident twin: d_feats on the device, results left in the batch's own device buffers
 * (d_best int32 [total], d_pen int32 [total][n_phones]; addresses returned through the
 * out-pointers, which may be NULL); asynchronous on the batch's stream. */
int psb_decode_batch_device(psb_batch_t *b, psb_phoneloop_t *p, const float *d_feats,
                            const int32_t *utt_off, int32_t n_utt, int32_t **d_best, int32_t **d_pen);

/* ------------------------------------------------------------------------------------ */
/* Senone-dump wire format (acmod_write_senfh_header / acmod_write_scores / acmod_read_scores,
 * acmod.c:335-346, 880-1017): lets GPU-computed scores drive the unmodified reference search
 * through ps_decode_senscr (pocketsphinx.c:1200) or `pocketsphinx_batch -senin yes`.  Host only.
 * write: all-senone frames.  read: returns frames read (<= max_frames) or <0; frames with partial
 * lists are expanded with SENSCR_DUMMY (0x7fff) like acmod_read_scores_internal. */
int psb_sendump_write(const char *path, const char *mdef_file, int32_t n_sen, double logbase,
                      const int16_t *senscr, int64_t n_frames);
int64_t psb_sendump_read(const char *path, int32_t *n_sen_out, int16_t *senscr, int64_t max_frames);

/* Number of sub-batches psb_decode_batch_* keeps in flight on separate streams.  0 = auto (the
 * default, also env PSB_PIPELINE): 2 for host buffers (copies overlap kernels), 1 for resident
 * features; 1 = one stream, which is what per-kernel timing wants; up to 8. */
int psb_batch_set_pipeline(psb_batch_t *b, int n);

/* ------------------------------------------------------------------------------------ */
/* Forced alignment for whole batches: state_align_search.c (start :43, step :184-219 =
 * renormalise, evaluate_hmms :64, prune_hmms :88, phone_transition :109, record_transitions :153;
 * finish :221-279 = backtrace).  Utterance u owns frames [utt_off[u], utt_off[u+1]) of the int16
 * score matrix [frames][n_sen] (all senones: -compallsen yes) and phones [ph_off[u], ph_off[u+1])
 * given as (ssid, tmatid) like hmm_init(hmmctx, hmm, FALSE, ssid, tmatid) (:455); sf / ef are the
 * per-phone alignment constraints of state_align_search_init (:462-469), NULL = always active.
 * Outputs per emitting state (index = phone * n_emit_state + j, ps_alignment_entry_t): start,
 * duration, score; -1 where the backtrace never visits the state.  status[u]: 0, -1 ("Failed to
 * reach final state"), -2 - frame ("Alignment failed in frame").  All arrays but d_senscr: host. */
int psb_align_batch_device(psb_hmmctx_t *c, const int16_t *d_senscr, const int32_t *utt_off,
                           int32_t n_utt, const int32_t *ph_off, const int32_t *ssid,
                           const int32_t *tmatid, const int32_t *sf, const int32_t *ef,
                           int32_t *st_start, int32_t *st_dur, int32_t *st_score, int32_t *status);
/* device time (CUDA events on the context's stream) of the last psb_align_batch_* kernel */
float psb_align_last_kernel_ms(const psb_hmmctx_t *c);
int psb_align_batch_host(psb_hmmctx_t *c, const int16_t *senscr, const int32_t *utt_off,
                         int32_t n_utt, const int32_t *ph_off, const int32_t *ssid,
                         const int32_t *tmatid, const int32_t *sf, const int32_t *ef,
                         int32_t *st_start, int32_t *st_dur, int32_t *st_score, int32_t *status);

/* ------------------------------------------------------------------------------------ */
/* Keyword spotting for whole batches: kws_search.c (start :577, step :599-628 = hmm_eval :194,
 * hmm_prune :234, trans :256-348) with one keyphrase set for all utterances.  The phone loop is
 * n_pl phones (ssid, tmatid) as kws_search_reinit builds it (:464-476, all CI phones); keyphrase k
 * owns the HMM chain [kp_off[k], kp_off[k+1]) of (kp_ssid, kp_tmat) (:510-538) and the threshold
 * kp_thresh[k]; beam and plp as kws_search_init computes them (:425-432).  d_senscr: device int16
 * [frames][n_sen], all senones.  Every detection the reference would pass to kws_detections_add
 * (:286-294) is returned as a row {frame, keyphrase, start frame, prob, ascr} in hits
 * [n_utt][cap_per_utt][5] (host), in the reference's order; n_hits[u] (host) counts them (rows past
 * cap_per_utt are dropped).  The host applies kws_detections_add unchanged. */
int psb_kws_batch_device(psb_hmmctx_t *c, const int16_t *d_senscr, const int32_t *utt_off, int32_t n_utt,
                         int32_t n_pl, const int32_t *pl_ssid, const int32_t *pl_tmat, int32_t n_kp,
                         const int32_t *kp_off, const int32_t *kp_thresh, const int32_t *kp_ssid,
                         const int32_t *kp_tmat, int32_t beam, int32_t plp, int32_t *hits,
                         int32_t cap_per_utt, int32_t *n_hits);

/* ------------------------------------------------------------------------------------ */
/* Phone decoding for whole batches: allphone_search.c without a phone LM (start :640-677, step
 * :700-722 = phmm_eval_all :349, phmm_exit :380, phmm_trans :458).  The PHMM graph is given in the
 * order the reference walks ci_phmm[] (ci-major, list order): node i = (ssid[i], tmatid[i]),
 * successors succ[succ_off[i] .. succ_off[i+1]) (plink_t lists, :186-262), `start` = the silence
 * PHMM entered by allphone_search_start; beam / pbeam / inspen as allphone_search_init computes
 * them (:581-602).  Every history_t the reference appends (:402-444) comes back as a row
 * {ef, node, predecessor entry, score} in hist [n_utt][cap_per_utt][4] (host), n_hist[u] counts
 * them; the host's allphone_backtrace (:765-840) works on that table unchanged.  Graphs up to a
 * few thousand nodes (shared memory): the context-independent graph has one node per phone. */
int psb_allphone_batch_device(psb_hmmctx_t *c, const int16_t *d_senscr, const int32_t *utt_off,
                              int32_t n_utt, int32_t n_nodes, const int32_t *ssid, const int32_t *tmatid,
                              const int32_t *succ_off, const int32_t *succ, int32_t start, int32_t beam,
                              int32_t pbeam, int32_t inspen, int32_t *hist, int32_t cap_per_utt,
                              int32_t *n_hist);
/* The same with a phone LM (-allphone <lm>): node_ci[n_nodes] maps nodes to CI phones, bg
 * [n_ci][n_ci] and tg [n_ci][n_ci][n_ci] are the LM scores >> SENSCR_SHIFT tabulated by the host
 * through its own LM object with the argument positions of phmm_exit / phmm_trans
 * (allphone_search.c:420-441, 497-513): bg[a][b] = ngram_bg_score(lm, wid[a], wid[b]),
 * tg[a][b][c] = ngram_tg_score(lm, wid[a], wid[b], wid[c]).  History rows have five columns:
 * {ef, node, predecessor entry, score, tscore}; cap_per_utt must hold every entry (n_hist[u] <=
 * cap_per_utt), because later frames look their predecessors up in the table. */
int psb_allphone_lm_batch_device(psb_hmmctx_t *c, const int16_t *d_senscr, const int32_t *utt_off,
                                 int32_t n_utt, int32_t n_nodes, const int32_t *ssid, const int32_t *tmatid,
                                 const int32_t *succ_off, const int32_t *succ, int32_t start, int32_t beam,
                                 int32_t pbeam, int32_t n_ci, const int32_t *node_ci, const int32_t *bg,
                                 const int32_t *tg, int32_t *hist, int32_t cap_per_utt, int32_t *n_hist);

/* Phone decoding over a PHMM net of any size, the context-dependent one (-allphone_ci no: one node per
 * distinct (CI phone, tmat, senone sequence) of the mdef, 29 324 on en-us) included, for whole
 * batches, with or without a phone LM.  The net is given in the reference's factored form, not as
 * links: node i (in the order of ci_phmm[], ci-major, list order) = (ssid[i], tmatid[i], node_ci[i],
 * lc[i], rc[i]), lc / rc the context bit vectors phmm_build fills (allphone_search.c:259-308; bit a
 * of lc: CI phone a may precede the node; a filler context sets every filler's bit; CI nodes have
 * all n_ci bits).  phmm_link's rule (:167-215) -- p links to p2 iff ci(p2) is in rc(p) and ci(p) in
 * lc(p2) -- is applied on the device.  n_ci <= 64; no mask bit at or above n_ci.  start = the
 * silence node allphone_search_start enters; beam / pbeam / inspen as allphone_search_init computes
 * them (inspen is ignored with an LM).  bg / tg: NULL for the unconstrained loop, else the phone LM's
 * tables as for psb_allphone_lm_batch_device.
 * The history table stays on the device (cap_per_utt rows of 16 bytes per utterance; at most
 * n_nodes entries per frame) and allphone_backtrace (:774-837) runs there.  Per utterance u:
 * res[u] = {status, n_hist, n_seg}, status 0 = ok, 1 = the history outgrew cap_per_utt (the search
 * of that utterance stopped; no segments; the other utterances are unaffected), 2 = more than
 * seg_cap segments (the first seg_cap are returned; T segments always suffice for T frames);
 * segs [n_utt][seg_cap][5] = (ci, sf, ef, score, tscore) in time order, as the reference's phseg_t
 * list.  hist: NULL, or [n_utt][cap_per_utt][4] host rows {ef, node, predecessor entry, score}
 * (for hosts that keep their own backtrace). */
int psb_allphone_net_batch_device(psb_hmmctx_t *c, const int16_t *d_senscr, const int32_t *utt_off,
                                  int32_t n_utt, int32_t n_nodes, const int32_t *ssid, const int32_t *tmatid,
                                  const int32_t *node_ci, const uint64_t *lc, const uint64_t *rc, int32_t n_ci,
                                  int32_t start, int32_t beam, int32_t pbeam, int32_t inspen, const int32_t *bg,
                                  const int32_t *tg, int32_t cap_per_utt, int32_t *res, int32_t *segs,
                                  int32_t seg_cap, int32_t *hist);

/* ------------------------------------------------------------------------------------ */
/* STATUS of the search entry points below (psb_fsg_batch_device, psb_ngram_*_batch_device): their phase
 * code reproduces the reference's tables in host emulation and is race-checked (tests/emul/), the kernels
 * themselves have not yet run on hardware (DESIGN.md 4.10-4.12); the reference-side export / import that
 * goes with them is integration/ps_search_cuda.c.
 *
 * Grammar decoding for whole batches: fsg_search.c (-fsg / -jsgf; start :770-817, step :683-761 =
 * hmm_eval :335, hmm_prune_prop :516, null_prop :566, word_trans :621) with fsg_history.c's
 * right-context bookkeeping (:132-240), every utterance against the same grammar.  The host keeps
 * fsg_search_init / fsg_lextree_init and flattens what they built (fsg_lextree.h:137-190;
 * integration/ps_search_cuda.c:cuda_fsg_export is the loop):
 *   pnodes [n_pnode][16] = ssid, tmatid, next (first successor, or the link id of a leaf, or -1),
 *                          sibling, logs2prob, ci_ext, ppos, leaf, ctxt.bv[8]; ids in alloc order
 *   roots  [n_state]      first root pnode of each state's lextree (-1: none)
 *   links  [n_link][5]    from_state, to_state, wid (-1: null), logs2prob, 1 if exits of this word
 *                          apply to every right context (filler or single-phone word, :468-474)
 *   nulloff [n_state+1], nullarc: the null arcs leaving each state as link ids, in fsg_model_arcs order
 *   beam / pbeam / wbeam as fsg_search_init computes them (beam_orig...), maxhmmpf (-1: off).
 * Every fsg_hist_entry_t the reference makes permanent comes back, in table order, as a row
 *   {link (-1: the start entry), frame, score, pred, lc, rc.bv[8]}
 * in hist [n_utt][cap_per_utt][13] (host); n_hist[u] counts them (rows past cap_per_utt are
 * dropped).  The host's fsg_search_find_exit / fsg_search_hyp / fsg_search_lattice work on that
 * table unchanged.  The lextree must be a tree under each state (it is, fsg_lextree.c:354-600). */
typedef struct psb_fsg_desc_s {
    int32_t n_pnode;  const int32_t *pnodes;
    int32_t n_state;  const int32_t *roots;
    int32_t n_link;   const int32_t *links;
    const int32_t *nulloff, *nullarc;
    int32_t n_ciphone, silcipid, start_state;
    int32_t beam, pbeam, wbeam, maxhmmpf;
} psb_fsg_desc_t;
int psb_fsg_batch_device(psb_hmmctx_t *c, const psb_fsg_desc_t *g, const int16_t *d_senscr,
                         const int32_t *utt_off, int32_t n_utt, int32_t *hist, int32_t cap_per_utt,
                         int32_t *n_hist);

/* ------------------------------------------------------------------------------------ */
/* N-gram decoding, first pass, for whole batches: ngram_search_fwdtree.c (search step :1454-1496,
 * start :470) with the backpointer-table half of ngram_search.c (save_bp :378, alloc_all_rc :593,
 * exit_score :655), every utterance against the same lextree, dictionary and language model.  The
 * host keeps ngram_search_init / ngram_fwdtree_init (create_search_channels :174) and flattens what
 * they built into int32 sections; integration/ps_search_cuda.c:cuda_ngram_export is that loop
 * (oracle/ref_driver.c:refdrv_fwdtree documents the layout):
 *   info  [40]  sizes (n_words, n_root_chan, n_nonroot_chan, n_1ph_words, n_1ph_LMwords, n_ciphone),
 *               beams (beam, pbeam, wbeam, lpbeam, lponlybeam), maxhmmpf, maxwpf, nwpen, pip, silpen,
 *               fillpen, <s> / </s> / <sil> ids, filler range, number of LM base words
 *   model       roots | non-root channels | words | single-phone words and their channels |
 *               dict2pid rssid (n_ssid, ssid[], cimap[]) | ldiph_lc | dense trigram scores
 *               tg[w][h1][h2] = ngram_tg_score(...) >> SENSCR_SHIFT over the LM's base words
 *   ci_tmat [n_ciphone]  bin_mdef_pid2tmatid of every CI phone
 * (the dense table limits this entry point to vocabularies of a few hundred words).  d_pen: optional
 * look-ahead: the phone loop's penalties after each of ITS frames ([total frames][n_ciphone], device:
 * what psb_decode_batch_device / psb_phoneloop_run_device leave behind = pls->penalties,
 * phone_loop_search.h:103) and its window pl_window; search frame t of an utterance of T frames runs
 * when the phone loop has seen frame min(t + pl_window, T - 1), as ps_search_forward / ps_end_utt
 * schedule it (pocketsphinx.c:1172-1195, 1329-1333).  Per utterance u the reference's own tables come back:
 *   bp      [n_utt][bp_cap_per_utt][10]  bptbl_t rows: frame, valid, wid, bp, score, s_idx, real_wid,
 *                                        prev_real_wid, last_phone, last2_phone
 *   bss     [n_utt][bss_cap_per_utt]     bscore_stack
 *   bp_idx  [total frames + n_utt]       bp_table_idx, utt_off[u] + u is utterance u's first slot
 *   result  [n_utt][3]                   entries, stack size, frames searched
 * on which ngram_search_find_exit / ngram_search_bp_hyp / the second pass work unchanged.  A full
 * table is an error (PSB_ERR_ARG): later frames read earlier entries.
 * Environment: PSB_NGS_BLOCKS / PSB_NGF_CHANNELS size the per-utterance fan-out pool of the first pass (default: one
 * block per multi-phone word, at most 8192) and the state area of the second (default: every LM word's
 * chain, at most 65536 channels); running out of either is reported as an error. */
typedef struct psb_ngram_desc_s {
    const int32_t *info;        /* [40] */
    const int32_t *model;       /* the sections, back to back */
    int64_t model_len;          /* int32 words in `model` (checked against the sizes info implies) */
    const int32_t *ci_tmat;     /* [n_ciphone] */
    const int32_t *ci_ssid;     /* [n_ciphone] bin_mdef_pid2ssid of every CI phone; second pass only (may be NULL for the first) */
    const int32_t *lm_arrays;   /* optional: the LM as sorted arrays (integration/ps_search_cuda.c:cuda_ngram_export_lm, layout
                                   there; scoring = pocketsphinx_b200/csrc/psb_lm_core.h); when given, trigram scores come from
                                   it, the dense table in `model` may be empty (info[26] = 0) and the LM's size no longer
                                   matters */
    int64_t lm_arrays_len;      /* int32 words in lm_arrays */
} psb_ngram_desc_t;
int psb_ngram_fwdtree_batch_device(psb_hmmctx_t *c, const psb_ngram_desc_t *g, const int16_t *d_senscr,
                                   const int32_t *d_pen, int32_t pl_window, const int32_t *utt_off, int32_t n_utt, int32_t *bp,
                                   int32_t bp_cap_per_utt, int32_t *bss, int32_t bss_cap_per_utt,
                                   int32_t *bp_idx, int32_t *result);
/* Second pass: ngram_search_fwdflat.c (start :371 with build_fwdflat_wordlist :224 and
 * build_fwdflat_chan :306, search step :813 = fwdflat_eval_chan :445, fwdflat_prune_chan :483,
 * fwdflat_word_transition :643) over whole utterances.  info / model as above, exported with the
 * second pass configured (info[28..33]: fwdflatbeam, fwdflatwbeam, fwdflatefwid, fwdflatsfwin, the
 * float32 bits of fwdflatlw / lw, pronunciation count; model continues with the LM-membership flags
 * and the pronunciations with their dict2pid_internal ssids).  bp_first [n_utt][first_cap_per_utt][10]
 * + n_first[n_utt]: every utterance's FIRST-pass table (the utterance vocabulary and the start-frame
 * windows come from it); n_first[u] = -1 runs the second pass alone (-fwdtree no: every LM word is in
 * the vocabulary and may follow every exit).  Outputs as for the first pass. */
int psb_ngram_fwdflat_batch_device(psb_hmmctx_t *c, const psb_ngram_desc_t *g, const int16_t *d_senscr,
                                   const int32_t *utt_off, int32_t n_utt, const int32_t *bp_first,
                                   int32_t first_cap_per_utt, const int32_t *n_first, int32_t *bp,
                                   int32_t bp_cap_per_utt, int32_t *bss, int32_t bss_cap_per_utt,
                                   int32_t *bp_idx, int32_t *result);

/* Both passes back to back with the first pass's tables staying on the device (what
 * ngram_search_finish does: fwdtree over the utterance, acmod_rewind, fwdflat over the same frames,
 * ngram_search.c:781-820).  Arguments as for the two entry points above; only the second pass's tables
 * come back (bp / bss / bp_idx / result), first_result [n_utt][3] (may be NULL) gets the first pass's
 * entry count, stack size and frames. */
int psb_ngram_two_pass_batch_device(psb_hmmctx_t *c, const psb_ngram_desc_t *g, const int16_t *d_senscr,
                                    const int32_t *d_pen, int32_t pl_window, const int32_t *utt_off, int32_t n_utt,
                                    int32_t first_cap_per_utt, int32_t first_bss_cap_per_utt, int32_t *bp,
                                    int32_t bp_cap_per_utt, int32_t *bss, int32_t bss_cap_per_utt, int32_t *bp_idx,
                                    int32_t *result, int32_t *first_result);

/* Reading the hypothesis out of the returned tables (host code, no device work: the reference does this
 * on the host as well, once per utterance).  Without -bestpath this is all of ps_get_hyp / ps_seg_iter;
 * with it the reference's lattice code takes the tables through integration/ps_search_cuda.c.
 *   psb_fsg_find_exit    fsg_search_find_exit (fsg_search.c:883-954): *entry = the best word exit in the
 *                        last frame <= frame_idx that has one (final != 0: only exits into final_state),
 *                        0 if there is no word exit yet, -1 if the final state was not reached
 *   psb_fsg_backtrace    fsg_search_seg_iter + fsg_seg_bp2itor (:1062-1091, :1122-1180): the predecessor
 *                        chain of `entry` in time order, seg [cap][7] = {entry, link, wid (-1: null
 *                        transition), sf, ef, ascr, lscr}; returns its length (>= 0) or an error
 *   psb_ngram_find_exit  ngram_search_find_exit, frame_idx = -1 (ngram_search.c:498-541): </s> in the last
 *                        frame with exits, else its best entry; *entry = -1 if no frame has exits
 *   psb_ngram_backtrace  ngram_search_bp_iter (:958-997): seg [cap][5] = {entry, wid, sf, ef, path score}
 *   psb_ngram_segments   the same chain with ngram_search_bp2itor's scores (:886-928), seg [cap][7] =
 *                        {entry, wid, sf, ef, path score, ascr, lscr}: needs the search description (first
 *                        phones, dict2pid cimap, LM) and the score stack; lwf = 1.0 after the first pass
 *                        alone, the float32 fwdflatlw / lw after a second pass (ngram_search_seg_iter :1033)
 * Filtering fillers / <s> / </s> out of the word string (dict_real_word) is the caller's: the dictionary's
 * strings never cross this interface. */
int psb_fsg_find_exit(const int32_t *hist, int32_t n_hist, const int32_t *links, int32_t n_link,
                      int32_t frame_idx, int32_t final_state, int32_t final, int32_t *entry, int32_t *score);
int32_t psb_fsg_backtrace(const int32_t *hist, int32_t n_hist, const int32_t *links, int32_t n_link,
                          int32_t entry, int32_t *seg, int32_t cap);
int psb_ngram_find_exit(const int32_t *bp, int32_t n_bp, const int32_t *bp_idx, int32_t n_frame,
                        int32_t finish_wid, int32_t *entry, int32_t *score);
int32_t psb_ngram_backtrace(const int32_t *bp, int32_t n_bp, int32_t entry, int32_t *seg, int32_t cap);
int32_t psb_ngram_segments(const psb_ngram_desc_t *g, const int32_t *bp, int32_t n_bp, const int32_t *bss, int32_t n_bss,
                           int32_t entry, float lwf, int32_t *seg, int32_t cap);

/* Self-test of the search kernels' block-wide exclusive scan (the one building block the host
 * emulation of their phase code cannot execute): scans a[0..n) in place on `device` with one CTA,
 * total[0] = the sum, total[1] = the result of an empty scan issued right behind it (must be 0). */
int psb_selftest_block_scan(int device, int32_t *a, int32_t n, int32_t *total);

/* ------------------------------------------------------------------------------------ */
/* Batched front end (SURVEY 8 row f-2): int16 PCM -> cepstra -> batch CMN -> 1s_c_d_dd features
 * for whole batches, every utterance a fresh stream (ps_start_stream + ps_process_raw(full_utt),
 * pocketsphinx.c:1073, acmod.c:528-560).  psb_fe_create_ex adds s2_4x / s3_1x39, live CMN and
 * dither, and sessions of utterances that carry their CMN and dither state.  The tables are the arrays the reference's own fe_t /
 * melfb_t hold after fe_init (fe_internal.h:100-180): a C host passes those pointers. */
typedef struct psb_fe_desc_s {
    int32_t frame_size, frame_shift, fft_size, fft_order;   /* fe_t */
    int32_t n_filt, n_cep;                                  /* melfb_t.num_filters, fe_t.num_cepstra */
    int32_t remove_dc, remove_noise;                        /* -remove_dc, -remove_noise (fe_noise.c) */
    int32_t transform;                                      /* 0 legacy, 1 dct, 2 htk (fe_internal.h) */
    int32_t lifter_val;                                     /* -lifter, 0 = none */
    int32_t window;                                         /* feat_window_size: 3 (1s_c_d_dd) */
    int32_t cmn;                                            /* 0 none, 1 batch (cmn.h) */
    int32_t n_coeffs;                                       /* sum of filt_width */
    float pre_emphasis_alpha, sqrt_inv_n, sqrt_inv_2n;
    const double *hamming;                                  /* [frame_size / 2] fe_t.hamming_window */
    const double *ccc, *sss;                                /* [fft_size / 4] FFT twiddles */
    const int16_t *spec_start, *filt_start, *filt_width;    /* [n_filt] */
    const float *filt_coeffs;                               /* [n_coeffs] */
    const float *mel_cosine;                                /* [n_cep][n_filt] */
    const float *lifter;                                    /* [n_cep] or NULL */
} psb_fe_desc_t;
typedef struct psb_fe_s psb_fe_t;
int psb_fe_create(const psb_fe_desc_t *d, int device, psb_fe_t **out);
void psb_fe_free(psb_fe_t *fe);
/* frames fe_process_frames + fe_end_utt produce for n_samples (fe_interface.c:352-545) */
int32_t psb_fe_n_frames(const psb_fe_t *fe, int64_t n_samples);
/* pcm: the utterances' samples back to back, samp_off int64[n_utt + 1] (host).  Outputs:
 * frame_off int32[n_utt + 1] (host), feats float [frames][psb_fe_feat_dim], mfcc (may be NULL) float
 * [frames][n_cep] = the cepstra after CMN and AGC (what the reference's buffers hold after
 * feat_cmn + feat_agc, which work in place).  *ms (may be NULL) = device time of the kernels. */
int psb_fe_process_host(psb_fe_t *fe, const int16_t *pcm, const int64_t *samp_off, int32_t n_utt,
                        float *feats, float *mfcc, int32_t *frame_off);
int psb_fe_process_device(psb_fe_t *fe, const int16_t *d_pcm, const int64_t *samp_off, int32_t n_utt,
                          float *d_feats, float *d_mfcc, int32_t *frame_off, float *ms);
/* device copy of the features of the last psb_fe_process_host call, and their dimension: 39 for
 * 1s_c_d_dd and s3_1x39, 51 for s2_4x (its four streams 12 + 24 + 3 + 12 back to back), the LDA
 * output dimension with a transform */
const float *psb_fe_device_feats(const psb_fe_t *fe);
int32_t psb_fe_feat_dim(const psb_fe_t *fe);

/* Feature type, CMN, AGC, LDA and dither options (feat_init, feat_read_lda, cmn_set_repr,
 * fe_init_dither).  With them, psb_fe_desc_t.window and .cmn are not read.  o == NULL is
 * psb_fe_create.  Per utterance the cepstra go through CMN (with -varnorm), then AGC on c0, then
 * the dynamic features, then the LDA transform (feat_s2mfc2feat_block_utt, feat.c:1277-1307).
 * All-zero AGC / LDA fields select neither. */
#define PSB_FE_MAX_CEP 32
enum { PSB_FEAT_1S_C_D_DD = 0, PSB_FEAT_S2_4X = 1, PSB_FEAT_S3_1X39 = 2 };   /* -feat (s3_1x39 = 1s_12c_12d_3p_12dd) */
enum { PSB_CMN_NONE = 0, PSB_CMN_BATCH = 1, PSB_CMN_LIVE = 2 };            /* -cmn (current = batch) */
enum { PSB_AGC_NONE = 0, PSB_AGC_MAX = 1, PSB_AGC_EMAX = 2, PSB_AGC_NOISE = 3 };   /* -agc (agc.h) */
typedef struct psb_fe_opts_s {
    int32_t feat;                          /* PSB_FEAT_*; s2_4x and s3_1x39 need n_cep == 13 */
    int32_t cmn;                           /* PSB_CMN_* */
    int32_t varnorm;                       /* -varnorm: 0 / 1, batch CMN only (live CMN refuses it) */
    int32_t dither;                        /* -dither: 0 / 1 */
    int32_t seed;                          /* -seed: the MT19937 seed, init_genrand((unsigned long)seed) */
    float cmn_init[PSB_FE_MAX_CEP];        /* -cmninit as cmn_set_repr parses it; unused entries 0 */
    int32_t agc;                           /* PSB_AGC_*; emax carries its estimate across a session */
    float agc_thresh;                      /* -agcthresh (agc_t.noise_thresh; the reference's default is 2.0),
                                              read by PSB_AGC_NOISE only */
    const float *lda;                      /* -lda: lda[0] of the feature_transform file, [lda_rows][lda_cols]
                                              row-major, eigenvectors in rows; NULL = no transform.  Copied
                                              by psb_fe_create_ex */
    int32_t lda_rows, lda_cols;            /* lda_cols must be the feature dimension; not with s2_4x */
    int32_t ldadim;                        /* -ldadim: rows used, if 0 < ldadim <= lda_rows; else lda_rows */
} psb_fe_opts_t;
int psb_fe_create_ex(const psb_fe_desc_t *d, const psb_fe_opts_t *o, int device, psb_fe_t **out);

/* What a ps_decoder_t carries from one utterance to the next: the live-CMN state (cmn_t), the
 * dither generator (genrand.c) and the emax AGC estimate (agc_t).  ps_start_stream resets none. */
typedef struct psb_fe_state_s {
    float cmn_mean[PSB_FE_MAX_CEP], cmn_sum[PSB_FE_MAX_CEP];
    int32_t cmn_nframe;
    int32_t mt_index;                      /* mti: 624 = a twist is due */
    uint32_t mt[624];
    float agc_max, agc_obs_max, agc_obs_max_sum;   /* agc_t.max, obs_max, obs_max_sum */
    int32_t agc_obs_frame, agc_obs_utt;            /* agc_t.obs_frame, obs_utt */
} psb_fe_state_t;
/* the state fe_init + cmn_set_repr + agc_init + agc_emax_set leave: mean = cmn_init, sum = mean * 500,
 * nframe = 500, init_genrand(seed), agc_max = 5 (10 with CMN none), the other AGC fields 0 */
int psb_fe_state_init(const psb_fe_t *fe, psb_fe_state_t *s);
/* Names the sessions of the next psb_fe_process_* / psb_decode_batch_pcm_host call: session s is
 * utterances sess_off[s] .. sess_off[s + 1] - 1 (in decode order; sess_off[0] = 0, sess_off[n_sess]
 * = that call's n_utt), starting from states_in[s] (NULL: psb_fe_state_init for every session).
 * Without this call every utterance is a session of its own from the initial state. */
int psb_fe_set_sessions(psb_fe_t *fe, const int32_t *sess_off, int32_t n_sess, const psb_fe_state_t *states_in);
/* the sessions' states after the last process call (n_sess of them, in session order) */
int psb_fe_get_states(const psb_fe_t *fe, psb_fe_state_t *states_out, int32_t n_sess);
/* From audio to phone-loop results in one call: front end, senone scores and Viterbi on the
 * device, features never leave it.  frame_off int32[n_utt + 1] (out) indexes best / pen / senscr
 * like utt_off of psb_decode_batch_host. */
int psb_decode_batch_pcm_host(psb_batch_t *b, psb_fe_t *fe, psb_phoneloop_t *p, const int16_t *pcm,
                              const int64_t *samp_off, int32_t n_utt, int32_t *frame_off,
                              int32_t *best, int32_t *pen, int16_t *senscr);

/* ------------------------------------------------------------------------------------ */
/* Voice activity detection and endpointing for whole batches of int16 streams (ps_vad.c,
 * ps_endpointer.c, common_audio/vad/).  For each stream: the decision of ps_vad_classify on every
 * full frame of a fresh ps_vad_init(mode, sample_rate, frame_length), and the segments a fresh
 * ps_endpointer_init(window, ratio, mode, sample_rate, frame_length) produces when
 * ps_endpointer_process is called on every full frame and ps_endpointer_end_stream once with the
 * remaining samples (0 <= r < frame size) -- also when r is 0, which the reference's Python
 * Segmenter skips.  Timestamp callbacks and state carried across calls are not implemented: every
 * call takes whole streams.
 * Refused like ps_vad_set_input_params (ps_vad.c:91-127) and ps_endpointer_init
 * (ps_endpointer.c:63-116): a rate with no supported rate within 50 % (8/16/32/48 kHz), frames other
 * than 10/20/30 ms at that rate, mode outside 0..3, ratios whose start_frames or end_frames fall
 * outside (0, maxlen).  Also refused, though the reference accepts them: rates whose closest supported
 * rate is 48 kHz (44.1 and 48 kHz input), whose 48->8 kHz resampler is not implemented; and windows of
 * more than 57 727 frames (maxlen; the endpointer's queue of decisions is kept in shared memory, four
 * streams per CTA: about 577 s at 10 ms frames).  Zero for sample_rate / frame_length /
 * window / ratio is the reference's default (16000, 0.03, 0.3, 0.9). */
typedef struct psb_vad_opts_s {
    int32_t mode;                 /* 0..3, ps_vad_mode_t */
    int32_t sample_rate;          /* Hz */
    double frame_length;          /* seconds */
    double window, ratio;         /* endpointer */
    int32_t warmup;               /* frames each parallel chunk of the filter bank runs ahead of its
                                     first frame: 0 = the frames of 0.5 s, -1 = none (every chunk
                                     boundary is then repaired); the result never depends on it */
} psb_vad_opts_t;
typedef struct psb_vad_s psb_vad_t;
int psb_vad_create(const psb_vad_opts_t *o, int device, psb_vad_t **out);
void psb_vad_free(psb_vad_t *v);
int32_t psb_vad_frame_size(const psb_vad_t *v);       /* samples per frame (ps_vad_frame_size) */
double psb_vad_frame_length(const psb_vad_t *v);      /* frame_size / sample_rate (vad.h:178) */
int32_t psb_vad_sample_rate(const psb_vad_t *v);
int32_t psb_vad_start_frames(const psb_vad_t *v);     /* ps_endpointer_t.start_frames / end_frames / maxlen */
int32_t psb_vad_end_frames(const psb_vad_t *v);
int32_t psb_vad_maxlen(const psb_vad_t *v);
int32_t psb_vad_warmup(const psb_vad_t *v);           /* the warm-up in frames after the default is applied */
int64_t psb_vad_last_repairs(const psb_vad_t *v);     /* chunk recomputations of the last call's repair passes */
int32_t psb_vad_last_passes(const psb_vad_t *v);      /* repair passes of the last call (the last one recomputes nothing) */
/* pcm: the streams' samples back to back, samp_off int64[n_streams + 1] (host, samp_off[0] = 0).
 * Outputs: frame_off int32[n_streams + 1] (host): stream s has frames frame_off[s] .. frame_off[s + 1] - 1;
 * flags int8[frames] (0 / 1); seg_n int32[n_streams]: stream s's segment count; its segments are
 * rows frame_off[s] .. frame_off[s] + seg_n[s] - 1 of segs int64[frames][2] (first sample, one past
 * the last, relative to the stream) and times double[frames][2] (ps_endpointer_speech_start /
 * speech_end); a stream has at most one segment per frame.  _device: pcm, flags, seg_n, segs and
 * times on the device, *ms (may be NULL) = device time of the kernels. */
int psb_vad_process_host(psb_vad_t *v, const int16_t *pcm, const int64_t *samp_off, int32_t n_streams,
                         int8_t *flags, int32_t *frame_off, int32_t *seg_n, int64_t *segs, double *times);
int psb_vad_process_device(psb_vad_t *v, const int16_t *d_pcm, const int64_t *samp_off, int32_t n_streams,
                           int8_t *d_flags, int32_t *frame_off, int32_t *d_seg_n, int64_t *d_segs, double *d_times,
                           float *ms);

/* number of kernels launched by this library in the calling process so far */
int64_t psb_kernel_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* PSB200_H */
