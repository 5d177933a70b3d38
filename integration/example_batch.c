/* integration/example_batch.c -- a plain-C host program against include/psb200.h: what a batch
 * front end (e.g. programs/pocketsphinx_batch.c of the reference) does with the library.  It is
 * compiled (C11, -Wall -Wextra -pedantic) by tests/test_abi.py to keep the header valid C; run it
 * on a machine with an H100:
 *     gcc -std=c11 -Iinclude integration/example_batch.c -Lpocketsphinx_b200 -lpsb200 -o example
 * The model arrays come from the host's own loaders (here: a caller-supplied descriptor). */
#include <stdio.h>
#include <stdlib.h>

#include "psb200.h"

/* Scores `n_utt` utterances of features and runs the phone loop; returns 0 on success. */
int
example_decode(const psb_model_desc_t *desc, const psb_fe_desc_t *fe_desc, const int16_t *pcm,
               const int64_t *samp_off, int32_t n_utt, const uint8_t *tp, int32_t n_tmat,
               const uint16_t *sseq, int32_t n_sseq, int32_t n_emit_state, const int32_t *ci_ssid,
               const int32_t *ci_tmat, int32_t n_ci)
{
    psb_model_t *model = NULL;
    psb_batch_t *batch = NULL;
    psb_fe_t *fe = NULL;
    psb_hmmctx_t *ctx = NULL;
    psb_phoneloop_t *pl = NULL;
    int32_t *frame_off = NULL, *best = NULL, *pen = NULL;
    int64_t frames = 0;
    int rc = -1, u;

    if (psb_device_count() < 1) {
        fprintf(stderr, "no CUDA device: %s\n", psb_last_error());
        return -1;
    }
    if (psb_model_create(desc, 0, &model) < 0) goto done;
    if (psb_fe_create(fe_desc, 0, &fe) < 0) goto done;
    for (u = 0; u < n_utt; ++u) frames += psb_fe_n_frames(fe, samp_off[u + 1] - samp_off[u]);
    if (psb_batch_create(model, n_utt, frames, &batch) < 0) goto done;
    if (psb_hmmctx_create(n_emit_state, tp, n_tmat, sseq, n_sseq, desc->n_sen, 0, &ctx) < 0) goto done;
    /* phone_loop_search defaults: window 5, beams from -pl_beam / -pl_pbeam, -pl_pip, -pl_weight */
    if (psb_phoneloop_create(ctx, n_ci, ci_ssid, ci_tmat, 5, -1080, -1080, 0, 3.0, &pl) < 0) goto done;
    frame_off = malloc(((size_t)n_utt + 1) * sizeof(*frame_off));
    best = malloc((size_t)frames * sizeof(*best));
    pen = malloc((size_t)frames * (size_t)n_ci * sizeof(*pen));
    if (!frame_off || !best || !pen) goto done;
    /* audio -> features -> senone scores -> phone-loop Viterbi, all on the device */
    if (psb_decode_batch_pcm_host(batch, fe, pl, pcm, samp_off, n_utt, frame_off, best, pen, NULL) < 0) goto done;
    for (u = 0; u < n_utt; ++u)
        printf("utterance %d: %d frames, best score of the last frame %d\n", u, frame_off[u + 1] - frame_off[u],
               frame_off[u + 1] > frame_off[u] ? best[frame_off[u + 1] - 1] : 0);
    rc = 0;
done:
    if (rc) fprintf(stderr, "error: %s\n", psb_last_error());
    free(frame_off); free(best); free(pen);
    psb_phoneloop_free(pl);
    psb_hmmctx_free(ctx);
    psb_batch_free(batch);
    psb_fe_free(fe);
    psb_model_free(model);
    return rc;
}
