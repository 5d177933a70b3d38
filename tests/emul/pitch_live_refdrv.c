/* pitch_live_refdrv.c -- one live stream through the compiled reference's yin_* (oracle/_ref/libpsref.so), fed in
 * chunks as audio arrives, with extract_pitch's buffering (programs/pocketsphinx_pitch.c): samples collect in a
 * frame buffer; when it holds flen of them yin_write and yin_read run, and the buffer keeps its last flen - fshift
 * samples.  A final chunk then runs yin_end and yin_read until it fails.  The yin_t lives across chunks; a reset is a
 * fresh yin_init. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct yin_s yin_t;
yin_t *yin_init(int frame_size, float search_threshold, float search_range, int smooth_window);
void yin_free(yin_t *pe);
void yin_start(yin_t *pe);
void yin_end(yin_t *pe);
void yin_write(yin_t *pe, int16_t const *frame);
int yin_read(yin_t *pe, uint16_t *out_period, uint16_t *out_bestdiff);

typedef struct {
    int flen, fshift, smooth_window;
    float voice_thresh, search_range;
    yin_t *yin;
    int16_t *buf;
    int nbuf;
    long frames, main_reads, reads;
    int ended;
} live_t;

static void live_fresh(live_t *h)
{
    if (h->yin) yin_free(h->yin);
    h->yin = yin_init(h->flen, h->voice_thresh, h->search_range, h->smooth_window);
    yin_start(h->yin);
    h->nbuf = 0;
    h->frames = h->main_reads = h->reads = 0;
    h->ended = 0;
}

void *refdrv_pitch_live_open(int flen, int fshift, float voice_thresh, float search_range, int smooth_window)
{
    live_t *h = (live_t *)calloc(1, sizeof(live_t));
    h->flen = flen, h->fshift = fshift, h->smooth_window = smooth_window;
    h->voice_thresh = voice_thresh, h->search_range = search_range;
    h->buf = (int16_t *)malloc(sizeof(int16_t) * (size_t)flen);
    live_fresh(h);
    return h;
}

void refdrv_pitch_live_free(void *p)
{
    live_t *h = (live_t *)p;
    yin_free(h->yin);
    free(h->buf);
    free(h);
}

void refdrv_pitch_live_reset(void *p) { live_fresh((live_t *)p); }

/* Feeds n samples, then ends the stream if `final`.  period / bestdiff: this chunk's reads (room for
 * ceil(n / fshift) + 2 * smooth_window); status: frames, main-loop reads and all reads so far, ended.  Returns the
 * chunk's reads, -1 if the stream has ended. */
long refdrv_pitch_live_feed(void *p, const int16_t *pcm, long n, int final, uint16_t *period, uint16_t *bestdiff,
                            int32_t *status)
{
    live_t *h = (live_t *)p;
    long k = 0, i = 0;
    if (h->ended) return -1;
    while (i < n) {
        long take = h->flen - h->nbuf;
        if (take > n - i) take = n - i;
        memcpy(h->buf + h->nbuf, pcm + i, sizeof(int16_t) * (size_t)take);
        h->nbuf += (int)take;
        i += take;
        if (h->nbuf < h->flen) break;
        yin_write(h->yin, h->buf);
        ++h->frames;
        if (yin_read(h->yin, &period[k], &bestdiff[k])) ++k, ++h->main_reads;
        memmove(h->buf, h->buf + h->fshift, sizeof(int16_t) * (size_t)(h->flen - h->fshift));
        h->nbuf = h->flen - h->fshift;
    }
    if (final) {
        yin_end(h->yin);
        while (yin_read(h->yin, &period[k], &bestdiff[k])) ++k;
        h->ended = 1;
    }
    h->reads += k;
    status[0] = (int32_t)h->frames;
    status[1] = (int32_t)h->main_reads;
    status[2] = (int32_t)h->reads;
    status[3] = h->ended;
    return k;
}
