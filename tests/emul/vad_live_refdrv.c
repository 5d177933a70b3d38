/* vad_live_refdrv.c -- one live stream through the compiled reference's endpointer, fed in chunks as
 * audio arrives: the samples after a chunk's last full frame wait for the next chunk,
 * ps_endpointer_process runs on every frame a chunk completes, and ps_endpointer_end_stream with the
 * waiting samples where a chunk is final (the stream then goes on with the same endpointer, as the
 * reference allows).  A ps_vad_t fed the same frames gives the decisions (ps_endpointer_end_stream
 * leaves the endpointer's own VAD alone, so the two stay equal).  Linked against libpsref.so; only
 * its public entry points are used, declared here.
 *
 * Sample positions count the samples of full frames since the stream was made fresh: frame f
 * starts at f * frame_size.  The driver knows which frame the endpointer returns from the queue
 * length, which follows from ps_endpointer_in_speech before and after each call (a push adds one
 * frame up to maxlen, a call that is or becomes in speech pops one, end_stream in speech empties
 * it), and checks every returned sample against the frame it claims. */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct ps_vad_s ps_vad_t;
typedef struct ps_endpointer_s ps_endpointer_t;
ps_vad_t *ps_vad_init(int mode, int sample_rate, double frame_length);
int ps_vad_free(ps_vad_t *vad);
size_t ps_vad_frame_size(ps_vad_t *vad);
int ps_vad_classify(ps_vad_t *vad, const short *frame);
ps_endpointer_t *ps_endpointer_init(double window, double ratio, int mode, int sample_rate, double frame_length);
int ps_endpointer_free(ps_endpointer_t *ep);
ps_vad_t *ps_endpointer_vad(ps_endpointer_t *ep);
const short *ps_endpointer_process(ps_endpointer_t *ep, const short *frame);
const short *ps_endpointer_end_stream(ps_endpointer_t *ep, const short *frame, size_t nsamp, size_t *out_nsamp);
int ps_endpointer_in_speech(ps_endpointer_t *ep);
double ps_endpointer_speech_start(ps_endpointer_t *ep);
double ps_endpointer_speech_end(ps_endpointer_t *ep);

typedef struct {
    double window, ratio, frame_length;
    int mode, rate, fs, maxlen, ring;
    ps_endpointer_t *ep;
    ps_vad_t *vad;
    short *frames;                /* the last `ring` frames, frame f at (f % ring) * fs */
    short *left;                  /* samples after the last full frame */
    int n_left, n;                /* waiting samples; the endpointer's queue length */
    int64_t pushed, start, pos;   /* frames so far; the open segment's first sample and its end so far */
} live_t;

static int live_fresh(live_t *h)
{
    if (h->ep) ps_endpointer_free(h->ep);
    if (h->vad) ps_vad_free(h->vad);
    h->ep = ps_endpointer_init(h->window, h->ratio, h->mode, h->rate, h->frame_length);
    h->vad = ps_vad_init(h->mode, h->rate, h->frame_length);
    h->n_left = h->n = 0;
    h->pushed = h->start = h->pos = 0;
    return h->ep && h->vad ? 0 : -1;
}

/* NULL where ps_endpointer_init refuses */
void *refdrv_live_open(double window, double ratio, int mode, int rate, double frame_length, int maxlen)
{
    live_t *h = (live_t *)calloc(1, sizeof(live_t));
    h->window = window, h->ratio = ratio, h->frame_length = frame_length, h->mode = mode, h->rate = rate;
    if (live_fresh(h)) {
        if (h->ep) ps_endpointer_free(h->ep);
        if (h->vad) ps_vad_free(h->vad);
        free(h);
        return NULL;
    }
    h->fs = (int)ps_vad_frame_size(ps_endpointer_vad(h->ep));
    h->maxlen = maxlen;
    h->ring = maxlen + 2;
    h->frames = (short *)malloc(sizeof(short) * (size_t)h->ring * h->fs);
    h->left = (short *)malloc(sizeof(short) * (size_t)h->fs);
    return h;
}

void refdrv_live_free(void *p)
{
    live_t *h = (live_t *)p;
    ps_endpointer_free(h->ep);
    ps_vad_free(h->vad);
    free(h->frames);
    free(h->left);
    free(h);
}

/* a fresh ps_endpointer_init for the same stream slot */
int refdrv_live_reset(void *p) { return live_fresh((live_t *)p); }

static void seg_out(live_t *h, int64_t *segs, double *times, long k)
{
    segs[2 * k] = h->start;
    segs[2 * k + 1] = h->pos;
    times[2 * k] = ps_endpointer_speech_start(h->ep);
    times[2 * k + 1] = ps_endpointer_speech_end(h->ep);
}

/* Feeds nsamp samples, then ends the stream if `final`.  flags: the decision of every frame the chunk completes
 * (status[2] - the previous call's status[2] of them); segs [k][2] / times [k][2]: the segments that ended;
 * status: in_speech, the open segment's first sample (-1 when not in speech), frames so far; st_times:
 * ps_endpointer_speech_start / _speech_end.  Returns the segment count, -2 if the returned audio is not the frames it
 * should be, -3 if cap is too small. */
long refdrv_live_feed(void *p, const short *pcm, long nsamp, int final, signed char *flags, int64_t *segs, double *times,
                      long cap, int64_t *status, double *st_times)
{
    live_t *h = (live_t *)p;
    const int fs = h->fs;
    long k = 0, nfl = 0;
    for (long i = 0; i < nsamp;) {
        long take = fs - h->n_left;
        if (take > nsamp - i) take = nsamp - i;
        memcpy(h->left + h->n_left, pcm + i, sizeof(short) * (size_t)take);
        h->n_left += (int)take;
        i += take;
        if (h->n_left < fs) break;
        const int64_t f = h->pushed;
        short *fr = h->frames + (size_t)(f % h->ring) * fs;
        memcpy(fr, h->left, sizeof(short) * (size_t)fs);
        h->n_left = 0;
        flags[nfl++] = (signed char)ps_vad_classify(h->vad, fr);
        const int before = ps_endpointer_in_speech(h->ep);
        const short *out = ps_endpointer_process(h->ep, fr);
        const int after = ps_endpointer_in_speech(h->ep);
        h->pushed++;
        const int n1 = h->n + 1 < h->maxlen ? h->n + 1 : h->maxlen;
        const int64_t head = h->pushed - n1;                     /* the queue's first frame before any pop */
        h->n = n1;
        if (!before && after) h->start = h->pos = head * fs;
        if (before || after) {
            h->n--;
            if (!out || memcmp(out, h->frames + (size_t)(head % h->ring) * fs, sizeof(short) * (size_t)fs)) return -2;
            h->pos += fs;
        } else if (out) {
            return -2;
        }
        if (before && !after) {
            if (k == cap) return -3;
            seg_out(h, segs, times, k++);
        }
    }
    if (final) {
        const int before = ps_endpointer_in_speech(h->ep);
        size_t got = 0;
        const short *out = ps_endpointer_end_stream(h->ep, h->left, (size_t)h->n_left, &got);
        if (before) {
            const int64_t head = h->pushed - h->n;
            const size_t whole = got / (size_t)fs * (size_t)fs;
            if (!out) return -2;
            for (size_t j = 0; j < whole; j += (size_t)fs)
                if (memcmp(out + j, h->frames + (size_t)((head + (int64_t)(j / fs)) % h->ring) * fs, sizeof(short) * (size_t)fs))
                    return -2;
            if (got > whole && memcmp(out + whole, h->left, sizeof(short) * (got - whole))) return -2;
            h->pos += (int64_t)got;
            h->n = 0;
            if (k == cap) return -3;
            seg_out(h, segs, times, k++);
        } else if (out) {
            return -2;
        }
        h->n_left = 0;
    }
    status[0] = ps_endpointer_in_speech(h->ep);
    status[1] = status[0] ? h->start : -1;
    status[2] = h->pushed;
    st_times[0] = ps_endpointer_speech_start(h->ep);
    st_times[1] = ps_endpointer_speech_end(h->ep);
    return k;
}
