/* vad_refdrv.c -- loops the compiled reference's VAD and endpointer over whole streams in C, so a
 * test makes one ctypes call per stream instead of one per frame.  Linked against the reference
 * library (libpsref.so); only its public entry points are used, declared here. */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

typedef struct ps_vad_s ps_vad_t;
typedef struct ps_endpointer_s ps_endpointer_t;
ps_vad_t *ps_vad_init(int mode, int sample_rate, double frame_length);
int ps_vad_free(ps_vad_t *vad);
size_t ps_vad_frame_size(ps_vad_t *vad);
int ps_vad_sample_rate(ps_vad_t *vad);
int ps_vad_classify(ps_vad_t *vad, const short *frame);
ps_endpointer_t *ps_endpointer_init(double window, double ratio, int mode, int sample_rate, double frame_length);
int ps_endpointer_free(ps_endpointer_t *ep);
ps_vad_t *ps_endpointer_vad(ps_endpointer_t *ep);
const short *ps_endpointer_process(ps_endpointer_t *ep, const short *frame);
const short *ps_endpointer_end_stream(ps_endpointer_t *ep, const short *frame, size_t nsamp, size_t *out_nsamp);
int ps_endpointer_in_speech(ps_endpointer_t *ep);
double ps_endpointer_speech_start(ps_endpointer_t *ep);
double ps_endpointer_speech_end(ps_endpointer_t *ep);

/* frame size and the rate ps_vad_init settles on; -1 where it refuses */
int refdrv_vad_params(int mode, int rate, double frame_length, int *frame_size, int *sample_rate)
{
    ps_vad_t *v = ps_vad_init(mode, rate, frame_length);
    if (!v) return -1;
    *frame_size = (int)ps_vad_frame_size(v);
    *sample_rate = ps_vad_sample_rate(v);
    ps_vad_free(v);
    return 0;
}

/* ps_vad_classify on every full frame of a fresh ps_vad_init(mode, rate, frame_length); with
 * `states` non-NULL, the first state_bytes of the instance (ps_vad_t starts with the VadInstT)
 * after every frame.  Returns the frame count, -1 if ps_vad_init refuses. */
long refdrv_vad_run(int mode, int rate, double frame_length, const short *pcm, long nsamp, signed char *flags,
                    unsigned char *states, long state_bytes)
{
    ps_vad_t *v = ps_vad_init(mode, rate, frame_length);
    if (!v) return -1;
    const long fs = (long)ps_vad_frame_size(v), nf = nsamp / fs;
    for (long f = 0; f < nf; ++f) {
        flags[f] = (signed char)ps_vad_classify(v, pcm + f * fs);
        if (states) memcpy(states + f * state_bytes, (const void *)v, (size_t)state_bytes);
    }
    ps_vad_free(v);
    return nf;
}

/* ps_endpointer_process on every full frame, then ps_endpointer_end_stream with the rest.
 * Segment i: segs[2i] = first sample, segs[2i + 1] = one past the last, times[2i], times[2i + 1] =
 * ps_endpointer_speech_start / _speech_end.  The first sample is the stream position of the
 * speech start time; every sample the endpointer returns is checked against the stream at the
 * position it claims.  Returns the segment count, -1 if ps_endpointer_init refuses, -2 if the
 * returned audio is not the stream's, -3 if cap is too small. */
long refdrv_endpoint_run(double window, double ratio, int mode, int rate, double frame_length, const short *pcm,
                         long nsamp, int64_t *segs, double *times, long cap)
{
    ps_endpointer_t *ep = ps_endpointer_init(window, ratio, mode, rate, frame_length);
    if (!ep) return -1;
    const long fs = (long)ps_vad_frame_size(ps_endpointer_vad(ep));
    const double fl = (double)fs / ps_vad_sample_rate(ps_endpointer_vad(ep));
    const long nf = nsamp / fs;
    long n = 0, rc = 0;
    int open = 0;
    int64_t start = 0, pos = 0;
    for (long f = 0; f <= nf && rc == 0; ++f) {
        size_t got = (size_t)fs;
        const short *out = f < nf ? ps_endpointer_process(ep, pcm + f * fs)
                                  : ps_endpointer_end_stream(ep, pcm + f * fs, (size_t)(nsamp - nf * fs), &got);
        if (!out) continue;
        if (!open) {
            if (n == cap) { rc = -3; break; }
            start = (int64_t)(ps_endpointer_speech_start(ep) / fl + 0.5) * fs;
            pos = start;
            open = 1;
        }
        if (pos + (int64_t)got > nsamp || memcmp(out, pcm + pos, got * sizeof(short)) != 0) { rc = -2; break; }
        pos += (int64_t)got;
        if (f == nf || !ps_endpointer_in_speech(ep)) {
            segs[2 * n] = start;
            segs[2 * n + 1] = pos;
            times[2 * n] = ps_endpointer_speech_start(ep);
            times[2 * n + 1] = ps_endpointer_speech_end(ep);
            ++n;
            open = 0;
        }
    }
    ps_endpointer_free(ep);
    return rc ? rc : n;
}
