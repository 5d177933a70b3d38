/* pitch_refdrv.c -- the loop of the reference's extract_pitch (programs/pocketsphinx_pitch.c) over the compiled
 * reference's yin_* (oracle/_ref/libpsref.so), for one stream in memory: yin_write and yin_read on every frame,
 * then yin_end and yin_read until it fails.  Frame f is samples f * fshift .. f * fshift + flen - 1, which is what
 * the program's memmove / fread loop hands yin_write. */
#include <stdint.h>

typedef struct yin_s yin_t;
yin_t *yin_init(int frame_size, float search_threshold, float search_range, int smooth_window);
void yin_free(yin_t *pe);
void yin_start(yin_t *pe);
void yin_end(yin_t *pe);
void yin_write(yin_t *pe, int16_t const *frame);
int yin_read(yin_t *pe, uint16_t *out_period, uint16_t *out_bestdiff);

/* period / bestdiff of every read that succeeds (room for one per frame); returns the reads, *n_main the main
 * loop's */
long refdrv_pitch_run(const int16_t *pcm, long n, int flen, int fshift, float voice_thresh, float search_range,
                      int smooth_window, uint16_t *period, uint16_t *bestdiff, long *n_main)
{
    yin_t *yin = yin_init(flen, voice_thresh, search_range, smooth_window);
    long nf = n >= flen ? 1 + (n - flen) / fshift : 0, k = 0, f;
    yin_start(yin);
    for (f = 0; f < nf; ++f) {
        yin_write(yin, pcm + f * fshift);
        if (yin_read(yin, &period[k], &bestdiff[k])) ++k;
    }
    *n_main = k;
    yin_end(yin);
    while (yin_read(yin, &period[k], &bestdiff[k])) ++k;
    yin_free(yin);
    return k;
}
