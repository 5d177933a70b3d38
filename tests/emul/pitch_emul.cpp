// pitch_emul.cpp -- pocketsphinx_b200/csrc/psb_pitch_core.h built for the host: the per-frame difference rows as
// pitch_diff_kernel computes them (lag sums, then the cum chain, then out_diff), and every read through the same
// schedule and decision pitch_read_kernel uses.  tests/test_pitch_oracle.py pins it against the compiled reference.
#include <stdint.h>

#include <vector>

#include "../../pocketsphinx_b200/csrc/psb_pitch_core.h"

extern "C" {

// frames of a stream as extract_pitch reads them
long pitch_emul_frames(long n, int flen, int fshift) { return n >= flen ? 1 + (n - flen) / fshift : 0; }

// One stream: period / bestdiff of every read (room for one per frame); returns the reads, *n_main the main loop's.
long pitch_emul_run(const int16_t *pcm, long n, int flen, int fshift, int threshold, int range, int smooth_window,
                    uint16_t *period, uint16_t *bestdiff, long *n_main)
{
    const int nf = (int)pitch_emul_frames(n, flen, fshift), ndiff = flen / 2, tscale = psb_pitch_tscale(ndiff);
    std::vector<int32_t> rows((size_t)nf * ndiff), per(nf), pd(nf);
    std::vector<uint32_t> dd(ndiff), dsh(ndiff);
    for (int f = 0; f < nf; ++f) {
        const int16_t *x = pcm + (long)f * fshift;
        int32_t *row = &rows[(size_t)f * ndiff];
        for (int t = 1; t < ndiff; ++t) psb_pitch_lag_sum(x, t, ndiff, tscale, &dd[t], &dsh[t]);
        row[0] = 32768;
        uint32_t cum = 0, cshift = 0;
        for (int t = 1; t < ndiff; ++t) {
            psb_pitch_cum_step(dd[t], dsh[t], tscale, &cum, &cshift);
            row[t] = psb_pitch_cmn(t, dd[t], dsh[t], cum, cshift, tscale);
        }
        per[f] = psb_pitch_search(row, threshold, 0, ndiff);
        pd[f] = row[per[f]];
    }
    const int reads = psb_pitch_n_reads(nf, smooth_window);
    for (int k = 0; k < reads; ++k) {
        const psb_pitch_read_t r = psb_pitch_read_at(k, nf, smooth_window);
        psb_pitch_decide(r, smooth_window, ndiff, threshold, range, per.data(), pd.data(),
                         [&](int32_t f) { return &rows[(size_t)f * ndiff]; }, period + k, bestdiff + k);
    }
    *n_main = psb_pitch_main_reads(nf, smooth_window);
    return reads;
}

}  // extern "C"
