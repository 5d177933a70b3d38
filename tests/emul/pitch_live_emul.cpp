// pitch_live_emul.cpp -- one live slot of psb_pitch_feed_* restated on the host over psb_pitch_core.h, with the state
// the device keeps between calls and nothing else: the samples from the next frame's start on, and the ring of the
// last wsize frames (row, period, diff at the period; frame f at f % wsize).  Each call stitches the leftover to the
// new samples, computes the new frames' rows as pitch_diff_kernel does, makes the call's reads through the schedule
// with earlier frames taken from the ring (psb_pitch_live_frames_t, as pitch_live_read_kernel), then stores the last
// min(wsize, new frames) frames and the new leftover, as pitch_store_kernel.
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "../../pocketsphinx_b200/csrc/psb_pitch_core.h"

namespace {

struct slot_t {
    int flen, fshift, ndiff, tscale, half, wsize;
    int32_t threshold, range;
    std::vector<int16_t> left;                 // the samples from the next frame's start on
    std::vector<int32_t> ring_rows, ring_period, ring_pdiff;
    int64_t samples = 0;
    int32_t frames = 0, reads = 0;
    int ended = 0;
};

}  // namespace

extern "C" {

void *pitch_live_emul_open(int flen, int fshift, int threshold, int range, int smooth_window)
{
    slot_t *h = new slot_t();
    h->flen = flen, h->fshift = fshift, h->ndiff = flen / 2, h->tscale = psb_pitch_tscale(h->ndiff);
    h->half = smooth_window, h->wsize = 2 * smooth_window + 1;
    h->threshold = threshold, h->range = range;
    h->ring_rows.assign((size_t)h->wsize * h->ndiff, 0);
    h->ring_period.assign((size_t)h->wsize, 0);
    h->ring_pdiff.assign((size_t)h->wsize, 0);
    return h;
}

void pitch_live_emul_free(void *p) { delete static_cast<slot_t *>(p); }

// a fresh slot: no samples, no frames (the ring's contents are never read before they are written)
void pitch_live_emul_reset(void *p)
{
    slot_t *h = static_cast<slot_t *>(p);
    h->left.clear();
    h->samples = 0, h->frames = 0, h->reads = 0, h->ended = 0;
}

// as refdrv_pitch_live_feed (tests/emul/pitch_live_refdrv.c)
long pitch_live_emul_feed(void *p, const int16_t *pcm, long n, int final, uint16_t *period, uint16_t *bestdiff,
                          int32_t *status)
{
    slot_t *h = static_cast<slot_t *>(p);
    if (h->ended) return -1;
    std::vector<int16_t> x(h->left);
    x.insert(x.end(), pcm, pcm + n);
    const int64_t len = (int64_t)x.size();
    const int32_t nf = len >= h->flen ? (int32_t)(1 + (len - h->flen) / h->fshift) : 0;
    const int32_t f0 = h->frames, f1 = f0 + nf, ndiff = h->ndiff;
    std::vector<int32_t> rows((size_t)nf * ndiff), per(nf), pd(nf);
    std::vector<uint32_t> dd(ndiff), dsh(ndiff);
    for (int f = 0; f < nf; ++f) {
        const int16_t *s = x.data() + (size_t)f * h->fshift;
        int32_t *row = &rows[(size_t)f * ndiff];
        for (int t = 1; t < ndiff; ++t) psb_pitch_lag_sum(s, t, ndiff, h->tscale, &dd[t], &dsh[t]);
        row[0] = 32768;
        uint32_t cum = 0, cshift = 0;
        for (int t = 1; t < ndiff; ++t) {
            psb_pitch_cum_step(dd[t], dsh[t], h->tscale, &cum, &cshift);
            row[t] = psb_pitch_cmn(t, dd[t], dsh[t], cum, cshift, h->tscale);
        }
        per[f] = psb_pitch_search(row, h->threshold, 0, ndiff);
        pd[f] = row[per[f]];
    }
    const int32_t k0 = psb_pitch_main_reads(f0, h->half), reads = psb_pitch_live_reads(f0, f1, h->half, final);
    const psb_pitch_live_frames_t pf{per.data(), h->ring_period.data(), f0, h->wsize, 1};
    const psb_pitch_live_frames_t df{pd.data(), h->ring_pdiff.data(), f0, h->wsize, 1};
    const psb_pitch_live_frames_t rf{rows.data(), h->ring_rows.data(), f0, h->wsize, ndiff};
    for (int32_t j = 0; j < reads; ++j) {
        const psb_pitch_read_t r = psb_pitch_read_at(k0 + j, f1, h->half);
        psb_pitch_decide(r, h->half, ndiff, h->threshold, h->range, pf, df, [&](int32_t f) { return rf.at(f); },
                         period + j, bestdiff + j);
    }
    // save: the last min(wsize, nf) frames into the ring, the samples from the next frame's start on
    const int keep = std::min<int32_t>(h->wsize, nf);
    for (int32_t f = f1 - keep; f < f1; ++f) {
        const int e = f % h->wsize, c = f - f0;
        std::copy(&rows[(size_t)c * ndiff], &rows[(size_t)(c + 1) * ndiff], &h->ring_rows[(size_t)e * ndiff]);
        h->ring_period[e] = per[c];
        h->ring_pdiff[e] = pd[c];
    }
    h->left.assign(x.begin() + (int64_t)nf * h->fshift, x.end());
    h->samples += n;
    h->frames = f1;
    h->reads += reads;
    h->ended = final ? 1 : 0;
    status[0] = h->frames;
    status[1] = psb_pitch_main_reads(h->frames, h->half);
    status[2] = h->reads;
    status[3] = h->ended;
    return reads;
}

}  // extern "C"
