// psb_pitch_core.h -- the integer arithmetic of the reference's YIN pitch tracker (fe/yin.c) and the
// read schedule of pocketsphinx_pitch's extract_pitch loop, as __host__ __device__ functions.  psb_pitch.cu's
// kernels and tests/emul/pitch_emul.cpp / pitch_live_emul.cpp (the CPU restatements the tests pin against the
// compiled reference) are built from this one file.
//
// Restated as gcc -O3 on x86-64 executes the reference (checked against its disassembly):
//   cmn_diff            yin.c:69-128   the square of a difference wraps in int; it is shifted arithmetically
//                                      by dshift & 31 (x86 masks 32-bit shift counts); the cum alignment shifts
//                                      by (dshift - cshift) & 31 or (cshift - dshift) & 31; the final 64-bit
//                                      shift count (tscale - 15 + cshift - dshift) is unsigned and masked to 63
//   thresholded_search  yin.c:171-192
//   yin_write/yin_read  yin.c:194-322  the ring of wsize slots: unsigned char pointers, a uint16 frame count
// CUDA clamps shift counts instead of masking them, so every mask is written out.
#ifndef PSB_PITCH_CORE_H
#define PSB_PITCH_CORE_H

#include <limits.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __CUDACC__
#define PSB_PITCH_HD __host__ __device__ __forceinline__
#define PSB_PITCH_MEMBER __host__ __device__ __forceinline__
#else
#define PSB_PITCH_HD static inline
#define PSB_PITCH_MEMBER inline
#endif

// how many bits t can be scaled up by in cmn_diff: one below the count of leading zeros of ndiff
PSB_PITCH_HD int psb_pitch_tscale(int ndiff)
{
    int tscale;
    for (tscale = 0; tscale < 32; ++tscale)
        if ((uint32_t)ndiff & (1u << (31 - tscale))) break;
    return tscale - 1;
}

// Lag t's sum of squared differences with its running renormalisation: *dd and *dshift as cmn_diff leaves them.
PSB_PITCH_HD void psb_pitch_lag_sum(const int16_t *sig, int t, int ndiff, int tscale, uint32_t *dd_out, uint32_t *dshift_out)
{
    const uint64_t lim = (uint64_t)1 << tscale;
    uint32_t dd = 0, dshift = 0;
    for (int j = 0; j < ndiff; ++j) {
        const int32_t diff = (int32_t)sig[j] - (int32_t)sig[t + j];
        if ((uint64_t)dd > lim) {
            dd >>= 1;
            ++dshift;
        }
        const int32_t sq = (int32_t)((uint32_t)diff * (uint32_t)diff);     // wraps for |diff| > 46340
        dd += (uint32_t)(sq >> (dshift & 31));                             // sar
    }
    *dd_out = dd;
    *dshift_out = dshift;
}

// One step of the cumulative sum over lags (sequential in t): adds lag t's dd at cum's scale, renormalises.
PSB_PITCH_HD void psb_pitch_cum_step(uint32_t dd, uint32_t dshift, int tscale, uint32_t *cum, uint32_t *cshift)
{
    const uint64_t lim = (uint64_t)1 << tscale;
    uint32_t c = *cum, cs = *cshift;
    if (dshift > cs) c += dd << ((dshift - cs) & 31);
    else c += dd >> ((cs - dshift) & 31);
    while ((uint64_t)c > lim) {
        c >>= 1;
        ++cs;
    }
    if (c == 0) c = 1;
    *cum = c;
    *cshift = cs;
}

// out_diff[t] from lag t's dd / dshift and the cum / cshift the chain had after lag t
PSB_PITCH_HD int32_t psb_pitch_cmn(int t, uint32_t dd, uint32_t dshift, uint32_t cum, uint32_t cshift, int tscale)
{
    const uint32_t norm = ((uint32_t)t << tscale) / cum;
    const uint32_t sh = ((uint32_t)(tscale - 15) + cshift - dshift) & 63;
    return (int32_t)(uint32_t)(((uint64_t)dd * norm) >> sh);               // the product is below 2^63: sar == shr
}

// thresholded_search: the first index in [start, end) below threshold, else the first index of the minimum
// (0 when the range is empty or every value is INT_MAX).  row == nullptr reads a never-written slot: zeros.
PSB_PITCH_HD int psb_pitch_search(const int32_t *row, int32_t threshold, int start, int end)
{
    int32_t mn = INT_MAX;
    int argmin = 0;
    for (int i = start; i < end; ++i) {
        const int32_t d = row ? row[i] : 0;
        if (d < threshold) return i;
        if (d < mn) {
            mn = d;
            argmin = i;
        }
    }
    return argmin;
}

// ---------------------------------------------------------------------------------------------------------------
// The read schedule (frame counts below 2^31).  extract_pitch calls yin_write then yin_read once per frame, then
// yin_end and yin_read until it fails.  Which reads succeed, which slot holds which frame, the current slot and the
// window depend only on the frame count, so each output can be placed without running the ring.

enum { PSB_PITCH_NFR_WRAP = 65536 };    // yin_t.nfr is a uint16

// reads that succeed inside the main loop of a stream of n_frames (half = smooth_window): a read after F frames
// succeeds when (uint16)F > half, so every 65 536 frames half + 1 reads fail
PSB_PITCH_HD int32_t psb_pitch_main_reads(int32_t n_frames, int half)
{
    if (half == 0) return n_frames;
    const int32_t per = PSB_PITCH_NFR_WRAP - 1 - half, r = n_frames % PSB_PITCH_NFR_WRAP;
    return n_frames / PSB_PITCH_NFR_WRAP * per + (r > half ? r - half : 0);
}

// all reads of a stream: the main loop's, then the drain until wcur reaches wstart (none without smoothing)
PSB_PITCH_HD int32_t psb_pitch_n_reads(int32_t n_frames, int half)
{
    const int32_t m = psb_pitch_main_reads(n_frames, half);
    if (half == 0) return m;
    const int wsize = 2 * half + 1;
    return m + ((n_frames - m) % wsize);
}

// reads of one live call that takes a slot from f0 to f1 frames: the main loop's reads of the new frames, and on a
// final call the drain after them (at most f1 - f0 + 2 * half)
PSB_PITCH_HD int32_t psb_pitch_live_reads(int32_t f0, int32_t f1, int half, int final)
{
    return (final ? psb_pitch_n_reads(f1, half) : psb_pitch_main_reads(f1, half)) - psb_pitch_main_reads(f0, half);
}

// the frame slot `slot` holds after F writes (frame f goes to slot f % wsize), -1 when never written
PSB_PITCH_HD int32_t psb_pitch_slot_frame(int slot, int32_t F, int wsize)
{
    return F > slot ? slot + (F - 1 - slot) / wsize * wsize : -1;
}

// Read k of a stream of n_frames: frames written at that read (*F), whether it is a main-loop read, the
// current slot and the window (first slot, length).
struct psb_pitch_read_t {
    int32_t F;
    int main_loop;
    int wcur, wstart, wlen;
};

PSB_PITCH_HD psb_pitch_read_t psb_pitch_read_at(int32_t k, int32_t n_frames, int half)
{
    psb_pitch_read_t r;
    const int wsize = 2 * half + 1;
    r.wcur = (int)(k % wsize);
    if (half == 0) {
        r.F = k + 1, r.main_loop = 1, r.wstart = 0, r.wlen = 0;
        return r;
    }
    const int32_t m = psb_pitch_main_reads(n_frames, half);
    if (k < m) {
        const int32_t per = PSB_PITCH_NFR_WRAP - 1 - half;
        r.F = k / per * PSB_PITCH_NFR_WRAP + half + 1 + k % per;
        r.main_loop = 1;
        const int nfr = (int)(r.F % PSB_PITCH_NFR_WRAP);
        if (nfr < wsize) r.wstart = 0, r.wlen = nfr;
        else r.wstart = (int)(r.F % wsize), r.wlen = wsize;
    } else {
        r.F = n_frames;
        r.main_loop = 0;
        r.wstart = (r.wcur + wsize - half) % wsize;
        const int ws = (int)(n_frames % wsize);
        r.wlen = ws - r.wstart;
        if (r.wlen < 0) r.wlen += wsize;
    }
    return r;
}

// A live slot's frames as one call's reads see them: frames f0 and later were written by this call and sit in `call`
// (frame f at f - f0), earlier ones in the slot's ring of wsize entries (frame f at f % wsize, as diff_window keeps
// them).  stride: values per frame, 1 for periods and diffs, ndiff for rows.  A read of this call needs no frame
// before f0 - wsize: its window ends at the frames written when it is made, never fewer than f0.
struct psb_pitch_live_frames_t {
    const int32_t *call, *ring;
    int32_t f0;
    int wsize, stride;
    PSB_PITCH_MEMBER const int32_t *at(int32_t f) const
    {
        return f >= f0 ? call + (size_t)(f - f0) * stride : ring + (size_t)(f % wsize) * stride;
    }
    PSB_PITCH_MEMBER int32_t operator[](int32_t f) const { return *at(f); }
};

// The decision of one yin_read.  period[f] / pdiff[f] are frame f's period and diff at that period; row(f) is frame
// f's diff row (ndiff values).  period / pdiff are arrays indexed by frame, or accessors with an operator[] that
// finds frame f elsewhere (a live slot's ring).  A never-written slot reads period 0, diff 0 and a row of zeros.
template <class PeriodOf, class DiffOf, class RowOf>
PSB_PITCH_HD void psb_pitch_decide(const psb_pitch_read_t &r, int half, int ndiff, int32_t threshold, int32_t range,
                                   const PeriodOf &period, const DiffOf &pdiff, RowOf row, uint16_t *out_period,
                                   uint16_t *out_bestdiff)
{
    const int wsize = 2 * half + 1;
    const int32_t cf = psb_pitch_slot_frame(r.wcur, r.F, wsize);
    const int cur_period = cf >= 0 ? period[cf] : 0;
    if (half == 0) {
        *out_period = (uint16_t)cur_period;
        *out_bestdiff = (uint16_t)(cf >= 0 ? pdiff[cf] : 0);
        return;
    }
    int best = cur_period;
    int32_t best_diff = cf >= 0 ? pdiff[cf] : 0;
    for (int i = 0; i < r.wlen; ++i) {
        const int32_t f = psb_pitch_slot_frame((r.wstart + i) % wsize, r.F, wsize);
        const int32_t d = f >= 0 ? pdiff[f] : 0;
        if (d < best_diff) {
            best_diff = d;
            best = f >= 0 ? period[f] : 0;
        }
    }
    if (best == cur_period) {
        *out_period = (uint16_t)best;
        *out_bestdiff = (uint16_t)best_diff;
        return;
    }
    int width = best * range / 32768;
    if (width == 0) width = 1;
    int lo = best - width, hi = best + width;
    if (lo < 0) lo = 0;
    if (hi > ndiff) hi = ndiff;
    const int32_t *cr = cf >= 0 ? row(cf) : nullptr;
    best = psb_pitch_search(cr, threshold, lo, hi);
    best_diff = cr ? cr[best] : 0;
    *out_period = (uint16_t)(best > 32768 ? 32768 : best);
    *out_bestdiff = (uint16_t)(best_diff > 32768 ? 32768 : best_diff);
}

#endif  // PSB_PITCH_CORE_H
