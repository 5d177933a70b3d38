// psb_pitch.cu -- YIN pitch tracking for whole batches of int16 streams (fe/yin.c driven as pocketsphinx_pitch's
// extract_pitch drives it, one fresh yin_t per stream).  The arithmetic is psb_pitch_core.h's; this file owns the
// launch shapes.
//
// Two stages, because a frame's difference row does not depend on any other frame and the smoothing only reads rows:
//   pitch_diff_kernel  one CTA per frame: the frame's samples in shared memory, one thread per lag for the
//                      sequential dd / dshift chain, thread 0 for the sequential cum / cshift chain over the lags
//                      (its truncating shifts do not reassociate), then every lag's out_diff in parallel and a block
//                      reduction for thresholded_search's answer.  Rows stay in device memory.
//   pitch_read_kernel  one thread per yin_read that succeeds: the schedule (psb_pitch_read_at) places the read from
//                      the stream's frame count alone; the window minimum and the narrowed search read the rows.
//
// Live calls (psb_pitch_feed_*) keep n_slots streams.  Per slot on the device: the samples from its next frame's start
// on (fewer than flen) and the ring of its last wsize frames (row, period, diff at the period, frame f at f % wsize);
// on the host: samples and frames so far and whether it has ended.  A call runs
//   pitch_stitch_kernel     each fed slot's leftover, then its new samples, into one buffer
//   pitch_diff_kernel       unchanged, over the stitched streams
//   pitch_live_read_kernel  as pitch_read_kernel, with frames before the call taken from the slot's ring
//   pitch_store_kernel      the call's last min(wsize, new frames) frames into the ring, the new leftover
// in stream order, so the ring is read before it is overwritten.
#include "psb_internal.cuh"
#include "psb_pitch_core.h"

#include <math.h>

#include <algorithm>
#include <memory>
#include <vector>

namespace {

constexpr int PITCH_MAX_THREADS = 512;
constexpr int PITCH_READ_THREADS = 256;
constexpr int PITCH_COPY_THREADS = 256;

// one fed slot of a live call: its frames before and after the call, and the index of its first read in this call
struct LiveSlot {
    int32_t slot, f0, f1, k0;
};

}  // namespace

struct psb_pitch_s {
    int device;
    int sample_rate, flen, fshift, ndiff, tscale, half, threads;
    int32_t threshold, range;      // Q15, as yin_init stores them
    size_t smem;
    Stream stream;                 // declared first: destroyed after the buffers below
    Event ev[2];
    DevBuf<int16_t> d_pcm;
    DevBuf<int64_t> d_samp_off;
    DevBuf<int32_t> d_frame_off, d_out_off;
    DevBuf<int32_t> d_rows;        // [frames][ndiff]: every frame's cumulative-mean-normalised difference row
    DevBuf<int32_t> d_period;      // [frames]: thresholded_search over the whole row
    DevBuf<int32_t> d_pdiff;       // [frames]: the row's value at that period
    DevBuf<uint16_t> d_out;        // _host: [2][reads] period, bestdiff
    // live slots (psb_pitch_live_open); the host mirrors each slot's samples, frames and ended flag
    int32_t n_slots = 0;
    std::vector<int64_t> samples;
    std::vector<int32_t> frames;
    std::vector<int8_t> ended;
    DevBuf<int16_t> d_left;        // [slots][flen]: the samples from the slot's next frame start on
    DevBuf<int32_t> d_ring_rows;   // [slots][wsize][ndiff]: the slot's frame f's row at f % wsize
    DevBuf<int32_t> d_ring_period; // [slots][wsize]
    DevBuf<int32_t> d_ring_pdiff;  // [slots][wsize]
    DevBuf<int16_t> d_stitch;      // a live call's streams: each fed slot's leftover, then its new samples
    DevBuf<int64_t> d_new_off;     // [n + 1]: the new samples' offsets
    DevBuf<LiveSlot> d_live;       // [n]
};

namespace {

// the last stream whose first index is at or before i (offsets of n streams, off[n] > i)
template <class T>
__device__ __forceinline__ int stream_of(const T *off, int n, T i)
{
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// shared memory of pitch_diff_kernel: dd, dshift, cum, cshift per lag, the reduction's 2 x 32 words, the samples
size_t diff_smem(int flen, int ndiff) { return (size_t)4 * ndiff * 4 + 64 * 8 + (((size_t)flen * 2 + 15) & ~(size_t)15); }

__global__ void __launch_bounds__(PITCH_MAX_THREADS) pitch_diff_kernel(
    const int16_t *__restrict__ pcm, const int64_t *__restrict__ samp_off, const int32_t *__restrict__ frame_off,
    int32_t n_streams, int flen, int fshift, int ndiff, int tscale, int32_t threshold, int32_t *__restrict__ rows,
    int32_t *__restrict__ period, int32_t *__restrict__ pdiff)
{
    extern __shared__ __align__(16) uint32_t pitch_sm[];
    uint32_t *s_dd = pitch_sm, *s_dsh = s_dd + ndiff, *s_cum = s_dsh + ndiff, *s_csh = s_cum + ndiff;
    unsigned long long *s_key = reinterpret_cast<unsigned long long *>(pitch_sm + ((4 * ndiff + 1) & ~1));
    uint32_t *s_thr = reinterpret_cast<uint32_t *>(s_key + 32);
    int16_t *s_sig = reinterpret_cast<int16_t *>(s_key + 64);
    const int g = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int s = stream_of(frame_off, n_streams, g);
    const int16_t *x = pcm + samp_off[s] + (int64_t)(g - frame_off[s]) * fshift;
    for (int i = tid; i < flen; i += nt) s_sig[i] = x[i];
    __syncthreads();
    for (int t = tid; t < ndiff; t += nt)
        if (t > 0) psb_pitch_lag_sum(s_sig, t, ndiff, tscale, &s_dd[t], &s_dsh[t]);
    __syncthreads();
    if (tid == 0) {
        uint32_t cum = 0, cshift = 0;
        for (int t = 1; t < ndiff; ++t) {
            psb_pitch_cum_step(s_dd[t], s_dsh[t], tscale, &cum, &cshift);
            s_cum[t] = cum;
            s_csh[t] = cshift;
        }
    }
    __syncthreads();
    // thresholded_search over [0, ndiff): the first lag below threshold, else the first lag of the minimum
    uint32_t thr = 0xffffffffu;
    unsigned long long key = ~0ull;                    // (value with its sign bit flipped, lag): ordered as (value, lag)
    int32_t *row = rows + (size_t)g * ndiff;
    for (int t = tid; t < ndiff; t += nt) {
        const int32_t v = t == 0 ? 32768 : psb_pitch_cmn(t, s_dd[t], s_dsh[t], s_cum[t], s_csh[t], tscale);
        row[t] = v;
        s_dd[t] = (uint32_t)v;
        if (v < threshold) thr = min(thr, (uint32_t)t);
        key = min(key, ((unsigned long long)((uint32_t)v ^ 0x80000000u) << 32) | (uint32_t)t);
    }
    thr = __reduce_min_sync(0xffffffffu, thr);
    for (int o = 16; o > 0; o >>= 1) key = min(key, __shfl_down_sync(0xffffffffu, key, o));
    const int warp = tid >> 5, lane = tid & 31, nw = (nt + 31) >> 5;
    if (lane == 0) s_thr[warp] = thr, s_key[warp] = key;
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < nw; ++w) thr = min(thr, s_thr[w]), key = min(key, s_key[w]);
        const int p = thr != 0xffffffffu ? (int)thr : (int)(uint32_t)key;
        period[g] = p;
        pdiff[g] = (int32_t)s_dd[p];
    }
}

__global__ void __launch_bounds__(PITCH_READ_THREADS) pitch_read_kernel(
    const int32_t *__restrict__ frame_off, const int32_t *__restrict__ out_off, int32_t n_streams, int32_t total,
    int half, int ndiff, int32_t threshold, int32_t range, const int32_t *__restrict__ rows,
    const int32_t *__restrict__ period, const int32_t *__restrict__ pdiff, uint16_t *__restrict__ out_period,
    uint16_t *__restrict__ out_bestdiff)
{
    const int o = blockIdx.x * PITCH_READ_THREADS + threadIdx.x;
    if (o >= total) return;
    const int s = stream_of(out_off, n_streams, o);
    const int base = frame_off[s];
    const psb_pitch_read_t r = psb_pitch_read_at(o - out_off[s], frame_off[s + 1] - base, half);
    const int32_t *srows = rows + (size_t)base * ndiff;
    psb_pitch_decide(r, half, ndiff, threshold, range, period + base, pdiff + base,
                     [=](int64_t f) { return srows + (size_t)f * ndiff; }, out_period + o, out_bestdiff + o);
}

// one thread per stitched sample: fed slot i's stream is its leftover, then its new samples
__global__ void __launch_bounds__(PITCH_COPY_THREADS) pitch_stitch_kernel(
    const int16_t *__restrict__ new_pcm, const int64_t *__restrict__ new_off, const int64_t *__restrict__ st_off,
    const LiveSlot *__restrict__ live, int32_t n, int64_t total, int flen, const int16_t *__restrict__ left,
    int16_t *__restrict__ out)
{
    const int64_t j = (int64_t)blockIdx.x * PITCH_COPY_THREADS + threadIdx.x;
    if (j >= total) return;
    const int i = stream_of(st_off, n, j);
    const int64_t p = j - st_off[i], nl = st_off[i + 1] - st_off[i] - (new_off[i + 1] - new_off[i]);
    out[j] = p < nl ? left[(size_t)live[i].slot * flen + p] : new_pcm[new_off[i] + p - nl];
}

// pitch_read_kernel for a live call: fed slot i's reads are k0 .. of a stream that has f1 frames at the end of the
// call; frames from f0 on are this call's (from frame_off[i] in rows / period / pdiff), earlier ones the ring's
__global__ void __launch_bounds__(PITCH_READ_THREADS) pitch_live_read_kernel(
    const LiveSlot *__restrict__ live, const int32_t *__restrict__ frame_off, const int32_t *__restrict__ out_off,
    int32_t n, int32_t total, int half, int ndiff, int32_t threshold, int32_t range, const int32_t *__restrict__ rows,
    const int32_t *__restrict__ period, const int32_t *__restrict__ pdiff, const int32_t *__restrict__ ring_rows,
    const int32_t *__restrict__ ring_period, const int32_t *__restrict__ ring_pdiff, uint16_t *__restrict__ out_period,
    uint16_t *__restrict__ out_bestdiff)
{
    const int o = blockIdx.x * PITCH_READ_THREADS + threadIdx.x;
    if (o >= total) return;
    const int i = stream_of(out_off, n, o);
    const LiveSlot s = live[i];
    const int wsize = 2 * half + 1, base = frame_off[i];
    const size_t ring = (size_t)s.slot * wsize;
    const psb_pitch_read_t r = psb_pitch_read_at(s.k0 + (o - out_off[i]), s.f1, half);
    const psb_pitch_live_frames_t per{period + base, ring_period + ring, s.f0, wsize, 1};
    const psb_pitch_live_frames_t pd{pdiff + base, ring_pdiff + ring, s.f0, wsize, 1};
    const psb_pitch_live_frames_t rw{rows + (size_t)base * ndiff, ring_rows + ring * ndiff, s.f0, wsize, ndiff};
    psb_pitch_decide(r, half, ndiff, threshold, range, per, pd, [=](int32_t f) { return rw.at(f); }, out_period + o,
                     out_bestdiff + o);
}

// block (i, j): entry j of fed slot i's last min(wsize, new frames) frames into the slot's ring; block (i, 0) also
// saves the samples from the slot's next frame start on as its leftover
__global__ void __launch_bounds__(PITCH_COPY_THREADS) pitch_store_kernel(
    const LiveSlot *__restrict__ live, const int32_t *__restrict__ frame_off, const int64_t *__restrict__ st_off,
    int half, int ndiff, int flen, int fshift, const int32_t *__restrict__ rows, const int32_t *__restrict__ period,
    const int32_t *__restrict__ pdiff, const int16_t *__restrict__ stitch, int32_t *__restrict__ ring_rows,
    int32_t *__restrict__ ring_period, int32_t *__restrict__ ring_pdiff, int16_t *__restrict__ left)
{
    const int i = blockIdx.x, j = blockIdx.y, tid = threadIdx.x;
    const LiveSlot s = live[i];
    const int wsize = 2 * half + 1, nf = s.f1 - s.f0, keep = min(wsize, nf);
    if (j < keep) {
        const int32_t f = s.f1 - keep + j, c = frame_off[i] + (f - s.f0);
        const size_t e = (size_t)s.slot * wsize + f % wsize;
        for (int t = tid; t < ndiff; t += PITCH_COPY_THREADS) ring_rows[e * ndiff + t] = rows[(size_t)c * ndiff + t];
        if (tid == 0) ring_period[e] = period[c], ring_pdiff[e] = pdiff[c];
    }
    if (j == 0) {
        const int64_t from = st_off[i] + (int64_t)nf * fshift, to = st_off[i + 1];
        for (int64_t p = from + tid; p < to; p += PITCH_COPY_THREADS) left[(size_t)s.slot * flen + (p - from)] = stitch[p];
    }
}

// frame_off / out_off (host, [n + 1]) from samp_off; refuses before any allocation or launch
int pitch_plan(const psb_pitch_t *h, const char *fn, const int64_t *samp_off, int32_t n, int32_t *frame_off, int32_t *out_off)
{
    PSB_REQUIRE(samp_off[0] == 0, "%s: samp_off[0] must be 0", fn);
    frame_off[0] = out_off[0] = 0;
    for (int s = 0; s < n; ++s) {
        const int64_t len = samp_off[s + 1] - samp_off[s];
        PSB_REQUIRE(len >= 0, "%s: samp_off not monotone at %d", fn, s);
        const int64_t nf = len >= h->flen ? 1 + (len - h->flen) / h->fshift : 0;
        PSB_REQUIRE((int64_t)frame_off[s] + nf < (int64_t)1 << 31, "%s: more than 2^31 - 1 frames in one call", fn);
        frame_off[s + 1] = frame_off[s] + (int32_t)nf;
        out_off[s + 1] = out_off[s] + (int32_t)psb_pitch_n_reads(nf, h->half);   // at most one read per frame
    }
    return PSB_OK;
}

int pitch_run(psb_pitch_t *h, const int16_t *d_pcm, const int64_t *samp_off, int32_t n, int32_t *out_off,
              uint16_t *d_period, uint16_t *d_bestdiff, float *ms)
{
    std::vector<int32_t> frame_off((size_t)n + 1);
    int rc = pitch_plan(h, "psb_pitch_process", samp_off, n, frame_off.data(), out_off);
    if (rc) return rc;
    const int32_t total_f = frame_off[n], total_o = out_off[n];
    rc = h->d_samp_off.reserve((size_t)n + 1);
    if (!rc) rc = h->d_frame_off.reserve((size_t)n + 1);
    if (!rc) rc = h->d_out_off.reserve((size_t)n + 1);
    if (!rc) rc = h->d_rows.reserve(std::max<size_t>((size_t)total_f * h->ndiff, 1));
    if (!rc) rc = h->d_period.reserve(std::max<size_t>((size_t)total_f, 1));
    if (!rc) rc = h->d_pdiff.reserve(std::max<size_t>((size_t)total_f, 1));
    if (rc) return rc;
    cudaStream_t st = h->stream;
    PSB_CUDA(cudaMemcpyAsync(h->d_samp_off, samp_off, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st));
    PSB_CUDA(cudaMemcpyAsync(h->d_frame_off, frame_off.data(), ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, st));
    PSB_CUDA(cudaMemcpyAsync(h->d_out_off, out_off, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, st));
    PSB_CUDA(cudaEventRecord(h->ev[0], st));
    if (total_f) {
        // the attribute belongs to the kernel, not to this handle: set it for this handle's frame size every launch
        PSB_CUDA(cudaFuncSetAttribute(pitch_diff_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem));
        pitch_diff_kernel<<<total_f, h->threads, h->smem, st>>>(d_pcm, h->d_samp_off, h->d_frame_off, n, h->flen, h->fshift,
                                                               h->ndiff, h->tscale, h->threshold, h->d_rows, h->d_period,
                                                               h->d_pdiff);
        PSB_LAUNCH_CHECK();
    }
    if (total_o) {
        pitch_read_kernel<<<(total_o + PITCH_READ_THREADS - 1) / PITCH_READ_THREADS, PITCH_READ_THREADS, 0, st>>>(
            h->d_frame_off, h->d_out_off, n, total_o, h->half, h->ndiff, h->threshold, h->range, h->d_rows, h->d_period,
            h->d_pdiff, d_period, d_bestdiff);
        PSB_LAUNCH_CHECK();
    }
    PSB_CUDA(cudaEventRecord(h->ev[1], st));
    PSB_CUDA(cudaStreamSynchronize(st));
    if (ms) PSB_CUDA(cudaEventElapsedTime(ms, h->ev[0], h->ev[1]));
    return PSB_OK;
}

// (uint16)(value * 32768) as yin_init computes it from the program's float option; -1 when it does not fit
int q15_of(double v)
{
    const float q = (float)v * 32768.0f;
    return q >= 0.0f && q < 65536.0f ? (int)(uint16_t)q : -1;
}

// A live call checked and laid out on the host: per fed slot, the stitched offsets, frames, reads and LiveSlot.
struct LivePlan {
    std::vector<int64_t> st_off;
    std::vector<int32_t> frame_off, out_off;
    std::vector<LiveSlot> live;
    int32_t max_new = 0;           // the most new frames of one slot
};

// refuses before any allocation or launch, and then the call changes no slot
int pitch_live_plan(const psb_pitch_t *h, const char *fn, const int32_t *slots, int32_t n, const int64_t *samp_off,
                    const int8_t *final, LivePlan *pl)
{
    PSB_REQUIRE(h->n_slots > 0, "%s: psb_pitch_live_open has not been called", fn);
    PSB_REQUIRE(n == 0 || slots, "%s: slots is null", fn);
    PSB_REQUIRE(samp_off[0] == 0, "%s: samp_off[0] must be 0", fn);
    std::vector<char> seen((size_t)h->n_slots, 0);
    pl->st_off.assign((size_t)n + 1, 0);
    pl->frame_off.assign((size_t)n + 1, 0);
    pl->out_off.assign((size_t)n + 1, 0);
    pl->live.resize((size_t)n);
    for (int i = 0; i < n; ++i) {
        const int s = slots[i];
        PSB_REQUIRE(s >= 0 && s < h->n_slots, "%s: slot %d out of range (0..%d)", fn, s, h->n_slots - 1);
        PSB_REQUIRE(!seen[s], "%s: slot %d fed twice in one call", fn, s);
        seen[s] = 1;
        PSB_REQUIRE(!h->ended[s], "%s: slot %d has ended (a final call ran); reset it before feeding it again", fn, s);
        const int64_t add = samp_off[i + 1] - samp_off[i];
        PSB_REQUIRE(add >= 0, "%s: samp_off not monotone at %d", fn, i);
        const int32_t f0 = h->frames[s];
        const int64_t len = h->samples[s] - (int64_t)f0 * h->fshift + add;   // the leftover is shorter than a frame
        const int64_t nf = len >= h->flen ? 1 + (len - h->flen) / h->fshift : 0;
        PSB_REQUIRE(f0 + nf < (int64_t)1 << 31, "%s: slot %d would pass 2^31 - 1 frames", fn, s);
        PSB_REQUIRE(pl->frame_off[i] + nf < (int64_t)1 << 31, "%s: more than 2^31 - 1 frames in one call", fn);
        const int32_t f1 = f0 + (int32_t)nf;
        pl->live[i] = LiveSlot{s, f0, f1, psb_pitch_main_reads(f0, h->half)};
        pl->st_off[i + 1] = pl->st_off[i] + len;
        pl->frame_off[i + 1] = pl->frame_off[i] + (int32_t)nf;
        pl->out_off[i + 1] = pl->out_off[i] + psb_pitch_live_reads(f0, f1, h->half, final && final[i]);
        pl->max_new = std::max(pl->max_new, (int32_t)nf);
    }
    return PSB_OK;
}

// runs a planned live call on new samples at d_new and updates the host mirror
int pitch_feed_run(psb_pitch_t *h, const LivePlan &pl, const int32_t *slots, int32_t n, const int16_t *d_new,
                   const int64_t *samp_off, const int8_t *final, uint16_t *d_period, uint16_t *d_bestdiff, float *ms)
{
    const int64_t total_s = pl.st_off[n];
    const int32_t total_f = pl.frame_off[n], total_o = pl.out_off[n];
    int rc = h->d_new_off.reserve((size_t)n + 1);
    if (!rc) rc = h->d_samp_off.reserve((size_t)n + 1);
    if (!rc) rc = h->d_frame_off.reserve((size_t)n + 1);
    if (!rc) rc = h->d_out_off.reserve((size_t)n + 1);
    if (!rc) rc = h->d_live.reserve(std::max<size_t>((size_t)n, 1));
    if (!rc) rc = h->d_stitch.reserve(std::max<size_t>((size_t)total_s, 1));
    if (!rc) rc = h->d_rows.reserve(std::max<size_t>((size_t)total_f * h->ndiff, 1));
    if (!rc) rc = h->d_period.reserve(std::max<size_t>((size_t)total_f, 1));
    if (!rc) rc = h->d_pdiff.reserve(std::max<size_t>((size_t)total_f, 1));
    if (rc) return rc;
    cudaStream_t st = h->stream;
    PSB_CUDA(cudaMemcpyAsync(h->d_new_off, samp_off, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st));
    PSB_CUDA(cudaMemcpyAsync(h->d_samp_off, pl.st_off.data(), ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st));
    PSB_CUDA(cudaMemcpyAsync(h->d_frame_off, pl.frame_off.data(), ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, st));
    PSB_CUDA(cudaMemcpyAsync(h->d_out_off, pl.out_off.data(), ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, st));
    if (n) PSB_CUDA(cudaMemcpyAsync(h->d_live, pl.live.data(), (size_t)n * sizeof(LiveSlot), cudaMemcpyHostToDevice, st));
    PSB_CUDA(cudaEventRecord(h->ev[0], st));
    if (total_s) {
        pitch_stitch_kernel<<<(unsigned)((total_s + PITCH_COPY_THREADS - 1) / PITCH_COPY_THREADS), PITCH_COPY_THREADS, 0,
                              st>>>(d_new, h->d_new_off, h->d_samp_off, h->d_live, n, total_s, h->flen, h->d_left,
                                    h->d_stitch);
        PSB_LAUNCH_CHECK();
    }
    if (total_f) {
        PSB_CUDA(cudaFuncSetAttribute(pitch_diff_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem));
        pitch_diff_kernel<<<total_f, h->threads, h->smem, st>>>(h->d_stitch, h->d_samp_off, h->d_frame_off, n, h->flen,
                                                               h->fshift, h->ndiff, h->tscale, h->threshold, h->d_rows,
                                                               h->d_period, h->d_pdiff);
        PSB_LAUNCH_CHECK();
    }
    if (total_o) {
        pitch_live_read_kernel<<<(total_o + PITCH_READ_THREADS - 1) / PITCH_READ_THREADS, PITCH_READ_THREADS, 0, st>>>(
            h->d_live, h->d_frame_off, h->d_out_off, n, total_o, h->half, h->ndiff, h->threshold, h->range, h->d_rows,
            h->d_period, h->d_pdiff, h->d_ring_rows, h->d_ring_period, h->d_ring_pdiff, d_period, d_bestdiff);
        PSB_LAUNCH_CHECK();
    }
    if (total_s) {                 // after the reads: they may need the ring entries this overwrites
        const dim3 grid((unsigned)n, (unsigned)std::max(1, std::min(2 * h->half + 1, pl.max_new)));
        pitch_store_kernel<<<grid, PITCH_COPY_THREADS, 0, st>>>(h->d_live, h->d_frame_off, h->d_samp_off, h->half, h->ndiff,
                                                                h->flen, h->fshift, h->d_rows, h->d_period, h->d_pdiff,
                                                                h->d_stitch, h->d_ring_rows, h->d_ring_period,
                                                                h->d_ring_pdiff, h->d_left);
        PSB_LAUNCH_CHECK();
    }
    PSB_CUDA(cudaEventRecord(h->ev[1], st));
    PSB_CUDA(cudaStreamSynchronize(st));
    if (ms) PSB_CUDA(cudaEventElapsedTime(ms, h->ev[0], h->ev[1]));
    for (int i = 0; i < n; ++i) {
        const int s = slots[i];
        h->samples[s] += samp_off[i + 1] - samp_off[i];
        h->frames[s] = pl.live[i].f1;
        h->ended[s] = final && final[i] ? 1 : 0;
    }
    return PSB_OK;
}

void pitch_live_status(const psb_pitch_t *h, const int32_t *slots, int32_t n, psb_pitch_live_status_t *status)
{
    for (int i = 0; i < n; ++i) {
        const int s = slots[i];
        psb_pitch_live_status_t &o = status[i];
        o.frames = h->frames[s];
        o.main_reads = psb_pitch_main_reads(h->frames[s], h->half);
        o.reads = h->ended[s] ? psb_pitch_n_reads(h->frames[s], h->half) : o.main_reads;
        o.ended = h->ended[s];
    }
}

}  // namespace

extern "C" void psb_pitch_free(psb_pitch_t *h)
{
    if (!h) return;
    cudaSetDevice(h->device);
    delete h;
}

extern "C" int psb_pitch_create(const psb_pitch_opts_t *o, int device, psb_pitch_t **out)
{
    PSB_REQUIRE(o && out, "psb_pitch_create: bad argument");
    *out = nullptr;
    PSB_REQUIRE(o->sample_rate > 0, "psb_pitch_create: sample_rate must be positive (got %d)", o->sample_rate);
    const double fl = 0.5 + o->sample_rate * o->flen, fs = 0.5 + o->sample_rate * o->fshift;
    PSB_REQUIRE(fl >= 0.0 && fl < 2147483648.0, "psb_pitch_create: flen %g s out of range", o->flen);
    PSB_REQUIRE(fs >= 0.0 && fs < 2147483648.0, "psb_pitch_create: fshift %g s out of range", o->fshift);
    const int flen = (int)(size_t)fl, fshift = (int)(size_t)fs;
    PSB_REQUIRE(flen / 2 >= 1, "psb_pitch_create: frame of %d samples; at least 2 are needed (ndiff = flen / 2 >= 1)", flen);
    PSB_REQUIRE(flen <= PSB_PITCH_MAX_FRAME,
                "psb_pitch_create: frame of %d samples; at most %d are implemented (one CTA's shared memory)", flen,
                PSB_PITCH_MAX_FRAME);
    PSB_REQUIRE(fshift >= 1, "psb_pitch_create: frame shift of 0 samples never advances");
    PSB_REQUIRE(fshift <= flen, "psb_pitch_create: frame shift of %d samples is longer than the %d-sample frame", fshift, flen);
    PSB_REQUIRE(o->smooth_window >= 0 && o->smooth_window <= 127,
                "psb_pitch_create: smooth_window %d out of range (0..127: the window of 2 * smooth_window + 1 frames is an "
                "unsigned char)", o->smooth_window);
    const int thr = q15_of(o->voice_thresh), range = q15_of(o->search_range);
    PSB_REQUIRE(thr >= 0, "psb_pitch_create: voice_thresh %g out of range (its Q15 value must fit 0..65535)", o->voice_thresh);
    PSB_REQUIRE(range >= 0, "psb_pitch_create: search_range %g out of range (its Q15 value must fit 0..65535)", o->search_range);
    PSB_CUDA(cudaSetDevice(device));
    std::unique_ptr<psb_pitch_t> h(new psb_pitch_t());
    h->device = device;
    h->sample_rate = o->sample_rate, h->flen = flen, h->fshift = fshift;
    h->ndiff = flen / 2;
    h->tscale = psb_pitch_tscale(h->ndiff);
    h->half = o->smooth_window;
    h->threshold = thr, h->range = range;
    h->threads = std::min(PITCH_MAX_THREADS, (h->ndiff + 31) / 32 * 32);
    h->smem = diff_smem(flen, h->ndiff);
    cudaError_t e = h->stream.create();
    if (e == cudaSuccess) e = h->ev[0].create();
    if (e == cudaSuccess) e = h->ev[1].create();
    if (e != cudaSuccess) {
        psb_set_error("psb_pitch_create: %s", cudaGetErrorString(e));
        return PSB_ERR_CUDA;
    }
    *out = h.release();
    return PSB_OK;
}

extern "C" int32_t psb_pitch_frame_size(const psb_pitch_t *h) { return h ? h->flen : -1; }
extern "C" int32_t psb_pitch_frame_shift(const psb_pitch_t *h) { return h ? h->fshift : -1; }
extern "C" int32_t psb_pitch_ndiff(const psb_pitch_t *h) { return h ? h->ndiff : -1; }

extern "C" int psb_pitch_process_device(psb_pitch_t *h, const int16_t *d_pcm, const int64_t *samp_off, int32_t n_streams,
                                        int32_t *out_off, uint16_t *d_period, uint16_t *d_bestdiff, float *ms)
{
    PSB_REQUIRE(h && samp_off && out_off && n_streams >= 0, "psb_pitch_process_device: bad argument");
    PSB_REQUIRE(d_pcm || samp_off[n_streams] == 0, "psb_pitch_process_device: pcm is null");
    PSB_REQUIRE(n_streams == 0 || (d_period && d_bestdiff), "psb_pitch_process_device: output is null");
    PSB_CUDA(cudaSetDevice(h->device));
    return pitch_run(h, d_pcm, samp_off, n_streams, out_off, d_period, d_bestdiff, ms);
}

extern "C" int psb_pitch_process_host(psb_pitch_t *h, const int16_t *pcm, const int64_t *samp_off, int32_t n_streams,
                                      int32_t *out_off, uint16_t *period, uint16_t *bestdiff, float *ms)
{
    PSB_REQUIRE(h && samp_off && out_off && n_streams >= 0, "psb_pitch_process_host: bad argument");
    const int64_t ns = samp_off[n_streams];
    PSB_REQUIRE(ns == 0 || pcm, "psb_pitch_process_host: pcm is null");
    PSB_REQUIRE(n_streams == 0 || (period && bestdiff), "psb_pitch_process_host: output is null");
    PSB_CUDA(cudaSetDevice(h->device));
    std::vector<int32_t> frame_off((size_t)n_streams + 1);
    int rc = pitch_plan(h, "psb_pitch_process_host", samp_off, n_streams, frame_off.data(), out_off);
    if (rc) return rc;
    const size_t reads = (size_t)out_off[n_streams];
    rc = h->d_pcm.reserve(std::max<size_t>((size_t)ns, 1));
    if (!rc) rc = h->d_out.reserve(std::max<size_t>(reads * 2, 1));
    if (rc) return rc;
    if (ns) PSB_CUDA(cudaMemcpyAsync(h->d_pcm, pcm, (size_t)ns * 2, cudaMemcpyHostToDevice, h->stream));
    rc = pitch_run(h, h->d_pcm, samp_off, n_streams, out_off, h->d_out, h->d_out + reads, ms);
    if (rc) return rc;
    if (reads) {
        PSB_CUDA(cudaMemcpy(period, h->d_out, reads * 2, cudaMemcpyDeviceToHost));
        PSB_CUDA(cudaMemcpy(bestdiff, h->d_out + reads, reads * 2, cudaMemcpyDeviceToHost));
    }
    return PSB_OK;
}

extern "C" int psb_pitch_live_open(psb_pitch_t *h, int32_t n_slots)
{
    PSB_REQUIRE(h && n_slots > 0, "psb_pitch_live_open: bad argument");
    PSB_CUDA(cudaSetDevice(h->device));
    PSB_CUDA(cudaStreamSynchronize(h->stream));
    h->n_slots = 0;                                              // until the table is whole again
    const size_t wsize = (size_t)(2 * h->half + 1);
    int rc = h->d_left.reserve((size_t)n_slots * h->flen);
    if (!rc) rc = h->d_ring_rows.reserve((size_t)n_slots * wsize * h->ndiff);
    if (!rc) rc = h->d_ring_period.reserve((size_t)n_slots * wsize);
    if (!rc) rc = h->d_ring_pdiff.reserve((size_t)n_slots * wsize);
    if (rc) return rc;
    // a fresh slot has no samples and no frames: the schedule reads its never-written ring entries as zeros, so the
    // device state needs no clearing
    h->samples.assign((size_t)n_slots, 0);
    h->frames.assign((size_t)n_slots, 0);
    h->ended.assign((size_t)n_slots, 0);
    h->n_slots = n_slots;
    return PSB_OK;
}

extern "C" int psb_pitch_live_reset(psb_pitch_t *h, const int32_t *slots, int32_t n)
{
    PSB_REQUIRE(h && n >= 0 && (n == 0 || slots), "psb_pitch_live_reset: bad argument");
    PSB_REQUIRE(h->n_slots > 0, "psb_pitch_live_reset: psb_pitch_live_open has not been called");
    for (int i = 0; i < n; ++i)
        PSB_REQUIRE(slots[i] >= 0 && slots[i] < h->n_slots, "psb_pitch_live_reset: slot %d out of range (0..%d)", slots[i],
                    h->n_slots - 1);
    for (int i = 0; i < n; ++i) {
        const int s = slots[i];
        h->samples[s] = 0, h->frames[s] = 0, h->ended[s] = 0;
    }
    return PSB_OK;
}

extern "C" int psb_pitch_feed_device(psb_pitch_t *h, const int32_t *slots, int32_t n, const int16_t *d_pcm,
                                     const int64_t *samp_off, const int8_t *final, int32_t *out_off, uint16_t *d_period,
                                     uint16_t *d_bestdiff, psb_pitch_live_status_t *status, float *ms)
{
    PSB_REQUIRE(h && samp_off && out_off && n >= 0, "psb_pitch_feed_device: bad argument");
    PSB_REQUIRE(d_pcm || samp_off[n] == 0, "psb_pitch_feed_device: pcm is null");
    PSB_REQUIRE(n == 0 || (d_period && d_bestdiff && status), "psb_pitch_feed_device: output is null");
    PSB_CUDA(cudaSetDevice(h->device));
    LivePlan pl;
    int rc = pitch_live_plan(h, "psb_pitch_feed_device", slots, n, samp_off, final, &pl);
    if (!rc) rc = pitch_feed_run(h, pl, slots, n, d_pcm, samp_off, final, d_period, d_bestdiff, ms);
    if (rc) return rc;
    std::copy(pl.out_off.begin(), pl.out_off.end(), out_off);
    pitch_live_status(h, slots, n, status);
    return PSB_OK;
}

extern "C" int psb_pitch_feed_host(psb_pitch_t *h, const int32_t *slots, int32_t n, const int16_t *pcm,
                                   const int64_t *samp_off, const int8_t *final, int32_t *out_off, uint16_t *period,
                                   uint16_t *bestdiff, psb_pitch_live_status_t *status, float *ms)
{
    PSB_REQUIRE(h && samp_off && out_off && n >= 0, "psb_pitch_feed_host: bad argument");
    const int64_t ns = samp_off[n];
    PSB_REQUIRE(ns == 0 || pcm, "psb_pitch_feed_host: pcm is null");
    PSB_REQUIRE(n == 0 || (period && bestdiff && status), "psb_pitch_feed_host: output is null");
    PSB_CUDA(cudaSetDevice(h->device));
    LivePlan pl;
    int rc = pitch_live_plan(h, "psb_pitch_feed_host", slots, n, samp_off, final, &pl);
    if (rc) return rc;
    const size_t reads = (size_t)pl.out_off[n];
    rc = h->d_pcm.reserve(std::max<size_t>((size_t)ns, 1));
    if (!rc) rc = h->d_out.reserve(std::max<size_t>(reads * 2, 1));
    if (rc) return rc;
    if (ns) PSB_CUDA(cudaMemcpyAsync(h->d_pcm, pcm, (size_t)ns * 2, cudaMemcpyHostToDevice, h->stream));
    rc = pitch_feed_run(h, pl, slots, n, h->d_pcm, samp_off, final, h->d_out, h->d_out + reads, ms);
    if (rc) return rc;
    if (reads) {
        PSB_CUDA(cudaMemcpy(period, h->d_out, reads * 2, cudaMemcpyDeviceToHost));
        PSB_CUDA(cudaMemcpy(bestdiff, h->d_out + reads, reads * 2, cudaMemcpyDeviceToHost));
    }
    std::copy(pl.out_off.begin(), pl.out_off.end(), out_off);
    pitch_live_status(h, slots, n, status);
    return PSB_OK;
}
