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
#include "psb_internal.cuh"
#include "psb_pitch_core.h"

#include <math.h>

#include <algorithm>
#include <memory>
#include <vector>

namespace {

constexpr int PITCH_MAX_THREADS = 512;
constexpr int PITCH_READ_THREADS = 256;

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
