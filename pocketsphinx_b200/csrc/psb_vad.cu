// psb_vad.cu -- voice activity detection and endpointing for whole batches of int16 streams
// (ps_vad_classify frame by frame on a fresh ps_vad_init, and ps_endpointer_process on every full
// frame followed by one ps_endpointer_end_stream; ps_vad.c, ps_endpointer.c, common_audio/vad/).
// The arithmetic is psb_vad_core.h's; this file owns the launch shapes.
//
// Two stages, because the filter-bank features do not depend on the decisions and the GMM does:
//   vad_feat_kernel    one thread per chunk of VAD_CHUNK (64) frames of a stream, started from the
//                      initial filter state `warmup` frames before the chunk; records its filter
//                      state at the chunk's first frame and at its end
//   vad_repair_kernel  one thread per chunk, in passes: every chunk whose start state differs from
//                      its predecessor's end state is recomputed from that state, in parallel; a
//                      recomputed chunk can change the end state its successor is checked against,
//                      so passes repeat until one recomputes nothing.  The features are exact by
//                      construction; isolated repairs take two passes.
//   vad_gmm_kernel     one warp per stream, sequential over frames: lanes 0..5 are the six
//                      channels (probabilities, FindMinimum, model update), the global decision
//                      goes through warp votes and a warp sum; lane 0 runs the endpointer.
// Live calls (psb_vad_feed_*) keep one psb_vad_slot_t per stream on the device.  vad_stitch_kernel
// puts each fed slot's leftover samples before its new ones and vad_keep_kernel saves the new
// leftover; stage A starts every chunk whose warm-up reaches back to the call's first frame from the
// slot's filter state; vad_gmm_kernel<true> loads the slot, runs the call's frames and stores it.
#include "psb_internal.cuh"
#include "psb_vad_core.h"

#include <math.h>

#include <algorithm>
#include <vector>

namespace {

constexpr int VAD_CHUNK = 64;          // frames per stage-A thread
constexpr int FEAT_THREADS = 32;       // stage-A CTA: 32 threads, strided scratch in shared memory
constexpr int GMM_WARPS = 4;
constexpr int GMM_RING_MAX = 227 * 1024 / GMM_WARPS - 1536 / GMM_WARPS;   // endpointer ring bytes per warp

// the decisions of the endpointer's queue, by stream frame number: frames pushed - maxlen .. pushed
struct FlagRing {
    int8_t *p;
    int m;                       // maxlen + 1: the frame being pushed never overwrites the one it evicts
    __device__ int8_t &operator[](int64_t f) const { return p[(int)f % m]; }   // f < 2^31 (checked per call)
};

}  // namespace

struct psb_vad_s {
    int device;
    int mode, sample_rate, closest, frame_size, maxlen, start_frames, end_frames, warmup;
    double frame_length, window, ratio;
    Stream stream;                // declared first: destroyed after the buffers below
    Event ev[2];
    DevBuf<int16_t> d_pcm;
    DevBuf<int16_t> d_feat;       // [frames][8]
    DevBuf<int8_t> d_flags;
    DevBuf<int64_t> d_segs;       // [frames][2]: a stream has at most one segment per frame
    DevBuf<double> d_times;
    DevBuf<int32_t> d_seg_n;
    DevBuf<int64_t> d_samp_off;
    DevBuf<int32_t> d_frame_off;
    DevBuf<int32_t> d_chunk_off;
    DevBuf<int32_t> d_chunk_stream;
    DevBuf<psb_vad_filt_t> d_st_start, d_st_end[2];
    DevBuf<unsigned long long> d_repairs;
    DevBuf<int> d_changed;        // repair pass flag, device and pinned host copy
    HostBuf<int> h_changed;
    int64_t last_repairs, last_passes;
    // live slots (psb_vad_live_open); the host mirrors each slot's leftover count and frame count
    int32_t n_slots = 0;
    std::vector<int32_t> left_n;
    std::vector<int64_t> pushed;
    DevBuf<psb_vad_slot_t> d_slot;
    DevBuf<int8_t> d_ring;        // [slot][maxlen + 1]: the endpointer queue's decisions
    DevBuf<int16_t> d_left;       // [slot][frame_size]: samples after the last full frame
    DevBuf<int16_t> d_stitch;     // per call: leftover + new samples of each fed slot
    DevBuf<int64_t> d_new_off;
    DevBuf<int32_t> d_slot_of;    // per call: [n] slot, [n .. 2n) samples kept as the new leftover
    DevBuf<int8_t> d_final;
    DevBuf<psb_vad_live_status_t> d_status;
};

namespace {

// one frame's features as the 16 bytes stage B reads (six Q4 log energies, total_power, zero)
union FrameFeat {
    int4 v;
    int16_t h[8];
};

// features of frames f0 .. f1 - 1 of one stream from filter state *f, which is left at frame f1
__device__ __forceinline__ void feat_frames(psb_vad_filt_t *f, int closest, const int16_t *x, int frame_size, int f0, int f1,
                                            psb_vad_buf scr, int16_t *out)
{
    for (int t = f0; t < f1; ++t) {
        FrameFeat u;
        psb_vad_frame_features(f, closest, x + (size_t)t * frame_size, frame_size, scr, u.h);
        u.h[7] = 0;
        *reinterpret_cast<int4 *>(out + (size_t)t * 8) = u.v;
    }
}

__global__ void __launch_bounds__(FEAT_THREADS) vad_feat_kernel(const int16_t *__restrict__ pcm, const int64_t *__restrict__ samp_off,
                                                                const int32_t *__restrict__ frame_off,
                                                                const int32_t *__restrict__ chunk_off,
                                                                const int32_t *__restrict__ chunk_stream, int32_t n_chunks,
                                                                int closest, int frame_size, int warmup, int16_t *__restrict__ feat,
                                                                psb_vad_filt_t *__restrict__ st_start, psb_vad_filt_t *__restrict__ st_end,
                                                                const psb_vad_slot_t *__restrict__ live, const int32_t *__restrict__ slot_of)
{
    extern __shared__ int16_t vad_scr[];
    const int c = blockIdx.x * FEAT_THREADS + threadIdx.x;
    if (c >= n_chunks) return;
    const int s = chunk_stream[c];
    const int nf = frame_off[s + 1] - frame_off[s];
    const int f0 = (c - chunk_off[s]) * VAD_CHUNK, f1 = min(f0 + VAD_CHUNK, nf);
    const int16_t *x = pcm + samp_off[s];
    const psb_vad_buf scr{vad_scr + threadIdx.x, FEAT_THREADS};
    psb_vad_filt_t f;
    if (live && f0 - warmup <= 0) f = live[slot_of[s]].filt;   // a live stream's exact state at the call's first frame
    else psb_vad_filt_init(&f);
    int16_t dummy[8];
    for (int t = max(0, f0 - warmup); t < f0; ++t)
        psb_vad_frame_features(&f, closest, x + (size_t)t * frame_size, frame_size, scr, dummy);
    st_start[c] = f;
    feat_frames(&f, closest, x, frame_size, f0, f1, scr, feat + (size_t)frame_off[s] * 8);
    st_end[c] = f;
}

// One repair pass, one thread per chunk: a chunk whose start state differs from its predecessor's end state
// (as the previous pass left it, end_in) is recomputed from that state.  end_out gets every chunk's end state
// after the pass; *changed is set when a chunk was recomputed.  Passes repeat until none is: after pass p the
// first p chunks of every stream are computed from their true state (induction over the boundaries), so the
// loop ends with every chunk exact; when repairs are isolated it ends after two passes.
__global__ void __launch_bounds__(FEAT_THREADS) vad_repair_kernel(const int16_t *__restrict__ pcm, const int64_t *__restrict__ samp_off,
                                                                  const int32_t *__restrict__ frame_off,
                                                                  const int32_t *__restrict__ chunk_off,
                                                                  const int32_t *__restrict__ chunk_stream, int32_t n_chunks,
                                                                  int closest, int frame_size, int warmup, int16_t *__restrict__ feat,
                                                                  psb_vad_filt_t *__restrict__ st_start,
                                                                  const psb_vad_filt_t *__restrict__ end_in,
                                                                  psb_vad_filt_t *__restrict__ end_out,
                                                                  unsigned long long *__restrict__ repairs, int *__restrict__ changed)
{
    extern __shared__ int16_t vad_scr[];
    const int c = blockIdx.x * FEAT_THREADS + threadIdx.x;
    if (c >= n_chunks) return;
    const int s = chunk_stream[c];
    const int k = c - chunk_off[s];
    psb_vad_filt_t e = end_in[c];
    if (k > 0 && k * VAD_CHUNK - warmup > 0) {               // otherwise the chunk started at the stream's beginning
        psb_vad_filt_t f = end_in[c - 1];
        const psb_vad_filt_t w = st_start[c];
        if (!psb_vad_filt_equal(&w, &f)) {
            st_start[c] = f;
            const int nf = frame_off[s + 1] - frame_off[s];
            const psb_vad_buf scr{vad_scr + threadIdx.x, FEAT_THREADS};
            feat_frames(&f, closest, pcm + samp_off[s], frame_size, k * VAD_CHUNK, min(k * VAD_CHUNK + VAD_CHUNK, nf), scr,
                        feat + (size_t)frame_off[s] * 8);
            e = f;
            atomicAdd(repairs, 1ull);
            *changed = 1;
        }
    }
    end_out[c] = e;
}

// per-call constants; the initial channel states and the mode's thresholds are built on the host
// (their tables indexed by lane would otherwise sit in each thread's stack)
struct GmmArgs {
    psb_vad_chan_t init[PSB_VAD_NCH];
    int16_t oh1, oh2, ind, tot;
    int frame_size, sample_rate, maxlen, start_frames, end_frames;
};

// the slot state of a live call (all null for whole streams)
struct LiveArgs {
    psb_vad_slot_t *slot;
    int8_t *ring;                       // [slot][maxlen + 1]
    const int32_t *slot_of;             // fed stream -> slot
    const int8_t *final;
    const psb_vad_filt_t *st_end;       // stage A's converged chunk end states
    const int32_t *chunk_off;
    psb_vad_live_status_t *status;
};

// Live = false: every stream starts fresh and ends with ps_endpointer_end_stream.  Live = true: stream s is slot
// slot_of[s], loaded at the start and stored at the end; end_stream runs where final[s] is set, and stream s's segment
// rows start at frame_off[s] + s (a final call ends one segment more than it has frames).
template <bool Live>
__global__ void __launch_bounds__(GMM_WARPS * 32, 1) vad_gmm_kernel(const int16_t *__restrict__ feat, const int64_t *__restrict__ samp_off,
                                                                 const int32_t *__restrict__ frame_off, int32_t n_streams, GmmArgs a,
                                                                 int8_t *flags, int32_t *__restrict__ seg_n,
                                                                 int64_t *__restrict__ segs, double *__restrict__ times, LiveArgs live)
{
    __shared__ int16_t sh_age[GMM_WARPS][PSB_VAD_NCH][16], sh_low[GMM_WARPS][PSB_VAD_NCH][16];
    extern __shared__ int8_t gmm_ring[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int s = blockIdx.x * GMM_WARPS + warp;
    if (s >= n_streams) return;                                 // whole warps leave together
    const unsigned FULL = 0xffffffffu;
    const int ch = lane < PSB_VAD_NCH ? lane : 0;
    int16_t *age = sh_age[warp][ch], *low = sh_low[warp][ch];
    psb_vad_chan_t c = a.init[ch];
    const FlagRing ring{gmm_ring + warp * (a.maxlen + 1), a.maxlen + 1};
    int32_t frame_counter = 0;
    int16_t over_hang = 0, num_of_speech = 0;
    psb_ep_t e;
    psb_vad_slot_t *rec = nullptr;
    int8_t *gring = nullptr;
    if (Live) {
        rec = live.slot + live.slot_of[s];
        gring = live.ring + (size_t)live.slot_of[s] * ring.m;
        psb_vad_slot_load_chan(rec, ch, &c);
        if (lane < PSB_VAD_NCH)
            for (int i = 0; i < 16; ++i) age[i] = rec->age[ch][i], low[i] = rec->low[ch][i];
        frame_counter = rec->frame_counter;
        over_hang = rec->over_hang, num_of_speech = rec->num_of_speech;
        e = rec->ep;
        for (int i = lane; i < ring.m; i += 32) ring.p[i] = gring[i];
    } else {
        if (lane < PSB_VAD_NCH)
            for (int i = 0; i < 16; ++i) age[i] = 0, low[i] = 10000;
        psb_ep_init(&e, a.maxlen, a.start_frames, a.end_frames, a.frame_size, a.sample_rate);
    }
    __syncwarp();
    const int16_t oh1 = a.oh1, oh2 = a.oh2, ind = a.ind, tot = a.tot;
    const int16_t sw = psb_vad_spectrum_weight(ch);
    const int fo = frame_off[s], nf = frame_off[s + 1] - fo;
    const int16_t *fp = feat + (size_t)fo * 8;
    int8_t *fl = flags + fo;
    const size_t so = Live ? (size_t)fo + s : (size_t)fo;      // the stream's first segment row
    psb_ep_seg_t sg;
    int n_seg = 0;
    int16_t v = lane < 7 && nf > 0 ? fp[lane] : 0;
    for (int t = 0; t < nf; ++t) {
        const int16_t x = v;
        if (t + 1 < nf && lane < 7) v = fp[(size_t)(t + 1) * 8 + lane];    // the next frame's value, ahead of the math
        const int16_t total = (int16_t)__shfl_sync(FULL, (int)x, 6);
        int vadflag = 0;
        if (total > PSB_VAD_MIN_ENERGY) {
            psb_vad_chan_probs_t p;
            if (lane < PSB_VAD_NCH) psb_vad_chan_probs(&c, x, &p);
            const int local = lane < PSB_VAD_NCH && p.llr * 4 > ind;
            const int sum = __reduce_add_sync(FULL, lane < PSB_VAD_NCH ? p.llr * sw : 0);
            vadflag = __any_sync(FULL, local) | (sum >= tot);
            if (lane < PSB_VAD_NCH) psb_vad_chan_update(&c, ch, age, low, x, vadflag, frame_counter, &p);
            frame_counter++;
        }
        vadflag = psb_vad_overhang(vadflag, &over_hang, &num_of_speech, oh1, oh2);
        if (lane == 0) {
            fl[t] = ring[e.pushed] = (int8_t)(vadflag > 0);     // e.pushed == t for a whole stream
            if (psb_ep_process(&e, ring, &sg)) {
                segs[2 * (so + n_seg)] = sg.start;
                segs[2 * (so + n_seg) + 1] = sg.end;
                times[2 * (so + n_seg)] = sg.start_time;
                times[2 * (so + n_seg) + 1] = sg.end_time;
                ++n_seg;
            }
        }
    }
    if (lane == 0) {
        const int tail = (int)(samp_off[s + 1] - samp_off[s] - (int64_t)nf * a.frame_size);
        if ((!Live || live.final[s]) && psb_ep_end_stream(&e, ring, tail, &sg)) {
            segs[2 * (so + n_seg)] = sg.start;
            segs[2 * (so + n_seg) + 1] = sg.end;
            times[2 * (so + n_seg)] = sg.start_time;
            times[2 * (so + n_seg) + 1] = sg.end_time;
            ++n_seg;
        }
        seg_n[s] = n_seg;
        if (Live) {
            psb_vad_live_status_t st;
            st.in_speech = e.in_speech;
            st.reserved = 0;
            st.start_sample = e.in_speech ? e.seg_start : -1;
            st.frames = e.pushed;
            st.speech_start = e.speech_start;
            st.speech_end = e.speech_end;
            live.status[s] = st;
            rec->ep = e;
            rec->frame_counter = frame_counter;
            rec->over_hang = over_hang, rec->num_of_speech = num_of_speech;
            if (nf > 0) rec->filt = live.st_end[live.chunk_off[s + 1] - 1];
        }
    }
    if (Live) {
        if (lane < PSB_VAD_NCH) {
            psb_vad_slot_store_chan(rec, ch, &c);
            for (int i = 0; i < 16; ++i) rec->age[ch][i] = age[i], rec->low[ch][i] = low[i];
        }
        __syncwarp();
        for (int i = lane; i < ring.m; i += 32) gring[i] = ring.p[i];
    }
}

// Live calls: fed stream i's samples are its slot's leftover followed by its new samples, back to back at `out`
// (samp_off: the stitched offsets, new_off: the new samples' offsets in pcm); one thread per output sample.
__global__ void vad_stitch_kernel(const int16_t *__restrict__ pcm, const int64_t *__restrict__ new_off,
                                  const int64_t *__restrict__ samp_off, const int32_t *__restrict__ slot_of, int32_t n,
                                  int64_t total, const int16_t *__restrict__ left, int frame_size, int16_t *__restrict__ out)
{
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < total; j += (int64_t)gridDim.x * blockDim.x) {
        int lo = 0, hi = n - 1;                                  // the last stream starting at or before j
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (samp_off[mid] <= j) lo = mid;
            else hi = mid - 1;
        }
        const int64_t k = j - samp_off[lo];
        const int64_t old = samp_off[lo + 1] - samp_off[lo] - (new_off[lo + 1] - new_off[lo]);
        out[j] = k < old ? left[(size_t)slot_of[lo] * frame_size + k] : pcm[new_off[lo] + k - old];
    }
}

// one CTA per fed stream: its last keep[i] stitched samples (none after a final call) become the slot's leftover
__global__ void vad_keep_kernel(const int16_t *__restrict__ stitched, const int64_t *__restrict__ samp_off,
                                const int32_t *__restrict__ slot_of, const int32_t *__restrict__ keep, int frame_size,
                                int16_t *__restrict__ left)
{
    const int i = blockIdx.x, k = keep[i];
    const int16_t *src = stitched + samp_off[i + 1] - k;
    int16_t *dst = left + (size_t)slot_of[i] * frame_size;
    for (int t = threadIdx.x; t < k; t += blockDim.x) dst[t] = src[t];
}

// the listed slots (all n when ids is null) become `fresh`; their queue rings need no clearing, since the
// endpointer reads only decisions it has written since
__global__ void vad_reset_kernel(psb_vad_slot_t *__restrict__ slot, const int32_t *__restrict__ ids, int32_t n,
                                 psb_vad_slot_t fresh)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) slot[ids ? ids[i] : i] = fresh;
}

size_t feat_smem(int closest) { return (size_t)FEAT_THREADS * psb_vad_scratch_elems(closest) * sizeof(int16_t); }

// a live call as psb_vad_feed_* hands it to vad_run
struct LiveCall {
    const int16_t *d_new;          // the new samples, new_off (host) [n + 1]
    const int64_t *new_off;
    const int32_t *slot_of;        // host [n]
    const int32_t *keep;           // host [n]: samples left after the last full frame that wait for the next call
    const int8_t *final;           // host [n] or null
    psb_vad_live_status_t *d_status;
};

// Stage A + B over streams whose samples are at d_pcm (for a live call: stitched from the slots' leftovers and
// lc->d_new, with samp_off the stitched offsets); frame_off (host) is filled here.
int vad_run(psb_vad_t *v, const int16_t *d_pcm, const int64_t *samp_off, int32_t n, int8_t *d_flags, int32_t *frame_off,
            int32_t *d_seg_n, int64_t *d_segs, double *d_times, float *ms, const LiveCall *lc = nullptr)
{
    std::vector<int32_t> chunk_off((size_t)n + 1), chunk_stream;
    frame_off[0] = 0;
    chunk_off[0] = 0;
    int max_nc = 0;
    for (int s = 0; s < n; ++s) {
        const int64_t len = samp_off[s + 1] - samp_off[s];
        PSB_REQUIRE(len >= 0, "psb_vad_process: samp_off not monotone at %d", s);
        const int64_t nf = len / v->frame_size;
        PSB_REQUIRE((int64_t)frame_off[s] + nf < (int64_t)1 << 31, "psb_vad_process: more than 2^31 frames in one call");
        frame_off[s + 1] = frame_off[s] + (int32_t)nf;
        const int nc = (int)((nf + VAD_CHUNK - 1) / VAD_CHUNK);
        max_nc = std::max(max_nc, nc);
        chunk_off[s + 1] = chunk_off[s] + nc;
        chunk_stream.insert(chunk_stream.end(), (size_t)nc, s);
    }
    const int32_t total = frame_off[n], n_chunks = chunk_off[n];
    int rc = v->d_feat.reserve(std::max<size_t>((size_t)total * 8, 1));
    if (!rc) rc = v->d_samp_off.reserve((size_t)n + 1);
    if (!rc) rc = v->d_frame_off.reserve((size_t)n + 1);
    if (!rc) rc = v->d_chunk_off.reserve((size_t)n + 1);
    if (!rc) rc = v->d_chunk_stream.reserve(std::max<size_t>((size_t)n_chunks, 1));
    if (!rc) rc = v->d_st_start.reserve(std::max<size_t>((size_t)n_chunks, 1));
    if (!rc) rc = v->d_st_end[0].reserve(std::max<size_t>((size_t)n_chunks, 1));
    if (!rc) rc = v->d_st_end[1].reserve(std::max<size_t>((size_t)n_chunks, 1));
    if (lc) {
        if (!rc) rc = v->d_stitch.reserve(std::max<size_t>((size_t)samp_off[n], 1));
        if (!rc) rc = v->d_new_off.reserve((size_t)n + 1);
        if (!rc) rc = v->d_slot_of.reserve(std::max<size_t>((size_t)n * 2, 1));
        if (!rc) rc = v->d_final.reserve(std::max<size_t>((size_t)n, 1));
    }
    if (rc) return rc;
    cudaStream_t st = v->stream;
    PSB_CUDA(cudaMemcpyAsync(v->d_samp_off, samp_off, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st));
    PSB_CUDA(cudaMemcpyAsync(v->d_frame_off, frame_off, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, st));
    PSB_CUDA(cudaMemcpyAsync(v->d_chunk_off, chunk_off.data(), ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, st));
    if (n_chunks)
        PSB_CUDA(cudaMemcpyAsync(v->d_chunk_stream, chunk_stream.data(), (size_t)n_chunks * 4, cudaMemcpyHostToDevice, st));
    LiveArgs live{};
    if (lc && n) {
        std::vector<int32_t> slot_keep(lc->slot_of, lc->slot_of + n);
        slot_keep.insert(slot_keep.end(), lc->keep, lc->keep + n);
        std::vector<int8_t> fin((size_t)n, 0);
        if (lc->final)
            for (int i = 0; i < n; ++i) fin[i] = lc->final[i] != 0;
        PSB_CUDA(cudaMemcpyAsync(v->d_new_off, lc->new_off, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st));
        PSB_CUDA(cudaMemcpyAsync(v->d_slot_of, slot_keep.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
        PSB_CUDA(cudaMemcpyAsync(v->d_final, fin.data(), (size_t)n, cudaMemcpyHostToDevice, st));
        live = LiveArgs{v->d_slot, v->d_ring, v->d_slot_of, v->d_final, nullptr, v->d_chunk_off, lc->d_status};
    }
    PSB_CUDA(cudaMemsetAsync(v->d_repairs, 0, sizeof(unsigned long long), st));
    PSB_CUDA(cudaEventRecord(v->ev[0], st));
    if (lc && n) {
        const int64_t ns = samp_off[n];
        if (ns) {
            const int blocks = (int)std::min<int64_t>((ns + 255) / 256, 4096);
            vad_stitch_kernel<<<blocks, 256, 0, st>>>(lc->d_new, v->d_new_off, v->d_samp_off, v->d_slot_of, n, ns, v->d_left,
                                                      v->frame_size, v->d_stitch);
            PSB_LAUNCH_CHECK();
            vad_keep_kernel<<<n, 128, 0, st>>>(v->d_stitch, v->d_samp_off, v->d_slot_of, v->d_slot_of + n, v->frame_size,
                                               v->d_left);
            PSB_LAUNCH_CHECK();
        }
        d_pcm = v->d_stitch;
    }
    const size_t smem = feat_smem(v->closest);
    const int grid = (n_chunks + FEAT_THREADS - 1) / FEAT_THREADS;
    v->last_passes = 0;
    int end_buf = 0;                                             // where the converged chunk end states are
    if (n_chunks) {
        PSB_CUDA(cudaFuncSetAttribute(vad_feat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        PSB_CUDA(cudaFuncSetAttribute(vad_repair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        vad_feat_kernel<<<grid, FEAT_THREADS, smem, st>>>(d_pcm, v->d_samp_off, v->d_frame_off, v->d_chunk_off, v->d_chunk_stream,
                                                          n_chunks, v->closest, v->frame_size, v->warmup, v->d_feat,
                                                          v->d_st_start, v->d_st_end[0], lc ? v->d_slot.get() : nullptr,
                                                          v->d_slot_of);
        PSB_LAUNCH_CHECK();
        // a live call whose streams have one chunk each has no boundary to repair: no passes, no host synchronisation
        for (int cur = 0; !lc || max_nc > 1; cur ^= 1) {
            PSB_CUDA(cudaMemsetAsync(v->d_changed, 0, sizeof(int), st));
            vad_repair_kernel<<<grid, FEAT_THREADS, smem, st>>>(d_pcm, v->d_samp_off, v->d_frame_off, v->d_chunk_off,
                                                                v->d_chunk_stream, n_chunks, v->closest, v->frame_size, v->warmup,
                                                                v->d_feat, v->d_st_start, v->d_st_end[cur], v->d_st_end[cur ^ 1],
                                                                v->d_repairs, v->d_changed);
            PSB_LAUNCH_CHECK();
            PSB_CUDA(cudaMemcpyAsync(v->h_changed, v->d_changed, sizeof(int), cudaMemcpyDeviceToHost, st));
            PSB_CUDA(cudaStreamSynchronize(st));
            ++v->last_passes;
            end_buf = cur ^ 1;
            if (!*v->h_changed) break;
        }
    }
    if (n) {
        const int l8 = v->frame_size / (v->closest / 8000);
        GmmArgs a;
        int16_t age[16], low[16];
        for (int ch = 0; ch < PSB_VAD_NCH; ++ch) psb_vad_chan_init(&a.init[ch], ch, age, low);
        psb_vad_thresholds(v->mode, l8 == 80 ? 0 : l8 == 160 ? 1 : 2, &a.oh1, &a.oh2, &a.ind, &a.tot);
        a.frame_size = v->frame_size, a.sample_rate = v->sample_rate, a.maxlen = v->maxlen;
        a.start_frames = v->start_frames, a.end_frames = v->end_frames;
        // the attribute belongs to the kernel, not to this handle: set it for this handle's ring before every launch
        const int ring = GMM_WARPS * (v->maxlen + 1);
        const int blocks = (n + GMM_WARPS - 1) / GMM_WARPS;
        if (lc) {
            live.st_end = v->d_st_end[end_buf];
            PSB_CUDA(cudaFuncSetAttribute(vad_gmm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ring));
            vad_gmm_kernel<true><<<blocks, GMM_WARPS * 32, (size_t)ring, st>>>(v->d_feat, v->d_samp_off, v->d_frame_off, n, a,
                                                                             d_flags, d_seg_n, d_segs, d_times, live);
        } else {
            PSB_CUDA(cudaFuncSetAttribute(vad_gmm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ring));
            vad_gmm_kernel<false><<<blocks, GMM_WARPS * 32, (size_t)ring, st>>>(v->d_feat, v->d_samp_off, v->d_frame_off, n, a,
                                                                              d_flags, d_seg_n, d_segs, d_times, live);
        }
        PSB_LAUNCH_CHECK();
    }
    PSB_CUDA(cudaEventRecord(v->ev[1], st));
    unsigned long long rep = 0;
    PSB_CUDA(cudaMemcpyAsync(&rep, v->d_repairs, sizeof(rep), cudaMemcpyDeviceToHost, st));
    PSB_CUDA(cudaStreamSynchronize(st));
    v->last_repairs = (int64_t)rep;
    if (ms) PSB_CUDA(cudaEventElapsedTime(ms, v->ev[0], v->ev[1]));
    return PSB_OK;
}

}  // namespace

extern "C" void psb_vad_free(psb_vad_t *v)
{
    if (!v) return;
    cudaSetDevice(v->device);
    delete v;
}

extern "C" int psb_vad_create(const psb_vad_opts_t *o, int device, psb_vad_t **out)
{
    PSB_REQUIRE(o && out, "psb_vad_create: bad argument");
    *out = nullptr;
    PSB_REQUIRE(o->mode >= 0 && o->mode <= 3, "psb_vad_create: invalid VAD mode %d (0..3)", o->mode);
    const int rate = o->sample_rate == 0 ? 16000 : o->sample_rate;
    const double fl = o->frame_length == 0.0 ? 0.03 : o->frame_length;
    int closest = 0;
    double best = 0.5;
    for (int r : {8000, 16000, 32000, 48000}) {
        const double d = fabs(1.0 - (double)r / rate);
        if (d < best) closest = r, best = d;
    }
    PSB_REQUIRE(closest != 0, "psb_vad_create: no suitable sampling rate found for %d", rate);
    PSB_REQUIRE(closest != 48000, "psb_vad_create: %d Hz maps to 48 kHz, whose 48->8 kHz resampler is not implemented", rate);
    PSB_REQUIRE(fl > 0.0 && fl < 1.0, "psb_vad_create: unsupported frame length %f", fl);
    const int frame_size = (int)(size_t)(closest * fl);
    PSB_REQUIRE(frame_size == closest / 100 || frame_size == closest / 50 || frame_size == closest * 3 / 100,
                "psb_vad_create: unsupported frame length %f (10, 20 or 30 ms)", fl);
    const double window = o->window == 0.0 ? 0.3 : o->window, ratio = o->ratio == 0.0 ? 0.9 : o->ratio;
    const double flen = (double)frame_size / rate;
    const double ml = window / flen + 0.5;
    PSB_REQUIRE(ml >= 0.0 && ml < 2147483647.0, "psb_vad_create: window %f out of range", window);
    const int maxlen = (int)ml;
    const int start_frames = (int)(ratio * maxlen), end_frames = (int)((1.0 - ratio) * maxlen + 0.5);
    PSB_REQUIRE(start_frames > 0 && start_frames < maxlen,
                "psb_vad_create: ratio %.2f makes start-pointing stupid or impossible (%d frames of %d)", ratio, start_frames, maxlen);
    PSB_REQUIRE(end_frames > 0 && end_frames < maxlen,
                "psb_vad_create: ratio %.2f makes end-pointing stupid or impossible (%d frames of %d)", ratio, end_frames, maxlen);
    PSB_REQUIRE(o->warmup >= -1, "psb_vad_create: warmup must be >= -1 (got %d)", o->warmup);
    PSB_REQUIRE(maxlen + 1 <= GMM_RING_MAX, "psb_vad_create: window of %d frames; at most %d are implemented", maxlen, GMM_RING_MAX - 1);
    PSB_CUDA(cudaSetDevice(device));
    std::unique_ptr<psb_vad_t> v(new psb_vad_t());
    v->device = device;
    v->mode = o->mode, v->sample_rate = rate, v->closest = closest, v->frame_size = frame_size;
    v->frame_length = flen, v->window = window, v->ratio = ratio;
    v->maxlen = maxlen, v->start_frames = start_frames, v->end_frames = end_frames;
    // default warm-up: the frames of 0.5 s of audio (a 0.2 s warm-up left 12 % of the 64-frame chunks of an hour of
    // speech and silence to repair at 10 ms frames; see DESIGN)
    v->warmup = o->warmup == 0 ? (int)ceil(0.5 / flen - 1e-9) : o->warmup < 0 ? 0 : o->warmup;
    cudaError_t e = v->stream.create();
    if (e == cudaSuccess) e = v->ev[0].create();
    if (e == cudaSuccess) e = v->ev[1].create();
    if (e != cudaSuccess) {
        psb_set_error("psb_vad_create: %s", cudaGetErrorString(e));
        return PSB_ERR_CUDA;
    }
    int rc = v->d_repairs.reserve(1);
    if (!rc) rc = v->d_changed.reserve(1);
    if (!rc) rc = v->h_changed.reserve(1);
    if (rc) return rc;
    *out = v.release();
    return PSB_OK;
}

extern "C" int32_t psb_vad_frame_size(const psb_vad_t *v) { return v ? v->frame_size : -1; }
extern "C" double psb_vad_frame_length(const psb_vad_t *v) { return v ? v->frame_length : -1.0; }
extern "C" int32_t psb_vad_sample_rate(const psb_vad_t *v) { return v ? v->sample_rate : -1; }
extern "C" int32_t psb_vad_start_frames(const psb_vad_t *v) { return v ? v->start_frames : -1; }
extern "C" int32_t psb_vad_end_frames(const psb_vad_t *v) { return v ? v->end_frames : -1; }
extern "C" int32_t psb_vad_maxlen(const psb_vad_t *v) { return v ? v->maxlen : -1; }
extern "C" int32_t psb_vad_warmup(const psb_vad_t *v) { return v ? v->warmup : -1; }
extern "C" int64_t psb_vad_last_repairs(const psb_vad_t *v) { return v ? v->last_repairs : -1; }
extern "C" int32_t psb_vad_last_passes(const psb_vad_t *v) { return v ? (int32_t)v->last_passes : -1; }

extern "C" int psb_vad_process_device(psb_vad_t *v, const int16_t *d_pcm, const int64_t *samp_off, int32_t n_streams,
                                      int8_t *d_flags, int32_t *frame_off, int32_t *d_seg_n, int64_t *d_segs,
                                      double *d_times, float *ms)
{
    PSB_REQUIRE(v && samp_off && frame_off && n_streams >= 0, "psb_vad_process_device: bad argument");
    PSB_REQUIRE(samp_off[0] == 0, "psb_vad_process_device: samp_off[0] must be 0");
    PSB_REQUIRE(d_pcm || samp_off[n_streams] == 0, "psb_vad_process_device: pcm is null");
    PSB_REQUIRE(n_streams == 0 || (d_flags && d_seg_n && d_segs && d_times), "psb_vad_process_device: output is null");
    PSB_CUDA(cudaSetDevice(v->device));
    return vad_run(v, d_pcm, samp_off, n_streams, d_flags, frame_off, d_seg_n, d_segs, d_times, ms);
}

extern "C" int psb_vad_process_host(psb_vad_t *v, const int16_t *pcm, const int64_t *samp_off, int32_t n_streams,
                                    int8_t *flags, int32_t *frame_off, int32_t *seg_n, int64_t *segs, double *times)
{
    PSB_REQUIRE(v && samp_off && frame_off && n_streams >= 0, "psb_vad_process_host: bad argument");
    PSB_REQUIRE(samp_off[0] == 0, "psb_vad_process_host: samp_off[0] must be 0");
    const int64_t ns = samp_off[n_streams];
    PSB_REQUIRE(ns == 0 || pcm, "psb_vad_process_host: pcm is null");
    PSB_REQUIRE(n_streams == 0 || (flags && seg_n && segs && times), "psb_vad_process_host: output is null");
    PSB_CUDA(cudaSetDevice(v->device));
    int64_t total = 0;
    for (int s = 0; s < n_streams; ++s) total += std::max<int64_t>(samp_off[s + 1] - samp_off[s], 0) / v->frame_size;
    int rc = v->d_pcm.reserve(std::max<size_t>((size_t)ns, 1));
    if (!rc) rc = v->d_flags.reserve(std::max<size_t>((size_t)total, 1));
    if (!rc) rc = v->d_seg_n.reserve(std::max<size_t>((size_t)n_streams, 1));
    if (!rc) rc = v->d_segs.reserve(std::max<size_t>((size_t)total * 2, 1));
    if (!rc) rc = v->d_times.reserve(std::max<size_t>((size_t)total * 2, 1));
    if (rc) return rc;
    if (ns) PSB_CUDA(cudaMemcpyAsync(v->d_pcm, pcm, (size_t)ns * 2, cudaMemcpyHostToDevice, v->stream));
    rc = vad_run(v, v->d_pcm, samp_off, n_streams, v->d_flags, frame_off, v->d_seg_n, v->d_segs, v->d_times, nullptr);
    if (rc) return rc;
    if (total) {
        PSB_CUDA(cudaMemcpy(flags, v->d_flags, (size_t)total, cudaMemcpyDeviceToHost));
        PSB_CUDA(cudaMemcpy(segs, v->d_segs, (size_t)total * 2 * sizeof(int64_t), cudaMemcpyDeviceToHost));
        PSB_CUDA(cudaMemcpy(times, v->d_times, (size_t)total * 2 * sizeof(double), cudaMemcpyDeviceToHost));
    }
    if (n_streams) PSB_CUDA(cudaMemcpy(seg_n, v->d_seg_n, (size_t)n_streams * 4, cudaMemcpyDeviceToHost));
    return PSB_OK;
}

namespace {

// the state of a fresh ps_endpointer_init into the listed slots (all n_slots when ids is null)
int vad_reset_slots(psb_vad_t *v, const int32_t *ids, int32_t n)
{
    if (ids) {
        PSB_REQUIRE(v->n_slots > 0, "psb_vad_live_reset: psb_vad_live_open has not been called");
        for (int i = 0; i < n; ++i)
            PSB_REQUIRE(ids[i] >= 0 && ids[i] < v->n_slots, "psb_vad_live_reset: slot %d out of range (0..%d)", ids[i], v->n_slots - 1);
        int rc = v->d_slot_of.reserve(std::max<size_t>((size_t)n * 2, 1));
        if (rc) return rc;
        if (n) PSB_CUDA(cudaMemcpyAsync(v->d_slot_of, ids, (size_t)n * 4, cudaMemcpyHostToDevice, v->stream));
    }
    psb_vad_slot_t fresh;
    psb_vad_slot_init(&fresh, v->maxlen, v->start_frames, v->end_frames, v->frame_size, v->sample_rate);
    if (n) {
        vad_reset_kernel<<<(n + 127) / 128, 128, 0, v->stream>>>(v->d_slot, ids ? v->d_slot_of.get() : nullptr, n, fresh);
        PSB_LAUNCH_CHECK();
    }
    PSB_CUDA(cudaStreamSynchronize(v->stream));
    for (int i = 0; i < n; ++i) {
        const int s = ids ? ids[i] : i;
        v->left_n[s] = 0;
        v->pushed[s] = 0;
    }
    return PSB_OK;
}

// checks a live call, computes the stitched offsets and runs it
int vad_feed(psb_vad_t *v, const char *fn, const int32_t *slots, int32_t n, const int16_t *d_new, const int64_t *samp_off,
             const int8_t *final, int8_t *d_flags, int32_t *frame_off, int32_t *d_seg_n, int64_t *d_segs, double *d_times,
             psb_vad_live_status_t *d_status, float *ms)
{
    PSB_REQUIRE(v->n_slots > 0, "%s: psb_vad_live_open has not been called", fn);
    PSB_REQUIRE(n == 0 || slots, "%s: slots is null", fn);
    PSB_REQUIRE(samp_off[0] == 0, "%s: samp_off[0] must be 0", fn);
    std::vector<char> seen((size_t)v->n_slots, 0);
    std::vector<int64_t> st_off((size_t)n + 1, 0);
    std::vector<int32_t> keep((size_t)n);
    for (int i = 0; i < n; ++i) {
        const int s = slots[i];
        PSB_REQUIRE(s >= 0 && s < v->n_slots, "%s: slot %d out of range (0..%d)", fn, s, v->n_slots - 1);
        PSB_REQUIRE(!seen[s], "%s: slot %d fed twice in one call", fn, s);
        seen[s] = 1;
        const int64_t add = samp_off[i + 1] - samp_off[i];
        PSB_REQUIRE(add >= 0, "%s: samp_off not monotone at %d", fn, i);
        const int64_t len = v->left_n[s] + add, nf = len / v->frame_size;
        PSB_REQUIRE(v->pushed[s] + nf < (int64_t)1 << 31, "%s: slot %d would pass 2^31 - 1 frames", fn, s);
        st_off[i + 1] = st_off[i] + len;
        keep[i] = final && final[i] ? 0 : (int32_t)(len - nf * v->frame_size);
    }
    const LiveCall lc{d_new, samp_off, slots, keep.data(), final, d_status};
    const int rc = vad_run(v, d_new, st_off.data(), n, d_flags, frame_off, d_seg_n, d_segs, d_times, ms, &lc);
    if (rc) return rc;
    for (int i = 0; i < n; ++i) {
        v->left_n[slots[i]] = keep[i];
        v->pushed[slots[i]] += frame_off[i + 1] - frame_off[i];
    }
    return PSB_OK;
}

}  // namespace

extern "C" int psb_vad_live_open(psb_vad_t *v, int32_t n_slots)
{
    PSB_REQUIRE(v && n_slots > 0, "psb_vad_live_open: bad argument");
    PSB_CUDA(cudaSetDevice(v->device));
    PSB_CUDA(cudaStreamSynchronize(v->stream));
    v->n_slots = 0;                                              // until the table is whole again
    int rc = v->d_slot.reserve((size_t)n_slots);
    if (!rc) rc = v->d_ring.reserve((size_t)n_slots * (v->maxlen + 1));
    if (!rc) rc = v->d_left.reserve((size_t)n_slots * v->frame_size);
    if (rc) return rc;
    v->left_n.assign((size_t)n_slots, 0);
    v->pushed.assign((size_t)n_slots, 0);
    rc = vad_reset_slots(v, nullptr, n_slots);
    if (!rc) v->n_slots = n_slots;
    return rc;
}

extern "C" int psb_vad_live_reset(psb_vad_t *v, const int32_t *slots, int32_t n)
{
    PSB_REQUIRE(v && n >= 0 && (n == 0 || slots), "psb_vad_live_reset: bad argument");
    PSB_CUDA(cudaSetDevice(v->device));
    return vad_reset_slots(v, slots, n);
}

extern "C" int psb_vad_feed_device(psb_vad_t *v, const int32_t *slots, int32_t n, const int16_t *d_pcm, const int64_t *samp_off,
                                   const int8_t *final, int8_t *d_flags, int32_t *frame_off, int32_t *d_seg_n, int64_t *d_segs,
                                   double *d_times, psb_vad_live_status_t *d_status, float *ms)
{
    PSB_REQUIRE(v && samp_off && frame_off && n >= 0, "psb_vad_feed_device: bad argument");
    PSB_REQUIRE(d_pcm || samp_off[n] == 0, "psb_vad_feed_device: pcm is null");
    PSB_REQUIRE(n == 0 || (d_flags && d_seg_n && d_segs && d_times && d_status), "psb_vad_feed_device: output is null");
    PSB_CUDA(cudaSetDevice(v->device));
    return vad_feed(v, "psb_vad_feed_device", slots, n, d_pcm, samp_off, final, d_flags, frame_off, d_seg_n, d_segs, d_times,
                    d_status, ms);
}

extern "C" int psb_vad_feed_host(psb_vad_t *v, const int32_t *slots, int32_t n, const int16_t *pcm, const int64_t *samp_off,
                                 const int8_t *final, int8_t *flags, int32_t *frame_off, int32_t *seg_n, int64_t *segs,
                                 double *times, psb_vad_live_status_t *status)
{
    PSB_REQUIRE(v && samp_off && frame_off && n >= 0, "psb_vad_feed_host: bad argument");
    const int64_t ns = samp_off[n];
    PSB_REQUIRE(ns == 0 || pcm, "psb_vad_feed_host: pcm is null");
    PSB_REQUIRE(n == 0 || (flags && seg_n && segs && times && status), "psb_vad_feed_host: output is null");
    PSB_CUDA(cudaSetDevice(v->device));
    int64_t cap = 0;                                             // frames at most: leftovers are shorter than a frame
    for (int i = 0; i < n; ++i) cap += (std::max<int64_t>(samp_off[i + 1] - samp_off[i], 0) + v->frame_size - 1) / v->frame_size;
    int rc = v->d_pcm.reserve(std::max<size_t>((size_t)ns, 1));
    if (!rc) rc = v->d_flags.reserve(std::max<size_t>((size_t)cap, 1));
    if (!rc) rc = v->d_seg_n.reserve(std::max<size_t>((size_t)n, 1));
    if (!rc) rc = v->d_segs.reserve(std::max<size_t>((size_t)(cap + n) * 2, 1));
    if (!rc) rc = v->d_times.reserve(std::max<size_t>((size_t)(cap + n) * 2, 1));
    if (!rc) rc = v->d_status.reserve(std::max<size_t>((size_t)n, 1));
    if (rc) return rc;
    if (ns) PSB_CUDA(cudaMemcpyAsync(v->d_pcm, pcm, (size_t)ns * 2, cudaMemcpyHostToDevice, v->stream));
    rc = vad_feed(v, "psb_vad_feed_host", slots, n, v->d_pcm, samp_off, final, v->d_flags, frame_off, v->d_seg_n, v->d_segs,
                  v->d_times, v->d_status, nullptr);
    if (rc) return rc;
    const size_t total = (size_t)frame_off[n], rows = total + (size_t)n;
    if (total) PSB_CUDA(cudaMemcpy(flags, v->d_flags, total, cudaMemcpyDeviceToHost));
    if (n) {
        PSB_CUDA(cudaMemcpy(segs, v->d_segs, rows * 2 * sizeof(int64_t), cudaMemcpyDeviceToHost));
        PSB_CUDA(cudaMemcpy(times, v->d_times, rows * 2 * sizeof(double), cudaMemcpyDeviceToHost));
        PSB_CUDA(cudaMemcpy(seg_n, v->d_seg_n, (size_t)n * 4, cudaMemcpyDeviceToHost));
        PSB_CUDA(cudaMemcpy(status, v->d_status, (size_t)n * sizeof(psb_vad_live_status_t), cudaMemcpyDeviceToHost));
    }
    return PSB_OK;
}
