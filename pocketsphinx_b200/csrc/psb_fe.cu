// psb_fe.cu -- batched front end on the device (SURVEY 8 row f-2): int16 PCM -> MFCC -> CMN ->
// dynamic features, for whole batches of utterances, each treated as a fresh stream
// (ps_start_stream + ps_process_raw(full_utt), pocketsphinx.c:1073, acmod.c:528-560) unless
// psb_fe_set_stream_starts carries the noise tracker from one utterance of a session to the next.
//
// Restates, operation for operation and in the reference's float32/float64 types and order:
//   fe_pre_emphasis_int16 / fe_hamming_window / fe_spch_to_frame     (fe_sigproc.c:726-853)
//   fe_fft_real (Sorensen real-valued FFT, float64)                  (:1062-1159)
//   fe_spec_magnitude / fe_mel_spec                                  (:1161-1242)
//   fe_remove_noise and its helpers                                  (fe_noise.c:109-364)
//   fe_mel_cep, fe_spec2cep / fe_dct2, fe_lifter                     (:1244-1349)
//   frame counting of fe_process_frames + fe_end_utt                 (fe_interface.c:352-545)
//   cmn (batch, with or without varnorm)                             (feat/cmn.c:165-232)
//   agc_max / agc_emax + agc_emax_update / agc_noise on c0           (feat/agc.c:110-216, feat.c:941-966)
//   feat_1s_c_d_dd_cep2feat with replicated edges                    (feat/feat.c:579-622, 1243-1330)
//   feat_s2_4x_cep2feat / feat_s3_1x39_cep2feat                      (feat/feat.c:425-538)
//   cmn_live + cmn_live_shiftwin + cmn_live_update over a session    (feat/cmn_live.c, feat.c:917-938)
//   dither: MT19937 (util/genrand.c) in the draw order of fe_process_frames + fe_end_utt
//   feat_lda_transform                                               (feat/lda.c:139-159)
// All tables (window, twiddles, mel filters, DCT cosines, lifter) are INPUTS: the host builds
// them with the reference's own init code / libm and passes them in psb_fe_desc_t.  The only
// operation that is not bit-reproducible is log(): device libm vs glibc can differ in the last
// bit of a float64, which survives the float32 rounding of the DCT sums only rarely (parity is
// asserted at 1e-4 relative as north_star allows for float paths; see tests/test_gpu_fe.py).
#include "psb_internal.cuh"

#include <string.h>

#include <algorithm>
#include <vector>

struct psb_fe_s {
    int device;
    int frame_size, frame_shift, fft_size, fft_order, n_filt, n_cep;
    int remove_dc, remove_noise, transform, lifter_val, window, cmn, n_coeffs;
    float alpha, sqrt_inv_n, sqrt_inv_2n;
    Stream stream;                // declared first: destroyed after the buffers below
    Event ev[2];
    DevBuf<double> d_hamming, d_ccc, d_sss;
    DevBuf<int16_t> d_spec_start, d_filt_start, d_filt_width;
    DevBuf<float> d_filt_coeffs, d_mel_cosine, d_lifter;
    DevBuf<int> d_rev;            // bit-reversal permutation [fft_size]
    // workspace
    DevBuf<double> d_mfspec;      // [frames][n_filt]
    DevBuf<float> d_mfcc;         // [frames][n_cep]
    DevBuf<int16_t> d_pcm;
    DevBuf<float> d_feats;
    DevBuf<int64_t> d_samp_off; DevBuf<int32_t> d_frame_off, d_frame_utt;
    // psb_fe_create_ex options and sessions
    int feat, feat_dim, dither, seed;
    int varnorm, agc, stream_dim;             // stream_dim: the features' dimension before LDA
    float agc_thresh;
    DevBuf<float> d_lda;                      // [feat_dim][stream_dim], NULL without LDA
    DevBuf<float> d_raw;                      // [frames][stream_dim]: the features LDA reads
    float cmn_init[PSB_FE_MAX_CEP];
    std::vector<int32_t> sess_off;            // set by psb_fe_set_sessions for the next call only
    std::vector<psb_fe_state_t> states;       // in: the next call's sessions; out: after it
    bool sess_pending;
    DevBuf<psb_fe_state_t> d_state;
    DevBuf<int32_t> d_sess_off;
    DevBuf<int64_t> d_draw;                   // per utterance: first tail sample, tail offset, main draws, tail draws
    DevBuf<int16_t> d_dpcm;                   // dithered samples of the full frames
    DevBuf<int16_t> d_tail;                   // freshly dithered samples of each utterance's last frame
    // psb_fe_set_stream_starts, for the next call only
    std::vector<uint8_t> starts;              // per utterance: 1 = ps_start_stream before it
    std::vector<psb_fe_noise_t> noise;        // in: the next call's trackers (empty: undefined); out: after it
    bool starts_pending, noise_out;           // noise_out: the last call set stream starts, noise holds its trackers
    DevBuf<psb_fe_noise_t> d_noise;           // [2][n_sess]: in, then out
    DevBuf<int4> d_chain;
    // psb_fe_set_filterbanks, for the next call only: n_bank banks of n_filt filters, bank[u] per utterance
    std::vector<int16_t> bank_spec_start, bank_filt_start, bank_filt_width;   // [n_bank][n_filt]
    std::vector<int32_t> bank_coeff_off, bank_of_utt;                          // [n_bank + 1], [n_utt]
    std::vector<float> bank_coeffs;
    bool banks_pending;
    DevBuf<int16_t> d_bank_spec_start, d_bank_filt_start, d_bank_filt_width;
    DevBuf<int32_t> d_bank_coeff_off, d_bank_of_utt;
    DevBuf<float> d_bank_coeffs;
};

namespace {

constexpr int FE_MAX_FILT = 64;
static_assert(FE_MAX_FILT == PSB_FE_MAX_FILT, "psb_fe_noise_t holds one entry per filter");
constexpr int FE_MAX_CEP = 32;

struct FeDev {
    int frame_size, frame_shift, fft_size, fft_order, n_filt, n_cep;
    int remove_dc, remove_noise, transform, lifter_val;
    float alpha, sqrt_inv_n, sqrt_inv_2n;
    const double *hamming, *ccc, *sss;
    const int16_t *spec_start, *filt_start, *filt_width;
    const float *filt_coeffs, *mel_cosine, *lifter;
    const int *rev;
};

// One CTA per frame: samples -> pre-emphasis -> window -> real FFT -> power spectrum -> mel.
// frame_utt[f] = utterance of flat frame f; frame_off[u] = first flat frame of utterance u.
// DITHER: pcm holds the dithered samples of the full frames, and the last frame of utterance u
// reads its own freshly dithered copy at tail + draw[4u + 1] (fe_end_utt re-reads the overflow
// samples); its pre-emphasis prior is still the full frames' sample before it.
// BANKS: p's filter tables hold several banks ([bank][n_filt], filt_start relative to the bank's first
// coefficient coeff_off[bank]), and utterance u reads bank bank_of_utt[u] (psb_fe_set_filterbanks).
template <bool DITHER, bool BANKS>
__global__ void __launch_bounds__(128)
fe_frame_kernel(FeDev p, const int16_t *__restrict__ pcm, const int64_t *__restrict__ samp_off,
                const int32_t *__restrict__ frame_off, const int32_t *__restrict__ frame_utt,
                double *__restrict__ mfspec, const int16_t *__restrict__ tail, const int64_t *__restrict__ draw,
                const int32_t *__restrict__ bank_of_utt, const int32_t *__restrict__ coeff_off)
{
    extern __shared__ double x[];             // [fft_size] frame, then [fft_size/2 + 1] power spectrum
    double *spec = x + p.fft_size;
    const int f = blockIdx.x;
    const int u = frame_utt[f];
    const int k = f - frame_off[u];           // frame index inside the utterance
    const int64_t s0 = samp_off[u], n = samp_off[u + 1] - s0;
    const int64_t start = (int64_t)k * p.frame_shift;
    int len = (int)min((int64_t)p.frame_size, n - start);
    const int16_t *in = pcm + s0 + start;
    const int16_t *src = in;
    if constexpr (DITHER)
        if (k == frame_off[u + 1] - frame_off[u] - 1) src = tail + draw[4 * u + 1];
    const int tid = threadIdx.x, nt = blockDim.x;
    const int half = p.frame_size / 2;

    // fe_spch_to_frame: pre-emphasis (prior = the sample just before the frame), zero padding,
    // Hamming window over frame_size; stored bit-reversed for the FFT below.
    if (!p.remove_dc) {
        for (int i = tid; i < p.fft_size; i += nt) {
            double v = 0.0;
            if (i < len) {
                if (p.alpha != 0.0f) {
                    const int16_t prev = i > 0 ? src[i - 1] : (start > 0 ? in[-1] : (int16_t)0);
                    v = (double)src[i] - (double)prev * (double)p.alpha;
                }
                else
                    v = (double)src[i];
            }
            if (i < half) v = v * p.hamming[i];
            else if (i >= p.frame_size - half && i < p.frame_size) v = v * p.hamming[p.frame_size - 1 - i];
            x[p.rev[i]] = v;
        }
    }
    else {
        // remove_dc needs the reference's sequential mean (fe_sigproc.c:805-812)
        for (int i = tid; i < p.fft_size; i += nt) {
            double v = 0.0;
            if (i < len) {
                if (p.alpha != 0.0f) {
                    const int16_t prev = i > 0 ? src[i - 1] : (start > 0 ? in[-1] : (int16_t)0);
                    v = (double)src[i] - (double)prev * (double)p.alpha;
                }
                else
                    v = (double)src[i];
            }
            x[i] = v;
        }
        __syncthreads();
        __shared__ double mean_s;
        if (tid == 0) {
            double mean = 0;
            for (int i = 0; i < p.frame_size; ++i) mean += x[i];
            mean_s = mean / p.frame_size;
        }
        __syncthreads();
        double keep[8];                                      // fft_size <= 8 * 128
        int c = 0;
        for (int i = tid; i < p.fft_size; i += nt) {
            double v = x[i];
            if (i < p.frame_size) v -= mean_s;
            if (i < half) v = v * p.hamming[i];
            else if (i >= p.frame_size - half && i < p.frame_size) v = v * p.hamming[p.frame_size - 1 - i];
            keep[c++] = v;
        }
        __syncthreads();
        c = 0;
        for (int i = tid; i < p.fft_size; i += nt) x[p.rev[i]] = keep[c++];
    }
    __syncthreads();

    // fe_fft_real.  Stage 0: 2-point butterflies.
    const int N = p.fft_size, m = p.fft_order;
    for (int i = 2 * tid; i < N; i += 2 * nt) {
        const double xt = x[i];
        x[i] = xt + x[i + 1];
        x[i + 1] = xt - x[i + 1];
    }
    __syncthreads();
    // Stages 1..m-1: N/4 independent work items each = (block, j)
    for (int kk = 1; kk < m; ++kk) {
        const int n4 = kk - 1, n2 = kk, n1 = kk + 1;
        const int per = 1 << n4;                             // items per block
        for (int w = tid; w < (N >> 2); w += nt) {
            const int b = w >> n4, j = w & (per - 1);
            const int i = b << n1;
            if (j == 0) {
                const double xt = x[i];
                x[i] = xt + x[i + (1 << n2)];
                x[i + (1 << n2)] = xt - x[i + (1 << n2)];
                x[i + (1 << n2) + (1 << n4)] = -x[i + (1 << n2) + (1 << n4)];
            }
            else {
                const int i1 = i + j, i2 = i + (1 << n2) - j, i3 = i + (1 << n2) + j, i4 = i + (1 << n2) + (1 << n2) - j;
                const double cc = p.ccc[j << (m - n1)], ss = p.sss[j << (m - n1)];
                const double x1 = x[i1], x2 = x[i2], x3 = x[i3], x4 = x[i4];
                const double t1 = x3 * cc + x4 * ss;
                const double t2 = x3 * ss - x4 * cc;
                x[i4] = x2 - t2;
                x[i3] = -x2 - t2;
                x[i2] = x1 - t1;
                x[i1] = x1 + t1;
            }
        }
        __syncthreads();
    }
    // fe_spec_magnitude
    for (int j = tid; j <= N / 2; j += nt)
        spec[j] = j == 0 ? x[0] * x[0] : x[j] * x[j] + x[N - j] * x[N - j];
    __syncthreads();
    // fe_mel_spec: one thread per filter, bins in ascending order; an empty filter (width 0) gives 0
    if (tid < p.n_filt) {
        int row = tid;
        const float *coeffs = p.filt_coeffs;
        if constexpr (BANKS) {
            const int b = bank_of_utt[u];
            row += b * p.n_filt;
            coeffs += coeff_off[b];
        }
        const int ss = p.spec_start[row], fs = p.filt_start[row], fw = p.filt_width[row];
        double acc = 0;
        for (int i = 0; i < fw; ++i) acc += spec[ss + i] * (double)coeffs[fs + i];
        mfspec[(size_t)f * p.n_filt + tid] = acc;
    }
}

// fe_remove_noise (fe_noise.c:270-364, float build) for one filter of one frame: the tracker's
// smoothers (power, noise, floor_, peak), and the gain (fe_noise_gain) and its +-4-filter smoothing
// (fe_noise_smooth) in two steps, since the smoothing reads the neighbours' gains.
// INIT: noise_stats->undefined (:290-305).
__device__ __forceinline__ double fe_noise_gain(double &power, double &noise, double &floor_, double &peak, double mval,
                                                bool init)
{
    // fe_noise.c constants (:64-75, :214-227)
    const double lambda_power = 0.7, comp_lambda_power = 1 - 0.7, lambda_a = 0.995, comp_lambda_a = 1 - 0.995,
                 lambda_b = 0.5, comp_lambda_b = 1 - 0.5, lambda_t = 0.85, mu_t = 0.2, max_gain = 20,
                 inv_max_gain = 1.0 / 20;
    if (init) {
        power = mval;
        noise = mval / max_gain;
        floor_ = mval / max_gain;
        peak = 0.0;
    }
    power = lambda_power * power + comp_lambda_power * mval;
    // fe_lower_envelope(power -> noise)
    if (power >= noise) noise = lambda_a * noise + comp_lambda_a * power;
    else noise = lambda_b * noise + comp_lambda_b * power;
    double signal = power - noise;
    if (signal < 1.0) signal = 1.0;
    // fe_lower_envelope(signal -> floor)
    if (signal >= floor_) floor_ = lambda_a * floor_ + comp_lambda_a * signal;
    else floor_ = lambda_b * floor_ + comp_lambda_b * signal;
    // fe_temp_masking
    const double cur_in = signal;
    peak *= lambda_t;
    if (signal < lambda_t * peak) signal = peak * mu_t;
    if (cur_in > peak) peak = cur_in;
    if (signal < floor_) signal = floor_;
    double g;
    if (signal < max_gain * power) g = signal / power;
    else g = max_gain;
    if (g < inv_max_gain) g = inv_max_gain;
    return g;
}

// fe_weight_smooth, window of +-4 filters: filter tid's value after noise removal
__device__ __forceinline__ double fe_noise_smooth(const double *gain, int tid, int nf, double mval)
{
    const int l1 = (tid - 4) > 0 ? (tid - 4) : 0;
    const int l2 = (tid + 4) < (nf - 1) ? (tid + 4) : (nf - 1);
    double coef = 0;
    for (int j = l1; j <= l2; ++j) coef += gain[j];
    return mval * (coef / (l2 - l1 + 1));
}

// One CTA (64 threads) per utterance: noise removal (sequential over frames), log, cepstral
// transform, lifter; then batch CMN (VARNORM: with variance normalisation); then the dynamic features.
template <bool VARNORM>
__global__ void __launch_bounds__(64)
fe_utt_kernel(FeDev p, const int32_t *__restrict__ frame_off, double *__restrict__ mfspec,
              float *__restrict__ mfcc, float *__restrict__ feats, int cmn, int window)
{
    __shared__ double gain[FE_MAX_FILT], lm[FE_MAX_FILT];
    __shared__ float mean_s[FE_MAX_CEP];
    const int u = blockIdx.x, tid = threadIdx.x;
    const int f0 = frame_off[u], T = frame_off[u + 1] - f0;
    if (T <= 0) return;
    const int nf = p.n_filt, nc = p.n_cep;
    double power = 0, noise = 0, floor_ = 0, peak = 0;
    for (int t = 0; t < T; ++t) {
        const size_t fr = (size_t)(f0 + t);
        double mval = tid < nf ? mfspec[fr * nf + tid] : 0.0;
        if (p.remove_noise) {
            if (tid < nf) gain[tid] = fe_noise_gain(power, noise, floor_, peak, mval, t == 0);
            __syncthreads();
            if (tid < nf) mval = fe_noise_smooth(gain, tid, nf, mval);
        }
        if (tid < nf) lm[tid] = log(mval + 1e-4);                        // fe_mel_cep, LOG_FLOOR
        __syncthreads();
        if (tid < nc) {
            float c;
            if (p.transform == 0) {                                      // fe_spec2cep (legacy)
                if (tid == 0) {
                    c = (float)(lm[0] / 2);
                    for (int j = 1; j < nf; ++j) c = (float)((double)c + lm[j]);
                    c = (float)((double)c / (double)nf);
                }
                else {
                    c = 0.f;
                    for (int j = 0; j < nf; ++j) {
                        const int beta = j == 0 ? 1 : 2;
                        c = (float)((double)c + (lm[j] * (double)p.mel_cosine[tid * nf + j]) * beta);
                    }
                    c = (float)((double)c / ((double)nf * 2));
                }
            }
            else {                                                       // fe_dct2
                if (tid == 0) {
                    c = (float)lm[0];
                    for (int j = 1; j < nf; ++j) c = (float)((double)c + lm[j]);
                    c = __fmul_rn(c, p.transform == 2 ? p.sqrt_inv_2n : p.sqrt_inv_n);
                }
                else {
                    c = 0.f;
                    for (int j = 0; j < nf; ++j) c = (float)((double)c + lm[j] * (double)p.mel_cosine[tid * nf + j]);
                    c = __fmul_rn(c, p.sqrt_inv_2n);
                }
            }
            if (p.lifter_val) c = __fmul_rn(c, p.lifter[tid]);           // fe_lifter
            mfcc[fr * nc + tid] = c;
        }
        __syncthreads();
    }
    // cmn() batch (cmn.c:136-176): float32 running sums over frames with c0 >= 0
    if (cmn == 1) {
        __threadfence_block();
        __syncthreads();
        if (tid < nc) {
            float sum = 0.f;
            int cnt = 0;
            for (int t = 0; t < T; ++t) {
                const float *row = mfcc + (size_t)(f0 + t) * nc;
                if (row[0] < 0) continue;
                sum = __fadd_rn(sum, row[tid]);
                ++cnt;
            }
            mean_s[tid] = __fdiv_rn(sum, (float)cnt);
        }
        __syncthreads();
        if constexpr (VARNORM) {
            // cmn.c:209-231: the variance sums over every frame, c0 >= 0 or not, in frame order;
            // inverse standard deviation (float)sqrt((double)n_frame / var)
            __shared__ float istd_s[FE_MAX_CEP];
            if (tid < nc) {
                float var = 0.f;
                for (int t = 0; t < T; ++t) {
                    const float d = __fsub_rn(mfcc[(size_t)(f0 + t) * nc + tid], mean_s[tid]);
                    var = __fadd_rn(var, __fmul_rn(d, d));
                }
                istd_s[tid] = __double2float_rn(__dsqrt_rn(__ddiv_rn((double)T, (double)var)));
            }
            __syncthreads();
            for (int i = tid; i < T * nc; i += blockDim.x) {
                float *v = mfcc + (size_t)f0 * nc + i;
                *v = __fmul_rn(__fsub_rn(*v, mean_s[i % nc]), istd_s[i % nc]);
            }
        }
        else {
            for (int i = tid; i < T * nc; i += blockDim.x) {
                float *v = mfcc + (size_t)f0 * nc + i;
                *v = __fsub_rn(*v, mean_s[i % nc]);
            }
        }
        __threadfence_block();
        __syncthreads();
    }
    // feat_1s_c_d_dd_cep2feat (feat.c:579-622); the frames before the first / after the last
    // are copies of it (feat_s2mfc2feat_live with beginutt / endutt, feat.c:1269-1300)
    if (feats) {
        const int W = window - 1;                                        // FEAT_DCEP_WIN = 2
        const int D = 3 * nc;
        for (int i = tid; i < T * nc; i += blockDim.x) {
            const int t = i / nc, c = i % nc;
            const float *base = mfcc + (size_t)f0 * nc + c;
#define CEP(tt) base[(size_t)min(max((tt), 0), T - 1) * nc]
            float *o = feats + (size_t)(f0 + t) * D;
            o[c] = CEP(t);
            o[nc + c] = __fsub_rn(CEP(t + W), CEP(t - W));
            const float d1 = __fsub_rn(CEP(t + W + 1), CEP(t - W + 1));
            const float d2 = __fsub_rn(CEP(t + W - 1), CEP(t - W - 1));
            o[2 * nc + c] = __fsub_rn(d1, d2);
#undef CEP
        }
    }
}

// The noise tracker carried across utterances (ps_start_stream only where a stream starts), in place
// on the mel spectra before fe_utt_kernel, which then runs without its own noise removal.  One CTA per
// chain: a chain is utterances chain.x .. chain.y - 1 of one session, whose frames are consecutive, with
// no stream start after its first utterance.  It starts from in[chain.z] (chain.z < 0: a stream start,
// noise_stats->undefined) and stores its tracker in out[chain.w] (chain.w < 0: a later chain of the
// session has the session's last state).  A stored tracker that is still undefined has zero arrays, so
// the bytes do not depend on how a session is cut into calls.
// Only the four smoothers are a recurrence over frames.  The chain is walked in runs of FE_NOISE_RUN
// frames: the run's spectra are staged in shared memory by all threads, one thread per filter runs the
// recurrence and each frame's gain through the run, then all threads smooth the gains and write the run.
constexpr int FE_NOISE_RUN = 32, FE_NOISE_THREADS = 128;

__global__ void __launch_bounds__(FE_NOISE_THREADS)
fe_noise_kernel(int nf, const int32_t *__restrict__ frame_off, const int4 *__restrict__ chain,
                const psb_fe_noise_t *__restrict__ in, psb_fe_noise_t *__restrict__ out, double *__restrict__ mfspec)
{
    __shared__ double ms[FE_NOISE_RUN * FE_MAX_FILT], gain[FE_NOISE_RUN][FE_MAX_FILT];
    const int4 c = chain[blockIdx.x];
    const int tid = threadIdx.x;
    const bool on = tid < nf;
    double power = 0, noise = 0, floor_ = 0, peak = 0;
    bool undef = true;
    if (c.z >= 0) {
        const psb_fe_noise_t *i = in + c.z;
        undef = i->undefined != 0;
        if (on && !undef) { power = i->power[tid]; noise = i->noise[tid]; floor_ = i->floor[tid]; peak = i->peak[tid]; }
    }
    const int f0 = frame_off[c.x], f1 = frame_off[c.y];
    for (int r0 = f0; r0 < f1; r0 += FE_NOISE_RUN) {
        const int n = min(FE_NOISE_RUN, f1 - r0);
        double *run = mfspec + (size_t)r0 * nf;
        for (int i = tid; i < n * nf; i += blockDim.x) ms[i] = run[i];
        __syncthreads();
        if (on)
            for (int k = 0; k < n; ++k) {
                gain[k][tid] = fe_noise_gain(power, noise, floor_, peak, ms[k * nf + tid], undef);
                undef = false;
            }
        undef = false;
        __syncthreads();
        for (int i = tid; i < n * nf; i += blockDim.x) {
            const int k = i / nf;
            run[i] = fe_noise_smooth(gain[k], i - k * nf, nf, ms[i]);
        }
        __syncthreads();
    }
    if (c.w >= 0) {
        psb_fe_noise_t *o = out + c.w;
        if (tid == 0) { o->undefined = undef; o->reserved = 0; }
        if (on) {
            o->power[tid] = undef ? 0.0 : power;
            o->noise[tid] = undef ? 0.0 : noise;
            o->floor[tid] = undef ? 0.0 : floor_;
            o->peak[tid] = undef ? 0.0 : peak;
        }
        for (int i = nf + tid; i < FE_MAX_FILT; i += blockDim.x)
            o->power[i] = o->noise[i] = o->floor[i] = o->peak[i] = 0.0;
    }
}

// One CTA per session: the session's MT19937 stream (genrand_int32, util/genrand.c), one draw per
// sample read.  Utterance u draws draw[4u + 2] times for its full frames (sample i <- draw i) and
// then draw[4u + 3] times for the samples of its last frame, from sample draw[4u] on (fe_end_utt).
// The twist of 624 words runs in three barrier-separated phases: words < 227 read only old
// words, words < 454 read the first phase's, the rest read the second's (and word 0).
constexpr int MT_N = 624, MT_M = 397, FE_DITHER_THREADS = 640;

__global__ void __launch_bounds__(FE_DITHER_THREADS)
fe_dither_kernel(const int16_t *__restrict__ pcm, const int64_t *__restrict__ samp_off,
                 const int32_t *__restrict__ sess_off, const int64_t *__restrict__ draw,
                 psb_fe_state_t *__restrict__ state, int16_t *__restrict__ dpcm, int16_t *__restrict__ tail)
{
    __shared__ uint32_t mt[MT_N];
    const int s = blockIdx.x, tid = threadIdx.x;
    psb_fe_state_t *st = state + s;
    for (int i = tid; i < MT_N; i += blockDim.x) mt[i] = st->mt[i];
    int mti = st->mt_index;
    __syncthreads();
    for (int u = sess_off[s]; u < sess_off[s + 1]; ++u) {
        const int64_t s0 = samp_off[u];
        for (int part = 0; part < 2; ++part) {
            const int64_t n = draw[4 * u + 2 + part];
            const int16_t *in = part ? pcm + s0 + draw[4 * u] : pcm + s0;
            int16_t *out = part ? tail + draw[4 * u + 1] : dpcm + s0;
            for (int64_t done = 0; done < n;) {
                if (mti >= MT_N) {
                    if (mti == MT_N + 1) {                       // never seeded: init_genrand(5489)
                        if (tid == 0) {
                            mt[0] = 5489u;
                            for (int i = 1; i < MT_N; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
                        }
                        __syncthreads();
                    }
                    for (int ph = 0; ph < 3; ++ph) {
                        const int lo = ph == 0 ? 0 : ph == 1 ? MT_N - MT_M : 2 * (MT_N - MT_M);
                        const int hi = ph == 0 ? MT_N - MT_M : ph == 1 ? 2 * (MT_N - MT_M) : MT_N;
                        const int kk = lo + tid;
                        uint32_t v = 0;
                        if (kk < hi) {
                            const uint32_t y = (mt[kk] & 0x80000000u) | (mt[kk + 1 < MT_N ? kk + 1 : 0] & 0x7fffffffu);
                            v = mt[kk + MT_M < MT_N ? kk + MT_M : kk + MT_M - MT_N] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
                        }
                        __syncthreads();
                        if (kk < hi) mt[kk] = v;
                        __syncthreads();
                    }
                    mti = 0;
                }
                const int64_t chunk = min((int64_t)(MT_N - mti), n - done);
                if (tid < chunk) {
                    uint32_t y = mt[mti + tid];
                    y ^= y >> 11;
                    y ^= (y << 7) & 0x9d2c5680u;
                    y ^= (y << 15) & 0xefc60000u;
                    y ^= y >> 18;
                    const int add = ((y >> 1) & 3u) == 0;        // !(genrand_int31() % 4)
                    const int64_t j = done + tid;
                    out[j] = (int16_t)(in[j] + add);             // int16 wrap, as fe_read_frame_int16
                }
                mti += (int)chunk;
                done += chunk;
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < MT_N; i += blockDim.x) st->mt[i] = mt[i];
    if (tid == 0) st->mt_index = mti;
}

// One warp per session, one lane per coefficient: cmn_live over each utterance's frames in order
// (frames with c0 < 0 are skipped), then cmn_live_shiftwin when more than CMN_WIN_HWM frames are
// counted and cmn_live_update (feat_cmn with endutt).  ps_end_utt's feat_update_stats repeats the
// update, which leaves the state as it is.
__global__ void __launch_bounds__(32)
fe_cmn_live_kernel(const int32_t *__restrict__ sess_off, const int32_t *__restrict__ frame_off,
                   float *__restrict__ mfcc, int nc, psb_fe_state_t *__restrict__ state)
{
    constexpr int CMN_WIN = 500, CMN_WIN_HWM = 800;
    psb_fe_state_t *st = state + blockIdx.x;
    const int c = threadIdx.x;
    const bool on = c < nc;
    float mean = on ? st->cmn_mean[c] : 0.f, sum = on ? st->cmn_sum[c] : 0.f;
    int nframe = st->cmn_nframe;
    for (int u = sess_off[blockIdx.x]; u < sess_off[blockIdx.x + 1]; ++u) {
        for (int f = frame_off[u]; f < frame_off[u + 1]; ++f) {
            float *row = mfcc + (size_t)f * nc;
            if (row[0] < 0) continue;
            if (on) {
                const float v = row[c];
                sum = __fadd_rn(sum, v);
                row[c] = __fsub_rn(v, mean);
            }
            ++nframe;
        }
        if (nframe > CMN_WIN_HWM) {                                      // cmn_live_shiftwin
            const float sf = (float)(1.0 / nframe);
            mean = __fdiv_rn(sum, (float)nframe);
            sum = __fmul_rn(sum, __fmul_rn((float)CMN_WIN, sf));
            nframe = CMN_WIN;
        }
        if (nframe > 0) mean = __fdiv_rn(sum, (float)nframe);           // cmn_live_update
    }
    if (on) { st->cmn_mean[c] = mean; st->cmn_sum[c] = sum; }
    if (c == 0) st->cmn_nframe = nframe;
}

// The dynamic features of every frame from its utterance's cepstra (after CMN), one thread per
// (frame, coefficient); frames past either end of the utterance are copies of its first / last
// (feat_s2mfc2feat_live with beginutt and endutt).
__global__ void fe_feat_kernel(const int32_t *__restrict__ frame_off, const int32_t *__restrict__ frame_utt,
                               const float *__restrict__ mfcc, float *__restrict__ feats, int nc, int feat, int dim,
                               int32_t total)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)total * nc) return;
    const int f = (int)(i / nc), c = (int)(i % nc);
    const int u = frame_utt[f], f0 = frame_off[u], T = frame_off[u + 1] - f0, t = f - f0;
    const float *base = mfcc + (size_t)f0 * nc + c;
#define CEP(dt) base[(size_t)min(max(t + (dt), 0), T - 1) * nc]
    float *o = feats + (size_t)f * dim;
    const float dd = __fsub_rn(__fsub_rn(CEP(3), CEP(-1)), __fsub_rn(CEP(1), CEP(-3)));
    if (feat == PSB_FEAT_1S_C_D_DD) {                                    // feat.c:579-622
        o[c] = CEP(0);
        o[nc + c] = __fsub_rn(CEP(2), CEP(-2));
        o[2 * nc + c] = dd;
    }
    else if (c == 0) {                                                   // POW: C0, DC0, D2C0
        float *pw = o + (feat == PSB_FEAT_S2_4X ? 36 : 24);
        pw[0] = CEP(0);
        pw[1] = __fsub_rn(CEP(2), CEP(-2));
        pw[2] = dd;
    }
    else if (feat == PSB_FEAT_S2_4X) {                                   // feat.c:425-484
        o[c - 1] = CEP(0);
        o[12 + c - 1] = __fsub_rn(CEP(2), CEP(-2));
        o[24 + c - 1] = __fsub_rn(CEP(4), CEP(-4));
        o[51 - 12 + c - 1] = dd;
    }
    else {                                                               // s3_1x39, feat.c:487-538
        o[c - 1] = CEP(0);
        o[12 + c - 1] = __fsub_rn(CEP(2), CEP(-2));
        o[27 + c - 1] = dd;
    }
#undef CEP
}

// The extreme of c0 over T frames as the reference's sequential scans find it: the running value is
// replaced only by a strictly greater (MAX) / smaller value, so ties keep the earliest frame and a NaN
// never replaces it.  SEED: the scan starts from frame 0's value, as agc_max and agc_noise do (a NaN
// there is kept); else it starts empty and skips NaNs (agc_emax compares against the running
// obs_max instead).  Each lane scans a contiguous run of frames; the runs are combined in frame
// order.  Returns in every lane whether any value was taken, and the value in *out.
template <bool MAX, bool SEED>
__device__ bool c0_extreme(const float *__restrict__ c0, int T, int nc, float *out)
{
    const int lane = threadIdx.x & 31, run = (T + 31) / 32;
    const int lo = min(lane * run, T), hi = min(lo + run, T);
    bool has = false;
    float v = 0.f;
    for (int t = lo; t < hi; ++t) {
        const float x = c0[(size_t)t * nc];
        if ((SEED && t == 0) || (!isnan(x) && (!has || (MAX ? x > v : x < v)))) { v = x; has = true; }
    }
    for (int s = 1; s < 32; s <<= 1) {
        const float ov = __shfl_down_sync(0xffffffffu, v, s);
        const bool oh = __shfl_down_sync(0xffffffffu, (int)has, s) != 0;
        if ((lane & (2 * s - 1)) == 0 && lane + s < 32 && oh && (!has || (MAX ? ov > v : ov < v))) { v = ov; has = true; }
    }
    *out = __shfl_sync(0xffffffffu, v, 0);
    return __shfl_sync(0xffffffffu, (int)has, 0) != 0;
}

// AGC on c0 after CMN (feat_agc with beginutt and endutt, feat.c:941-966), one warp per utterance
// (max, noise) or per session (emax: its utterances in order, agc_emax then agc_emax_update each;
// the update ps_end_utt repeats through feat_update_stats finds obs_frame 0 and changes nothing).
template <int AGC>
__global__ void __launch_bounds__(32)
fe_agc_kernel(const int32_t *__restrict__ sess_off, const int32_t *__restrict__ frame_off, float *__restrict__ mfcc,
              int nc, float thresh, psb_fe_state_t *__restrict__ state)
{
    const int lane = threadIdx.x;
    int u0 = blockIdx.x, u1 = blockIdx.x + 1;
    float emax = 0.f, obs_max = 0.f, obs_sum = 0.f;
    int obs_frame = 0, obs_utt = 0;
    if constexpr (AGC == PSB_AGC_EMAX) {
        const psb_fe_state_t *st = state + blockIdx.x;
        u0 = sess_off[blockIdx.x]; u1 = sess_off[blockIdx.x + 1];
        emax = st->agc_max; obs_max = st->agc_obs_max; obs_sum = st->agc_obs_max_sum;
        obs_frame = st->agc_obs_frame; obs_utt = st->agc_obs_utt;
    }
    for (int u = u0; u < u1; ++u) {
        const int f0 = frame_off[u], T = frame_off[u + 1] - f0;
        float *c0 = mfcc + (size_t)f0 * nc;
        float sub = 0.f, m;
        bool apply = T > 0;
        if constexpr (AGC == PSB_AGC_MAX) {                              // agc_max (agc.c:110-127)
            if (T > 0) c0_extreme<true, true>(c0, T, nc, &sub);
        }
        else if constexpr (AGC == PSB_AGC_NOISE) {                       // agc_noise (agc.c:181-216)
            if (T > 0) {
                c0_extreme<false, true>(c0, T, nc, &m);
                const float lim = __fadd_rn(m, thresh);
                float sum = 0.f;
                int cnt = 0;
                if (lane == 0)
                    for (int t = 0; t < T; ++t) {
                        const float x = c0[(size_t)t * nc];
                        if (x < lim) { sum = __fadd_rn(sum, x); ++cnt; }
                    }
                cnt = __shfl_sync(0xffffffffu, cnt, 0);
                sub = __shfl_sync(0xffffffffu, cnt > 0 ? __fdiv_rn(sum, (float)cnt) : 0.f, 0);
                apply = cnt > 0;
            }
        }
        else {                                                           // agc_emax + agc_emax_update (agc.c:143-178)
            sub = emax;
            if (T > 0 && c0_extreme<true, false>(c0, T, nc, &m) && m > obs_max) { obs_max = m; obs_frame = 1; }
            if (obs_frame) {
                obs_sum = __fadd_rn(obs_sum, obs_max);
                ++obs_utt;
                emax = __fdiv_rn(obs_sum, (float)obs_utt);
                if (obs_utt == 16) { obs_sum = __fdiv_rn(obs_sum, 2.f); obs_utt = 8; }
            }
            obs_frame = 0;
            obs_max = -1000.f;
        }
        if (apply)
            for (int t = lane; t < T; t += 32) c0[(size_t)t * nc] = __fsub_rn(c0[(size_t)t * nc], sub);
    }
    if constexpr (AGC == PSB_AGC_EMAX)
        if (lane == 0) {
            psb_fe_state_t *st = state + blockIdx.x;
            st->agc_max = emax; st->agc_obs_max = obs_max; st->agc_obs_max_sum = obs_sum;
            st->agc_obs_frame = obs_frame; st->agc_obs_utt = obs_utt;
        }
}

// feat_lda_transform (lda.c:139-159): out[j] = sum over ascending k of x[k] * lda[j][k] in float32,
// one thread per (frame, output row), the rows used in shared memory.  in [total][n] -> out [total][m].
__global__ void __launch_bounds__(256)
fe_lda_kernel(const float *__restrict__ in, const float *__restrict__ lda, float *__restrict__ out, int n, int m,
              int32_t total)
{
    extern __shared__ float a_s[];                                       // [m][n]
    for (int i = threadIdx.x; i < m * n; i += blockDim.x) a_s[i] = lda[i];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)total * m) return;
    const float *x = in + (size_t)(i / m) * n, *a = a_s + (i % m) * n;
    float acc = 0.f;
    for (int k = 0; k < n; ++k) acc = __fadd_rn(acc, __fmul_rn(x[k], a[k]));
    out[i] = acc;
}

static FeDev dev_fe(const psb_fe_t *fe)
{
    FeDev p;
    p.frame_size = fe->frame_size; p.frame_shift = fe->frame_shift; p.fft_size = fe->fft_size; p.fft_order = fe->fft_order;
    p.n_filt = fe->n_filt; p.n_cep = fe->n_cep; p.remove_dc = fe->remove_dc; p.remove_noise = fe->remove_noise;
    p.transform = fe->transform; p.lifter_val = fe->lifter_val; p.alpha = fe->alpha;
    p.sqrt_inv_n = fe->sqrt_inv_n; p.sqrt_inv_2n = fe->sqrt_inv_2n;
    p.hamming = fe->d_hamming; p.ccc = fe->d_ccc; p.sss = fe->d_sss;
    p.spec_start = fe->d_spec_start; p.filt_start = fe->d_filt_start; p.filt_width = fe->d_filt_width;
    p.filt_coeffs = fe->d_filt_coeffs; p.mel_cosine = fe->d_mel_cosine; p.lifter = fe->d_lifter; p.rev = fe->d_rev;
    return p;
}

template <typename T>
static int up(DevBuf<T> &dst, const T *src, size_t n)
{
    const int rc = dst.reserve(std::max<size_t>(n, 1));
    if (rc) return rc;
    if (n) PSB_CUDA(cudaMemcpy(dst, src, n * sizeof(T), cudaMemcpyHostToDevice));
    return PSB_OK;
}

// the workspace's growth rule
template <typename T>
static int grow(DevBuf<T> &b, size_t need)
{
    return b.reserve(need, need / 8 + 64);
}

}  // namespace

extern "C" void psb_fe_free(psb_fe_t *fe)
{
    if (!fe) return;
    cudaSetDevice(fe->device);
    if (fe->stream) cudaStreamSynchronize(fe->stream);
    delete fe;
}

extern "C" int psb_fe_create(const psb_fe_desc_t *d, int device, psb_fe_t **out)
{
    return psb_fe_create_ex(d, nullptr, device, out);
}

extern "C" int psb_fe_create_ex(const psb_fe_desc_t *d, const psb_fe_opts_t *o, int device, psb_fe_t **out)
{
    PSB_REQUIRE(d && out, "psb_fe_create: bad argument");
    PSB_REQUIRE(d->frame_size > 1 && d->frame_shift > 0 && d->frame_size >= d->frame_shift, "psb_fe_create: bad frame size / shift");
    PSB_REQUIRE(d->fft_size == (1 << d->fft_order) && d->fft_size >= d->frame_size && d->fft_size >= 8 && d->fft_size <= 1024,
                "psb_fe_create: fft_size must be a power of two in [max(8, frame_size), 1024] (got %d)", d->fft_size);
    PSB_REQUIRE(d->n_filt > 0 && d->n_filt <= FE_MAX_FILT && d->n_cep > 0 && d->n_cep <= FE_MAX_CEP && d->n_cep <= d->n_filt,
                "psb_fe_create: need n_cep <= n_filt <= %d and n_cep <= %d", FE_MAX_FILT, FE_MAX_CEP);
    PSB_REQUIRE(d->transform >= 0 && d->transform <= 2, "psb_fe_create: transform must be 0 (legacy), 1 (dct) or 2 (htk)");
    if (!o) {
        PSB_REQUIRE(d->cmn == 0 || d->cmn == 1, "psb_fe_create: cmn must be 0 (none) or 1 (batch); live CMN needs psb_fe_create_ex");
        PSB_REQUIRE(d->window == 3, "psb_fe_create: only the 1s_c_d_dd feature type (window 3) is built; s2_4x and s3_1x39 need psb_fe_create_ex");
    }
    else {
        PSB_REQUIRE(o->feat >= PSB_FEAT_1S_C_D_DD && o->feat <= PSB_FEAT_S3_1X39,
                    "psb_fe_create_ex: feat must be 0 (1s_c_d_dd), 1 (s2_4x) or 2 (s3_1x39)");
        PSB_REQUIRE(o->feat == PSB_FEAT_1S_C_D_DD || d->n_cep == 13, "psb_fe_create_ex: s2_4x and s3_1x39 need n_cep 13 (got %d)", d->n_cep);
        PSB_REQUIRE(o->cmn >= PSB_CMN_NONE && o->cmn <= PSB_CMN_LIVE, "psb_fe_create_ex: cmn must be 0 (none), 1 (batch) or 2 (live)");
        PSB_REQUIRE(o->varnorm == 0 || o->varnorm == 1, "psb_fe_create_ex: varnorm must be 0 or 1");
        PSB_REQUIRE(!o->varnorm || o->cmn == PSB_CMN_BATCH,
                    o->cmn == PSB_CMN_LIVE ? "psb_fe_create_ex: variance normalization is not implemented in live mode"
                                           : "psb_fe_create_ex: variance normalization needs batch CMN");
        PSB_REQUIRE(o->dither == 0 || o->dither == 1, "psb_fe_create_ex: dither must be 0 or 1");
        PSB_REQUIRE(o->agc >= PSB_AGC_NONE && o->agc <= PSB_AGC_NOISE, "psb_fe_create_ex: agc must be 0 (none), 1 (max), 2 (emax) or 3 (noise)");
        if (o->lda) {
            const int dim = o->feat == PSB_FEAT_1S_C_D_DD ? 3 * d->n_cep : 39;
            PSB_REQUIRE(o->feat != PSB_FEAT_S2_4X, "psb_fe_create_ex: LDA needs single-stream features; s2_4x has four streams");
            PSB_REQUIRE(o->lda_cols == dim, "psb_fe_create_ex: the LDA matrix has %d columns, the features %d dimensions", o->lda_cols, dim);
            PSB_REQUIRE(o->lda_rows > 0, "psb_fe_create_ex: the LDA matrix has %d rows", o->lda_rows);
            const int m = o->ldadim > 0 && o->ldadim <= o->lda_rows ? o->ldadim : o->lda_rows;
            PSB_REQUIRE(m <= dim, "psb_fe_create_ex: %d LDA outputs from %d-dimensional features", m, dim);
        }
    }
    PSB_REQUIRE(d->hamming && d->ccc && d->sss && d->spec_start && d->filt_start && d->filt_width && d->filt_coeffs &&
                d->mel_cosine && (d->lifter_val == 0 || d->lifter), "psb_fe_create: missing table");
    int n_coeffs = 0;
    for (int i = 0; i < d->n_filt; ++i) {
        PSB_REQUIRE(d->filt_start[i] == n_coeffs && d->filt_width[i] >= 0 && d->spec_start[i] >= 0 &&
                    d->spec_start[i] + d->filt_width[i] <= d->fft_size / 2 + 1, "psb_fe_create: mel filter %d out of range", i);
        n_coeffs += d->filt_width[i];
    }
    PSB_REQUIRE(n_coeffs == d->n_coeffs, "psb_fe_create: n_coeffs %d != sum of filter widths %d", d->n_coeffs, n_coeffs);
    PSB_CUDA(cudaSetDevice(device));
    std::unique_ptr<psb_fe_t> fe(new psb_fe_t());
    fe->device = device;
    fe->frame_size = d->frame_size; fe->frame_shift = d->frame_shift; fe->fft_size = d->fft_size; fe->fft_order = d->fft_order;
    fe->n_filt = d->n_filt; fe->n_cep = d->n_cep; fe->remove_dc = d->remove_dc; fe->remove_noise = d->remove_noise;
    fe->transform = d->transform; fe->lifter_val = d->lifter_val; fe->window = d->window; fe->cmn = d->cmn;
    fe->feat = PSB_FEAT_1S_C_D_DD; fe->seed = -1;
    if (o) {
        fe->feat = o->feat; fe->cmn = o->cmn; fe->dither = o->dither; fe->seed = o->seed;
        fe->window = o->feat == PSB_FEAT_S2_4X ? 4 : 3;
        memcpy(fe->cmn_init, o->cmn_init, sizeof(fe->cmn_init));
        fe->varnorm = o->varnorm; fe->agc = o->agc; fe->agc_thresh = o->agc_thresh;
    }
    fe->stream_dim = fe->feat_dim = fe->feat == PSB_FEAT_S2_4X ? 51 : 3 * fe->n_cep;
    if (o && o->lda) fe->feat_dim = o->ldadim > 0 && o->ldadim <= o->lda_rows ? o->ldadim : o->lda_rows;   // feat_read_lda
    fe->n_coeffs = n_coeffs; fe->alpha = d->pre_emphasis_alpha; fe->sqrt_inv_n = d->sqrt_inv_n; fe->sqrt_inv_2n = d->sqrt_inv_2n;
    std::vector<int> rev((size_t)d->fft_size);
    for (int i = 0; i < d->fft_size; ++i) {
        int r = 0;
        for (int b = 0; b < d->fft_order; ++b) r |= ((i >> b) & 1) << (d->fft_order - 1 - b);
        rev[(size_t)i] = r;
    }
    int rc = up(fe->d_hamming, d->hamming, (size_t)d->frame_size / 2);
    if (!rc) rc = up(fe->d_ccc, d->ccc, (size_t)d->fft_size / 4);
    if (!rc) rc = up(fe->d_sss, d->sss, (size_t)d->fft_size / 4);
    if (!rc) rc = up(fe->d_spec_start, d->spec_start, (size_t)d->n_filt);
    if (!rc) rc = up(fe->d_filt_start, d->filt_start, (size_t)d->n_filt);
    if (!rc) rc = up(fe->d_filt_width, d->filt_width, (size_t)d->n_filt);
    if (!rc) rc = up(fe->d_filt_coeffs, d->filt_coeffs, (size_t)n_coeffs);
    if (!rc) rc = up(fe->d_mel_cosine, d->mel_cosine, (size_t)d->n_cep * d->n_filt);
    if (!rc) rc = up(fe->d_lifter, d->lifter, d->lifter_val ? (size_t)d->n_cep : 0);
    if (!rc) rc = up(fe->d_rev, rev.data(), rev.size());
    if (!rc && o && o->lda) rc = up(fe->d_lda, o->lda, (size_t)fe->feat_dim * fe->stream_dim);
    if (rc) return rc;
    cudaError_t e = fe->stream.create();
    if (e == cudaSuccess) e = fe->ev[0].create();
    if (e == cudaSuccess) e = fe->ev[1].create();
    if (e != cudaSuccess) {
        psb_set_error("psb_fe_create: %s", cudaGetErrorString(e));
        return PSB_ERR_CUDA;
    }
    *out = fe.release();
    return PSB_OK;
}

extern "C" int32_t psb_fe_n_frames(const psb_fe_t *fe, int64_t n_samples)
{
    // fe_process_frames (full frames) + fe_end_utt (one more from the leftover samples)
    if (!fe || n_samples <= 0) return 0;
    const int64_t full = n_samples >= fe->frame_size ? 1 + (n_samples - fe->frame_size) / fe->frame_shift : 0;
    return (int32_t)(full + 1);
}

static void state_init(const psb_fe_t *fe, psb_fe_state_t *s)
{
    // cmn_set_repr (cmn.c:119-146) and init_genrand((unsigned long)seed) (genrand.c)
    memset(s, 0, sizeof(*s));
    for (int i = 0; i < fe->n_cep; ++i) {
        s->cmn_mean[i] = fe->cmn_init[i];
        s->cmn_sum[i] = fe->cmn_init[i] * 500;
    }
    s->cmn_nframe = 500;
    s->mt[0] = (uint32_t)fe->seed;
    for (int i = 1; i < 624; ++i) s->mt[i] = 1812433253u * (s->mt[i - 1] ^ (s->mt[i - 1] >> 30)) + (uint32_t)i;
    s->mt_index = 624;
    s->agc_max = fe->cmn != PSB_CMN_NONE ? 5.f : 10.f;                 // feat_init's agc_emax_set (feat.c:879)
}

// what fe_init and ps_start_stream leave (fe_reset_noisestats): the next frame initialises the tracker
static psb_fe_noise_t noise_undefined()
{
    psb_fe_noise_t z;
    memset(&z, 0, sizeof(z));
    z.undefined = 1;
    return z;
}

static int fe_run(psb_fe_t *fe, const int16_t *d_pcm, const int64_t *samp_off, int32_t n_utt, float *d_feats,
                  float *d_mfcc_out, int32_t *frame_off, float *ms)
{
    // sessions: the ones psb_fe_set_sessions named for this call, else one per utterance
    const bool pending = fe->sess_pending, carry = fe->starts_pending, banks = fe->banks_pending;
    fe->sess_pending = fe->starts_pending = fe->noise_out = fe->banks_pending = false;
    if (banks)
        PSB_REQUIRE(fe->bank_of_utt.size() == (size_t)n_utt, "psb_fe: the filter banks name %d utterances, the call has %d",
                    (int)fe->bank_of_utt.size(), n_utt);
    if (pending) {
        PSB_REQUIRE(fe->sess_off.back() == n_utt, "psb_fe: the sessions cover %d utterances, the call has %d", fe->sess_off.back(), n_utt);
    }
    else {
        fe->sess_off.resize((size_t)n_utt + 1);
        for (int u = 0; u <= n_utt; ++u) fe->sess_off[(size_t)u] = u;
        fe->states.clear();
    }
    const int32_t n_sess = (int32_t)fe->sess_off.size() - 1;
    const bool live = fe->cmn == PSB_CMN_LIVE, emax = fe->agc == PSB_AGC_EMAX, stateful = live || fe->dither || emax;
    if (stateful && fe->states.empty()) {
        fe->states.resize((size_t)n_sess);
        for (auto &st : fe->states) state_init(fe, &st);
    }
    // stream starts: the ones psb_fe_set_stream_starts named for this call, else one before every utterance.
    // noise_next: each session's tracker where none of its frames changes it -- the incoming one, undefined
    // after a stream start; fe_noise_kernel overwrites the sessions whose frames it walks.
    std::vector<int4> chains;
    std::vector<psb_fe_noise_t> noise_next;
    if (carry) {
        PSB_REQUIRE(fe->starts.size() == (size_t)n_utt, "psb_fe: the stream starts cover %d utterances, the call has %d",
                    (int)fe->starts.size(), n_utt);
        PSB_REQUIRE(fe->noise.empty() || fe->noise.size() == (size_t)n_sess, "psb_fe: %d noise trackers for %d sessions",
                    (int)fe->noise.size(), n_sess);
        if (fe->noise.empty()) fe->noise.resize((size_t)n_sess, noise_undefined());
        noise_next = fe->noise;
        for (int s = 0; s < n_sess; ++s) {
            const int u0 = fe->sess_off[(size_t)s], u1 = fe->sess_off[(size_t)s + 1];
            for (int u = u0; u < u1; ++u) {
                if (fe->starts[(size_t)u]) noise_next[(size_t)s] = noise_undefined();
                if (u == u0 || fe->starts[(size_t)u]) chains.push_back(make_int4(u, u + 1, u == u0 && !fe->starts[(size_t)u] ? s : -1, -1));
                else chains.back().y = u + 1;
            }
            if (u1 > u0) chains.back().w = s;
        }
        if (!fe->remove_noise) chains.clear();
    }
    std::vector<int32_t> foff((size_t)n_utt + 1);
    foff[0] = 0;
    for (int u = 0; u < n_utt; ++u) {
        PSB_REQUIRE(samp_off[u + 1] >= samp_off[u], "psb_fe: samp_off not monotone at %d", u);
        const int64_t t = (int64_t)foff[(size_t)u] + psb_fe_n_frames(fe, samp_off[u + 1] - samp_off[u]);
        PSB_REQUIRE(t < (1ll << 31), "psb_fe: more than 2^31 frames in one batch");
        foff[(size_t)u + 1] = (int32_t)t;
    }
    const int32_t total = foff[(size_t)n_utt];
    if (frame_off) memcpy(frame_off, foff.data(), foff.size() * sizeof(int32_t));
    if (ms) *ms = 0.f;
    if (total == 0) chains.clear();
    if (chains.empty()) fe->noise.swap(noise_next);
    fe->noise_out = carry && chains.empty();
    // live CMN and emax AGC update their state even after an utterance without frames (cmn_live_update,
    // agc_emax_update)
    if (total == 0 && !((live || emax) && n_sess > 0)) return PSB_OK;
    std::vector<int32_t> futt((size_t)total);
    for (int u = 0; u < n_utt; ++u)
        for (int32_t f = foff[(size_t)u]; f < foff[(size_t)u + 1]; ++f) futt[(size_t)f] = u;
    int rc = grow(fe->d_mfspec, (size_t)total * fe->n_filt);
    if (!rc) rc = grow(fe->d_mfcc, (size_t)total * fe->n_cep);
    if (!rc) rc = fe->d_samp_off.reserve((size_t)n_utt + 1, 64);
    if (!rc) rc = fe->d_frame_off.reserve((size_t)n_utt + 1, 64);
    if (!rc) rc = grow(fe->d_frame_utt, (size_t)std::max(total, 1));
    if (!rc && fe->d_lda && d_feats) rc = grow(fe->d_raw, (size_t)std::max(total, 1) * fe->stream_dim);
    // dither: per utterance the first sample of its last frame, where its copy goes, and the draws
    // of fe_process_frames (every sample the full frames read) and of fe_end_utt (the last frame's)
    std::vector<int64_t> draw;
    int64_t n_tail = 0;
    if (fe->dither) {
        draw.resize((size_t)n_utt * 4);
        for (int u = 0; u < n_utt; ++u) {
            const int64_t n = samp_off[u + 1] - samp_off[u];
            const int64_t full = n >= fe->frame_size ? 1 + (n - fe->frame_size) / fe->frame_shift : 0;
            const int64_t main = full ? fe->frame_size + (full - 1) * fe->frame_shift : 0;
            const int64_t t0 = full * fe->frame_shift;
            draw[4 * (size_t)u] = t0;
            draw[4 * (size_t)u + 1] = n_tail;
            draw[4 * (size_t)u + 2] = main;
            draw[4 * (size_t)u + 3] = n > 0 ? n - t0 : 0;
            n_tail += draw[4 * (size_t)u + 3];
        }
        if (!rc) rc = grow(fe->d_draw, draw.size() + 1);
        if (!rc) rc = grow(fe->d_dpcm, (size_t)std::max<int64_t>(samp_off[n_utt], 1));
        if (!rc) rc = grow(fe->d_tail, (size_t)std::max<int64_t>(n_tail, 1));
    }
    if (stateful) {
        if (!rc) rc = grow(fe->d_state, (size_t)n_sess);
        if (!rc) rc = grow(fe->d_sess_off, (size_t)n_sess + 1);
    }
    if (!chains.empty()) {
        if (!rc) rc = grow(fe->d_noise, 2 * (size_t)n_sess);
        if (!rc) rc = grow(fe->d_chain, chains.size());
    }
    if (banks) {
        if (!rc) rc = grow(fe->d_bank_spec_start, fe->bank_spec_start.size());
        if (!rc) rc = grow(fe->d_bank_filt_start, fe->bank_filt_start.size());
        if (!rc) rc = grow(fe->d_bank_filt_width, fe->bank_filt_width.size());
        if (!rc) rc = grow(fe->d_bank_coeff_off, fe->bank_coeff_off.size());
        if (!rc) rc = grow(fe->d_bank_coeffs, std::max<size_t>(fe->bank_coeffs.size(), 1));
        if (!rc) rc = grow(fe->d_bank_of_utt, std::max<size_t>(fe->bank_of_utt.size(), 1));
    }
    if (rc) return rc;
    PSB_CUDA(cudaMemcpyAsync(fe->d_samp_off, samp_off, ((size_t)n_utt + 1) * 8, cudaMemcpyHostToDevice, fe->stream));
    PSB_CUDA(cudaMemcpyAsync(fe->d_frame_off, foff.data(), foff.size() * 4, cudaMemcpyHostToDevice, fe->stream));
    if (total) PSB_CUDA(cudaMemcpyAsync(fe->d_frame_utt, futt.data(), futt.size() * 4, cudaMemcpyHostToDevice, fe->stream));
    if (fe->dither) PSB_CUDA(cudaMemcpyAsync(fe->d_draw, draw.data(), draw.size() * 8, cudaMemcpyHostToDevice, fe->stream));
    if (stateful) {
        PSB_CUDA(cudaMemcpyAsync(fe->d_state, fe->states.data(), (size_t)n_sess * sizeof(psb_fe_state_t), cudaMemcpyHostToDevice, fe->stream));
        PSB_CUDA(cudaMemcpyAsync(fe->d_sess_off, fe->sess_off.data(), ((size_t)n_sess + 1) * 4, cudaMemcpyHostToDevice, fe->stream));
    }
    const size_t noise_bytes = (size_t)n_sess * sizeof(psb_fe_noise_t);
    if (!chains.empty()) {
        PSB_CUDA(cudaMemcpyAsync(fe->d_noise, fe->noise.data(), noise_bytes, cudaMemcpyHostToDevice, fe->stream));
        PSB_CUDA(cudaMemcpyAsync(fe->d_noise.get() + n_sess, noise_next.data(), noise_bytes, cudaMemcpyHostToDevice, fe->stream));
        PSB_CUDA(cudaMemcpyAsync(fe->d_chain, chains.data(), chains.size() * sizeof(int4), cudaMemcpyHostToDevice, fe->stream));
    }
    FeDev p = dev_fe(fe);
    if (banks) {
        PSB_CUDA(cudaMemcpyAsync(fe->d_bank_spec_start, fe->bank_spec_start.data(), fe->bank_spec_start.size() * 2,
                                 cudaMemcpyHostToDevice, fe->stream));
        PSB_CUDA(cudaMemcpyAsync(fe->d_bank_filt_start, fe->bank_filt_start.data(), fe->bank_filt_start.size() * 2,
                                 cudaMemcpyHostToDevice, fe->stream));
        PSB_CUDA(cudaMemcpyAsync(fe->d_bank_filt_width, fe->bank_filt_width.data(), fe->bank_filt_width.size() * 2,
                                 cudaMemcpyHostToDevice, fe->stream));
        PSB_CUDA(cudaMemcpyAsync(fe->d_bank_coeff_off, fe->bank_coeff_off.data(), fe->bank_coeff_off.size() * 4,
                                 cudaMemcpyHostToDevice, fe->stream));
        if (!fe->bank_coeffs.empty())
            PSB_CUDA(cudaMemcpyAsync(fe->d_bank_coeffs, fe->bank_coeffs.data(), fe->bank_coeffs.size() * 4,
                                     cudaMemcpyHostToDevice, fe->stream));
        if (n_utt) PSB_CUDA(cudaMemcpyAsync(fe->d_bank_of_utt, fe->bank_of_utt.data(), (size_t)n_utt * 4, cudaMemcpyHostToDevice, fe->stream));
        p.spec_start = fe->d_bank_spec_start; p.filt_start = fe->d_bank_filt_start; p.filt_width = fe->d_bank_filt_width;
        p.filt_coeffs = fe->d_bank_coeffs;
    }
    // with the noise tracker carried, fe_noise_kernel removes the noise and fe_utt_kernel does not
    FeDev pu = p;
    if (!chains.empty()) pu.remove_noise = 0;
    const size_t smem = ((size_t)fe->fft_size + fe->fft_size / 2 + 1) * sizeof(double);
    // the features of 1s_c_d_dd without live CMN, AGC or LDA come out of fe_utt_kernel; every other
    // configuration normalises and builds them in the kernels behind it
    const bool utt_feats = fe->feat == PSB_FEAT_1S_C_D_DD && !live && fe->agc == PSB_AGC_NONE && !fe->d_lda;
    PSB_CUDA(cudaEventRecord(fe->ev[0], fe->stream));
    if (fe->dither && n_sess) {
        fe_dither_kernel<<<(unsigned)n_sess, FE_DITHER_THREADS, 0, fe->stream>>>(d_pcm, fe->d_samp_off, fe->d_sess_off, fe->d_draw,
                                                                            fe->d_state, fe->d_dpcm, fe->d_tail);
        PSB_LAUNCH_CHECK();
    }
    if (total) {
        const int16_t *src = fe->dither ? fe->d_dpcm.get() : d_pcm;
        const int16_t *tail = fe->dither ? fe->d_tail.get() : nullptr;
        const int64_t *draw_d = fe->dither ? fe->d_draw.get() : nullptr;
        const int32_t *bank_of_utt = banks ? fe->d_bank_of_utt.get() : nullptr, *coeff_off = banks ? fe->d_bank_coeff_off.get() : nullptr;
        auto kern = fe->dither ? (banks ? fe_frame_kernel<true, true> : fe_frame_kernel<true, false>)
                               : (banks ? fe_frame_kernel<false, true> : fe_frame_kernel<false, false>);
        kern<<<(unsigned)total, 128, smem, fe->stream>>>(p, src, fe->d_samp_off, fe->d_frame_off, fe->d_frame_utt, fe->d_mfspec,
                                                          tail, draw_d, bank_of_utt, coeff_off);
        PSB_LAUNCH_CHECK();
        if (!chains.empty()) {
            fe_noise_kernel<<<(unsigned)chains.size(), FE_NOISE_THREADS, 0, fe->stream>>>(
                fe->n_filt, fe->d_frame_off, fe->d_chain, fe->d_noise, fe->d_noise.get() + n_sess, fe->d_mfspec);
            PSB_LAUNCH_CHECK();
        }
        if (fe->varnorm)
            fe_utt_kernel<true><<<(unsigned)n_utt, 64, 0, fe->stream>>>(pu, fe->d_frame_off, fe->d_mfspec, fe->d_mfcc,
                                                                       utt_feats ? d_feats : nullptr, fe->cmn, fe->window);
        else
            fe_utt_kernel<false><<<(unsigned)n_utt, 64, 0, fe->stream>>>(pu, fe->d_frame_off, fe->d_mfspec, fe->d_mfcc,
                                                                        utt_feats ? d_feats : nullptr, live ? 0 : fe->cmn, fe->window);
        PSB_LAUNCH_CHECK();
    }
    if (live) {
        fe_cmn_live_kernel<<<(unsigned)n_sess, 32, 0, fe->stream>>>(fe->d_sess_off, fe->d_frame_off, fe->d_mfcc, fe->n_cep, fe->d_state);
        PSB_LAUNCH_CHECK();
    }
    if (fe->agc == PSB_AGC_MAX && total) {
        fe_agc_kernel<PSB_AGC_MAX><<<(unsigned)n_utt, 32, 0, fe->stream>>>(nullptr, fe->d_frame_off, fe->d_mfcc, fe->n_cep, 0.f, nullptr);
        PSB_LAUNCH_CHECK();
    }
    else if (fe->agc == PSB_AGC_NOISE && total) {
        fe_agc_kernel<PSB_AGC_NOISE><<<(unsigned)n_utt, 32, 0, fe->stream>>>(nullptr, fe->d_frame_off, fe->d_mfcc, fe->n_cep,
                                                                           fe->agc_thresh, nullptr);
        PSB_LAUNCH_CHECK();
    }
    else if (emax && n_sess) {
        fe_agc_kernel<PSB_AGC_EMAX><<<(unsigned)n_sess, 32, 0, fe->stream>>>(fe->d_sess_off, fe->d_frame_off, fe->d_mfcc, fe->n_cep,
                                                                           0.f, fe->d_state);
        PSB_LAUNCH_CHECK();
    }
    if (!utt_feats && d_feats && total) {
        const int64_t work = (int64_t)total * fe->n_cep;
        fe_feat_kernel<<<(unsigned)((work + 255) / 256), 256, 0, fe->stream>>>(fe->d_frame_off, fe->d_frame_utt, fe->d_mfcc,
                                                                           fe->d_lda ? fe->d_raw : d_feats, fe->n_cep, fe->feat,
                                                                           fe->stream_dim, total);
        PSB_LAUNCH_CHECK();
        if (fe->d_lda) {
            const int64_t outs = (int64_t)total * fe->feat_dim;
            fe_lda_kernel<<<(unsigned)((outs + 255) / 256), 256, (size_t)fe->feat_dim * fe->stream_dim * sizeof(float), fe->stream>>>(
                fe->d_raw, fe->d_lda, d_feats, fe->stream_dim, fe->feat_dim, total);
            PSB_LAUNCH_CHECK();
        }
    }
    PSB_CUDA(cudaEventRecord(fe->ev[1], fe->stream));
    if (d_mfcc_out && total)
        PSB_CUDA(cudaMemcpyAsync(d_mfcc_out, fe->d_mfcc, (size_t)total * fe->n_cep * 4, cudaMemcpyDeviceToDevice, fe->stream));
    if (stateful)
        PSB_CUDA(cudaMemcpyAsync(fe->states.data(), fe->d_state, (size_t)n_sess * sizeof(psb_fe_state_t), cudaMemcpyDeviceToHost, fe->stream));
    if (!chains.empty())
        PSB_CUDA(cudaMemcpyAsync(fe->noise.data(), fe->d_noise.get() + n_sess, noise_bytes, cudaMemcpyDeviceToHost, fe->stream));
    PSB_CUDA(cudaStreamSynchronize(fe->stream));
    fe->noise_out = carry;
    if (ms) PSB_CUDA(cudaEventElapsedTime(ms, fe->ev[0], fe->ev[1]));
    return PSB_OK;
}

extern "C" int psb_fe_process_device(psb_fe_t *fe, const int16_t *d_pcm, const int64_t *samp_off, int32_t n_utt,
                                     float *d_feats, float *d_mfcc, int32_t *frame_off, float *ms)
{
    PSB_REQUIRE(fe && samp_off && n_utt >= 0 && (d_pcm || samp_off[n_utt] == samp_off[0]), "psb_fe_process_device: bad argument");
    PSB_REQUIRE(samp_off[0] == 0, "psb_fe_process_device: samp_off[0] must be 0");
    PSB_CUDA(cudaSetDevice(fe->device));
    return fe_run(fe, d_pcm, samp_off, n_utt, d_feats, d_mfcc, frame_off, ms);
}

extern "C" int psb_fe_process_host(psb_fe_t *fe, const int16_t *pcm, const int64_t *samp_off, int32_t n_utt,
                                   float *feats, float *mfcc, int32_t *frame_off)
{
    PSB_REQUIRE(fe && samp_off && n_utt >= 0 && frame_off, "psb_fe_process_host: bad argument");
    PSB_REQUIRE(samp_off[0] == 0, "psb_fe_process_host: samp_off[0] must be 0");
    PSB_CUDA(cudaSetDevice(fe->device));
    const int64_t ns = samp_off[n_utt];
    PSB_REQUIRE(ns == 0 || pcm, "psb_fe_process_host: pcm is null");
    int64_t total = 0;
    for (int u = 0; u < n_utt; ++u) total += psb_fe_n_frames(fe, samp_off[u + 1] - samp_off[u]);
    int rc = grow(fe->d_pcm, (size_t)std::max<int64_t>(ns, 1));
    if (!rc) rc = grow(fe->d_feats, (size_t)std::max<int64_t>(total, 1) * fe->feat_dim);
    if (rc) return rc;
    if (ns) PSB_CUDA(cudaMemcpyAsync(fe->d_pcm, pcm, (size_t)ns * 2, cudaMemcpyHostToDevice, fe->stream));
    rc = fe_run(fe, fe->d_pcm, samp_off, n_utt, fe->d_feats, nullptr, frame_off, nullptr);
    if (rc) return rc;
    if (total && feats) PSB_CUDA(cudaMemcpy(feats, fe->d_feats, (size_t)total * fe->feat_dim * 4, cudaMemcpyDeviceToHost));
    if (total && mfcc) PSB_CUDA(cudaMemcpy(mfcc, fe->d_mfcc, (size_t)total * fe->n_cep * 4, cudaMemcpyDeviceToHost));
    return PSB_OK;
}

extern "C" const float *psb_fe_device_feats(const psb_fe_t *fe)
{
    return fe ? fe->d_feats.get() : nullptr;
}

extern "C" int32_t psb_fe_feat_dim(const psb_fe_t *fe)
{
    return fe ? fe->feat_dim : 0;
}

extern "C" int psb_fe_state_init(const psb_fe_t *fe, psb_fe_state_t *s)
{
    PSB_REQUIRE(fe && s, "psb_fe_state_init: bad argument");
    state_init(fe, s);
    return PSB_OK;
}

extern "C" int psb_fe_set_sessions(psb_fe_t *fe, const int32_t *sess_off, int32_t n_sess, const psb_fe_state_t *states_in)
{
    PSB_REQUIRE(fe && sess_off && n_sess >= 0, "psb_fe_set_sessions: bad argument");
    PSB_REQUIRE(sess_off[0] == 0, "psb_fe_set_sessions: sess_off[0] must be 0");
    for (int s = 0; s < n_sess; ++s)
        PSB_REQUIRE(sess_off[s + 1] >= sess_off[s], "psb_fe_set_sessions: sess_off not monotone at %d", s);
    if (states_in)
        for (int s = 0; s < n_sess; ++s)
            PSB_REQUIRE(states_in[s].mt_index >= 0 && states_in[s].mt_index <= 625 && states_in[s].cmn_nframe >= 0,
                        "psb_fe_set_sessions: state %d is not a front-end state", s);
    fe->sess_off.assign(sess_off, sess_off + n_sess + 1);
    fe->states.clear();
    if (states_in) fe->states.assign(states_in, states_in + n_sess);
    fe->sess_pending = true;
    return PSB_OK;
}

extern "C" int psb_fe_get_states(const psb_fe_t *fe, psb_fe_state_t *states_out, int32_t n_sess)
{
    PSB_REQUIRE(fe && states_out && n_sess >= 0, "psb_fe_get_states: bad argument");
    PSB_REQUIRE(!fe->sess_off.empty() && n_sess == (int32_t)fe->sess_off.size() - 1,
                "psb_fe_get_states: the last call had %d sessions", fe->sess_off.empty() ? 0 : (int)fe->sess_off.size() - 1);
    for (int s = 0; s < n_sess; ++s) {
        if (fe->states.empty()) state_init(fe, &states_out[s]);     // nothing carried: the state is the initial one
        else states_out[s] = fe->states[(size_t)s];
    }
    return PSB_OK;
}

extern "C" int psb_fe_set_stream_starts(psb_fe_t *fe, const uint8_t *start, int32_t n_utt, const psb_fe_noise_t *noise_in,
                                        int32_t n_sess)
{
    PSB_REQUIRE(fe && n_utt >= 0 && (start || n_utt == 0) && (!noise_in || n_sess >= 0), "psb_fe_set_stream_starts: bad argument");
    for (int u = 0; u < n_utt; ++u)
        PSB_REQUIRE(start[u] <= 1, "psb_fe_set_stream_starts: start[%d] is %d, not 0 or 1", u, start[u]);
    if (noise_in)
        for (int s = 0; s < n_sess; ++s)
            PSB_REQUIRE(noise_in[s].undefined == 0 || noise_in[s].undefined == 1,
                        "psb_fe_set_stream_starts: tracker %d is not a noise tracker (undefined = %d)", s, noise_in[s].undefined);
    fe->starts.assign(start, start + n_utt);
    fe->noise.clear();
    if (noise_in) {
        fe->noise.assign(noise_in, noise_in + n_sess);
        for (auto &z : fe->noise)                       // an undefined tracker's arrays are never read
            if (z.undefined) z = noise_undefined();
    }
    fe->starts_pending = true;
    return PSB_OK;
}

extern "C" int psb_fe_get_noise_states(const psb_fe_t *fe, psb_fe_noise_t *noise_out, int32_t n_sess)
{
    PSB_REQUIRE(fe && noise_out && n_sess >= 0, "psb_fe_get_noise_states: bad argument");
    PSB_REQUIRE(fe->noise_out, "psb_fe_get_noise_states: the last process call set no stream starts");
    PSB_REQUIRE(n_sess == (int32_t)fe->noise.size(), "psb_fe_get_noise_states: the last call had %d sessions", (int)fe->noise.size());
    memcpy(noise_out, fe->noise.data(), (size_t)n_sess * sizeof(psb_fe_noise_t));
    return PSB_OK;
}

// One bank of n_filt filters in fe_build_melfilters' layout: every filter either covers DFT points inside the
// spectrum with filt_start the running coefficient count, or is empty (width 0) -- at spec_start -1 with
// filt_start 0, as a filter no DFT point falls in is left, or at any start with the running count.  Returns the
// first filter that is neither, or -1; *n_coeffs = the sum of the widths.
static int bank_bad_filter(int n_filt, int fft_size, const int16_t *ss, const int16_t *fs, const int16_t *fw, int32_t *n_coeffs)
{
    int32_t n = 0;
    for (int i = 0; i < n_filt; ++i) {
        const bool empty_calloc = ss[i] == -1 && fw[i] == 0 && fs[i] == 0;
        if (!empty_calloc && !(fw[i] >= 0 && ss[i] >= 0 && ss[i] + fw[i] <= fft_size / 2 + 1 && fs[i] == n)) return i;
        n += fw[i];
    }
    *n_coeffs = n;
    return -1;
}

extern "C" int psb_fe_set_filterbanks(psb_fe_t *fe, int32_t n_bank, const int16_t *spec_start, const int16_t *filt_start,
                                      const int16_t *filt_width, const int32_t *coeff_off, const float *coeffs,
                                      const int32_t *bank, int32_t n_utt)
{
    PSB_REQUIRE(fe && n_bank > 0 && spec_start && filt_start && filt_width && coeff_off && n_utt >= 0 && (bank || n_utt == 0),
                "psb_fe_set_filterbanks: bad argument");
    PSB_REQUIRE(coeff_off[0] == 0, "psb_fe_set_filterbanks: coeff_off[0] must be 0 (got %d)", coeff_off[0]);
    const int nf = fe->n_filt;
    for (int b = 0; b < n_bank; ++b) {
        const size_t o = (size_t)b * nf;
        int32_t n = 0;
        PSB_REQUIRE(coeff_off[b + 1] >= coeff_off[b], "psb_fe_set_filterbanks: coeff_off not monotone at bank %d", b);
        const int bad = bank_bad_filter(nf, fe->fft_size, spec_start + o, filt_start + o, filt_width + o, &n);
        PSB_REQUIRE(bad < 0, "psb_fe_set_filterbanks: bank %d, mel filter %d out of range", b, bad);
        PSB_REQUIRE(n == coeff_off[b + 1] - coeff_off[b], "psb_fe_set_filterbanks: bank %d has %d coefficients, coeff_off says %d",
                    b, n, coeff_off[b + 1] - coeff_off[b]);
    }
    PSB_REQUIRE(coeff_off[n_bank] == 0 || coeffs, "psb_fe_set_filterbanks: coeffs is null");
    for (int u = 0; u < n_utt; ++u)
        PSB_REQUIRE(bank[u] >= 0 && bank[u] < n_bank, "psb_fe_set_filterbanks: utterance %d names bank %d of %d", u, bank[u], n_bank);
    const size_t n = (size_t)n_bank * nf;
    fe->bank_spec_start.assign(spec_start, spec_start + n);
    fe->bank_filt_start.assign(filt_start, filt_start + n);
    fe->bank_filt_width.assign(filt_width, filt_width + n);
    fe->bank_coeff_off.assign(coeff_off, coeff_off + n_bank + 1);
    fe->bank_coeffs.assign(coeffs, coeffs + coeff_off[n_bank]);
    fe->bank_of_utt.assign(bank, bank + n_utt);
    fe->banks_pending = true;
    return PSB_OK;
}

extern "C" int psb_fe_cancel_settings(psb_fe_t *fe)
{
    PSB_REQUIRE(fe, "psb_fe_cancel_settings: bad argument");
    // the setters overwrote the last call's states / trackers with the next call's inputs: report neither
    if (fe->sess_pending) { fe->sess_off.clear(); fe->states.clear(); }
    if (fe->starts_pending) { fe->noise.clear(); fe->noise_out = false; }
    fe->sess_pending = fe->starts_pending = fe->banks_pending = false;
    return PSB_OK;
}
