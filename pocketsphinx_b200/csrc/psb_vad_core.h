// psb_vad_core.h -- the per-frame fixed-point arithmetic of the reference's voice activity
// detector (PocketSphinx 5's WebRTC-derived VAD) and of its endpointer, as __host__ __device__
// functions.  psb_vad.cu's kernels and tests/emul/vad_emul.cpp / vad_live_emul.cpp (the CPU
// restatements the tests pin against the compiled reference) are built from this one file.
//
// Restated, in the reference's int16 / int32 types, truncations and wrap-arounds:
//   WebRtcVad_Downsampling                                 (common_audio/vad/vad_sp.c:25-53)
//   HighPassFilter / AllPassFilter / SplitFilter /
//   LogOfEnergy / WebRtcVad_CalculateFeatures              (vad_filterbank.c:39-329)
//   WebRtcSpl_Energy + WebRtcSpl_GetScalingSquare          (signal_processing/energy.c,
//                                                           get_scaling_square.c)
//   WebRtcVad_GaussianProbability                          (vad_gmm.c:29-82)
//   WebRtcVad_FindMinimum                                  (vad_sp.c:58-176)
//   GmmProbability, one channel at a time                  (vad_core.c:133-489)
//   ep_push / ep_pop / ps_endpointer_process / _end_stream (ps_endpointer.c:209-440)
// Every intermediate that can leave its type in the reference is computed here with an explicit
// wrap (the reference relies on the compiler's two's-complement behaviour for those).
#ifndef PSB_VAD_CORE_H
#define PSB_VAD_CORE_H

#include <stdint.h>

#ifdef __CUDACC__
#define PSB_VAD_HD __host__ __device__ __forceinline__
#define PSB_VAD_MEMBER __host__ __device__ __forceinline__
#else
#define PSB_VAD_HD static inline
#define PSB_VAD_MEMBER inline
#endif

enum { PSB_VAD_NCH = 6, PSB_VAD_MIN_ENERGY = 10 };

// The filter memories the features depend on (the part of VadInstT stage A owns).  Two runs
// whose psb_vad_filt_t agree produce the same features from then on.
struct psb_vad_filt_t {
    int32_t ds[4];               // downsampling_filter_states: [0..1] 16->8 kHz, [2..3] 32->16 kHz
    int16_t upper[5], lower[5];  // split-filter all-pass states, Q(-1)
    int16_t hp[4];               // 80 Hz high-pass
};

PSB_VAD_HD void psb_vad_filt_init(psb_vad_filt_t *f)
{
    for (int i = 0; i < 4; ++i) f->ds[i] = 0, f->hp[i] = 0;
    for (int i = 0; i < 5; ++i) f->upper[i] = 0, f->lower[i] = 0;
}

PSB_VAD_HD bool psb_vad_filt_equal(const psb_vad_filt_t *a, const psb_vad_filt_t *b)
{
    bool eq = true;
    for (int i = 0; i < 4; ++i) eq &= a->ds[i] == b->ds[i] && a->hp[i] == b->hp[i];
    for (int i = 0; i < 5; ++i) eq &= a->upper[i] == b->upper[i] && a->lower[i] == b->lower[i];
    return eq;
}

// two's-complement helpers: the reference's int arithmetic where it can overflow
PSB_VAD_HD int32_t vw_add(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
PSB_VAD_HD int32_t vw_sub(int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); }
PSB_VAD_HD int32_t vw_mul(int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); }
PSB_VAD_HD int vw_clz(uint32_t x)
{
#ifdef __CUDA_ARCH__
    return __clz((int)x);
#else
    return x ? __builtin_clz(x) : 32;
#endif
}
// WebRtcSpl_NormW32 (spl_inl.h:136)
PSB_VAD_HD int vw_norm_w32(int32_t a) { return a == 0 ? 0 : vw_clz((uint32_t)(a < 0 ? ~a : a)) - 1; }
// WebRtcSpl_DivW32W16 (division_operations.c:39-49): C division, 0x7FFFFFFF for a zero divisor
PSB_VAD_HD int32_t vw_div(int32_t num, int16_t den)
{
    if (den == 0) return 0x7FFFFFFF;
    if (num == INT32_MIN && den == -1) return INT32_MIN;
    return num / den;
}

// Strided scratch: element i of a buffer lives at p[i * s] (s = 1 on the host, the CTA's thread
// count on the device, so that a warp's threads touch consecutive shared-memory halves).
struct psb_vad_buf {
    int16_t *p;
    int s;
    PSB_VAD_MEMBER int16_t &operator[](int i) const { return p[i * s]; }
};

// 2:1 downsampler: two all-pass branches on the even / odd samples, summed.
template <typename In>
PSB_VAD_HD void psb_vad_downsample(In in, psb_vad_buf out, int32_t *st, int in_len)
{
    int32_t s1 = st[0], s2 = st[1];
    for (int n = 0; n < in_len / 2; ++n) {
        const int32_t a = in[2 * n], b = in[2 * n + 1];
        const int16_t u = (int16_t)((s1 >> 1) + ((5243 * a) >> 14));
        s1 = a - ((5243 * u) >> 12);
        const int16_t l = (int16_t)((s2 >> 1) + ((1392 * b) >> 14));
        s2 = b - ((1392 * l) >> 12);
        out[n] = (int16_t)(u + l);
    }
    st[0] = s1;
    st[1] = s2;
}

// one all-pass branch over every other sample; the state is kept in Q(-1) between frames
template <typename In>
PSB_VAD_HD void psb_vad_allpass(In in, int first, int len, int32_t coef, int16_t *state, psb_vad_buf out)
{
    int32_t s = vw_mul(*state, 65536);
    for (int i = 0; i < len; ++i) {
        const int32_t x = in[first + 2 * i];
        const int16_t y = (int16_t)(vw_add(s, coef * x) >> 16);
        out[i] = y;
        s = vw_mul(vw_sub(x * 16384, coef * y), 2);
    }
    *state = (int16_t)(s >> 16);
}

template <typename In>
PSB_VAD_HD void psb_vad_split(In in, int len, int16_t *up, int16_t *lo, psb_vad_buf hp, psb_vad_buf lp)
{
    const int half = len >> 1;
    psb_vad_allpass(in, 0, half, 20972, up, hp);
    psb_vad_allpass(in, 1, half, 5571, lo, lp);
    for (int i = 0; i < half; ++i) {
        const int16_t h = hp[i], l = lp[i];
        hp[i] = (int16_t)(h - l);
        lp[i] = (int16_t)(l + h);
    }
}

PSB_VAD_HD void psb_vad_highpass(psb_vad_buf in, int len, int16_t *st, psb_vad_buf out)
{
    for (int i = 0; i < len; ++i) {
        const int32_t x = in[i];
        int32_t acc = 6631 * x - 13262 * st[0] + 6631 * st[1];
        st[1] = st[0];
        st[0] = (int16_t)x;
        acc -= -7756 * st[2] + 5620 * st[3];
        st[3] = st[2];
        st[2] = (int16_t)(acc >> 14);
        out[i] = st[2];
    }
}

// WebRtcSpl_Energy: every square is shifted by a scaling taken from the band-frame's largest
// magnitude before it is summed, so the maximum must be known first (two passes over the band).
PSB_VAD_HD void psb_vad_log_energy(psb_vad_buf x, int len, int16_t offset, int16_t *total, int16_t *out)
{
    int16_t smax = -1;
    for (int i = 0; i < len; ++i) {
        const int16_t v = x[i];
        const int16_t a = (int16_t)(v > 0 ? v : -v);           // -(-32768) stays -32768, as in the reference
        smax = a > smax ? a : smax;
    }
    int scaling = 0;
    if (smax != 0) {
        const int nbits = 32 - vw_clz((uint32_t)len);
        const int t = vw_norm_w32((int32_t)smax * smax);
        scaling = t > nbits ? 0 : nbits - t;
    }
    uint32_t en = 0;
    for (int i = 0; i < len; ++i) {
        const int32_t v = x[i];
        en += (uint32_t)((v * v) >> scaling);
    }
    if (en == 0) {
        *out = offset;
        return;
    }
    const int norm = 17 - vw_clz(en);
    int tot = scaling + norm;
    uint32_t e = norm < 0 ? en << -norm : en >> norm;
    const int16_t log2e = (int16_t)(14336 + (int16_t)((e & 0x3FFF) >> 4));
    int16_t le = (int16_t)(((24660 * log2e) >> 19) + ((tot * 24660) >> 9));
    if (le < 0) le = 0;
    *out = (int16_t)(le + offset);
    if (*total <= PSB_VAD_MIN_ENERGY) {
        if (tot >= 0) *total = (int16_t)(*total + PSB_VAD_MIN_ENERGY + 1);
        else *total = (int16_t)(*total + (int16_t)(e >> -tot));
    }
}

// Scratch elements one frame's features need at `closest` Hz: the 8 kHz signal (none at 8 kHz,
// where the input is read in place; the 32 kHz path halves its 16 kHz buffer in place) and the
// four band buffers of WebRtcVad_CalculateFeatures (120 + 120 + 60 + 60).
PSB_VAD_HD int psb_vad_scratch_elems(int closest)
{
    return (closest == 8000 ? 0 : closest == 16000 ? 240 : 480) + 360;
}

// The six Q4 log energies and total_power of one frame (feat[0..5], feat[6]).  `pcm` holds
// frame_size samples at `closest` Hz.
template <typename In>
PSB_VAD_HD void psb_vad_frame_features(psb_vad_filt_t *f, int closest, In pcm, int frame_size, psb_vad_buf scr,
                                       int16_t *feat)
{
    const int nb = closest == 8000 ? 0 : closest == 16000 ? 240 : 480;
    psb_vad_buf hp120{scr.p + (nb + 0) * scr.s, scr.s}, lp120{scr.p + (nb + 120) * scr.s, scr.s};
    psb_vad_buf hp60{scr.p + (nb + 240) * scr.s, scr.s}, lp60{scr.p + (nb + 300) * scr.s, scr.s};
    int16_t total = 0;
    int L;
    if (closest == 8000) {
        L = frame_size;
        psb_vad_split(pcm, L, &f->upper[0], &f->lower[0], hp120, lp120);
    } else {
        psb_vad_buf x{scr.p, scr.s};
        if (closest == 16000) {
            psb_vad_downsample(pcm, x, &f->ds[0], frame_size);
            L = frame_size / 2;
        } else {
            psb_vad_downsample(pcm, x, &f->ds[2], frame_size);
            psb_vad_downsample(x, x, &f->ds[0], frame_size / 2);    // in place: out[n] after in[2n], in[2n+1]
            L = frame_size / 4;
        }
        psb_vad_split(x, L, &f->upper[0], &f->lower[0], hp120, lp120);
    }
    const int half = L >> 1;
    psb_vad_split(hp120, half, &f->upper[1], &f->lower[1], hp60, lp60);
    psb_vad_log_energy(hp60, half >> 1, 176, &total, &feat[5]);
    psb_vad_log_energy(lp60, half >> 1, 176, &total, &feat[4]);
    psb_vad_split(lp120, half, &f->upper[2], &f->lower[2], hp60, lp60);
    psb_vad_log_energy(hp60, half >> 1, 176, &total, &feat[3]);
    psb_vad_split(lp60, half >> 1, &f->upper[3], &f->lower[3], hp120, lp120);
    psb_vad_log_energy(hp120, half >> 2, 272, &total, &feat[2]);
    psb_vad_split(lp120, half >> 2, &f->upper[4], &f->lower[4], hp60, lp60);
    psb_vad_log_energy(hp60, half >> 3, 368, &total, &feat[1]);
    psb_vad_highpass(lp60, half >> 3, f->hp, hp120);
    psb_vad_log_energy(hp120, half >> 3, 368, &total, &feat[0]);
    feat[6] = total;
}

// ---- stage B: the GMM, one channel at a time ----------------------------------------------

// GMM state of one channel: Gaussians k = 0, 1 (VadInstT's arrays at [channel + 6 k]) and the
// smoothed minimum; the 16-entry age / minimum memory is passed separately (shared memory on
// the device).
struct psb_vad_chan_t {
    int16_t nm[2], sm[2], ns[2], ss[2];
    int16_t mean_value;
    // the channel's constants (vad_core.c:19-54), looked up once
    int16_t wn[2], ws[2], min_diff, max_speech, max_noise, maxspe;
};

// everything GmmProbability keeps per frame for one channel between the decision and the update
struct psb_vad_chan_probs_t {
    int16_t llr;        // log-likelihood ratio (shifts_h0 - shifts_h1)
    int16_t ngp[2], sgp[2], dn[2], ds[2];
};

PSB_VAD_HD void psb_vad_chan_init(psb_vad_chan_t *c, int ch, int16_t *age, int16_t *low)
{
    const int16_t nm[12] = {6738, 4892, 7065, 6715, 6771, 3369, 7646, 3863, 7820, 7266, 5020, 4362};
    const int16_t sm[12] = {8306, 10085, 10078, 11823, 11843, 6309, 9473, 9571, 10879, 7581, 8180, 7483};
    const int16_t ns[12] = {378, 1064, 493, 582, 688, 593, 474, 697, 475, 688, 421, 455};
    const int16_t ss[12] = {555, 505, 567, 524, 585, 1231, 509, 828, 492, 1540, 1079, 850};
    const int16_t wn[12] = {34, 62, 72, 66, 53, 25, 94, 66, 56, 62, 75, 103};
    const int16_t ws[12] = {48, 82, 45, 87, 50, 47, 80, 46, 83, 41, 78, 81};
    const int16_t min_diff[6] = {544, 544, 576, 576, 576, 576};
    const int16_t max_speech[6] = {11392, 11392, 11520, 11520, 11520, 11520};
    const int16_t max_noise[6] = {9216, 9088, 8960, 8832, 8704, 8576};
    for (int k = 0; k < 2; ++k) {
        const int g = ch + 6 * k;
        c->nm[k] = nm[g], c->sm[k] = sm[g], c->ns[k] = ns[g], c->ss[k] = ss[g];
        c->wn[k] = wn[g], c->ws[k] = ws[g];
    }
    c->mean_value = 1600;
    c->min_diff = min_diff[ch];
    c->max_speech = max_speech[ch];
    c->max_noise = max_noise[ch];
    // GmmProbability's maxspe is 12800 for channel 0 and the previous channel's limit after it
    c->maxspe = ch == 0 ? (int16_t)12800 : max_speech[ch - 1];
    for (int i = 0; i < 16; ++i) age[i] = 0, low[i] = 10000;
}

// Mode thresholds (WebRtcVad_set_mode_core) for the frame length index fi (0: 80, 1: 160, 2: 240
// samples at 8 kHz): over_hang_max_1, over_hang_max_2, individual, total.
PSB_VAD_HD void psb_vad_thresholds(int mode, int fi, int16_t *oh1, int16_t *oh2, int16_t *ind, int16_t *tot)
{
    const int16_t t[4][4][3] = {
        {{8, 4, 3}, {14, 7, 5}, {24, 21, 24}, {57, 48, 57}},
        {{8, 4, 3}, {14, 7, 5}, {37, 32, 37}, {100, 80, 100}},
        {{6, 3, 2}, {9, 5, 3}, {82, 78, 82}, {285, 260, 285}},
        {{6, 3, 2}, {9, 5, 3}, {94, 94, 94}, {1100, 1050, 1100}}};
    *oh1 = t[mode][0][fi];
    *oh2 = t[mode][1][fi];
    *ind = t[mode][2][fi];
    *tot = t[mode][3][fi];
}

// WebRtcVad_GaussianProbability: the Q20 probability and delta = (x - m) / s^2 in Q11
PSB_VAD_HD int32_t psb_vad_gauss(int16_t x, int16_t mean, int16_t std, int16_t *delta)
{
    const int16_t inv_std = (int16_t)vw_div(131072 + (std >> 1), std);
    int16_t t = (int16_t)(inv_std >> 2);
    const int16_t inv_std2 = (int16_t)((t * t) >> 2);
    t = (int16_t)(x << 3);
    t = (int16_t)(t - mean);
    *delta = (int16_t)((inv_std2 * t) >> 10);
    const int32_t e = (*delta * t) >> 9;
    int16_t ev = 0;
    if (e < 22005) {
        int16_t u = (int16_t)((5909 * e) >> 12);
        u = (int16_t)-u;
        ev = (int16_t)(0x0400 | (u & 0x03FF));
        u = (int16_t)(u ^ 0xFFFF);
        u = (int16_t)(u >> 10);
        u = (int16_t)(u + 1);
        ev = (int16_t)(ev >> u);
    }
    return inv_std * ev;
}

// First half of GmmProbability for one channel: probabilities under both models, the
// log-likelihood ratio, and the per-Gaussian shares used by the update.
PSB_VAD_HD void psb_vad_chan_probs(const psb_vad_chan_t *c, int16_t x, psb_vad_chan_probs_t *p)
{
    int32_t h0 = 0, h1 = 0, np0 = 0, sp0 = 0;
    for (int k = 0; k < 2; ++k) {
        const int32_t pn = c->wn[k] * psb_vad_gauss(x, c->nm[k], c->ns[k], &p->dn[k]);
        const int32_t ps = c->ws[k] * psb_vad_gauss(x, c->sm[k], c->ss[k], &p->ds[k]);
        h0 += pn;
        h1 += ps;
        if (k == 0) np0 = pn, sp0 = ps;
    }
    const int s0 = h0 == 0 ? 31 : vw_norm_w32(h0);
    const int s1 = h1 == 0 ? 31 : vw_norm_w32(h1);
    p->llr = (int16_t)(s0 - s1);
    const int16_t q0 = (int16_t)(h0 >> 12), q1 = (int16_t)(h1 >> 12);
    if (q0 > 0) {
        p->ngp[0] = (int16_t)vw_div((int32_t)(((uint32_t)np0 & 0xFFFFF000u) << 2), q0);
        p->ngp[1] = (int16_t)(16384 - p->ngp[0]);
    } else {
        p->ngp[0] = 16384;
        p->ngp[1] = 0;
    }
    if (q1 > 0) {
        p->sgp[0] = (int16_t)vw_div((int32_t)(((uint32_t)sp0 & 0xFFFFF000u) << 2), q1);
        p->sgp[1] = (int16_t)(16384 - p->sgp[0]);
    } else {
        p->sgp[0] = 0;
        p->sgp[1] = 0;
    }
}

PSB_VAD_HD int16_t psb_vad_spectrum_weight(int ch) { return (int16_t)(6 + 2 * ch); }

// WebRtcVad_FindMinimum for one channel; frame_counter is the count before this frame.
PSB_VAD_HD int16_t psb_vad_find_minimum(psb_vad_chan_t *c, int16_t *age, int16_t *low, int16_t x, int32_t frame_counter)
{
    for (int i = 0; i < 16; ++i) {
        if (age[i] != 100) {
            age[i] = (int16_t)(age[i] + 1);
        } else {
            for (int j = i; j < 15; ++j) low[j] = low[j + 1], age[j] = age[j + 1];
            age[15] = 101;
            low[15] = 10000;
        }
    }
    int pos = -1;
    if (x < low[7]) {
        if (x < low[3]) pos = x < low[1] ? (x < low[0] ? 0 : 1) : (x < low[2] ? 2 : 3);
        else pos = x < low[5] ? (x < low[4] ? 4 : 5) : (x < low[6] ? 6 : 7);
    } else if (x < low[15]) {
        if (x < low[11]) pos = x < low[9] ? (x < low[8] ? 8 : 9) : (x < low[10] ? 10 : 11);
        else pos = x < low[13] ? (x < low[12] ? 12 : 13) : (x < low[14] ? 14 : 15);
    }
    if (pos > -1) {
        for (int i = 15; i > pos; --i) low[i] = low[i - 1], age[i] = age[i - 1];
        low[pos] = x;
        age[pos] = 1;
    }
    int16_t median = 1600;
    if (frame_counter > 2) median = low[2];
    else if (frame_counter > 0) median = low[0];
    int16_t alpha = 0;
    if (frame_counter > 0) alpha = median < c->mean_value ? 6553 : 32439;
    int32_t t = (alpha + 1) * c->mean_value;
    t += (32767 - alpha) * median;
    t += 16384;
    c->mean_value = (int16_t)(t >> 15);
    return c->mean_value;
}

// Second half of GmmProbability for one channel: model adaptation after the frame's decision.
PSB_VAD_HD void psb_vad_chan_update(psb_vad_chan_t *c, int ch, int16_t *age, int16_t *low, int16_t x, int vadflag,
                                    int32_t frame_counter, const psb_vad_chan_probs_t *p)
{
    const int16_t maxspe = c->maxspe;
    const int16_t fmin = psb_vad_find_minimum(c, age, low, x, frame_counter);
    int32_t ngm = c->nm[0] * c->wn[0] + c->nm[1] * c->wn[1];
    const int16_t ngm8 = (int16_t)(ngm >> 6);
    for (int k = 0; k < 2; ++k) {
        const int16_t nmk = c->nm[k], smk = c->sm[k];
        int16_t nsk = c->ns[k], ssk = c->ss[k];
        int16_t nmk2 = nmk;
        if (!vadflag) {
            const int16_t delt = (int16_t)((p->ngp[k] * p->dn[k]) >> 11);
            nmk2 = (int16_t)(nmk + (int16_t)((delt * 655) >> 22));
        }
        const int16_t ndelt = (int16_t)((fmin << 4) - ngm8);
        int16_t nmk3 = (int16_t)(nmk2 + (int16_t)((ndelt * 154) >> 9));
        const int16_t lo = (int16_t)((k + 5) << 7), hi = (int16_t)((72 + k - ch) << 7);
        if (nmk3 < lo) nmk3 = lo;
        if (nmk3 > hi) nmk3 = hi;
        c->nm[k] = nmk3;
        if (vadflag) {
            const int16_t delt = (int16_t)((p->sgp[k] * p->ds[k]) >> 11);
            int16_t t = (int16_t)((delt * 6554) >> 21);
            int16_t smk2 = (int16_t)(smk + ((t + 1) >> 1));
            const int16_t maxmu = (int16_t)(maxspe + 640);
            const int16_t minmu = k == 0 ? (int16_t)640 : (int16_t)768;
            if (smk2 < minmu) smk2 = minmu;
            if (smk2 > maxmu) smk2 = maxmu;
            c->sm[k] = smk2;
            t = (int16_t)((smk + 4) >> 3);
            t = (int16_t)(x - t);
            int32_t a = (p->ds[k] * t) >> 3;
            a = a - 4096;
            const int16_t sg = (int16_t)(p->sgp[k] >> 2);
            a = vw_mul(sg, a) >> 4;
            const int16_t den = (int16_t)(ssk * 10);
            if (a > 0) t = (int16_t)vw_div(a, den);
            else t = (int16_t)-(int16_t)vw_div(vw_sub(0, a), den);
            t = (int16_t)(t + 128);
            ssk = (int16_t)(ssk + (t >> 8));
            if (ssk < 384) ssk = 384;
            c->ss[k] = ssk;
        } else {
            int16_t t = (int16_t)(x - (nmk >> 3));
            int32_t a = (p->dn[k] * t) >> 3;
            a -= 4096;
            t = (int16_t)((p->ngp[k] + 2) >> 2);
            a = vw_mul(t, a) >> 14;
            if (a > 0) t = (int16_t)vw_div(a, nsk);
            else t = (int16_t)-(int16_t)vw_div(vw_sub(0, a), nsk);
            t = (int16_t)(t + 32);
            nsk = (int16_t)(nsk + (t >> 6));
            if (nsk < 384) nsk = 384;
            c->ns[k] = nsk;
        }
    }
    ngm = c->nm[0] * c->wn[0] + c->nm[1] * c->wn[1];
    int32_t sgm = c->sm[0] * c->ws[0] + c->sm[1] * c->ws[1];
    const int16_t diff = (int16_t)((int16_t)(sgm >> 9) - (int16_t)(ngm >> 9));
    if (diff < c->min_diff) {
        const int16_t t = (int16_t)(c->min_diff - diff);
        const int16_t up = (int16_t)((13 * t) >> 2), dn = (int16_t)((3 * t) >> 2);
        sgm = 0;
        ngm = 0;
        for (int k = 0; k < 2; ++k) {
            c->sm[k] = (int16_t)(c->sm[k] + up);
            sgm += c->sm[k] * c->ws[k];
            c->nm[k] = (int16_t)(c->nm[k] - dn);
            ngm += c->nm[k] * c->wn[k];
        }
    }
    int16_t t = (int16_t)(sgm >> 7);
    if (t > c->max_speech) {
        t = (int16_t)(t - c->max_speech);
        for (int k = 0; k < 2; ++k) c->sm[k] = (int16_t)(c->sm[k] - t);
    }
    t = (int16_t)(ngm >> 7);
    if (t > c->max_noise) {
        t = (int16_t)(t - c->max_noise);
        for (int k = 0; k < 2; ++k) c->nm[k] = (int16_t)(c->nm[k] - t);
    }
}

// the hysteresis at the end of GmmProbability; returns the frame's raw decision (0, 1, or 2 +
// the overhang left); ps_vad_classify reports it as 0 / 1
PSB_VAD_HD int psb_vad_overhang(int vadflag, int16_t *over_hang, int16_t *num_of_speech, int16_t oh1, int16_t oh2)
{
    if (!vadflag) {
        if (*over_hang > 0) {
            vadflag = 2 + *over_hang;
            *over_hang = (int16_t)(*over_hang - 1);
        }
        *num_of_speech = 0;
    } else {
        *num_of_speech = (int16_t)(*num_of_speech + 1);
        if (*num_of_speech > 6) {
            *num_of_speech = 6;
            *over_hang = oh2;
        } else {
            *over_hang = oh1;
        }
    }
    return vadflag;
}

// ---- the endpointer -------------------------------------------------------------------------

// ps_endpointer_t without the sample ring: the queue is frames head .. head + n - 1 of the
// stream, and their decisions are read back through `flags` (any type indexed by the stream's
// frame number: the per-frame output on the host, a ring of maxlen + 1 entries on the device).
struct psb_ep_t {
    int maxlen, start_frames, end_frames, frame_size, sample_rate;
    double frame_length;
    int n, speech_count, in_speech;
    int64_t head, pushed;
    double qstart_time, last_audio_timestamp, speech_start, speech_end;
    int64_t seg_start;
};

struct psb_ep_seg_t {
    int64_t start, end;          // samples [start, end)
    double start_time, end_time; // ps_endpointer_speech_start / _speech_end
};

PSB_VAD_HD void psb_ep_init(psb_ep_t *e, int maxlen, int start_frames, int end_frames, int frame_size, int sample_rate)
{
    e->maxlen = maxlen, e->start_frames = start_frames, e->end_frames = end_frames;
    e->frame_size = frame_size, e->sample_rate = sample_rate;
    e->frame_length = (double)frame_size / sample_rate;
    e->n = e->speech_count = e->in_speech = 0;
    e->head = e->pushed = 0;
    e->qstart_time = e->last_audio_timestamp = e->speech_start = e->speech_end = 0.0;
    e->seg_start = 0;
}

template <typename Flags>
PSB_VAD_HD int psb_ep_pop(psb_ep_t *e, const Flags &flags)
{
    e->qstart_time += e->frame_length;
    const int s = flags[e->head];
    if (s) e->speech_count--;
    e->head++;
    e->n--;
    return s;
}

// ps_endpointer_process on frame e->pushed, whose decision flags[e->pushed] has been written.
// Returns 1 and fills *seg when a segment ends with this frame.
template <typename Flags>
PSB_VAD_HD int psb_ep_process(psb_ep_t *e, const Flags &flags, psb_ep_seg_t *seg)
{
    const bool full = e->n == e->maxlen;
    if (full && flags[e->head]) e->speech_count--;       // the oldest frame is overwritten
    if (flags[e->pushed]) e->speech_count++;
    if (full) {
        e->qstart_time += e->frame_length;
        e->head++;
    } else {
        e->n++;
    }
    e->pushed++;
    e->last_audio_timestamp += e->frame_length;
    if (e->in_speech) {
        if (e->speech_count < e->end_frames) {
            psb_ep_pop(e, flags);
            e->speech_end = e->qstart_time;
            e->in_speech = 0;
            seg->start = e->seg_start;
            seg->end = e->head * e->frame_size;
            seg->start_time = e->speech_start;
            seg->end_time = e->speech_end;
            return 1;
        }
    } else if (e->speech_count > e->start_frames) {
        e->speech_start = e->qstart_time;
        e->speech_end = 0;
        e->in_speech = 1;
        e->seg_start = e->head * e->frame_size;
    }
    if (e->in_speech) psb_ep_pop(e, flags);
    return 0;
}

// ps_endpointer_end_stream with the nsamp (< frame_size) samples after the last full frame.
template <typename Flags>
PSB_VAD_HD int psb_ep_end_stream(psb_ep_t *e, const Flags &flags, int nsamp, psb_ep_seg_t *seg)
{
    if (!e->in_speech) return 0;
    e->in_speech = 0;
    e->speech_end = e->qstart_time;
    int64_t end = e->head * e->frame_size;
    while (e->n > 0) {
        if (!psb_ep_pop(e, flags)) break;
        e->speech_end = e->qstart_time;
        end = e->head * e->frame_size;
    }
    if (e->n == 0 && e->speech_end == e->qstart_time) {
        e->last_audio_timestamp += (double)nsamp / e->sample_rate;
        e->speech_end = e->last_audio_timestamp;
        end += nsamp;
    }
    // ep_clear: the rest of the queue is dropped without advancing qstart_time (the times of a stream that goes on
    // lag by the dropped frames, as the reference's do), while frame numbers stay the stream's own
    e->n = 0;
    e->speech_count = 0;
    e->head = e->pushed;
    seg->start = e->seg_start;
    seg->end = end;
    seg->start_time = e->speech_start;
    seg->end_time = e->speech_end;
    return 1;
}

// ---- live streams -----------------------------------------------------------------------------

// Everything a ps_endpointer_t (and the ps_vad_t inside it) carries from one frame to the next,
// except the decisions of its queue (a ring of maxlen + 1 int8 indexed by frame number, kept beside
// the record) and the samples after the last full frame (fewer than frame_size, also kept beside
// it).  A stream saved here after any frame and restored goes on exactly as if it had not stopped.
struct psb_vad_slot_t {
    psb_vad_filt_t filt;
    int16_t nm[PSB_VAD_NCH][2], sm[PSB_VAD_NCH][2], ns[PSB_VAD_NCH][2], ss[PSB_VAD_NCH][2];
    int16_t mean_value[PSB_VAD_NCH];
    int16_t age[PSB_VAD_NCH][16], low[PSB_VAD_NCH][16];
    int32_t frame_counter;
    int16_t over_hang, num_of_speech;
    psb_ep_t ep;
};

// the state of a fresh ps_endpointer_init
PSB_VAD_HD void psb_vad_slot_init(psb_vad_slot_t *s, int maxlen, int start_frames, int end_frames, int frame_size,
                                  int sample_rate)
{
    psb_vad_filt_init(&s->filt);
    for (int ch = 0; ch < PSB_VAD_NCH; ++ch) {
        psb_vad_chan_t c;
        psb_vad_chan_init(&c, ch, s->age[ch], s->low[ch]);
        for (int k = 0; k < 2; ++k) s->nm[ch][k] = c.nm[k], s->sm[ch][k] = c.sm[k], s->ns[ch][k] = c.ns[k], s->ss[ch][k] = c.ss[k];
        s->mean_value[ch] = c.mean_value;
    }
    s->frame_counter = 0;
    s->over_hang = s->num_of_speech = 0;
    psb_ep_init(&s->ep, maxlen, start_frames, end_frames, frame_size, sample_rate);
}

// channel ch's adapted GMM into *c, whose constants psb_vad_chan_init has set
PSB_VAD_HD void psb_vad_slot_load_chan(const psb_vad_slot_t *s, int ch, psb_vad_chan_t *c)
{
    for (int k = 0; k < 2; ++k) c->nm[k] = s->nm[ch][k], c->sm[k] = s->sm[ch][k], c->ns[k] = s->ns[ch][k], c->ss[k] = s->ss[ch][k];
    c->mean_value = s->mean_value[ch];
}

PSB_VAD_HD void psb_vad_slot_store_chan(psb_vad_slot_t *s, int ch, const psb_vad_chan_t *c)
{
    for (int k = 0; k < 2; ++k) s->nm[ch][k] = c->nm[k], s->sm[ch][k] = c->sm[k], s->ns[ch][k] = c->ns[k], s->ss[ch][k] = c->ss[k];
    s->mean_value[ch] = c->mean_value;
}

#endif  // PSB_VAD_CORE_H
