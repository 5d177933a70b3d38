// vad_emul.cpp -- pocketsphinx_b200/csrc/psb_vad_core.h (the arithmetic psb_vad.cu's kernels are
// compiled from) built for the host, for the CPU tests against the compiled reference:
//   vad_emul_run       the sequential run, with the whole VadInstT (reference layout) after every frame
//   vad_emul_features  stage A as the device runs it: chunks of C frames, each from the initial
//                      filter state `warmup` frames early, then the boundary walk with repairs
//   vad_emul_segments  stage B + the endpointer over given features
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../pocketsphinx_b200/csrc/psb_vad_core.h"

// VadInstT (common_audio/vad/vad_core.h:25-51), field for field
struct ref_vadinst_t {
    int32_t vad;
    int32_t downsampling_filter_states[4];
    int32_t state_48_to_8[40];
    int16_t noise_means[12], speech_means[12], noise_stds[12], speech_stds[12];
    int32_t frame_counter;
    int16_t over_hang, num_of_speech;
    int16_t index_vector[96], low_value_vector[96];
    int16_t mean_value[6];
    int16_t upper_state[5], lower_state[5], hp_filter_state[4];
    int16_t over_hang_max_1[3], over_hang_max_2[3], individual[3], total[3];
    int32_t init_flag;
};
static_assert(sizeof(ref_vadinst_t) == 736, "VadInstT layout");

namespace {

struct Gmm {
    psb_vad_chan_t ch[6];
    int16_t age[6][16], low[6][16];
    int32_t frame_counter = 0;
    int16_t over_hang = 0, num_of_speech = 0;
    int vad = 1;
    int mode, fi;
    Gmm(int mode_, int len8k) : mode(mode_), fi(len8k == 80 ? 0 : len8k == 160 ? 1 : 2)
    {
        for (int c = 0; c < 6; ++c) psb_vad_chan_init(&ch[c], c, age[c], low[c]);
    }
    int step(const int16_t *feat)
    {
        int16_t oh1, oh2, ind, tot;
        psb_vad_thresholds(mode, fi, &oh1, &oh2, &ind, &tot);
        int vadflag = 0;
        if (feat[6] > PSB_VAD_MIN_ENERGY) {
            psb_vad_chan_probs_t p[6];
            int32_t sum = 0;
            for (int c = 0; c < 6; ++c) {
                psb_vad_chan_probs(&ch[c], feat[c], &p[c]);
                sum += p[c].llr * psb_vad_spectrum_weight(c);
                if (p[c].llr * 4 > ind) vadflag = 1;
            }
            vadflag |= sum >= tot;
            for (int c = 0; c < 6; ++c) psb_vad_chan_update(&ch[c], c, age[c], low[c], feat[c], vadflag, frame_counter, &p[c]);
            frame_counter++;
        }
        vad = psb_vad_overhang(vadflag, &over_hang, &num_of_speech, oh1, oh2);
        return vad > 0;
    }
    void dump(const psb_vad_filt_t &f, ref_vadinst_t *r) const
    {
        memset(r, 0, sizeof(*r));
        r->vad = vad;
        for (int i = 0; i < 4; ++i) r->downsampling_filter_states[i] = f.ds[i], r->hp_filter_state[i] = f.hp[i];
        for (int i = 0; i < 5; ++i) r->upper_state[i] = f.upper[i], r->lower_state[i] = f.lower[i];
        for (int c = 0; c < 6; ++c) {
            for (int k = 0; k < 2; ++k) {
                r->noise_means[c + 6 * k] = ch[c].nm[k], r->speech_means[c + 6 * k] = ch[c].sm[k];
                r->noise_stds[c + 6 * k] = ch[c].ns[k], r->speech_stds[c + 6 * k] = ch[c].ss[k];
            }
            for (int i = 0; i < 16; ++i) r->index_vector[16 * c + i] = age[c][i], r->low_value_vector[16 * c + i] = low[c][i];
            r->mean_value[c] = ch[c].mean_value;
        }
        r->frame_counter = frame_counter;
        r->over_hang = over_hang;
        r->num_of_speech = num_of_speech;
        for (int i = 0; i < 3; ++i)
            psb_vad_thresholds(mode, i, &r->over_hang_max_1[i], &r->over_hang_max_2[i], &r->individual[i], &r->total[i]);
        r->init_flag = 42;
    }
};

int len8k(int closest, int frame_size) { return frame_size / (closest / 8000); }

}  // namespace

extern "C" {

// the state ps_vad_init leaves (mode's thresholds, nothing processed)
void vad_emul_init_state(int mode, ref_vadinst_t *out)
{
    Gmm g(mode, 80);
    psb_vad_filt_t f;
    psb_vad_filt_init(&f);
    g.dump(f, out);
}

long vad_emul_run(int mode, int closest, int frame_size, const int16_t *pcm, long n_frames, int8_t *flags,
                  ref_vadinst_t *states)
{
    Gmm g(mode, len8k(closest, frame_size));
    psb_vad_filt_t f;
    psb_vad_filt_init(&f);
    std::vector<int16_t> scr(psb_vad_scratch_elems(closest));
    for (long t = 0; t < n_frames; ++t) {
        int16_t feat[8];
        psb_vad_frame_features(&f, closest, pcm + t * frame_size, frame_size, psb_vad_buf{scr.data(), 1}, feat);
        flags[t] = (int8_t)g.step(feat);
        if (states) g.dump(f, &states[t]);
    }
    return n_frames;
}

// feat [n_frames][8]; returns the number of chunk recomputations, *passes the repair passes.  The passes
// are vad_repair_kernel's: every chunk reads its predecessor's end state as the previous pass left it.
long vad_emul_features(int closest, int frame_size, const int16_t *pcm, long n_frames, int chunk, int warmup,
                       int16_t *feat, int *passes)
{
    std::vector<int16_t> scr(psb_vad_scratch_elems(closest)), dummy(8);
    psb_vad_buf b{scr.data(), 1};
    const long n_chunks = (n_frames + chunk - 1) / chunk;
    std::vector<psb_vad_filt_t> st_start(n_chunks), end_in(n_chunks), end_out(n_chunks);
    auto run = [&](psb_vad_filt_t f, long k) {
        const long f0 = k * chunk, f1 = f0 + chunk < n_frames ? f0 + chunk : n_frames;
        for (long t = f0; t < f1; ++t) psb_vad_frame_features(&f, closest, pcm + t * frame_size, frame_size, b, feat + 8 * t);
        return f;
    };
    for (long k = 0; k < n_chunks; ++k) {
        psb_vad_filt_t f;
        psb_vad_filt_init(&f);
        const long f0 = k * chunk, w0 = f0 - warmup > 0 ? f0 - warmup : 0;
        for (long t = w0; t < f0; ++t) psb_vad_frame_features(&f, closest, pcm + t * frame_size, frame_size, b, dummy.data());
        st_start[k] = f;
        end_in[k] = run(f, k);
    }
    long repairs = 0;
    *passes = 0;
    for (bool changed = n_chunks > 0; changed;) {
        changed = false;
        ++*passes;
        for (long k = 0; k < n_chunks; ++k) {
            end_out[k] = end_in[k];
            if (k == 0 || k * chunk - warmup <= 0) continue;      // started from the stream's own beginning
            if (psb_vad_filt_equal(&st_start[k], &end_in[k - 1])) continue;
            st_start[k] = end_in[k - 1];
            end_out[k] = run(end_in[k - 1], k);
            ++repairs;
            changed = true;
        }
        end_in.swap(end_out);
    }
    return repairs;
}

// stage B over feat [n_frames][8]: flags, then the endpointer; segs [n][2], times [n][2]
long vad_emul_segments(int mode, int closest, int frame_size, int sample_rate, int maxlen, int start_frames,
                       int end_frames, const int16_t *feat, long n_frames, int nsamp_tail, int8_t *flags,
                       int64_t *segs, double *times)
{
    Gmm g(mode, len8k(closest, frame_size));
    psb_ep_t e;
    psb_ep_init(&e, maxlen, start_frames, end_frames, frame_size, sample_rate);
    long n = 0;
    psb_ep_seg_t s;
    const int8_t *fl = flags;
    for (long t = 0; t < n_frames; ++t) {
        flags[t] = (int8_t)g.step(feat + 8 * t);
        if (psb_ep_process(&e, fl, &s)) {
            segs[2 * n] = s.start, segs[2 * n + 1] = s.end, times[2 * n] = s.start_time, times[2 * n + 1] = s.end_time;
            ++n;
        }
    }
    if (psb_ep_end_stream(&e, fl, nsamp_tail, &s)) {
        segs[2 * n] = s.start, segs[2 * n + 1] = s.end, times[2 * n] = s.start_time, times[2 * n + 1] = s.end_time;
        ++n;
    }
    return n;
}

}  // extern "C"
