// vad_live_emul.cpp -- a live stream as psb_vad_feed_* runs one slot, built for the host from
// pocketsphinx_b200/csrc/psb_vad_core.h: between calls the stream exists only as its saved
// psb_vad_slot_t, its queue ring of maxlen + 1 decisions and its leftover samples.  A call puts the
// leftover before the new samples, computes the features in chunks of 64 frames (chunk 0, and every
// chunk whose warm-up reaches back to the call's first frame, from the saved filter state; the
// others from the initial state `warmup` frames early, then vad_repair_kernel's passes), loads the
// GMM and endpointer, runs the frames, ends the stream where final, and saves everything back.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../pocketsphinx_b200/csrc/psb_vad_core.h"

namespace {

constexpr int CHUNK = 64;

struct Ring {
    int8_t *p;
    int m;
    int8_t &operator[](int64_t f) const { return p[(int)f % m]; }
};

struct Live {
    int mode, closest, frame_size, sample_rate, maxlen, start_frames, end_frames, warmup;
    psb_vad_slot_t slot;
    std::vector<int8_t> ring;
    std::vector<int16_t> left;
    void fresh()
    {
        psb_vad_slot_init(&slot, maxlen, start_frames, end_frames, frame_size, sample_rate);
        ring.assign((size_t)maxlen + 1, 0);
        left.clear();
    }
};

// features of frames f0 .. f1 - 1 from *f
void run_frames(psb_vad_filt_t *f, const Live &L, const int16_t *x, long f0, long f1, int16_t *feat)
{
    std::vector<int16_t> scr(psb_vad_scratch_elems(L.closest));
    int16_t dummy[8];
    for (long t = f0; t < f1; ++t)
        psb_vad_frame_features(f, L.closest, x + t * L.frame_size, L.frame_size, psb_vad_buf{scr.data(), 1},
                               feat ? feat + 8 * t : dummy);
}

}  // namespace

extern "C" {

void *vad_live_emul_open(int mode, int closest, int frame_size, int sample_rate, int maxlen, int start_frames,
                         int end_frames, int warmup)
{
    Live *L = new Live{mode, closest, frame_size, sample_rate, maxlen, start_frames, end_frames, warmup, {}, {}, {}};
    L->fresh();
    return L;
}

void vad_live_emul_free(void *p) { delete (Live *)p; }
void vad_live_emul_reset(void *p) { ((Live *)p)->fresh(); }

// outputs as tests/emul/vad_live_refdrv.c's refdrv_live_feed; returns the segment count
long vad_live_emul_feed(void *p, const int16_t *pcm, long nsamp, int final, int8_t *flags, int64_t *segs, double *times,
                        int64_t *status, double *st_times)
{
    Live &L = *(Live *)p;
    std::vector<int16_t> x(L.left);
    x.insert(x.end(), pcm, pcm + nsamp);
    const long len = (long)x.size(), nf = len / L.frame_size, n_chunks = (nf + CHUNK - 1) / CHUNK;

    // stage A
    std::vector<int16_t> feat((size_t)nf * 8 + 8);
    std::vector<psb_vad_filt_t> st_start(n_chunks), end_in(n_chunks), end_out(n_chunks);
    for (long k = 0; k < n_chunks; ++k) {
        const long f0 = k * CHUNK, w0 = f0 - L.warmup > 0 ? f0 - L.warmup : 0;
        psb_vad_filt_t f;
        if (w0 == 0) f = L.slot.filt;
        else psb_vad_filt_init(&f);
        run_frames(&f, L, x.data(), w0, f0, nullptr);
        st_start[k] = f;
        run_frames(&f, L, x.data(), f0, f0 + CHUNK < nf ? f0 + CHUNK : nf, feat.data());
        end_in[k] = f;
    }
    for (bool changed = n_chunks > 1; changed;) {
        changed = false;
        for (long k = 0; k < n_chunks; ++k) {
            end_out[k] = end_in[k];
            if (k == 0 || k * CHUNK - L.warmup <= 0 || psb_vad_filt_equal(&st_start[k], &end_in[k - 1])) continue;
            psb_vad_filt_t f = st_start[k] = end_in[k - 1];
            run_frames(&f, L, x.data(), k * CHUNK, k * CHUNK + CHUNK < nf ? k * CHUNK + CHUNK : nf, feat.data());
            end_out[k] = f;
            changed = true;
        }
        end_in.swap(end_out);
    }
    if (n_chunks) L.slot.filt = end_in[n_chunks - 1];

    // stage B from the saved slot
    const int l8 = L.frame_size / (L.closest / 8000);
    int16_t oh1, oh2, ind, tot;
    psb_vad_thresholds(L.mode, l8 == 80 ? 0 : l8 == 160 ? 1 : 2, &oh1, &oh2, &ind, &tot);
    psb_vad_slot_t &s = L.slot;
    psb_vad_chan_t ch[PSB_VAD_NCH];
    int16_t scratch_age[16], scratch_low[16];
    for (int c = 0; c < PSB_VAD_NCH; ++c) {
        psb_vad_chan_init(&ch[c], c, scratch_age, scratch_low);
        psb_vad_slot_load_chan(&s, c, &ch[c]);
    }
    const Ring ring{L.ring.data(), L.maxlen + 1};
    long n = 0;
    psb_ep_seg_t sg;
    for (long t = 0; t < nf; ++t) {
        const int16_t *ft = feat.data() + 8 * t;
        int vadflag = 0;
        if (ft[6] > PSB_VAD_MIN_ENERGY) {
            psb_vad_chan_probs_t pr[PSB_VAD_NCH];
            int32_t sum = 0;
            for (int c = 0; c < PSB_VAD_NCH; ++c) {
                psb_vad_chan_probs(&ch[c], ft[c], &pr[c]);
                sum += pr[c].llr * psb_vad_spectrum_weight(c);
                if (pr[c].llr * 4 > ind) vadflag = 1;
            }
            vadflag |= sum >= tot;
            for (int c = 0; c < PSB_VAD_NCH; ++c)
                psb_vad_chan_update(&ch[c], c, s.age[c], s.low[c], ft[c], vadflag, s.frame_counter, &pr[c]);
            s.frame_counter++;
        }
        vadflag = psb_vad_overhang(vadflag, &s.over_hang, &s.num_of_speech, oh1, oh2);
        flags[t] = ring[s.ep.pushed] = (int8_t)(vadflag > 0);
        if (psb_ep_process(&s.ep, ring, &sg)) {
            segs[2 * n] = sg.start, segs[2 * n + 1] = sg.end, times[2 * n] = sg.start_time, times[2 * n + 1] = sg.end_time;
            ++n;
        }
    }
    const long tail = len - nf * L.frame_size;
    if (final && psb_ep_end_stream(&s.ep, ring, (int)tail, &sg)) {
        segs[2 * n] = sg.start, segs[2 * n + 1] = sg.end, times[2 * n] = sg.start_time, times[2 * n + 1] = sg.end_time;
        ++n;
    }
    for (int c = 0; c < PSB_VAD_NCH; ++c) psb_vad_slot_store_chan(&s, c, &ch[c]);
    L.left.assign(final ? x.end() : x.end() - tail, x.end());

    status[0] = s.ep.in_speech;
    status[1] = s.ep.in_speech ? s.ep.seg_start : -1;
    status[2] = s.ep.pushed;
    st_times[0] = s.ep.speech_start;
    st_times[1] = s.ep.speech_end;
    return n;
}

}  // extern "C"
