// tests/emul/apn_emul.cpp -- TEST INFRASTRUCTURE.  Compiles the phase code of the device phone
// decoder over a factored PHMM net (pocketsphinx_b200/csrc/psb_apn_core.h, the source
// allphone_net_kernel is built from) for the host and runs it one "thread" at a time: every
// block-wide loop to completion, in ascending or (-DPSB_FSG_EMUL_REVERSE) descending order.  Only the
// HMM update comes from the oracle (the device's own hmm_step is covered by the GPU tests).  Never
// linked into libpsb200.so.
#define PSB_FSG_HOST_EMUL 1
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../pocketsphinx_b200/csrc/psb_apn_core.h"
extern "C" {
#include "../../oracle/ps_oracle.h"
}

namespace {
struct OracleEval {
    pso_hmmctx_t ctx;
    const ApnNet *G;
    const int32_t *ssid, *tmatid;
    int operator()(const ApnWork &W, int p)
    {
        pso_hmm_t h;
        const int N = G->n_emit, H = G->H;
        pso_hmm_init(&ctx, &h, 0, ssid[p], tmatid[p]);
        for (int s = 0; s < N; ++s) { h.score[s] = W.score[s * H + p]; h.history[s] = W.hist[s * H + p]; }
        h.out_score = W.out_score[p]; h.out_history = W.out_hist[p]; h.bestscore = W.best[p];
        const int b = pso_hmm_vit_eval(&ctx, &h);
        for (int s = 0; s < N; ++s) { W.score[s * H + p] = h.score[s]; W.hist[s * H + p] = h.history[s]; }
        W.out_score[p] = h.out_score; W.out_hist[p] = h.out_history; W.best[p] = h.bestscore;
        return b;
    }
};
}

// One utterance.  res = (status: 0 ok / 1 history overflow, n_hist, n_seg).  Returns 0.
extern "C" int32_t
apn_emul_run(int32_t n_emit_state, const uint8_t *tp, const uint16_t *sseq, int32_t H, const int32_t *ssid,
             const int32_t *tmatid, const int32_t *ci, const uint64_t *lc, const uint64_t *rc, int32_t n_ci,
             int32_t start, int32_t beam, int32_t pbeam, int32_t inspen, const int32_t *bg, const int32_t *tg,
             const int16_t *senscr, int32_t n_sen, int32_t T, int32_t *hist_out, int32_t cap, int32_t *segs,
             int32_t seg_cap, int32_t *res)
{
    ApnNet G;
    memset(&G, 0, sizeof(G));
    G.H = H; G.n_ci = n_ci; G.n_emit = n_emit_state; G.start = start;
    G.beam = beam; G.pbeam = pbeam; G.inspen = inspen;
    G.ci = ci; G.lc = (const unsigned long long *)lc; G.rc = (const unsigned long long *)rc; G.bg = bg; G.tg = tg;
    std::vector<int32_t> work(apn_work_words(H, n_emit_state), 0x5a5a5a5a);   // poison: nothing may rely on zeroed scratch
    std::vector<int32_t> tab(2 * (size_t)n_ci * n_ci, 0x5a5a5a5a);
    ApnWork W;
    apn_work_carve(work.data(), G, W);
    W.msc = tab.data(); W.mix = tab.data() + (size_t)n_ci * n_ci;
    W.hist_out = hist_out; W.cap = cap;
    ApnScalars S;
    memset((void *)&S, 0x5a, sizeof(S));
    OracleEval ev;
    memset(&ev.ctx, 0, sizeof(ev.ctx));
    ev.ctx.n_emit_state = n_emit_state; ev.ctx.tp = tp; ev.ctx.sseq = sseq;
    ev.G = &G; ev.ssid = ssid; ev.tmatid = tmatid;
    FSG_SYNC();
    apn_start(G, W, &S);
    for (int t = 0; t < T && !S.overflow; ++t) {
        ev.ctx.senscore = senscr + (size_t)t * n_sen;
        apn_step(G, W, &S, t, ev);
    }
    res[0] = S.overflow ? 1 : 0;
    res[1] = S.n_hist;
    res[2] = S.overflow ? 0 : apn_backtrace(G, W, &S, segs, seg_cap);
    return 0;
}

extern "C" long emul_race_count(void)
{
#ifdef PSB_FSG_RACECHECK
    return fsgrace::st().n_races;
#else
    return -1;
#endif
}
