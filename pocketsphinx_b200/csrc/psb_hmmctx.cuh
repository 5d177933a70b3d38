// psb_hmmctx.cuh -- the HMM context object behind psb_hmmctx_t, shared by psb_hmm.cu (hmm_vit_eval,
// phone loop, alignment, keyword spotting, phone decoding) and psb_search.cu (grammar / n-gram search),
// and the plumbing its whole-utterance entry points share.
#pragma once
#include "psb_hmm.cuh"

#include <initializer_list>

// A context serves one host thread at a time.  Every entry point that runs on its stream returns with the
// stream idle, so the next call, whichever entry point it is, may reuse the workspace slots.
struct psb_hmmctx_s {
    int device;
    int n_emit, n_tmat, n_sseq, n_sen;
    Stream stream;                // declared first: destroyed after the buffers below
    DevBuf<uint8_t> d_tp;
    DevBuf<uint16_t> d_sseq;      // [n_sseq][n_emit], on the device and on the host
    std::vector<uint16_t> h_sseq;
    // staging for psb_hmm_vit_eval_batch
    DevBuf<psb_hmm_t> d_hmms;
    HostBuf<psb_hmm_t> h_hmms;
    DevBuf<int16_t> d_senscr;
    HostBuf<int16_t> h_senscr;
    DevBuf<int32_t> d_best;
    HostBuf<int32_t> h_best;
    Event al_ev[2];               // around the last psb_align_batch_* kernel
    float last_align_ms;
    int64_t last_align_tok_bytes; // the token arena of the last psb_align_batch_* call (ids and scores)
    // grow-only device workspace of the whole-utterance entry points (srch_reserve)
    DevBuf<unsigned char> srch[10];
};

static inline HmmCtxDev dev_ctx(const psb_hmmctx_t *c)
{
    HmmCtxDev d;
    d.n_emit = c->n_emit; d.n_sen = c->n_sen; d.tp = c->d_tp; d.sseq = c->d_sseq;
    return d;
}

// Grow-only device workspace kept in the context: repeated calls (one per batch) do not pay
// an allocation again.
template <class T>
static int srch_reserve(psb_hmmctx_t *c, int slot, size_t count, T **out)
{
    const size_t bytes = (count > 0 ? count : 1) * sizeof(T);
    const int rc = c->srch[slot].reserve(bytes, bytes / 4);
    *out = reinterpret_cast<T *>(c->srch[slot].get());
    return rc;
}

// The utterances of a whole-utterance entry point: offsets from 0 that never decrease, and scores wherever
// there are frames.
static inline int ctx_check_utts(const char *fn, const int32_t *utt_off, int32_t n_utt, const void *senscr)
{
    const int rc = psb_check_utt_off(fn, utt_off, n_utt);
    if (rc) return rc;
    PSB_REQUIRE(senscr || utt_off[n_utt] == 0, "%s: scores missing", fn);
    return PSB_OK;
}

// hmm_init of n non-multiplexed HMMs (hmm.c:99-102): HMM i = (ssid[i], tmatid[i]) gets the senone ids of
// its senone sequence, state s at senid[i * hmm_stride + s * state_stride].
static inline int ctx_senids(const psb_hmmctx_t *c, const char *what, int n, const int32_t *ssid, const int32_t *tmatid,
                             uint16_t *senid, size_t hmm_stride, size_t state_stride)
{
    const int N = c->n_emit;
    for (int i = 0; i < n; ++i) {
        PSB_REQUIRE(ssid[i] >= 0 && ssid[i] < c->n_sseq, "%s: ssid[%d] = %d out of range", what, i, ssid[i]);
        PSB_REQUIRE(tmatid[i] >= 0 && tmatid[i] < c->n_tmat, "%s: tmatid[%d] = %d out of range", what, i, tmatid[i]);
        for (int s = 0; s < N; ++s) {
            const uint16_t v = c->h_sseq[(size_t)ssid[i] * N + s];
            PSB_REQUIRE(v < c->n_sen, "%s: senone id %d out of range", what, v);
            senid[i * hmm_stride + s * state_stride] = v;
        }
    }
    return PSB_OK;
}

struct CtxCopy {
    void *dst;
    const void *src;
    size_t bytes;
};

// The end of a whole-utterance entry point, after its launches (made only when e was cudaSuccess): count
// them, copy the results back to the host, wait for the stream -- also after an error, so that the next
// call finds it idle -- and turn a CUDA error into a message naming fn.
static inline int ctx_finish(psb_hmmctx_t *c, const char *fn, cudaError_t e, int launches, std::initializer_list<CtxCopy> out)
{
    if (e == cudaSuccess) {
        g_psb_launches.fetch_add(launches, std::memory_order_relaxed);
        e = cudaGetLastError();
    }
    for (const CtxCopy &o : out)
        if (e == cudaSuccess && o.bytes) e = cudaMemcpyAsync(o.dst, o.src, o.bytes, cudaMemcpyDeviceToHost, c->stream);
    const cudaError_t s = cudaStreamSynchronize(c->stream);
    if (e == cudaSuccess) e = s;
    if (e != cudaSuccess) {
        psb_set_error("%s: %s", fn, cudaGetErrorString(e));
        return PSB_ERR_CUDA;
    }
    return PSB_OK;
}
