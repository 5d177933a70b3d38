// psb_search.cu -- the search modules that run whole utterances on the device: grammar decoding
// (fsg_search.c) and both passes of n-gram decoding (ngram_search_fwdtree.c, ngram_search_fwdflat.c).
// The kernels are thin shells around phase code shared with the host emulation harnesses under
// tests/emul/ (psb_fsg_core.h, psb_ngs_core.h, psb_ngf_core.h).
#include "psb_hmmctx.cuh"

#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

// ---------------------------------------------------------------------------------------
// Grammar decoding: fsg_search.c for whole batches (SURVEY 8 row f-1, the lextree search that is
// small enough to live entirely on the device).  One CTA per utterance; the phases and the
// reasoning that makes them equal to the reference's list walks are in psb_fsg_core.h, which a host
// harness (tests/emul/) runs against the reference's golden history tables.  HMM state and the
// per-frame scratch live in global memory (L2-resident: ~80 KB per utterance for a 250-node
// lextree); only the frame scalars are in shared memory.
#include "psb_fsg_host.h"

namespace {

struct FsgDevEval {
    HmmCtxDev c;
    const uint16_t *senid_g;
    const int32_t *tmatid_g;
    const int16_t *row;
    int P;
    __device__ __forceinline__ int operator()(const FsgWork &W, int p) const
    {
        const HmmSoA<> V{W.score, W.hist, W.out_score, W.out_hist, W.best, P};
        const int N = c.n_emit;
        HmmReg h;
        V.load(h, p, N, senid_g + (size_t)p * N, 1);
        const int b = hmm_step(h, c, tmatid_g[p], false, row);
        V.store(h, p, N);
        return b;
    }
};

constexpr int SRCH_THREADS = 128;
constexpr int FSG_THREADS = SRCH_THREADS;

__global__ void __launch_bounds__(FSG_THREADS)
fsg_search_kernel(const int16_t *__restrict__ senscr, const int32_t *__restrict__ utt_off, HmmCtxDev c, FsgGraph G,
                  const uint16_t *__restrict__ senid_g, const int32_t *__restrict__ tmatid_g,
                  int32_t *work, size_t work_words, int32_t *hist_out, int cap, int32_t *n_hist)
{
    __shared__ FsgScalars S;
    const int u = (int)blockIdx.x;
    const long long f0 = utt_off[u];
    const int T = utt_off[u + 1] - utt_off[u];
    FsgWork W;
    fsg_work_carve(work + (size_t)u * work_words, G, W);
    W.hist_out = hist_out + (size_t)u * cap * FSG_ROW;
    W.cap = cap;
    FsgDevEval ev{c, senid_g, tmatid_g, nullptr, G.P};
    fsg_start(G, W, &S);
    for (int f = 0; f < T; ++f) {
        if (S.overflow) break;                               // uniform: written before the last barrier of the step
        ev.row = senscr + (f0 + f) * c.n_sen;
        fsg_step(G, W, &S, f, ev);
    }
    FSG_IF_LEADER n_hist[u] = S.overflow ? -1 : S.n_hist;
}

}  // namespace

static_assert(FSG_WORST_SCORE == PSB_WORST_SCORE, "score floor");
static_assert(FSG_MAX_NSTATE == PSB_HMM_MAX_NSTATE, "state count");

extern "C" int psb_fsg_batch_device(psb_hmmctx_t *c, const psb_fsg_desc_t *g, const int16_t *d_senscr,
                                    const int32_t *utt_off, int32_t n_utt, int32_t *hist, int32_t cap_per_utt,
                                    int32_t *n_hist)
{
    PSB_REQUIRE(c && g && utt_off && n_utt >= 0 && hist && n_hist && cap_per_utt > 0, "psb_fsg_batch_device: bad argument");
    if (n_utt == 0) return PSB_OK;
    int rc = ctx_check_utts("psb_fsg_batch_device", utt_off, n_utt, d_senscr);
    if (rc) return rc;
    PSB_REQUIRE(g->start_state >= 0 && g->start_state < g->n_state, "psb_fsg_batch_device: start state out of range");
    PSB_REQUIRE(g->silcipid >= 0 && g->silcipid < g->n_ciphone, "psb_fsg_batch_device: silence phone out of range");
    FsgFlat flat;
    std::string err;
    if (fsg_flatten(g->n_pnode, g->pnodes, g->n_state, g->roots, g->n_link, g->links, g->nulloff, g->nullarc,
                    g->n_ciphone, flat, err) != 0) {
        psb_set_error("psb_fsg_batch_device: %s", err.c_str());
        return PSB_ERR_ARG;
    }
    const int N = c->n_emit, P = flat.P;
    PSB_CUDA(cudaSetDevice(c->device));
    std::vector<uint16_t> senid((size_t)P * N);
    rc = ctx_senids(c, "psb_fsg_batch_device (pnodes)", P, flat.ssid.data(), flat.tmatid.data(), senid.data(), N, 1);
    if (rc) return rc;
    // one int32 block: graph | tmatid[P] | utt_off[n_utt+1] | n_hist[n_utt]
    std::vector<int32_t> ibuf(flat.buf);
    const size_t o_tm = ibuf.size();
    ibuf.insert(ibuf.end(), flat.tmatid.begin(), flat.tmatid.end());
    const size_t o_uo = ibuf.size();
    ibuf.insert(ibuf.end(), utt_off, utt_off + n_utt + 1);
    const size_t o_nh = ibuf.size();
    ibuf.resize(o_nh + (size_t)n_utt, 0);
    const size_t work_words = fsg_work_words(flat, N);
    const size_t hist_n = (size_t)n_utt * cap_per_utt * FSG_ROW;
    int32_t *d_i = nullptr, *d_hist = nullptr, *d_work = nullptr;
    uint16_t *d_senid = nullptr;
    rc = srch_reserve(c, 0, ibuf.size(), &d_i);
    if (!rc) rc = srch_reserve(c, 1, hist_n, &d_hist);
    if (!rc) rc = srch_reserve(c, 2, work_words * (size_t)n_utt, &d_work);
    if (!rc) rc = srch_reserve(c, 3, senid.size(), &d_senid);
    if (rc) return rc;
    cudaStream_t st = c->stream;
    cudaError_t e = cudaMemcpyAsync(d_i, ibuf.data(), ibuf.size() * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_senid, senid.data(), senid.size() * 2, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        FsgGraph G;
        memset(&G, 0, sizeof(G));
        fsg_graph_bind(flat, d_i, G);
        G.n_ci = g->n_ciphone; G.n_emit = N; G.silcipid = g->silcipid; G.start_state = g->start_state;
        G.beam = g->beam; G.pbeam = g->pbeam; G.wbeam = g->wbeam; G.maxhmmpf = g->maxhmmpf;
        fsg_search_kernel<<<n_utt, FSG_THREADS, 0, st>>>(d_senscr, d_i + o_uo, dev_ctx(c), G, d_senid, d_i + o_tm, d_work, work_words,
                                                         d_hist, cap_per_utt, d_i + o_nh);
    }
    rc = ctx_finish(c, "psb_fsg_batch_device", e, 1, {{hist, d_hist, hist_n * 4}, {n_hist, d_i + o_nh, (size_t)n_utt * 4}});
    if (rc) return rc;
    for (int u = 0; u < n_utt; ++u)
        PSB_REQUIRE(n_hist[u] >= 0, "psb_fsg_batch_device: scratch overflow in utterance %d (internal)", u);
    return PSB_OK;
}

// ---------------------------------------------------------------------------------------
// N-gram decoding, first pass (ngram_search_fwdtree.c) for whole batches: SURVEY 8 row f-1 proper.
// One CTA per utterance, every utterance against the same lextree / dictionary / LM tables; the
// phases are in psb_ngs_core.h (host-emulated against the reference's backpointer tables by
// tests/emul/ngs_emul.cpp).  All state is in global memory; the backpointer table, the
// right-context score stack and bp_table_idx of every utterance are the outputs.
#include "psb_ngs_host.h"

namespace {

// hmm_vit_eval on channel `ch` of a channel-indexed SoA work area (first and second pass share it):
// multiplexed channels carry their per-state senone sequences in W.mss, the others use G.senid.
template <class GraphT, class WorkT>
struct ChanDevEval {
    HmmCtxDev c;
    const GraphT *G;
    const int16_t *row;
    __device__ __forceinline__ int operator()(const WorkT &W, int ch, bool mpx, int sid = -1) const      // sid: static-table index
    {
        const HmmSoA<> V{W.score, W.hist, W.out_score, W.out_hist, W.best, G->M};
        const int N = c.n_emit;
        if (sid < 0) sid = ch;
        HmmReg h;
        V.load(h, ch, N, G->senid + (size_t)sid * N, 1, mpx ? W.mss : nullptr);
        const int b = hmm_step(h, c, G->tmatid[sid], mpx, row);
        V.store(h, ch, N, mpx ? W.mss : nullptr);
        return b;
    }
};
typedef ChanDevEval<NgsGraph, NgsWork> NgsDevEval;

constexpr int NGS_THREADS = SRCH_THREADS;

__global__ void __launch_bounds__(NGS_THREADS)
ngs_fwdtree_kernel(const int16_t *__restrict__ senscr, const int32_t *__restrict__ utt_off, HmmCtxDev c, NgsGraph G,
                   int32_t *work, size_t work_words, const int32_t *pen, int pl_window, int32_t *bp_out, int bp_cap, int32_t *bss_out,
                   int bss_cap, int32_t *bp_idx_out, int32_t *result /* [n_utt][3]: bpidx, bss_head, frames done (or -error) */)
{
    __shared__ NgsScalars S;
    const int u = (int)blockIdx.x;
    const long long f0 = utt_off[u];
    const int T = utt_off[u + 1] - utt_off[u];
    NgsWork W;
    ngs_work_carve(work + (size_t)u * work_words, G, W);
    W.bp = bp_out + (size_t)u * bp_cap * NGS_BP_ROW;
    W.bss = bss_out + (size_t)u * bss_cap;
    W.bp_idx = bp_idx_out + f0 + u;                          // T + 1 slots per utterance
    W.pen = pen ? pen + (size_t)f0 * G.n_ci : nullptr;
    W.pl_window = pl_window; W.T = T;
    W.bp_cap = bp_cap; W.bss_cap = bss_cap;
    NgsDevEval ev{c, &G, nullptr};
    ngs_start(G, W, &S);
    for (int f = 0; f < T; ++f) {
        if (S.stop || S.error) break;                        // uniform: set before a barrier
        ev.row = senscr + (f0 + f) * c.n_sen;
        ngs_step(G, W, &S, f, ev);
    }
    FSG_SYNC();
    FSG_IF_LEADER {
        W.bp_idx[S.n_done] = S.bpidx;                        // ngram_fwdtree_finish :1507
        result[u * 3] = S.bpidx; result[u * 3 + 1] = S.bss_head; result[u * 3 + 2] = S.error ? -S.error : S.n_done;
    }
}

}  // namespace

extern "C" int psb_ngram_fwdtree_batch_device(psb_hmmctx_t *c, const psb_ngram_desc_t *g, const int16_t *d_senscr,
                                              const int32_t *d_pen, int32_t pl_window, const int32_t *utt_off, int32_t n_utt, int32_t *bp,
                                              int32_t bp_cap_per_utt, int32_t *bss, int32_t bss_cap_per_utt,
                                              int32_t *bp_idx, int32_t *result)
{
    PSB_REQUIRE(c && g && g->info && g->model && g->ci_tmat && utt_off && n_utt >= 0 && bp && bss && bp_idx && result &&
                bp_cap_per_utt > 0 && bss_cap_per_utt > 0, "psb_ngram_fwdtree_batch_device: bad argument");
    if (n_utt == 0) return PSB_OK;
    int rc = ctx_check_utts("psb_ngram_fwdtree_batch_device", utt_off, n_utt, d_senscr);
    if (rc) return rc;
    PSB_REQUIRE(pl_window >= 0, "psb_ngram_fwdtree_batch_device: negative look-ahead window");
    PSB_CUDA(cudaSetDevice(c->device));
    const int N = c->n_emit;
    NgsFlat flat;
    std::string err;
    if (ngs_flatten(g->info, g->model, (long long)g->model_len, g->lm_arrays, (long long)g->lm_arrays_len, g->ci_tmat, c->h_sseq.data(), c->n_sseq, N, c->n_tmat, c->n_sen, flat, err) != 0) {
        psb_set_error("psb_ngram_fwdtree_batch_device: %s", err.c_str());
        return PSB_ERR_ARG;
    }
    std::vector<int32_t> ibuf(flat.buf);
    const size_t o_uo = ibuf.size();
    ibuf.insert(ibuf.end(), utt_off, utt_off + n_utt + 1);
    const size_t o_res = ibuf.size();
    ibuf.resize(o_res + (size_t)n_utt * 3, 0);
    const size_t work_words = ngs_work_words(flat.G);
    const size_t total_frames = (size_t)utt_off[n_utt];
    const size_t n_bp = (size_t)n_utt * bp_cap_per_utt * NGS_BP_ROW, n_bss = (size_t)n_utt * bss_cap_per_utt,
                 n_idx = total_frames + (size_t)n_utt;
    int32_t *d_i = nullptr, *d_work = nullptr, *d_bp = nullptr, *d_bss = nullptr, *d_idx = nullptr;
    rc = srch_reserve(c, 0, ibuf.size(), &d_i);
    if (!rc) rc = srch_reserve(c, 1, work_words * (size_t)n_utt, &d_work);
    if (!rc) rc = srch_reserve(c, 2, n_bp, &d_bp);
    if (!rc) rc = srch_reserve(c, 3, n_bss, &d_bss);
    if (!rc) rc = srch_reserve(c, 4, n_idx, &d_idx);
    if (rc) return rc;
    cudaStream_t st = c->stream;
    cudaError_t e = cudaMemcpyAsync(d_i, ibuf.data(), ibuf.size() * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_idx, 0, n_idx * 4, st);
    if (e == cudaSuccess) {
        ngs_bind(flat, d_i);
        ngs_fwdtree_kernel<<<n_utt, NGS_THREADS, 0, st>>>(d_senscr, d_i + o_uo, dev_ctx(c), flat.G, d_work, work_words, d_pen, pl_window,
                                                          d_bp, bp_cap_per_utt, d_bss, bss_cap_per_utt, d_idx, d_i + o_res);
    }
    rc = ctx_finish(c, "psb_ngram_fwdtree_batch_device", e, 1,
                    {{bp, d_bp, n_bp * 4}, {bss, d_bss, n_bss * 4}, {bp_idx, d_idx, n_idx * 4}, {result, d_i + o_res, (size_t)n_utt * 12}});
    if (rc) return rc;
    for (int u = 0; u < n_utt; ++u) {
        PSB_REQUIRE(result[u * 3 + 2] != -1, "psb_ngram_fwdtree_batch_device: utterance %d overflowed the backpointer table "
                    "or the score stack (%d entries / %d scores allowed)", u, bp_cap_per_utt, bss_cap_per_utt);
        PSB_REQUIRE(result[u * 3 + 2] != -3, "psb_ngram_fwdtree_batch_device: utterance %d ran out of fan-out blocks "
                    "(PSB_NGS_BLOCKS)", u);
        PSB_REQUIRE(result[u * 3 + 2] >= 0, "psb_ngram_fwdtree_batch_device: utterance %d: internal error (search status %d)",
                    u, result[u * 3 + 2]);
    }
    return PSB_OK;
}

// ---------------------------------------------------------------------------------------
// N-gram decoding, second pass (ngram_search_fwdflat.c) for whole batches: SURVEY 8 row f-4.  One
// CTA per utterance, one thread per active word (psb_ngf_core.h, host-emulated against the
// reference's second-pass backpointer tables by tests/emul/ngf_emul.cpp).  Input: every
// utterance's first-pass backpointer table (from psb_ngram_fwdtree_batch_device or the host).
#include "psb_ngf_host.h"

namespace {

typedef ChanDevEval<NgfGraph, NgfWork> NgfDevEval;

__global__ void __launch_bounds__(NGS_THREADS)
ngs_fwdflat_kernel(const int16_t *__restrict__ senscr, const int32_t *__restrict__ utt_off, HmmCtxDev c, NgfGraph G,
                   int32_t *work, size_t work_words, const int32_t *bp_in, int in_cap, const int32_t *n_in, int n_in_stride,
                   int32_t *bp_out, int bp_cap, int32_t *bss_out, int bss_cap, int32_t *bp_idx_out, int32_t *result)
{
    __shared__ NgfScalars S;
    const int u = (int)blockIdx.x;
    const long long f0 = utt_off[u];
    const int T = utt_off[u + 1] - utt_off[u];
    NgfWork W;
    ngf_work_carve(work + (size_t)u * work_words, G, T, in_cap, W);
    W.bp = bp_out + (size_t)u * bp_cap * NGS_BP_ROW;
    W.bss = bss_out + (size_t)u * bss_cap;
    W.bp_idx = bp_idx_out + f0 + u;
    W.bp_in = bp_in + (size_t)u * in_cap * NGS_BP_ROW;
    W.n_bp_in = n_in[(size_t)u * n_in_stride];
    if (W.n_bp_in > in_cap) W.n_bp_in = 0;                      // (negative: no first pass, -fwdtree no)
    W.bp_cap = bp_cap; W.bss_cap = bss_cap;
    NgfDevEval ev{c, &G, nullptr};
    ngf_start(G, W, &S);
    for (int f = 0; f < T; ++f) {
        if (S.stop || S.error) break;
        ev.row = senscr + (f0 + f) * c.n_sen;
        ngf_step(G, W, &S, f, ev);
    }
    FSG_SYNC();
    FSG_IF_LEADER {
        W.bp_idx[S.n_done] = S.bpidx;                        // ngram_fwdflat_finish :937
        result[u * 3] = S.bpidx; result[u * 3 + 1] = S.bss_head; result[u * 3 + 2] = S.error ? -S.error : S.n_done;
    }
}

}  // namespace

extern "C" int psb_ngram_fwdflat_batch_device(psb_hmmctx_t *c, const psb_ngram_desc_t *g, const int16_t *d_senscr,
                                              const int32_t *utt_off, int32_t n_utt, const int32_t *bp_first,
                                              int32_t first_cap_per_utt, const int32_t *n_first, int32_t *bp,
                                              int32_t bp_cap_per_utt, int32_t *bss, int32_t bss_cap_per_utt,
                                              int32_t *bp_idx, int32_t *result)
{
    PSB_REQUIRE(c && g && g->info && g->model && g->ci_tmat && g->ci_ssid && utt_off && n_utt >= 0 && bp_first && n_first && bp &&
                bss && bp_idx && result && first_cap_per_utt > 0 && bp_cap_per_utt > 0 && bss_cap_per_utt > 0,
                "psb_ngram_fwdflat_batch_device: bad argument (the descriptor needs ci_ssid for this pass)");
    if (n_utt == 0) return PSB_OK;
    int rc = ctx_check_utts("psb_ngram_fwdflat_batch_device", utt_off, n_utt, d_senscr);
    if (rc) return rc;
    int t_max = 0;
    for (int u = 0; u < n_utt; ++u) {
        PSB_REQUIRE(n_first[u] >= -1 && n_first[u] <= first_cap_per_utt, "psb_ngram_fwdflat_batch_device: n_first[%d] out of range", u);
        const int32_t *b = bp_first + (size_t)u * first_cap_per_utt * NGS_BP_ROW;
        const int T = utt_off[u + 1] - utt_off[u];
        for (int i = 0; i < n_first[u]; ++i) {
            const int32_t *r = b + (size_t)i * NGS_BP_ROW;
            PSB_REQUIRE(r[3] >= -1 && r[3] < i && r[2] >= 0 && r[2] < g->info[1] && r[0] >= 0 && r[0] < (T > 0 ? T : 1),
                        "psb_ngram_fwdflat_batch_device: utterance %d: first-pass entry %d is inconsistent", u, i);
        }
        if (T > t_max) t_max = T;
    }
    PSB_CUDA(cudaSetDevice(c->device));
    const int N = c->n_emit;
    NgfFlat flat;
    std::string err;
    if (ngf_flatten(g->info, g->model, (long long)g->model_len, g->lm_arrays, (long long)g->lm_arrays_len, g->ci_tmat, g->ci_ssid, c->h_sseq.data(), c->n_sseq, N, c->n_tmat, c->n_sen, flat, err) != 0) {
        psb_set_error("psb_ngram_fwdflat_batch_device: %s", err.c_str());
        return PSB_ERR_ARG;
    }
    std::vector<int32_t> ibuf(flat.buf);
    const size_t o_uo = ibuf.size();
    ibuf.insert(ibuf.end(), utt_off, utt_off + n_utt + 1);
    const size_t o_nin = ibuf.size();
    ibuf.insert(ibuf.end(), n_first, n_first + n_utt);
    const size_t o_res = ibuf.size();
    ibuf.resize(o_res + (size_t)n_utt * 3, 0);
    const size_t work_words = ngf_work_words(flat.G, t_max, first_cap_per_utt);
    const size_t total_frames = (size_t)utt_off[n_utt];
    const size_t n_in = (size_t)n_utt * first_cap_per_utt * NGS_BP_ROW, n_bp = (size_t)n_utt * bp_cap_per_utt * NGS_BP_ROW,
                 n_bss = (size_t)n_utt * bss_cap_per_utt, n_idx = total_frames + (size_t)n_utt;
    int32_t *d_i = nullptr, *d_work = nullptr, *d_in = nullptr, *d_bp = nullptr, *d_bss = nullptr, *d_idx = nullptr;
    rc = srch_reserve(c, 0, ibuf.size(), &d_i);
    if (!rc) rc = srch_reserve(c, 1, work_words * (size_t)n_utt, &d_work);
    if (!rc) rc = srch_reserve(c, 2, n_in, &d_in);
    if (!rc) rc = srch_reserve(c, 3, n_bp, &d_bp);
    if (!rc) rc = srch_reserve(c, 4, n_bss, &d_bss);
    if (!rc) rc = srch_reserve(c, 5, n_idx, &d_idx);
    if (rc) return rc;
    cudaStream_t st = c->stream;
    cudaError_t e = cudaMemcpyAsync(d_i, ibuf.data(), ibuf.size() * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_in, bp_first, n_in * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_idx, 0, n_idx * 4, st);
    if (e == cudaSuccess) {
        ngf_bind(flat, d_i);
        ngs_fwdflat_kernel<<<n_utt, NGS_THREADS, 0, st>>>(d_senscr, d_i + o_uo, dev_ctx(c), flat.G, d_work, work_words, d_in, first_cap_per_utt,
                                                          d_i + o_nin, 1, d_bp, bp_cap_per_utt, d_bss, bss_cap_per_utt, d_idx, d_i + o_res);
    }
    rc = ctx_finish(c, "psb_ngram_fwdflat_batch_device", e, 1,
                    {{bp, d_bp, n_bp * 4}, {bss, d_bss, n_bss * 4}, {bp_idx, d_idx, n_idx * 4}, {result, d_i + o_res, (size_t)n_utt * 12}});
    if (rc) return rc;
    for (int u = 0; u < n_utt; ++u) {
        PSB_REQUIRE(result[u * 3 + 2] != -1, "psb_ngram_fwdflat_batch_device: utterance %d overflowed the backpointer table "
                    "or the score stack (%d entries / %d scores allowed)", u, bp_cap_per_utt, bss_cap_per_utt);
        PSB_REQUIRE(result[u * 3 + 2] != -3, "psb_ngram_fwdflat_batch_device: utterance %d: its vocabulary does not fit the state "
                    "area (PSB_NGF_CHANNELS)", u);
        PSB_REQUIRE(result[u * 3 + 2] >= 0, "psb_ngram_fwdflat_batch_device: utterance %d: internal error (search status %d)",
                    u, result[u * 3 + 2]);
    }
    return PSB_OK;
}

// Both passes back to back, the first pass's tables staying on the device (ngram_search_finish :781-820:
// fwdtree, acmod_rewind, fwdflat over the same frames).  Only the second pass's tables come back, plus
// the first pass's entry counts for diagnostics.
extern "C" int psb_ngram_two_pass_batch_device(psb_hmmctx_t *c, const psb_ngram_desc_t *g, const int16_t *d_senscr,
                                               const int32_t *d_pen, int32_t pl_window, const int32_t *utt_off, int32_t n_utt,
                                               int32_t first_cap_per_utt, int32_t first_bss_cap_per_utt, int32_t *bp,
                                               int32_t bp_cap_per_utt, int32_t *bss, int32_t bss_cap_per_utt, int32_t *bp_idx,
                                               int32_t *result, int32_t *first_result)
{
    PSB_REQUIRE(c && g && g->info && g->model && g->ci_tmat && g->ci_ssid && utt_off && n_utt >= 0 && bp && bss && bp_idx && result &&
                first_cap_per_utt > 0 && first_bss_cap_per_utt > 0 && bp_cap_per_utt > 0 && bss_cap_per_utt > 0 && pl_window >= 0,
                "psb_ngram_two_pass_batch_device: bad argument");
    if (n_utt == 0) return PSB_OK;
    int rc = ctx_check_utts("psb_ngram_two_pass_batch_device", utt_off, n_utt, d_senscr);
    if (rc) return rc;
    int t_max = 0;
    for (int u = 0; u < n_utt; ++u)
        if (utt_off[u + 1] - utt_off[u] > t_max) t_max = utt_off[u + 1] - utt_off[u];
    PSB_CUDA(cudaSetDevice(c->device));
    const int N = c->n_emit;
    NgsFlat f1;
    NgfFlat f2;
    std::string err;
    if (ngs_flatten(g->info, g->model, (long long)g->model_len, g->lm_arrays, (long long)g->lm_arrays_len, g->ci_tmat, c->h_sseq.data(), c->n_sseq, N, c->n_tmat, c->n_sen, f1, err) != 0 ||
        ngf_flatten(g->info, g->model, (long long)g->model_len, g->lm_arrays, (long long)g->lm_arrays_len, g->ci_tmat, g->ci_ssid, c->h_sseq.data(), c->n_sseq, N, c->n_tmat, c->n_sen, f2, err) != 0) {
        psb_set_error("psb_ngram_two_pass_batch_device: %s", err.c_str());
        return PSB_ERR_ARG;
    }
    // one int32 block: first-pass graph | second-pass graph | utt_off | result1 [n_utt][3] | result2 [n_utt][3]
    std::vector<int32_t> ibuf(f1.buf);
    const size_t o_g2 = ibuf.size();
    ibuf.insert(ibuf.end(), f2.buf.begin(), f2.buf.end());
    const size_t o_uo = ibuf.size();
    ibuf.insert(ibuf.end(), utt_off, utt_off + n_utt + 1);
    const size_t o_r1 = ibuf.size();
    ibuf.resize(o_r1 + (size_t)n_utt * 6, 0);
    const size_t o_r2 = o_r1 + (size_t)n_utt * 3;
    const size_t ww1 = ngs_work_words(f1.G), ww2 = ngf_work_words(f2.G, t_max, first_cap_per_utt), ww = ww1 > ww2 ? ww1 : ww2;
    const size_t total_frames = (size_t)utt_off[n_utt], n_idx = total_frames + (size_t)n_utt;
    const size_t n_bp1 = (size_t)n_utt * first_cap_per_utt * NGS_BP_ROW, n_bss1 = (size_t)n_utt * first_bss_cap_per_utt,
                 n_bp2 = (size_t)n_utt * bp_cap_per_utt * NGS_BP_ROW, n_bss2 = (size_t)n_utt * bss_cap_per_utt;
    int32_t *d_i = nullptr, *d_work = nullptr, *d_bp1 = nullptr, *d_bss1 = nullptr, *d_idx1 = nullptr, *d_bp2 = nullptr, *d_bss2 = nullptr,
            *d_idx2 = nullptr;
    rc = srch_reserve(c, 0, ibuf.size(), &d_i);
    if (!rc) rc = srch_reserve(c, 1, ww * (size_t)n_utt, &d_work);
    if (!rc) rc = srch_reserve(c, 2, n_bp1, &d_bp1);
    if (!rc) rc = srch_reserve(c, 3, n_bss1, &d_bss1);
    if (!rc) rc = srch_reserve(c, 4, n_idx, &d_idx1);
    if (!rc) rc = srch_reserve(c, 5, n_bp2, &d_bp2);
    if (!rc) rc = srch_reserve(c, 6, n_bss2, &d_bss2);
    if (!rc) rc = srch_reserve(c, 7, n_idx, &d_idx2);
    if (rc) return rc;
    cudaStream_t st = c->stream;
    cudaError_t e = cudaMemcpyAsync(d_i, ibuf.data(), ibuf.size() * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_idx1, 0, n_idx * 4, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_idx2, 0, n_idx * 4, st);
    if (e == cudaSuccess) {
        ngs_bind(f1, d_i);
        ngf_bind(f2, d_i + o_g2);
        ngs_fwdtree_kernel<<<n_utt, NGS_THREADS, 0, st>>>(d_senscr, d_i + o_uo, dev_ctx(c), f1.G, d_work, ww, d_pen, pl_window, d_bp1,
                                                          first_cap_per_utt, d_bss1, first_bss_cap_per_utt, d_idx1, d_i + o_r1);
        ngs_fwdflat_kernel<<<n_utt, NGS_THREADS, 0, st>>>(d_senscr, d_i + o_uo, dev_ctx(c), f2.G, d_work, ww, d_bp1, first_cap_per_utt,
                                                          d_i + o_r1, 3, d_bp2, bp_cap_per_utt, d_bss2, bss_cap_per_utt, d_idx2, d_i + o_r2);
    }
    std::vector<int32_t> r1((size_t)n_utt * 3);
    rc = ctx_finish(c, "psb_ngram_two_pass_batch_device", e, 2,
                    {{bp, d_bp2, n_bp2 * 4}, {bss, d_bss2, n_bss2 * 4}, {bp_idx, d_idx2, n_idx * 4},
                     {result, d_i + o_r2, (size_t)n_utt * 12}, {r1.data(), d_i + o_r1, (size_t)n_utt * 12}});
    if (rc) return rc;
    if (first_result) memcpy(first_result, r1.data(), r1.size() * 4);
    for (int u = 0; u < n_utt; ++u) {
        PSB_REQUIRE(r1[(size_t)u * 3 + 2] != -1, "psb_ngram_two_pass_batch_device: utterance %d: first pass overflowed its tables (%d entries / %d scores)",
                    u, first_cap_per_utt, first_bss_cap_per_utt);
        PSB_REQUIRE(result[u * 3 + 2] != -1, "psb_ngram_two_pass_batch_device: utterance %d: second pass overflowed its tables (%d entries / %d scores)",
                    u, bp_cap_per_utt, bss_cap_per_utt);
        PSB_REQUIRE(r1[(size_t)u * 3 + 2] != -3 && result[u * 3 + 2] != -3, "psb_ngram_two_pass_batch_device: utterance %d ran out of fan-out blocks "
                    "(PSB_NGS_BLOCKS) or state channels (PSB_NGF_CHANNELS)", u);
        PSB_REQUIRE(r1[(size_t)u * 3 + 2] >= 0 && result[u * 3 + 2] >= 0,
                    "psb_ngram_two_pass_batch_device: utterance %d: internal error (search status %d in the first pass, %d in "
                    "the second)", u, r1[(size_t)u * 3 + 2], result[u * 3 + 2]);
    }
    return PSB_OK;
}

// ---------------------------------------------------------------------------------------
// Self-test hook for the one building block of the search kernels that host emulation cannot run:
// the block-wide exclusive scan (fsg_exscan, psb_fsg_core.h).  One CTA scans a[0..n) in place.
namespace {
__global__ void __launch_bounds__(NGS_THREADS)
exscan_selftest_kernel(int32_t *a, int n, int32_t *total)
{
    __shared__ int scan[34];
    const int t = fsg_exscan(a, n, scan);
    const int t2 = fsg_exscan(a + n, 0, scan);               // an empty scan right behind it (scan[33] reuse)
    if (threadIdx.x == blockDim.x - 1) { total[0] = t; total[1] = t2; }
}
}  // namespace

extern "C" int psb_selftest_block_scan(int device, int32_t *a, int32_t n, int32_t *total)
{
    PSB_REQUIRE(a && total && n >= 0, "psb_selftest_block_scan: bad argument");
    PSB_CUDA(cudaSetDevice(device));
    DevBuf<int32_t> d;
    const int rc = d.reserve((size_t)n + 2);
    if (rc) return rc;
    cudaError_t e = cudaMemcpy(d, a, (size_t)n * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        exscan_selftest_kernel<<<1, NGS_THREADS>>>(d, n, d + n);
        g_psb_launches.fetch_add(1, std::memory_order_relaxed);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(a, d, (size_t)n * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(total, d + n, 8, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) {
        psb_set_error("psb_selftest_block_scan: %s", cudaGetErrorString(e));
        return PSB_ERR_CUDA;
    }
    return PSB_OK;
}
