// psb_apn_core.h -- phone decoding over a PHMM net given in the reference's factored form
// (allphone_search.c with -allphone_ci no or yes), one utterance as a sequence of block-wide,
// data-parallel phases.
//
// phmm_link (allphone_search.c:167-215) links p -> p2 exactly when ci(p2) is in rc(p) and ci(p) is
// in lc(p2).  The net is therefore given per node as (ssid, tmatid, ci, lc, rc) with 64-bit context
// masks, in the order of ci_phmm[] (ci-major, list order), which is the order phmm_exit numbers
// history entries in.  No link list is walked:
//
//  * phmm_eval_all (:349-376) and phmm_exit (:378-467): every node active in the frame is
//    evaluated; those inside pbeam append a history entry, numbered in node order by a block
//    scan, the others are cleared.  With a phone LM the entry's tscore reads the SAME entry as
//    pred and pred_pred (:417-444); it is not stored but recomputed where it is needed.
//  * phmm_trans (:469-523) enters target p2 with the FIRST maximum, in history order, of
//    out_score + tscore over its exited predecessors, if that beats the beam and p2's state-0
//    score.  The first maximum is the lexicographic max of (score, -history index), which is
//    associative, and a predecessor's candidate for p2 depends on p2 only through ci(p2) (no LM:
//    out_score + inspen; LM: out_score + tg[pci][ci(p)][ci(p2)] or bg[ci(p)][ci(p2)], pci the CI
//    phone of p's own predecessor entry).  So each frame builds an n_ci x n_ci class table:
//    M[a][b] = lexmax over exited p with ci(p) = a and b in rc(p) -- an atomic max of the score,
//    then an atomic min of the index among the entries that reach it -- and each target takes the
//    lexmax of M[a][ci(p2)] over a in lc(p2).  The beam and the state-0 tests are monotone, so
//    applying them after the max is the same as applying them link by link.
//  * allphone_backtrace (:774-837): the best entry of the last frame that has entries (strict >
//    scanning down: the highest index among equal scores; entry 0 never counts), then the chain
//    of predecessors down to entry 0, which is never emitted.
//
// The same source is compiled by nvcc into allphone_net_kernel (psb_hmm.cu) and by g++ into a TEST
// harness (tests/emul/apn_emul.cpp), which runs the phases one "thread" at a time in ascending or
// descending order, with the race check of psb_fsg_racecheck.h when asked.
#pragma once
#include "psb_fsg_core.h"

#if defined(__CUDACC__) && !defined(PSB_FSG_HOST_EMUL)
#define APN_CTZ64(m) (__ffsll((long long)(m)) - 1)
#define APN_RAW(a) (a)
#else
#define APN_CTZ64(m) __builtin_ctzll(m)
#define APN_RAW(a) FSG_RAW(a)
#endif

#define APN_ROW 4               // history row: ef, node, predecessor entry, score
#define APN_NONE INT_MAX        // class-table entry no exited node reaches
#define APN_SEG 5               // segment: ci, sf, ef, score, tscore

// The net and the search parameters, read-only, shared by every utterance.
struct ApnNet {
    int H, n_ci, n_emit, start;
    int beam, pbeam, inspen;
    const int32_t *ci;              // [H]
    const unsigned long long *lc;   // [H] bit a: a predecessor of CI phone a may enter this node
    const unsigned long long *rc;   // [H] bit b: this node may enter nodes of CI phone b
    const int32_t *bg, *tg;         // phone LM (nullptr: none): [n_ci][n_ci], [n_ci][n_ci][n_ci]
};

// Per-utterance state in global memory; msc / mix may live in shared memory.
struct ApnWork {
    fsg_wp score, hist;                          // [n_emit][H]
    fsg_wp out_score, out_hist, best, frame;     // [H]
    fsg_wp ex;                                   // [H] exit flag, then the history index of this frame's entry or -1
    fsg_wp pci;                                  // [H] CI phone of the predecessor of this frame's entry, or -1
    fsg_wp msc, mix;                             // [n_ci * n_ci] the frame's class table
    fsg_wp hist_out;                             // [cap][APN_ROW]
    int cap;
};

struct ApnScalars {
    fsg_int best, n_hist, last_start, overflow, bt_score, bt_idx;
    int scan[34];
};

// Words of global scratch per utterance (score, hist, out_score, out_hist, best, frame, ex, pci).
FSG_HDH size_t apn_work_words(int H, int n_emit) { return (size_t)(2 * n_emit + 6) * (size_t)H; }

FSG_HD void apn_work_carve(int32_t *b, const ApnNet &G, ApnWork &W)
{
    const size_t H = (size_t)G.H, N = (size_t)G.n_emit;
    W.score = b; b += N * H;  W.hist = b; b += N * H;
    W.out_score = b; b += H;  W.out_hist = b; b += H;  W.best = b; b += H;  W.frame = b; b += H;
    W.ex = b; b += H;  W.pci = b;
}

#if defined(__CUDACC__) && !defined(PSB_FSG_HOST_EMUL)
// In-place exclusive scan of a[0..n) by the whole block, one contiguous chunk per thread (n is
// tens of thousands: one pass, two barriers); returns the total to every thread.
__device__ inline int apn_exscan(fsg_wp a, int n, int *scan /* [34], shared */)
{
    const int tid = (int)threadIdx.x, nt = (int)blockDim.x, lane = tid & 31, w = tid >> 5;
    const int chunk = (n + nt - 1) / nt, c0 = min(n, tid * chunk), c1 = min(n, c0 + chunk);
    int cnt = 0;
    for (int i = c0; i < c1; ++i) cnt += a[i];
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) scan[w] = incl;
    __syncthreads();
    int base = 0, total = 0;
    for (int j = 0; j < (nt >> 5); ++j) {
        if (j < w) base += scan[j];
        total += scan[j];
    }
    int run = base + incl - cnt;
    for (int i = c0; i < c1; ++i) { const int v = a[i]; a[i] = run; run += v; }
    __syncthreads();                                  // scan[] is reused by the next call
    return total;
}
#else
static inline int apn_exscan(fsg_wp a, int n, int *scan)
{
    int run = 0;
    (void)scan;
    FSG_COLLECTIVE_BEGIN();
    for (int i = 0; i < n; ++i) { const int v = APN_RAW(a)[i]; APN_RAW(a)[i] = run; run += v; }
    FSG_COLLECTIVE_END();
    return run;
}
#endif

FSG_HD void apn_clear_node(const ApnNet &G, const ApnWork &W, int p)        /* hmm_clear, hmm.c:180-196 */
{
    for (int s = 0; s < G.n_emit; ++s) { W.score[s * G.H + p] = FSG_WORST_SCORE; W.hist[s * G.H + p] = -1; }
    W.out_score[p] = FSG_WORST_SCORE; W.out_hist[p] = -1; W.best[p] = FSG_WORST_SCORE; W.frame[p] = -1;
}

// The tscore phmm_exit gives history entry k (:413-453), from the table itself.
FSG_HDH int apn_entry_tscore(const ApnNet &G, const int32_t *hist_out, int k)
{
    if (!G.bg) return G.inspen;
    const int hh = hist_out[(size_t)k * APN_ROW + 2];
    if (hh <= 0) return 0;
    const int n = G.n_ci, pc = G.ci[hist_out[(size_t)hh * APN_ROW + 1]], c = G.ci[hist_out[(size_t)k * APN_ROW + 1]];
    return hist_out[(size_t)hh * APN_ROW + 2] > 0 ? G.tg[((size_t)pc * n + pc) * n + c] : G.bg[(size_t)pc * n + c];
}

// allphone_search_start (:669-707): every node cleared, the silence node entered with 0.
FSG_HD void apn_start(const ApnNet &G, const ApnWork &W, ApnScalars *S)
{
    FSG_FOR(i, G.H) apn_clear_node(G, W, i);
    FSG_SYNC();
    FSG_IF_LEADER {
        W.score[G.start] = 0; W.hist[G.start] = 0; W.frame[G.start] = 0;
        S->best = FSG_WORST_SCORE; S->n_hist = 0; S->last_start = 0; S->overflow = 0;
    }
    FSG_SYNC();
}

// phmm_trans's candidate of exited node p for targets of CI phone b.
FSG_HD int apn_cand(const ApnNet &G, const ApnWork &W, int p, int a, int b)
{
    if (!G.bg) return W.out_score[p] + G.inspen;
    const int n = G.n_ci, pc = W.pci[p];
    return W.out_score[p] + (pc >= 0 ? G.tg[((size_t)pc * n + a) * n + b] : G.bg[(size_t)a * n + b]);
}

// allphone_search_step (:727-748) for frame t.  Eval(W, p) runs hmm_vit_eval on node p against this
// frame's senone scores and returns its best score.
template <class Eval>
FSG_HD void apn_step(const ApnNet &G, const ApnWork &W, ApnScalars *S, int t, Eval &ev)
{
    const int H = G.H, n = G.n_ci, nf = t + 1;
    FSG_FOR(i, H) {                                                          // phmm_eval_all
        if (W.frame[i] == t) {
            const int b = ev(W, i);
            FSG_ATOMIC_MAX(&S->best, b);
        }
    }
    FSG_SYNC();
    const int best = S->best, th = best + G.pbeam, nh0 = S->n_hist;
    FSG_FOR(i, H) W.ex[i] = (W.frame[i] == t && W.best[i] >= th) ? 1 : 0;   // phmm_exit: numbering
    FSG_SYNC();
    const int n_new = apn_exscan(W.ex, H, S->scan);
    FSG_FOR(i, H) {                                                          // phmm_exit: entries
        if (W.frame[i] != t) { W.ex[i] = -1; continue; }
        if (W.best[i] >= th) {
            const int k = nh0 + W.ex[i], hh = W.out_hist[i];
            if (G.bg) W.pci[i] = hh > 0 ? G.ci[W.hist_out[(size_t)hh * APN_ROW + 1]] : -1;
            if (k < W.cap) {
                W.hist_out[(size_t)k * APN_ROW + 0] = t; W.hist_out[(size_t)k * APN_ROW + 1] = i;
                W.hist_out[(size_t)k * APN_ROW + 2] = hh; W.hist_out[(size_t)k * APN_ROW + 3] = W.out_score[i];
            }
            W.ex[i] = k;
            W.frame[i] = nf;
        }
        else {
            apn_clear_node(G, W, i);
            W.ex[i] = -1;
        }
    }
    FSG_FOR(k, n * n) { W.msc[k] = INT_MIN; W.mix[k] = APN_NONE; }
    FSG_IF_LEADER S->best = FSG_WORST_SCORE;
    FSG_SYNC();
    FSG_FOR(i, H) {                                                          // class table: scores
        if (W.ex[i] < 0) continue;
        const int a = G.ci[i];
        for (unsigned long long m = G.rc[i]; m; m &= m - 1) {
            const int b = APN_CTZ64(m);
            FSG_ATOMIC_MAX_AT(W.msc, a * n + b, apn_cand(G, W, i, a, b));
        }
    }
    FSG_IF_LEADER {
        S->n_hist = nh0 + n_new;
        if (n_new > 0) S->last_start = nh0;
        if (nh0 + n_new > W.cap) S->overflow = 1;
    }
    FSG_SYNC();
    FSG_FOR(i, H) {                                                          // class table: first index at the max
        if (W.ex[i] < 0) continue;
        const int a = G.ci[i];
        for (unsigned long long m = G.rc[i]; m; m &= m - 1) {
            const int b = APN_CTZ64(m);
            if (apn_cand(G, W, i, a, b) == W.msc[a * n + b]) FSG_ATOMIC_MIN_AT(W.mix, a * n + b, (int)W.ex[i]);
        }
    }
    FSG_SYNC();
    const int floor_ = best + G.beam;
    FSG_FOR(i, H) {                                                          // phmm_trans, pulled per target
        const int b = G.ci[i];
        int bs = INT_MIN, bi = APN_NONE;
        for (unsigned long long m = G.lc[i]; m; m &= m - 1) {
            const int a = APN_CTZ64(m);
            const int x = W.mix[a * n + b];
            if (x == APN_NONE) continue;
            const int s = W.msc[a * n + b];
            if (s > bs || (s == bs && x < bi)) { bs = s; bi = x; }
        }
        if (bi != APN_NONE && bs > floor_ && bs > W.score[i]) { W.score[i] = bs; W.hist[i] = bi; W.frame[i] = nf; }   // hmm_enter
    }
    FSG_SYNC();
}

// allphone_backtrace (:774-837) over the utterance's table after its last frame.  Writes at most
// seg_cap segments (ci, sf, ef, score, tscore) in time order and returns their number.
FSG_HD int apn_backtrace(const ApnNet &G, const ApnWork &W, ApnScalars *S, int32_t *segs, int seg_cap)
{
    const int nh = S->n_hist;
    const int lo = S->last_start > 1 ? (int)S->last_start : 1;
    FSG_IF_LEADER { S->bt_score = INT_MIN; S->bt_idx = -1; }
    FSG_SYNC();
    FSG_FOR(j, nh - lo) FSG_ATOMIC_MAX(&S->bt_score, (int)W.hist_out[(size_t)(lo + j) * APN_ROW + 3]);
    FSG_SYNC();
    const int bsc = S->bt_score;
    FSG_FOR(j, nh - lo) {
        if (W.hist_out[(size_t)(lo + j) * APN_ROW + 3] == bsc) FSG_ATOMIC_MAX(&S->bt_idx, lo + j);
    }
    FSG_SYNC();
    int n_seg = 0;
    FSG_IF_LEADER {
        const int32_t *h = APN_RAW(W.hist_out);
        int len = 0;
        for (int k = S->bt_idx; k > 0; k = h[(size_t)k * APN_ROW + 2]) ++len;
        int j = len;
        for (int k = S->bt_idx; k > 0; k = h[(size_t)k * APN_ROW + 2]) {
            --j;
            if (j >= seg_cap) continue;
            const int hh = h[(size_t)k * APN_ROW + 2], ts = apn_entry_tscore(G, h, k);
            int32_t *s = segs + (size_t)j * APN_SEG;
            s[0] = G.ci[h[(size_t)k * APN_ROW + 1]];
            s[1] = hh > 0 ? h[(size_t)hh * APN_ROW + 0] + 1 : 0;
            s[2] = h[(size_t)k * APN_ROW + 0];
            s[3] = h[(size_t)k * APN_ROW + 3] - (hh > 0 ? h[(size_t)hh * APN_ROW + 3] : 0) - ts;   // ascore (:750-761)
            s[4] = ts;
        }
        n_seg = len;
    }
    return n_seg;
}
