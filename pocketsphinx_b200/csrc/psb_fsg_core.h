// psb_fsg_core.h -- grammar (FSG) decoding of ONE utterance as a sequence of block-wide,
// data-parallel phases: fsg_search.c + fsg_history.c re-thought for a CTA, not translated.
//
// The reference walks linked lists one node at a time (fsg_search_step, fsg_search.c:683-761);
// every rule below is the closed form of what those sequential walks compute, so that all nodes
// of a phase can be handled at once and the result -- the complete history table -- is identical:
//
//  * active list.  glist_add_ptr PREPENDS, so the reference visits nodes in reverse insertion
//    order.  Lists are kept here in insertion order; "walk position" w = n_act-1-index.
//  * pnode_trans (:410-441).  The lextree under a state is a tree: every non-root pnode has one
//    parent, so "enter the child if the new score beats the beam and its state-0 score" has a
//    single writer per child -- no ties, no atomics.
//  * who inserts a node into the next list (this fixes the next frame's walk order, and through
//    it the order of equal-score word exits -- homophones tie exactly): a surviving node inserts
//    itself at its own walk position unless its parent, standing EARLIER in the walk, entered it
//    first; a parent inserts every child it enters that has not already inserted itself.  Per
//    walk position that is a count; an exclusive block scan turns counts into list offsets.
//  * fsg_history_entry_add (fsg_history.c:132-213) keeps, per (destination state, left context),
//    a list sorted by score (ties: insertion order) in which every entry's right-context set loses
//    the sets of all entries before it, empty ones being dropped.  Whatever the insertion order,
//    the outcome is: rc_final(e) = rc(e) minus the union of rc(e') over all e' of the same group
//    that precede e in (score descending, walk order), and fsg_history_end_frame (:220-240) emits
//    the groups by (state, lc) ascending.  So: one candidate per thread, an O(E^2) sweep for the
//    set difference, another for the rank.  E (word exits in a frame) is tens.
//  * null_prop (:566-614) = the same resolve step over (new entry x null arc) candidates;
//    word_trans (:621-680) is pulled per root: the first maximum over this frame's entries.
//
// The same source is compiled twice: by nvcc into fsg_search_kernel (psb_search.cu), and by g++ with
// PSB_FSG_HOST_EMUL into a TEST harness (tests/emul/fsg_emul.cpp) that runs every FSG_FOR loop to
// completion, forwards or (PSB_FSG_EMUL_REVERSE) backwards, to check the phase logic -- including
// its freedom from intra-phase ordering assumptions -- against the reference's golden history
// tables without a GPU.  libpsb200.so contains no host execution path of the phase code (only the LM
// lookup helpers of psb_lm_core.h / ngs_tg are __host__ __device__: psb_result.cu scores segments with them).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <limits.h>

#if defined(__CUDACC__) && !defined(PSB_FSG_HOST_EMUL)
#define FSG_HD __device__ __forceinline__
#define FSG_HDH __host__ __device__ __forceinline__
#define FSG_FOR(i, n) for (int i = (int)threadIdx.x; i < (n); i += (int)blockDim.x)   /* one CTA per utterance */
#define FSG_SYNC() __syncthreads()
#define FSG_IF_LEADER if (threadIdx.x == 0)
#define FSG_ATOMIC_MAX(p, v) atomicMax((p), (v))
#define FSG_ATOMIC_ADD(p, v) atomicAdd((p), (v))
#define FSG_ATOMIC_MIN(p, v) atomicMin((p), (v))
#define FSG_ATOMIC_MAX_AT(a, i, v) atomicMax(&(a)[i], (v))
#define FSG_ATOMIC_MIN_AT(a, i, v) atomicMin(&(a)[i], (v))
#define FSG_ATOMIC_ADD_AT(a, i, v) atomicAdd(&(a)[i], (v))
#define FSG_ATOMIC_FETCH_ADD_AT(a, i, v) atomicAdd(&(a)[i], (v))
#ifdef __CUDA_ARCH__
#define FSG_FADD(a, b) __fadd_rn((a), (b))
#define FSG_FMUL(a, b) __fmul_rn((a), (b))
#else                                   /* host half of the few __host__ __device__ helpers (LM lookups of psb_result.cu): */
#define FSG_FADD(a, b) ((a) + (b))      /* x86-64 scalar SSE, one rounding per operation, no contraction without -mfma */
#define FSG_FMUL(a, b) ((a) * (b))
#endif
typedef int32_t *fsg_wp;
typedef uint32_t *fsg_wup;
typedef int fsg_int;
typedef float fsg_float;
typedef long long fsg_ll;
#else
#define FSG_HD static inline
#define FSG_HDH static inline
#ifdef PSB_FSG_RACECHECK                /* tests only: tests/emul/psb_fsg_racecheck.h, see tests/test_emul_racecheck.py */
#include "psb_fsg_racecheck.h"
#else
#ifdef PSB_FSG_EMUL_REVERSE
#define FSG_FOR(i, n) for (int i = (n) - 1; i >= 0; --i)
#else
#define FSG_FOR(i, n) for (int i = 0; i < (n); ++i)
#endif
#define FSG_SYNC() ((void)0)
#define FSG_IF_LEADER
static inline void fsg_host_max(int *p, int v) { if (v > *p) *p = v; }
static inline void fsg_host_min(int *p, int v) { if (v < *p) *p = v; }
#define FSG_ATOMIC_MAX(p, v) fsg_host_max((p), (v))
#define FSG_ATOMIC_ADD(p, v) (*(p) += (v))
#define FSG_ATOMIC_MIN(p, v) fsg_host_min((p), (v))
#define FSG_ATOMIC_MAX_AT(a, i, v) fsg_host_max(&(a)[i], (v))
#define FSG_ATOMIC_MIN_AT(a, i, v) fsg_host_min(&(a)[i], (v))
#define FSG_ATOMIC_ADD_AT(a, i, v) ((a)[i] += (v))
static inline int fsg_host_fetch_add(int *p, int v) { const int o = *p; *p = o + v; return o; }
#define FSG_ATOMIC_FETCH_ADD_AT(a, i, v) fsg_host_fetch_add(&(a)[i], (v))
#define FSG_COLLECTIVE_BEGIN() ((void)0)
#define FSG_COLLECTIVE_END() ((void)0)
#define FSG_RAW(a) (a)
typedef int32_t *fsg_wp;            /* pointer into an utterance's mutable state */
typedef uint32_t *fsg_wup;
typedef int fsg_int;                /* block-shared scalar */
typedef float fsg_float;
typedef long long fsg_ll;
#endif
#define FSG_FADD(a, b) ((a) + (b))      /* harnesses are built with -ffp-contract=off */
#define FSG_FMUL(a, b) ((a) * (b))
#endif

#define FSG_WORST_SCORE ((int)0xE0000000)
#define FSG_ROW 13              /* history row: link, frame, score, pred, lc, rc.bv[8] */
#define FSG_MAX_NSTATE 5

// The flattened lextree and grammar, read-only, shared by every utterance (fsg_lextree.h:137-190).
struct FsgGraph {
    int P, R, n_state, n_ci, n_emit;
    int silcipid, start_state, beam, pbeam, wbeam, maxhmmpf;
    int CC;                     // capacity of the per-frame candidate / new-entry scratch
    const int32_t *lp;          // [P] logs2prob (already >> SENSCR_SHIFT, wip/pip included)
    const int32_t *next;        // [P] first child, or the fsg link of a leaf
    const int32_t *sib;         // [P] next sibling or -1
    const int32_t *ci_ext;      // [P]
    const int32_t *leaf;        // [P]
    const int32_t *parent;      // [P] -1 for roots
    const uint32_t *ctxt;       // [P][8]
    const int32_t *root_list;   // [R] roots, state by state, in sibling order
    const int32_t *root_state;  // [R]
    const int32_t *link_to;     // [L] destination state
    const int32_t *link_all;    // [L] filler or single-phone word: exits apply to all right contexts
    const int32_t *link_nlp;    // [L] logs2prob >> SENSCR_SHIFT (used for null arcs)
    const int32_t *nulloff;     // [n_state+1]
    const int32_t *nullarc;     // [n_null] link ids
};

// Per-utterance state in global memory.
struct FsgWork {
    fsg_wp score, hist;                          // [n_emit][P]
    fsg_wp out_score, out_hist, best, frame;   // [P]
    fsg_wp pos, posf;                            // [P] walk position in the frame posf
    fsg_wp act[2];                                // [P] active lists, insertion order
    fsg_wp cnt, ecnt, kflag;                    // [CC+1]
    fsg_wp c_link, c_score, c_pred, c_lc, c_grp, c_alive;   // [CC] candidates
    fsg_wup c_rc, c_rcf;                         // [CC][8]
    fsg_wp ne_dest, ne_score, ne_lc;            // [CC] this frame's history entries
    fsg_wup ne_rc;                                // [CC][8]
    fsg_wp rfirst, rcnt, rnew;                    // [R] (+1)
    fsg_wp hist_out;                              // [cap][FSG_ROW]
    int cap;
};

struct FsgScalars {
    fsg_int cur, n_act, n_ins, n_exit, n_newroot;
    fsg_int best, beam, pbeam, wbeam, thresh, pth, wth;
    fsg_int n_hist, bp_start, n_new, n_res, overflow;
    fsg_float beam_factor;
    int scan[34];
};

#if defined(__CUDACC__) && !defined(PSB_FSG_HOST_EMUL)
// In-place exclusive scan of a[0..n) by the whole block; returns the total to every thread.
__device__ inline int fsg_exscan(fsg_wp a, int n, int *scan /* [34], shared */)
{
    const int tid = (int)threadIdx.x, nt = (int)blockDim.x, lane = tid & 31, w = tid >> 5;
    if (tid == 0) scan[33] = 0;
    __syncthreads();
    for (int base = 0; base < n; base += nt) {
        const int i = base + tid;
        const int v = i < n ? a[i] : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) scan[w] = incl;
        __syncthreads();
        const int carry = scan[33];
        int wbase = 0;
        for (int j = 0; j < w; ++j) wbase += scan[j];
        if (i < n) a[i] = carry + wbase + incl - v;
        __syncthreads();
        if (tid == nt - 1) scan[33] = carry + wbase + incl;
        __syncthreads();
    }
    const int total = scan[33];
    __syncthreads();                                  // the next scan resets scan[33]
    return total;
}
#else
static inline int fsg_exscan(fsg_wp a, int n, int *scan)
{
    int run = 0;
    (void)scan;
    FSG_COLLECTIVE_BEGIN();                            /* the device scan starts and ends with a barrier */
    for (int i = 0; i < n; ++i) { const int v = FSG_RAW(a)[i]; FSG_RAW(a)[i] = run; run += v; }
    FSG_COLLECTIVE_END();
    return run;
}
#endif

// Carve one utterance's scratch (fsg_work_words() int32 words, psb_fsg_host.h) into its arrays.
FSG_HD void fsg_work_carve(int32_t *b, const FsgGraph &G, FsgWork &W)
{
    const size_t P = (size_t)G.P, CC = (size_t)G.CC, N = (size_t)G.n_emit;
    W.score = b; b += N * P;  W.hist = b; b += N * P;
    W.out_score = b; b += P;  W.out_hist = b; b += P;  W.best = b; b += P;  W.frame = b; b += P;
    W.pos = b; b += P;  W.posf = b; b += P;  W.act[0] = b; b += P;  W.act[1] = b; b += P;
    W.cnt = b; b += CC + 1;  W.ecnt = b; b += CC + 1;  W.kflag = b; b += CC + 1;
    W.c_link = b; b += CC;  W.c_score = b; b += CC;  W.c_pred = b; b += CC;  W.c_lc = b; b += CC;
    W.c_grp = b; b += CC;  W.c_alive = b; b += CC;
    W.c_rc = fsg_wup((uint32_t *)b); b += 8 * CC;  W.c_rcf = fsg_wup((uint32_t *)b); b += 8 * CC;
    W.ne_dest = b; b += CC;  W.ne_score = b; b += CC;  W.ne_lc = b; b += CC;
    W.ne_rc = fsg_wup((uint32_t *)b); b += 8 * CC;
    W.rfirst = b; b += (size_t)G.R + 1;  W.rcnt = b; b += (size_t)G.R + 1;  W.rnew = b;
}

FSG_HD void fsg_clear_node(const FsgGraph &G, const FsgWork &W, int p)        /* hmm_clear, hmm.c:180-196 */
{
    for (int s = 0; s < G.n_emit; ++s) { W.score[s * G.P + p] = FSG_WORST_SCORE; W.hist[s * G.P + p] = -1; }
    W.out_score[p] = FSG_WORST_SCORE; W.out_hist[p] = -1; W.best[p] = FSG_WORST_SCORE; W.frame[p] = -1;
}

// Does p's parent, active in frame f, transition into p?  (prune_prop :540-548 + pnode_trans :425-428,
// evaluated on the state hmm_eval left; nothing a phase reads here is written in that phase.)
FSG_HD bool fsg_parent_enters(const FsgGraph &G, const FsgWork &W, const FsgScalars *S, int p, int f)
{
    const int par = G.parent[p];
    if (par < 0 || W.posf[par] != f) return false;
    if (W.best[par] < S->thresh || W.out_score[par] < S->pth) return false;
    const int ns = W.out_score[par] + G.lp[p];
    return ns > S->thresh && ns > W.score[p];
}

// Resolve n candidates (c_*) into history entries appended to this frame's scratch at ne_base and
// to the table at bp_start + ne_base: fsg_history_entry_add for each, then fsg_history_end_frame.
// direct: the frame < 0 shortcut (fsg_history.c:143-156), entries are appended as they come.
FSG_HD void fsg_resolve(const FsgGraph &G, const FsgWork &W, FsgScalars *S, int n, int ne_base, int frame, bool direct)
{
    FSG_IF_LEADER S->n_res = 0;
    FSG_SYNC();
    FSG_FOR(i, n) {
        uint32_t rc[8], any = 0;
        for (int q = 0; q < 8; ++q) rc[q] = W.c_rc[i * 8 + q];
        if (!direct) {
            const int g = W.c_grp[i], sc = W.c_score[i];
            for (int j = 0; j < n; ++j) {
                if (j == i || W.c_grp[j] != g) continue;
                const int sj = W.c_score[j];
                if (sj > sc || (sj == sc && j < i))
                    for (int q = 0; q < 8; ++q) rc[q] &= ~W.c_rc[j * 8 + q];
            }
        }
        for (int q = 0; q < 8; ++q) { W.c_rcf[i * 8 + q] = rc[q]; any |= rc[q]; }
        W.c_alive[i] = (direct || any != 0) ? 1 : 0;
    }
    FSG_SYNC();
    FSG_FOR(i, n) {
        if (!W.c_alive[i]) continue;
        int rank = 0;
        if (direct) rank = i;
        else {
            const int g = W.c_grp[i], sc = W.c_score[i];
            for (int j = 0; j < n; ++j) {
                if (j == i || !W.c_alive[j]) continue;
                const int gj = W.c_grp[j], sj = W.c_score[j];
                if (gj < g || (gj == g && (sj > sc || (sj == sc && j < i)))) ++rank;
            }
        }
        const int e = ne_base + rank, l = W.c_link[i];
        if (e < G.CC) {
            W.ne_dest[e] = l >= 0 ? G.link_to[l] : G.start_state;
            W.ne_score[e] = W.c_score[i];
            W.ne_lc[e] = W.c_lc[i];
            for (int q = 0; q < 8; ++q) W.ne_rc[e * 8 + q] = W.c_rcf[i * 8 + q];
        }
        const int bp = S->bp_start + e;
        if (bp < W.cap) {
            fsg_wp r = W.hist_out + (size_t)bp * FSG_ROW;
            r[0] = l; r[1] = frame; r[2] = W.c_score[i]; r[3] = W.c_pred[i]; r[4] = W.c_lc[i];
            for (int q = 0; q < 8; ++q) r[5 + q] = (int32_t)W.c_rcf[i * 8 + q];
        }
        FSG_ATOMIC_ADD(&S->n_res, 1);
    }
    FSG_SYNC();
}

// null_prop (:566-614) over this frame's first n1 entries, then word_trans (:621-680) over all of
// them; roots that become active are appended to the next list after its first n_ins nodes.
FSG_HD void fsg_cross_word(const FsgGraph &G, const FsgWork &W, FsgScalars *S, int n1, int frame)
{
    const int th = S->best + S->wbeam, nf = frame + 1;
    FSG_FOR(b, n1) {
        const int d = W.ne_dest[b];
        int c = 0;
        for (int k = G.nulloff[d]; k < G.nulloff[d + 1]; ++k)
            if (W.ne_score[b] + G.link_nlp[G.nullarc[k]] >= th) ++c;
        W.cnt[b] = c;
    }
    FSG_SYNC();
    const int n2c = fsg_exscan(W.cnt, n1, S->scan);
    if (n2c > G.CC || n1 + n2c > G.CC) {                                  // cannot happen: CC = P * (1 + widest null fan-out)
        FSG_IF_LEADER S->overflow = 1;
        FSG_SYNC();
        return;
    }
    FSG_FOR(b, n1) {
        const int d = W.ne_dest[b];
        int o = W.cnt[b];
        for (int k = G.nulloff[d]; k < G.nulloff[d + 1]; ++k) {
            const int l = G.nullarc[k], ns = W.ne_score[b] + G.link_nlp[l];
            if (ns < th) continue;
            W.c_link[o] = l; W.c_score[o] = ns; W.c_pred[o] = S->bp_start + b; W.c_lc[o] = W.ne_lc[b];
            W.c_grp[o] = G.link_to[l] * G.n_ci + W.ne_lc[b];
            for (int q = 0; q < 8; ++q) W.c_rc[o * 8 + q] = W.ne_rc[b * 8 + q];
            ++o;
        }
    }
    FSG_SYNC();
    fsg_resolve(G, W, S, n2c, n1, frame, frame < 0);
    const int n_new = n1 + S->n_res;
    const int thresh = S->best + S->beam;
    fsg_wp nxt = W.act[S->cur ^ 1];
    FSG_FOR(ri, G.R) {
        const int p = G.root_list[ri], d = G.root_state[ri], rc = G.ci_ext[p];
        int cur = W.score[p], first = -1, h = -1;
        for (int b = 0; b < n_new; ++b) {
            if (W.ne_dest[b] != d) continue;
            const int lc = W.ne_lc[b];
            if (!((G.ctxt[p * 8 + (lc >> 5)] >> (lc & 31)) & 1u) || !((W.ne_rc[b * 8 + (rc >> 5)] >> (rc & 31)) & 1u)) continue;
            const int ns = W.ne_score[b] + G.lp[p];
            if (ns > thresh && ns > cur) {
                if (first < 0) first = b;
                cur = ns; h = S->bp_start + b;
            }
        }
        int key = -1;
        if (first >= 0) {
            if (W.frame[p] < nf) key = first;                               // newly activated
            W.score[p] = cur; W.hist[p] = h; W.frame[p] = nf;                // hmm_enter
        }
        W.rfirst[ri] = key;
    }
    // newly activated roots, compacted in root order (scan), then ranked among themselves by (first entering
    // entry, sibling order): K is small even when the grammar has thousands of roots
    FSG_SYNC();
    FSG_FOR(ri, G.R) W.rcnt[ri] = W.rfirst[ri] >= 0 ? 1 : 0;
    FSG_SYNC();
    const int K = fsg_exscan(W.rcnt, G.R, S->scan);
    FSG_FOR(ri, G.R) if (W.rfirst[ri] >= 0) W.rnew[W.rcnt[ri]] = ri;
    FSG_SYNC();
    FSG_FOR(k, K) {
        const int ri = W.rnew[k], key = W.rfirst[ri];
        int rank = 0;
        for (int j = 0; j < K; ++j) {
            const int rj = W.rnew[j], kj = W.rfirst[rj];
            if (kj < key || (kj == key && rj < ri)) ++rank;
        }
        nxt[S->n_ins + rank] = G.root_list[ri];
    }
    FSG_IF_LEADER S->n_newroot = K;
    FSG_SYNC();
    FSG_IF_LEADER {
        S->n_hist += n_new;
        S->n_act = S->n_ins + S->n_newroot;
        S->cur ^= 1;
    }
    FSG_SYNC();
}

// fsg_search_start (:770-817): everything inactive, the dummy entry leading to the start state,
// its null transitions and the first word transitions.
FSG_HD void fsg_start(const FsgGraph &G, const FsgWork &W, FsgScalars *S)
{
    FSG_FOR(p, G.P) { fsg_clear_node(G, W, p); W.pos[p] = -1; W.posf[p] = -2; }
    FSG_IF_LEADER {
        S->cur = 0; S->n_act = 0; S->n_ins = 0; S->n_exit = 0; S->n_newroot = 0;
        S->best = 0; S->beam = G.beam; S->pbeam = G.pbeam; S->wbeam = G.wbeam; S->beam_factor = 1.0f;
        S->n_hist = 0; S->bp_start = 0; S->overflow = 0;
        W.c_link[0] = -1; W.c_score[0] = 0; W.c_pred[0] = -1; W.c_lc[0] = G.silcipid; W.c_grp[0] = 0;
        for (int q = 0; q < 8; ++q) W.c_rc[q] = 0xffffffffu;
    }
    FSG_SYNC();
    fsg_resolve(G, W, S, 1, 0, -1, true);
    fsg_cross_word(G, W, S, 1, -1);
}

// fsg_search_step (:683-761) for frame f.  Eval(W, p) runs hmm_vit_eval on node p against this
// frame's senone scores and returns its best score.
template <class Eval>
FSG_HD void fsg_step(const FsgGraph &G, const FsgWork &W, FsgScalars *S, int f, Eval &eval)
{
    const int n_act = S->n_act, nf = f + 1;
    const fsg_wp act = W.act[S->cur];
    fsg_wp nxt = W.act[S->cur ^ 1];
    FSG_IF_LEADER { S->best = FSG_WORST_SCORE; S->bp_start = S->n_hist; }
    FSG_SYNC();
    FSG_FOR(w, n_act) {                                                      // hmm_eval :335-373
        const int p = act[n_act - 1 - w];
        W.pos[p] = w; W.posf[p] = f;
        const int b = eval(W, p);
        FSG_ATOMIC_MAX(&S->best, b);
    }
    FSG_SYNC();
    FSG_IF_LEADER {                                                      // :378-400
        if (G.maxhmmpf != -1 && n_act > G.maxhmmpf) {
            if (S->beam_factor > 0.1) {
                S->beam_factor *= 0.9f;
                S->beam = (int32_t)(G.beam * S->beam_factor);
                S->pbeam = (int32_t)(G.pbeam * S->beam_factor);
                S->wbeam = (int32_t)(G.wbeam * S->beam_factor);
            }
        }
        else { S->beam_factor = 1.0f; S->beam = G.beam; S->pbeam = G.pbeam; S->wbeam = G.wbeam; }
        S->thresh = S->best + S->beam; S->pth = S->best + S->pbeam; S->wth = S->best + S->wbeam;
    }
    FSG_SYNC();
    const int thresh = S->thresh, pth = S->pth, wth = S->wth;
    FSG_FOR(w, n_act) {                                                      // prune_prop :516-560, decisions only
        const int p = act[n_act - 1 - w];
        int c = 0, e = 0, flag = 0;
        if (W.best[p] >= thresh) {
            const int par = G.parent[p];
            bool by_parent = false;
            if (par >= 0 && W.posf[par] == f && W.pos[par] < w) by_parent = fsg_parent_enters(G, W, S, p, f);
            if (!by_parent) { c = 1; flag |= 1; }
            if (!G.leaf[p]) {
                if (W.out_score[p] >= pth) {
                    flag |= 2;
                    for (int ch = G.next[p]; ch >= 0; ch = G.sib[ch]) {
                        const int ns = W.out_score[p] + G.lp[ch];
                        if (ns > thresh && ns > W.score[ch]) {
                            const bool already = W.posf[ch] == f && W.pos[ch] < w && W.best[ch] >= thresh;
                            if (!already) ++c;
                        }
                    }
                }
            }
            else if (W.out_score[p] >= wth) { e = 1; flag |= 4; }
        }
        W.cnt[w] = c; W.ecnt[w] = e; W.kflag[w] = flag;
    }
    FSG_SYNC();
    const int n_ins = fsg_exscan(W.cnt, n_act, S->scan);
    const int n_exit = fsg_exscan(W.ecnt, n_act, S->scan);
    FSG_IF_LEADER { S->n_ins = n_ins; S->n_exit = n_exit; }
    FSG_FOR(w, n_act) {                                                      // ... applied
        const int p = act[n_act - 1 - w], flag = W.kflag[w];
        int o = W.cnt[w];
        if (flag & 1) nxt[o++] = p;
        if (W.best[p] >= thresh) W.frame[p] = nf;
        if (flag & 2) {
            for (int ch = G.next[p]; ch >= 0; ch = G.sib[ch]) {
                const int ns = W.out_score[p] + G.lp[ch];
                if (ns > thresh && ns > W.score[ch]) {
                    const bool already = W.posf[ch] == f && W.pos[ch] < w && W.best[ch] >= thresh;
                    if (!already) nxt[o++] = ch;
                    W.score[ch] = ns; W.hist[ch] = W.out_hist[p]; W.frame[ch] = nf;     // hmm_enter
                }
            }
        }
        if (flag & 4) {                                                      // pnode_exit :444-507
            const int j = W.ecnt[w], l = G.next[p];
            W.c_link[j] = l; W.c_score[j] = W.out_score[p]; W.c_pred[j] = W.out_hist[p]; W.c_lc[j] = G.ci_ext[p];
            W.c_grp[j] = G.link_to[l] * G.n_ci + G.ci_ext[p];
            for (int q = 0; q < 8; ++q) W.c_rc[j * 8 + q] = G.link_all[l] ? 0xffffffffu : G.ctxt[p * 8 + q];
        }
    }
    FSG_SYNC();
    fsg_resolve(G, W, S, n_exit, 0, f, false);
    const int n1 = S->n_res;
    fsg_cross_word(G, W, S, n1, f);                                          // flips S->cur, sets S->n_act
    FSG_FOR(k, n_act) {                                                      // :736-748
        const int p = act[k];
        if (W.frame[p] == f) fsg_clear_node(G, W, p);
    }
    FSG_SYNC();
}
