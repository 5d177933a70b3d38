// psb_hmm.cuh -- device-side Viterbi step for one HMM instance (register resident).
//
// One call = one hmm_vit_eval (hmm.c:787-805): s_i = score[i] + (-senscore[senid_i]), each
// target state takes the max over its (at most three) predecessors with the reference's
// exact tie order, history (and, for multiplexed HMMs, the senone-sequence id) follows the
// winner, everything is floored at WORST_SCORE, and the exit state is fed by the top two
// emitting states.  The five reference specialisations differ in which blocks are guarded
// and in how a missing skip arc is treated, so each is restated separately.
#pragma once
#include "psb_internal.cuh"

struct HmmCtxDev {
    int n_emit;
    int n_sen;
    const uint8_t *tp;        // [n_tmat][n_emit][n_emit+1]
    const uint16_t *sseq;     // [n_sseq][n_emit]
};

struct HmmReg {
    int score[PSB_HMM_MAX_NSTATE];
    int hist[PSB_HMM_MAX_NSTATE];
    int out_score, out_hist;
    int senid[PSB_HMM_MAX_NSTATE];   // senone ids (non-mpx) or per-state sseq ids (mpx)
    int best;
};

__device__ __forceinline__ int hmm_pick3(int t0, int t1, int t2, int &out)
{
    // hmm.c:257-271 and twins: returns 0 (self loop), 1 (state below), 2 (skip)
    if (t0 > t1) {
        if (t2 > t0) { out = t2; return 2; }
        out = t0; return 0;
    }
    if (t2 > t1) { out = t2; return 2; }
    out = t1; return 1;
}

#define PSB_FLOOR(s) do { if ((s) < PSB_WORST_SCORE) (s) = PSB_WORST_SCORE; } while (0)
#define PSB_RAISE(b, s) do { if ((s) > (b)) (b) = (s); } while (0)

// obs[i] = -senscore[senone of state i] (already negated), valid for non-mpx HMMs.
// hmm_vit_eval_3st_lr (hmm.c:530-607)
__device__ __forceinline__ int hmm_step_3st(HmmReg &h, const uint8_t *tp, const int (&obs)[PSB_HMM_MAX_NSTATE])
{
#define TP(i, j) (-(int)tp[(i) * 4 + (j)])
    int s0, s1, s2, s3, t0, t1, t2, best = PSB_WORST_SCORE;
    s2 = h.score[2] + obs[2];
    s1 = h.score[1] + obs[1];
    s0 = h.score[0] + obs[0];
    t2 = INT_MIN;                            // stale-t2 quirk, SURVEY A.1.5
    if (s1 > PSB_WORST_SCORE) {
        t1 = s2 + TP(2, 3);
        if (TP(1, 3) > PSB_TMAT_WORST) t2 = s1 + TP(1, 3);
        if (t1 > t2) { s3 = t1; h.out_hist = h.hist[2]; }
        else { s3 = t2; h.out_hist = h.hist[1]; }
        PSB_FLOOR(s3);
        h.out_score = s3;
        best = s3;
    }
    t0 = s2 + TP(2, 2);
    t1 = s1 + TP(1, 2);
    if (TP(0, 2) > PSB_TMAT_WORST) t2 = s0 + TP(0, 2);
    {
        int w = hmm_pick3(t0, t1, t2, s2);
        if (w == 2) h.hist[2] = h.hist[0];
        else if (w == 1) h.hist[2] = h.hist[1];
    }
    PSB_FLOOR(s2); PSB_RAISE(best, s2);
    h.score[2] = s2;
    t0 = s1 + TP(1, 1);
    t1 = s0 + TP(0, 1);
    if (t0 > t1) s1 = t0;
    else { s1 = t1; h.hist[1] = h.hist[0]; }
    PSB_FLOOR(s1); PSB_RAISE(best, s1);
    h.score[1] = s1;
    s0 = s0 + TP(0, 0);
    PSB_FLOOR(s0); PSB_RAISE(best, s0);
    h.score[0] = s0;
    h.best = best;
    return best;
#undef TP
}

// hmm_step_3st for a kernel that runs the same instance over many frames (the fused sweep,
// psb_hmm.cu): the transition bytes are decoded once per instance into ready-to-add ints, the
// two "is this arc allowed" tests (TP(1,3), TP(0,2) against TMAT_WORST) into all-ones / zero
// masks, and every tie-ordered pick is a compare + select with no branch.  The other kernels
// see each instance once per launch and keep hmm_step_3st, which reads the bytes in place.
// Same bits as hmm_step_3st, the floor and the stale-t2 quirk included: an absent arc yields
// INT_MIN by masking, never by arithmetic on a sentinel.
struct HmmTp3 {
    int p00, p01, p11, p12, p22, p23, p02, p13;   // -tp[i][j]
    int m02, m13;                                 // -1: the arc exists (tp byte != 255), 0: it does not
};

__device__ __forceinline__ HmmTp3 hmm_tp3_decode(const uint8_t *tp)
{
    HmmTp3 k;
    k.p00 = -(int)tp[0]; k.p01 = -(int)tp[1]; k.p02 = -(int)tp[2];
    k.p11 = -(int)tp[5]; k.p12 = -(int)tp[6]; k.p13 = -(int)tp[7];
    k.p22 = -(int)tp[10]; k.p23 = -(int)tp[11];
    // opaque to the compiler, so that the masks stay in registers instead of being re-derived from the bytes every frame
    asm("mov.b32 %0, %1;" : "=r"(k.m02) : "r"(k.p02 > PSB_TMAT_WORST ? -1 : 0));
    asm("mov.b32 %0, %1;" : "=r"(k.m13) : "r"(k.p13 > PSB_TMAT_WORST ? -1 : 0));
    return k;
}

// Transitions for a padding slot (scores at WORST_SCORE, any senone): every candidate falls below the floor whatever
// int16 score the slot gathers (WORST - (-32768) + PAD stays under WORST), so the slot's best score is WORST_SCORE in
// every frame and never shows in a maximum -- no per-frame "is this slot an instance" test.
__device__ __forceinline__ HmmTp3 hmm_tp3_padding()
{
    constexpr int PAD = -0x100000;
    HmmTp3 k;
    k.p00 = k.p01 = k.p02 = k.p11 = k.p12 = k.p13 = k.p22 = k.p23 = PAD;
    k.m02 = k.m13 = -1;
    return k;
}

// (m ? a : b) for an all-ones / zero mask m: one LOP3
__device__ __forceinline__ int hmm_msel(int m, int a, int b) { return (a & m) | (b & ~m); }

// x_i = senscore of state i's senone (not negated); returns the instance's best score.  S1_LIVE: the caller has
// established sc[1] - x1 > WORST_SCORE (the exit state is evaluated), so the four selects on that test fold away.
template <bool S1_LIVE = false>
__device__ __forceinline__ int hmm_step_3st_dec(int (&sc)[3], int (&hi)[3], int &osc, int &ohi, const HmmTp3 &k,
                                                int x0, int x1, int x2)
{
    const int s2 = sc[2] - x2, s1 = sc[1] - x1, s0 = sc[0] - x0;
    // exit state, only when s1 > WORST (hmm.c:545-556)
    const bool a = S1_LIVE || s1 > PSB_WORST_SCORE;
    const int e1 = s2 + k.p23;
    const int e2 = hmm_msel(k.m13, s1 + k.p13, INT_MIN);
    const int s3 = max(max(e1, e2), PSB_WORST_SCORE);
    const int oh = e1 > e2 ? hi[2] : hi[1];
    osc = a ? s3 : osc;
    ohi = a ? oh : ohi;
    // state 2: t2 keeps its exit-state value (or INT_MIN) when TP(0,2) is absent
    const int u2 = hmm_msel(k.m02, s0 + k.p02, a ? e2 : INT_MIN);
    const int u0 = s2 + k.p22, u1 = s1 + k.p12;
    const int m01 = max(u0, u1);
    const int n2 = max(max(m01, u2), PSB_WORST_SCORE);
    const int h2 = u2 > m01 ? hi[0] : (u0 > u1 ? hi[2] : hi[1]);      // hmm_pick3's tie order
    // state 1
    const int v0 = s1 + k.p11, v1 = s0 + k.p01;
    const int n1 = max(max(v0, v1), PSB_WORST_SCORE);
    const int h1 = v0 > v1 ? hi[1] : hi[0];
    // state 0
    const int n0 = max(s0 + k.p00, PSB_WORST_SCORE);
    sc[0] = n0; sc[1] = n1; sc[2] = n2;
    hi[1] = h1; hi[2] = h2;
    return max(max(a ? s3 : PSB_WORST_SCORE, n2), max(n1, n0));
}

// hmm_vit_eval_5st_lr (hmm.c:223-353)
__device__ __forceinline__ int hmm_step_5st(HmmReg &h, const uint8_t *tp, const int (&obs)[PSB_HMM_MAX_NSTATE])
{
#define TP(i, j) (-(int)tp[(i) * 6 + (j)])
    int s0, s1, s2, s3, s4, s5, t0, t1, t2, best = PSB_WORST_SCORE;
    s4 = h.score[4] + obs[4];
    s3 = h.score[3] + obs[3];
    if (s3 > PSB_WORST_SCORE) {
        t1 = s4 + TP(4, 5);
        t2 = s3 + TP(3, 5);
        if (t1 > t2) { s5 = t1; h.out_hist = h.hist[4]; }
        else { s5 = t2; h.out_hist = h.hist[3]; }
        PSB_FLOOR(s5);
        h.out_score = s5;
        best = s5;
    }
    s2 = h.score[2] + obs[2];
    if (s2 > PSB_WORST_SCORE) {
        int w = hmm_pick3(s4 + TP(4, 4), s3 + TP(3, 4), s2 + TP(2, 4), s4);
        if (w == 2) h.hist[4] = h.hist[2];
        else if (w == 1) h.hist[4] = h.hist[3];
        PSB_FLOOR(s4); PSB_RAISE(best, s4);
        h.score[4] = s4;
    }
    s1 = h.score[1] + obs[1];
    if (s1 > PSB_WORST_SCORE) {
        int w = hmm_pick3(s3 + TP(3, 3), s2 + TP(2, 3), s1 + TP(1, 3), s3);
        if (w == 2) h.hist[3] = h.hist[1];
        else if (w == 1) h.hist[3] = h.hist[2];
        PSB_FLOOR(s3); PSB_RAISE(best, s3);
        h.score[3] = s3;
    }
    s0 = h.score[0] + obs[0];
    {
        int w = hmm_pick3(s2 + TP(2, 2), s1 + TP(1, 2), s0 + TP(0, 2), s2);
        if (w == 2) h.hist[2] = h.hist[0];
        else if (w == 1) h.hist[2] = h.hist[1];
        PSB_FLOOR(s2); PSB_RAISE(best, s2);
        h.score[2] = s2;
    }
    t0 = s1 + TP(1, 1);
    t1 = s0 + TP(0, 1);
    if (t0 > t1) s1 = t0;
    else { s1 = t1; h.hist[1] = h.hist[0]; }
    PSB_FLOOR(s1); PSB_RAISE(best, s1);
    h.score[1] = s1;
    s0 = s0 + TP(0, 0);
    PSB_FLOOR(s0); PSB_RAISE(best, s0);
    h.score[0] = s0;
    h.best = best;
    return best;
#undef TP
}

// Multiplexed HMMs: senid[] holds one senone-sequence id per state (BAD_SSID = empty); the
// observation of state st is -senscore[sseq[senid[st]][st]] (hmm.h:199-209).
__device__ __forceinline__ int mpx_obs(const HmmCtxDev &c, const int16_t *senscr, const HmmReg &h, int st)
{
    return -(int)senscr[c.sseq[(size_t)h.senid[st] * c.n_emit + st]];
}

// hmm_vit_eval_3st_lr_mpx (hmm.c:610-706)
__device__ __forceinline__ int hmm_step_3st_mpx(HmmReg &h, const HmmCtxDev &c, const uint8_t *tp, const int16_t *senscr)
{
#define TP(i, j) (-(int)tp[(i) * 4 + (j)])
    int s0, s1, s2, s3, t0, t1, t2, best, w;
    t2 = INT_MIN;
    if (h.senid[2] == PSB_BAD_SSID) s2 = t1 = PSB_WORST_SCORE;
    else { s2 = h.score[2] + mpx_obs(c, senscr, h, 2); t1 = s2 + TP(2, 3); }
    if (h.senid[1] == PSB_BAD_SSID) s1 = t2 = PSB_WORST_SCORE;
    else {
        s1 = h.score[1] + mpx_obs(c, senscr, h, 1);
        if (TP(1, 3) > PSB_TMAT_WORST) t2 = s1 + TP(1, 3);
    }
    if (t1 > t2) { s3 = t1; h.out_hist = h.hist[2]; }
    else { s3 = t2; h.out_hist = h.hist[1]; }
    PSB_FLOOR(s3);
    h.out_score = s3;
    best = s3;
    s0 = h.score[0] + mpx_obs(c, senscr, h, 0);
    t0 = t1 = PSB_WORST_SCORE;
    if (s2 != PSB_WORST_SCORE) t0 = s2 + TP(2, 2);
    if (s1 != PSB_WORST_SCORE) t1 = s1 + TP(1, 2);
    if (TP(0, 2) > PSB_TMAT_WORST) t2 = s0 + TP(0, 2);
    w = hmm_pick3(t0, t1, t2, s2);
    if (w == 2) { h.hist[2] = h.hist[0]; h.senid[2] = h.senid[0]; }
    else if (w == 1) { h.hist[2] = h.hist[1]; h.senid[2] = h.senid[1]; }
    PSB_FLOOR(s2); PSB_RAISE(best, s2);
    h.score[2] = s2;
    t0 = PSB_WORST_SCORE;
    if (s1 != PSB_WORST_SCORE) t0 = s1 + TP(1, 1);
    t1 = s0 + TP(0, 1);
    if (t0 > t1) s1 = t0;
    else { s1 = t1; h.hist[1] = h.hist[0]; h.senid[1] = h.senid[0]; }
    PSB_FLOOR(s1); PSB_RAISE(best, s1);
    h.score[1] = s1;
    s0 += TP(0, 0);
    PSB_FLOOR(s0); PSB_RAISE(best, s0);
    h.score[0] = s0;
    h.best = best;
    return best;
#undef TP
}

// hmm_vit_eval_5st_lr_mpx (hmm.c:356-525)
__device__ __forceinline__ int hmm_step_5st_mpx(HmmReg &h, const HmmCtxDev &c, const uint8_t *tp, const int16_t *senscr)
{
#define TP(i, j) (-(int)tp[(i) * 6 + (j)])
    int s0, s1, s2, s3, s4, s5, t0, t1, t2, best, w;
    if (h.senid[4] == PSB_BAD_SSID) s4 = t1 = PSB_WORST_SCORE;
    else { s4 = h.score[4] + mpx_obs(c, senscr, h, 4); t1 = s4 + TP(4, 5); }
    if (h.senid[3] == PSB_BAD_SSID) s3 = t2 = PSB_WORST_SCORE;
    else { s3 = h.score[3] + mpx_obs(c, senscr, h, 3); t2 = s3 + TP(3, 5); }
    if (t1 > t2) { s5 = t1; h.out_hist = h.hist[4]; }
    else { s5 = t2; h.out_hist = h.hist[3]; }
    PSB_FLOOR(s5);
    h.out_score = s5;
    best = s5;

    if (h.senid[2] == PSB_BAD_SSID) s2 = t2 = PSB_WORST_SCORE;
    else { s2 = h.score[2] + mpx_obs(c, senscr, h, 2); t2 = s2 + TP(2, 4); }
    t0 = t1 = PSB_WORST_SCORE;
    if (s4 != PSB_WORST_SCORE) t0 = s4 + TP(4, 4);
    if (s3 != PSB_WORST_SCORE) t1 = s3 + TP(3, 4);
    w = hmm_pick3(t0, t1, t2, s4);
    if (w == 2) { h.hist[4] = h.hist[2]; h.senid[4] = h.senid[2]; }
    else if (w == 1) { h.hist[4] = h.hist[3]; h.senid[4] = h.senid[3]; }
    PSB_FLOOR(s4); PSB_RAISE(best, s4);
    h.score[4] = s4;

    if (h.senid[1] == PSB_BAD_SSID) s1 = t2 = PSB_WORST_SCORE;
    else { s1 = h.score[1] + mpx_obs(c, senscr, h, 1); t2 = s1 + TP(1, 3); }
    t0 = t1 = PSB_WORST_SCORE;
    if (s3 != PSB_WORST_SCORE) t0 = s3 + TP(3, 3);
    if (s2 != PSB_WORST_SCORE) t1 = s2 + TP(2, 3);
    w = hmm_pick3(t0, t1, t2, s3);
    if (w == 2) { h.hist[3] = h.hist[1]; h.senid[3] = h.senid[1]; }
    else if (w == 1) { h.hist[3] = h.hist[2]; h.senid[3] = h.senid[2]; }
    PSB_FLOOR(s3); PSB_RAISE(best, s3);
    h.score[3] = s3;

    s0 = h.score[0] + mpx_obs(c, senscr, h, 0);
    t0 = t1 = PSB_WORST_SCORE;
    if (s2 != PSB_WORST_SCORE) t0 = s2 + TP(2, 2);
    if (s1 != PSB_WORST_SCORE) t1 = s1 + TP(1, 2);
    t2 = s0 + TP(0, 2);
    w = hmm_pick3(t0, t1, t2, s2);
    if (w == 2) { h.hist[2] = h.hist[0]; h.senid[2] = h.senid[0]; }
    else if (w == 1) { h.hist[2] = h.hist[1]; h.senid[2] = h.senid[1]; }
    PSB_FLOOR(s2); PSB_RAISE(best, s2);
    h.score[2] = s2;

    t0 = PSB_WORST_SCORE;
    if (s1 != PSB_WORST_SCORE) t0 = s1 + TP(1, 1);
    t1 = s0 + TP(0, 1);
    if (t0 > t1) s1 = t0;
    else { s1 = t1; h.hist[1] = h.hist[0]; h.senid[1] = h.senid[0]; }
    PSB_FLOOR(s1); PSB_RAISE(best, s1);
    h.score[1] = s1;

    s0 += TP(0, 0);
    PSB_FLOOR(s0); PSB_RAISE(best, s0);
    h.score[0] = s0;
    h.best = best;
    return best;
#undef TP
}

// hmm_vit_eval_anytopo (hmm.c:709-784) for n_emit in 1..5, mpx or not.
__device__ __forceinline__ int hmm_step_any(HmmReg &h, const HmmCtxDev &c, const uint8_t *tp, const int16_t *senscr, bool mpx)
{
    const int n = c.n_emit;
    int st[PSB_HMM_MAX_NSTATE];
#define TP(i, j) (-(int)tp[(i) * (n + 1) + (j)])
#pragma unroll
    for (int from = 0; from < PSB_HMM_MAX_NSTATE; ++from) {
        if (from < n) {
            int sid;
            if (mpx)
                sid = h.senid[from] == PSB_BAD_SSID ? PSB_BAD_SSID : c.sseq[(size_t)h.senid[from] * n + from];
            else
                sid = h.senid[from];
            const int o = sid == PSB_BAD_SSID ? PSB_WORST_SCORE : -(int)senscr[sid];
            int v = h.score[from] + o;
            if (from > 0 && v < PSB_WORST_SCORE) v = PSB_WORST_SCORE;
            st[from] = v;
        }
    }
    int scr = PSB_WORST_SCORE, bestfrom = -1, nscr, best;
#pragma unroll
    for (int from = PSB_HMM_MAX_NSTATE - 1; from >= 0; --from)
        if (from < n && TP(from, n) > PSB_TMAT_WORST && (nscr = st[from] + TP(from, n)) > scr) {
            scr = nscr;
            bestfrom = from;
        }
    h.out_score = scr;
#pragma unroll
    for (int q = 0; q < PSB_HMM_MAX_NSTATE; ++q)
        if (q == bestfrom) h.out_hist = h.hist[q];
    best = scr;
#pragma unroll
    for (int to = PSB_HMM_MAX_NSTATE - 1; to >= 0; --to) {
        if (to < n) {
            scr = TP(to, to) > PSB_TMAT_WORST ? st[to] + TP(to, to) : PSB_WORST_SCORE;
            bestfrom = -1;
#pragma unroll
            for (int from = PSB_HMM_MAX_NSTATE - 1; from >= 0; --from)
                if (from < to && TP(from, to) > PSB_TMAT_WORST && (nscr = st[from] + TP(from, to)) > scr) {
                    scr = nscr;
                    bestfrom = from;
                }
            h.score[to] = scr;
#pragma unroll
            for (int q = 0; q < PSB_HMM_MAX_NSTATE; ++q)
                if (q == bestfrom) {
                    h.hist[to] = h.hist[q];
                    if (mpx) h.senid[to] = h.senid[q];
                }
            if (best < scr) best = scr;
        }
    }
    h.best = best;
    return best;
#undef TP
}

// Dispatcher (hmm.c:786-805).  senscr: the frame's int16 scores.
__device__ __forceinline__ int hmm_step(HmmReg &h, const HmmCtxDev &c, int tmatid, bool mpx, const int16_t *senscr)
{
    const int n = c.n_emit;
    const uint8_t *tp = c.tp + (size_t)tmatid * n * (n + 1);
    if (!mpx && (n == 3 || n == 5)) {
        int obs[PSB_HMM_MAX_NSTATE];
#pragma unroll
        for (int i = 0; i < PSB_HMM_MAX_NSTATE; ++i) obs[i] = i < n ? -(int)senscr[h.senid[i]] : 0;
        return n == 3 ? hmm_step_3st(h, tp, obs) : hmm_step_5st(h, tp, obs);
    }
    if (mpx && n == 3) return hmm_step_3st_mpx(h, c, tp, senscr);
    if (mpx && n == 5) return hmm_step_5st_mpx(h, c, tp, senscr);
    return hmm_step_any(h, c, tp, senscr, mpx);
}

// An HMM set the whole-utterance kernels keep as a struct of arrays (shared or global memory): state s of
// HMM i at [s * stride + i], the exit state and the best score at [i].  BEST = false: the caller keeps no
// best score (best is not used), and a loaded HMM starts from WORST_SCORE.
template <bool BEST = true>
struct HmmSoA {
    int *score, *hist;            // [n_emit][stride]
    int *out_score, *out_hist;    // [stride]
    int *best;                    // [stride]
    int stride;

    // HMM i into registers.  Its senone ids are sen[s * sen_stride]; for a multiplexed channel (mss given)
    // its per-state senone-sequence ids are mss[s * stride + i] instead.
    template <class SenT>
    __device__ __forceinline__ void load(HmmReg &h, int i, int n, const SenT *sen, int sen_stride, const int *mss = nullptr) const
    {
#pragma unroll
        for (int s = 0; s < PSB_HMM_MAX_NSTATE; ++s) {
            h.score[s] = s < n ? score[s * stride + i] : PSB_WORST_SCORE;
            h.hist[s] = s < n ? hist[s * stride + i] : -1;
            h.senid[s] = s < n ? (mss ? mss[s * stride + i] : sen[s * sen_stride]) : PSB_BAD_SSID;
        }
        h.out_score = out_score[i]; h.out_hist = out_hist[i]; h.best = BEST ? best[i] : PSB_WORST_SCORE;
    }
    // HMM i back from registers; a multiplexed channel's senone-sequence ids, which follow the winning
    // predecessors, go back to mss
    __device__ __forceinline__ void store(const HmmReg &h, int i, int n, int *mss = nullptr) const
    {
#pragma unroll
        for (int s = 0; s < PSB_HMM_MAX_NSTATE; ++s)
            if (s < n) {
                score[s * stride + i] = h.score[s]; hist[s * stride + i] = h.hist[s];
                if (mss) mss[s * stride + i] = h.senid[s];
            }
        out_score[i] = h.out_score; out_hist[i] = h.out_hist;
        if (BEST) best[i] = h.best;
    }
    // hmm_clear (hmm.c:180-196) of HMM i; each caller resets its own frame field
    __device__ __forceinline__ void clear(int i, int n) const
    {
        for (int s = 0; s < n; ++s) { score[s * stride + i] = PSB_WORST_SCORE; hist[s * stride + i] = -1; }
        out_score[i] = PSB_WORST_SCORE; out_hist[i] = -1;
        if (BEST) best[i] = PSB_WORST_SCORE;
    }
};
