// psb_tm.cuh -- the tied-mixture senone arithmetic: one definition of each rule the reference applies after the top-N
// lists, shared by the batch senone kernels (psb_ptm.cu) and the per-frame scorer (psb_scorer.cu).
#pragma once
#include "psb_internal.cuh"

namespace {

constexpr int TOPN = 4;               // the batch kernels are specialised for -topn 4 (the default)
constexpr int SEN_BIAS = 64;          // > 3 * tab[0] for any 8-bit add table the 16x2 senone kernels accept

// fast_logmath_add (tied_mgau_common.h:111-127) on negated logs.  mixw + normalised score can
// reach 255 + 96, so |x - y| can exceed the reference's 256-entry table (logmath.c:116-120):
// the reference then reads past its allocation (undefined); the add table is identically 0 from
// entry ~30 on, so the kernels continue it with zeros up to PSB_LOGADD8_N entries.
__device__ __forceinline__ int logadd8(const uint8_t *tab, int x, int y)
{
    return min(x, y) - tab[abs(x - y)];
}

// One fast_logmath_add on two senones at once (unsigned 16x2): x holds the running values of two senones, the bytes of
// w that `sel` picks their next mixture weights, nvj the codeword's normalised score.  Every value carries SEN_BIAS so
// that the slightly negative intermediate results (>= -3 * tab[0]) stay non-negative halfwords: min, max and |x - y|
// are bias-free, min - tab[d] carries it.
__device__ __forceinline__ unsigned logadd8_16x2(const uint8_t *tab, unsigned x, unsigned w, unsigned sel, unsigned nvj)
{
    const unsigned y = __byte_perm(w, 0u, sel);
    const unsigned mn = __viaddmin_u16x2(y, nvj, x);
    const unsigned mx = __viaddmax_u16x2(y, nvj, x);
    const unsigned d = mx - mn;
    const unsigned t = (unsigned)tab[d & 0xffffu] | ((unsigned)tab[d >> 16] << 16);
    return mn - t;
}

// 4-bit mixture weights, two per byte, looked up in the 16-entry cluster table.  PTM picks the nibble by the low bit of
// the byte itself (ptm_mgau.c:376-377, sic); semi-continuous by the senone's parity (s2_semi_mgau.c:813-814).
__device__ __forceinline__ int ptm_weight4(const uint8_t *cb16, int b)
{
    return cb16[(b & 1) ? b >> 4 : b & 0x0f];
}
__device__ __forceinline__ int semi_weight4(const uint8_t *cb16, int b, int s)
{
    return cb16[(s & 1) ? b >> 4 : b & 0x0f];
}

// Byte offset of the weight row of codeword byte j of record bytes cwb, stream f, in the [f][cw][mixw_stride] table.
__device__ __forceinline__ unsigned tm_row(unsigned cwb, int j, int f, int nd, int mixw_stride)
{
    return ((unsigned)f * nd + ((cwb >> (8 * j)) & 0xff)) * (unsigned)mixw_stride;
}

// The 16x2 kernels' copy of four normalised scores: score + SEN_BIAS in both halfwords.
__device__ __forceinline__ uint4 sen_bias16x2(const unsigned (&nv)[TOPN])
{
    return make_uint4((nv[0] + SEN_BIAS) * 0x10001u, (nv[1] + SEN_BIAS) * 0x10001u,
                      (nv[2] + SEN_BIAS) * 0x10001u, (nv[3] + SEN_BIAS) * 0x10001u);
}

// ptm_mgau_codebook_norm (ptm_mgau.c:266-295), all codebooks active, over one frame's PTM top-N records (.x = best
// score >> 10, .y = codeword bytes, .z = bytes best - score_j, see psb_ptm.cu).  Thread tid < K takes pair tid: norm[f]
// becomes stream f's best score over the codebooks (norm[] preset to PSB_WORST_SCORE before a barrier, ptm_mgau.c:273),
// then rowoff[tid] = the listed codewords' weight rows, nsc[tid] = min(96, norm - (score_j >> 10)) (:277-291) and,
// for the 16x2 kernels (X2), nvp[tid] = their 16x2 copy.  The caller's barrier publishes rowoff / nsc / nvp.
template <bool X2>
__device__ __forceinline__ void ptm_norm_rows(const int4 *__restrict__ topn, long long frame, int K, int n_feat, int nd,
                                              int mixw_stride, int *norm, uint4 *rowoff, uint4 *nsc, uint4 *nvp)
{
    const int tid = threadIdx.x;
    int4 r = make_int4(0, 0, 0, 0);
    if (tid < K) {
        r = topn[frame * K + tid];
        atomicMax(&norm[tid % n_feat], r.x);
    }
    __syncthreads();
    if (tid < K) {
        const int f = tid % n_feat;
        const int base = norm[f] - r.x;
        const unsigned eb = (unsigned)r.z, cwb = (unsigned)r.y;
        unsigned ro[TOPN], nv[TOPN];
#pragma unroll
        for (int j = 0; j < TOPN; ++j) {
            int v = base + (int)((eb >> (8 * j)) & 0xff);
            nv[j] = (unsigned)(v > PSB_MAX_NEG_ASCR ? PSB_MAX_NEG_ASCR : v);
            ro[j] = tm_row(cwb, j, f, nd, mixw_stride);
        }
        rowoff[tid] = make_uint4(ro[0], ro[1], ro[2], ro[3]);
        nsc[tid] = make_uint4(nv[0], nv[1], nv[2], nv[3]);
        if (X2) nvp[tid] = sen_bias16x2(nv);
    }
}

// One frame's semi-continuous top-N records, already normalised by mgau_norm (s2_semi_mgau.c:186-203; .x = entries
// inside topn_beam, .y = codeword bytes, .z = normalised score bytes).  Thread tid < n_feat takes stream tid: rowoff,
// nsc, nvp (X2) as in ptm_norm_rows, cnt[tid] = the count.  The caller's barrier publishes them.
template <bool X2>
__device__ __forceinline__ void semi_rows(const int4 *__restrict__ topn, long long frame, int n_feat, int nd,
                                          int mixw_stride, uint4 *rowoff, uint4 *nsc, uint4 *nvp, int *cnt)
{
    const int tid = threadIdx.x;
    if (tid < n_feat) {
        const int4 r = topn[frame * n_feat + tid];
        const unsigned cwb = (unsigned)r.y, eb = (unsigned)r.z;
        unsigned ro[TOPN], nv[TOPN];
#pragma unroll
        for (int j = 0; j < TOPN; ++j) {
            ro[j] = tm_row(cwb, j, tid, nd, mixw_stride);
            nv[j] = (eb >> (8 * j)) & 0xff;
        }
        rowoff[tid] = make_uint4(ro[0], ro[1], ro[2], ro[3]);
        nsc[tid] = make_uint4(nv[0], nv[1], nv[2], nv[3]);
        if (X2) nvp[tid] = sen_bias16x2(nv);
        cnt[tid] = r.x;
    }
}

// ptm_mgau_senone_eval's chain for one senone and stream (ptm_mgau.c:366-392): log-add mixw + normalised score over
// the four listed codewords.  mw: the senone's column (byte s, or s / 2 for 4-bit weights); ro / nv: rowoff / nsc.
template <bool FOURBIT>
__device__ __forceinline__ int ptm_mix(const uint8_t *__restrict__ mw, uint4 ro, uint4 nv, const uint8_t *tab,
                                       const uint8_t *cb16)
{
    int w0 = mw[ro.x], w1 = mw[ro.y], w2 = mw[ro.z], w3 = mw[ro.w];
    if (FOURBIT) {
        w0 = ptm_weight4(cb16, w0); w1 = ptm_weight4(cb16, w1);
        w2 = ptm_weight4(cb16, w2); w3 = ptm_weight4(cb16, w3);
    }
    int fden = w0 + (int)nv.x;
    fden = logadd8(tab, fden, w1 + (int)nv.y);
    fden = logadd8(tab, fden, w2 + (int)nv.z);
    fden = logadd8(tab, fden, w3 + (int)nv.w);
    return fden;
}

// get_scores_{8b,4b}_feat_all's chain for senone s and one stream (s2_semi_mgau.c:425-444, 797-831): log-add mixw +
// normalised score over the first n listed codewords, at least one.
template <bool FOURBIT>
__device__ __forceinline__ int semi_mix(const uint8_t *__restrict__ mixw, int s, uint4 ro, uint4 nv, int n,
                                        const uint8_t *tab, const uint8_t *cb16)
{
    const unsigned rr[TOPN] = {ro.x, ro.y, ro.z, ro.w}, vv[TOPN] = {nv.x, nv.y, nv.z, nv.w};
    int tmp = 0;
#pragma unroll
    for (int k = 0; k < TOPN; ++k) {
        if (k == 0 || k < n) {
            const int w = FOURBIT ? semi_weight4(cb16, mixw[rr[k] + (unsigned)(s >> 1)], s) : mixw[rr[k] + (unsigned)s];
            const int v = w + (int)vv[k];
            tmp = k == 0 ? v : logadd8(tab, tmp, v);
        }
    }
    return tmp;
}

// The end of ptm_mgau_senone_eval (ptm_mgau.c:398-400): the block-wide minimum of every thread's `best` (through
// red[], one int per warp), then dst[s] = asc[s] - best for every senone.
__device__ __forceinline__ void store_relative_to_best(int best, int *red, const int16_t *asc, int16_t *dst, int n_sen)
{
    const int tid = threadIdx.x;
    best = __reduce_min_sync(0xffffffffu, best);
    if ((tid & 31) == 0) red[tid >> 5] = best;
    __syncthreads();
    if (tid < 32) {
        int v = tid < (int)(blockDim.x >> 5) ? red[tid] : 0x7fffffff;
        v = __reduce_min_sync(0xffffffffu, v);
        if (tid == 0) red[0] = v;
    }
    __syncthreads();
    best = red[0];
    for (int s = tid; s < n_sen; s += blockDim.x)
        dst[s] = (int16_t)(asc[s] - best);
}

}  // namespace
