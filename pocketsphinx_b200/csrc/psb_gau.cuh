// psb_gau.cuh -- the Gaussian exponent with the reference's roundings, shared by the top-N kernels
// (psb_ptm.cu: scans over time; psb_ptm_tc.cu: tensor-core filter + exact rescoring; psb_scorer.cu: per frame).
#pragma once
#include "psb_internal.cuh"

namespace {

__device__ __forceinline__ int f2i_clamped(float d)
{
    // (int32)d, clamped first like ptm_mgau.c:129-132,219-222.  cvt.rzi saturates, which is
    // the same thing for d < INT_MIN; d > INT_MAX cannot occur (d <= det).
    return __float2int_rz(d);
}

// FIXED_POINT build of the reference (mfcc_t = int32 Q12, SURVEY A.1.11).  FIXMUL (fe/fixpoint.h:98-100) is the
// 64-bit product shifted right by 12 and truncated to 32 bits; GMMSUB (tied_mgau_common.h:62-66) as gcc compiles it
// is (b < 0) ? INT_MIN : wrap32(a - b).
__device__ __forceinline__ int fx_mul(int a, int b)
{
    return (int)(unsigned)(((long long)a * (long long)b) >> 12);
}
__device__ __forceinline__ int fx_gmmsub(int a, int b)
{
    return b < 0 ? INT_MIN : (int)((unsigned)a - (unsigned)b);
}

// dpen (optional) = the partial sum before the last dimension's term: the semi-continuous
// back-end's early-exit test sees that value (s2_semi_mgau.c:137-143, SURVEY A.1.3).
template <int FL, bool PEN = false>
__device__ __forceinline__ float gau_dist(const float4 *__restrict__ r, const float (&x)[FL], float *dpen = nullptr)
{
    constexpr int RECF = (1 + 2 * FL + 3) / 4 * 4;
    float rr[RECF];
#pragma unroll
    for (int q = 0; q < RECF / 4; ++q) {
        float4 v = r[q];
        rr[4 * q + 0] = v.x; rr[4 * q + 1] = v.y; rr[4 * q + 2] = v.z; rr[4 * q + 3] = v.w;
    }
    float d = rr[0];
#pragma unroll
    for (int j = 0; j < FL; ++j) {
        float diff = __fsub_rn(x[j], rr[1 + 2 * j]);
        float sq = __fmul_rn(diff, diff);
        float c = __fmul_rn(sq, rr[2 + 2 * j]);
        if (PEN && j == FL - 1) *dpen = d;
        d = __fsub_rn(d, c);
    }
    return d;
}

// ---------------------------------------------------------------------------------------
// Pair variant (psb_fadd2_rn/psb_fmul2_rn: two scalar .rn operations each on sm_90): two *codewords* per
// instruction.  Records are stored pair-interleaved with NEGATED means and variance terms,
//   {detA, detB, -muA_0, -muB_0, -vA_0, -vB_0, -muA_1, ...}            (psb_api.cu build_records)
// so that the reference's sub / mul / mul / sub chain becomes add / mul / mul / add on float2:
//   x - mu == x + (-mu),  (sq * v) negated == sq * (-v),  d - c == d + (-c)   -- all exact in IEEE,
// and each half rounds exactly like __fadd_rn/__fmul_rn; one record load serves two codewords.
// The final accumulation stays SCALAR, as in gau_dist.
template <int FL, bool PEN = false>
__device__ __forceinline__ float2 gau_dist2(const float4 *__restrict__ r, const float2 (&xx)[FL], float2 *dpen = nullptr)
{
    constexpr int RECF2 = (2 + 4 * FL + 3) / 4 * 4;
    float2 rr[RECF2 / 2];
#pragma unroll
    for (int q = 0; q < RECF2 / 4; ++q) {
        const float4 v = r[q];
        rr[2 * q] = make_float2(v.x, v.y);
        rr[2 * q + 1] = make_float2(v.z, v.w);
    }
    float2 d = rr[0];
#pragma unroll
    for (int j = 0; j < FL; ++j) {
        float2 t = psb_fadd2_rn(xx[j], rr[1 + 2 * j]);
        t = psb_fmul2_rn(t, t);
        t = psb_fmul2_rn(t, rr[2 + 2 * j]);
        if (PEN && j == FL - 1) *dpen = d;
        d.x = __fadd_rn(d.x, t.x);
        d.y = __fadd_rn(d.y, t.y);
    }
    return d;
}


}  // namespace
