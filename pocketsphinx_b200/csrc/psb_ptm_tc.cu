// psb_ptm_tc.cu -- PTM top-N selection without the recurrence over time: a tensor-core filter,
// exact rescoring of the few survivors, and a sequential fix-up for exact ties.
//
// What the reference computes per frame and (codebook, stream) pair is a list of four codewords:
// eval_topn re-scores last frame's four, eval_cb scans all codewords in order and inserts every one
// whose distance beats the current worst (ptm_mgau.c:88-226).  ptm_topnq_kernel (psb_ptm.cu)
// follows that literally: time is sequential, every frame evaluates all 256 distances.  Two facts
// make most of that work unnecessary, with the SAME bits in the result:
//
//  (1) The list does not depend on the previous frame unless scores tie.  Let s(1) >= s(2) >= ...
//      be the truncated integer scores of ALL codewords of the pair in this frame.  The worst
//      listed score only rises during a scan and every codeword that is rejected or evicted has a
//      score <= the final worst, so the final worst is >= s(4).  If s(1) > s(2) > s(3) > s(4) > s(5),
//      each of the four best is accepted when the scan (or eval_topn) meets it -- at most three
//      listed scores exceed its own and none equals it, so the worst listed score is smaller and
//      `d >= (float)worst` holds -- and can never be evicted.  The list is then exactly those four
//      in descending order, whatever the seeds were.  Only when two of the five best integer scores
//      coincide do the order-dependent rules (`>=` shifting, strict `>` in eval_topn,
//      skip-if-listed) matter; those frames are flagged and redone by ptm_fixup_warp_kernel, which
//      replays the reference's loop literally with the previous frame's list as seeds.
//  (2) The five best can be found without computing 256 exact distances.  With y = x - m (m = the
//      codebook's mean centre) the exponent d = det - sum_j v_j (y_j - mu'_j)^2 is the inner product
//      of X = (y_j^2, y_j, 1) with W_c = (-v_cj, 2 v_cj mu'_cj, det_c - sum_j v_cj mu'_cj^2): one
//      [frames x 32] x [32 x n_density] GEMM per pair on the tensor cores, as 3 x TF32 (lo*hi + hi*lo
//      + hi*hi; W is split into TF32 halves on the host) with warpgroup MMA (ptm_wgmma_kernel).
//      Its result a_c differs from the reference's float d_c by at most
//      eps = ERR * (sum_j Amax_j y_j^2 + Bmax_j |y_j| + Cmax), a bound every row computes for itself
//      (Amax/Bmax/Cmax: per-pair maxima of |W| entries).  Five distinct codewords with a_c >= L0 (the
//      fifth largest of eight group maxima of the row) give the integer L' = floor(L0 - eps) - 1 <= s(5) - 1,
//      and every codeword with s_c >= s(5) has d_c > L', hence a_c >= L' - eps: the candidate set C
//      (about seven of 256 on the BASELINE shape).
//
// A row is then decided from the filter values alone when its five largest a_c are more than 2 eps + 1
// apart and the `>> 10` of the four best is the same at both ends of [a - eps, a + eps]: the record
// is certain without one exact distance.  Otherwise the row's candidate codewords (all of them when
// C has more than TC_CAP members) get the reference's exact float arithmetic, one thread per row, from
// ptm_wgmma_kernel's work list served by ptm_tc_exact_kernel.
//
// Nothing here is approximate in its output: tests/test_gpu_parity.py compares every record with the
// oracle's lists, PSB_TC_CHECK=1 makes the filter kernel measure max |a_c - d_c| / eps on the device.
#include "psb_gau.cuh"
#include "psb_internal.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace {

constexpr int TC_ROWS = 128;          // frames per CTA and tile (2 warpgroups x 64 rows)
constexpr int TC_K = 32;              // GEMM depth: 2 * FL + 1 <= 32
constexpr int TC_CAP = 18;            // candidate codewords per row: the byte list a work-list item carries
constexpr float TC_ERR = 1.0f / 262144.f;  // 2^-18 of the magnitude sum S: 3 x TF32 leaves 3 * 2^-22 per product, the rest is
                                           // room for the tensor core's fp32 accumulation (<= 2^-23 per step assumed, 12 steps per
                                           // chain) and the reference's own 52 roundings; PSB_TC_CHECK=1 measures what is used of it

// PSB_TC_CHECK builds only: 64-bit counters at byte 16 of the batch's debug block (psb_batch_tc_counters)
enum {
    ST_ROWS, ST_FILTER_ALONE, ST_EXACT_DIST, ST_TIE_FLAGS,
    ST_OVER_CAP,                                   // rows with more than TC_CAP candidates
    ST_LANE_OVER,                                  // rows where one quad lane stored more than TC_CAP pairs
    ST_FALLBACK_LISTED, ST_FALLBACK_ALL,           // rows in doubt rescored in the filter kernel (work list full)
    ST_SPLIT,                                      // rows in doubt whose candidate bytes came from both threads
    ST_FAIL_GAP, ST_FAIL_STRADDLE, ST_FAIL_SIGN, ST_FAIL_SAT,   // listed rows failing each certainty test
    ST_N
};
constexpr size_t TC_CHECK_BYTES = 16 + 8 * ST_N;

__device__ __forceinline__ float to_tf32(float x)
{
    unsigned r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

struct Top5 {
    int s[5];
    unsigned c;           // codewords of entries 0..3, byte j = entry j
    int c4;               // codeword of entry 4 (unused by the record)
    int n;
};

__device__ __forceinline__ void top5_insert(Top5 &t, int s, int c)
{
    // sorted descending; equal scores keep arrival order (irrelevant: ties are redone by the fix-up)
    int p = 0;
#pragma unroll
    for (int j = 0; j < 5; ++j) p += (j < t.n && t.s[j] >= s) ? 1 : 0;
    if (p >= 5) return;
#pragma unroll
    for (int j = 4; j >= 1; --j)
        if (j > p) t.s[j] = t.s[j - 1];
#pragma unroll
    for (int j = 0; j < 5; ++j)
        if (j == p) t.s[j] = s;
    // codeword bytes: entries p..3 move up one byte, entry 3 falls into c4
    if (p < 4) {
        const unsigned lowmask = p == 0 ? 0u : (0xffffffffu >> (32 - 8 * p));
        t.c4 = (int)(t.c >> 24);
        t.c = (t.c & lowmask) | ((unsigned)c << (8 * p)) | ((t.c << 8) & ~(lowmask | (0xffu << (8 * p))));
    }
    else
        t.c4 = c;
    if (t.n < 5) ++t.n;
}

// ---------------------------------------------------------------------------------------
// The filter on Hopper's warpgroup MMA: each warpgroup issues twelve wgmma.mma_async m64nNDk8 TF32 (lo*hi, hi*lo,
// hi*hi over four K steps) per 64 frames, A (X rows split into TF32 halves) and B (W, both halves) straight from shared
// memory in the canonical K-major no-swizzle layout, the fp32 accumulator in registers.  A frame's row is spread over the
// four lanes of a quad: group maxima meet by shuffles; each lane then stores, without a branch or an atomic, the column
// pairs of its rows whose larger value passes the threshold (predicated stores to its own slots, one mask bit per pair),
// and two threads per row -- all four warps -- pick the five largest candidates and decide the row.  The two warpgroups of
// a CTA share W and run their 64-frame halves independently (named barriers), so the GEMM of one overlaps the selection
// of the other, and each issues its next tile's GEMM before it resolves the rows of the current one; a CTA walks
// `tiles_per_cta` consecutive tiles of its pair.
constexpr int WG_ROWS = 64;                                                   // frames per warpgroup and tile
constexpr int WG_SLOTS = (TC_CAP + 1) * WG_ROWS * 4;                         // candidate pairs: [slot][row][quad lane], slot TC_CAP absorbs overflow
constexpr int WG_EXTRA = WG_SLOTS * 8 + WG_ROWS * 4 * 4 + WG_ROWS * 4 + 2 * WG_ROWS * 4 + WG_ROWS * 20;   // pairs, masks, thresholds, bounds, codewords

__device__ __forceinline__ uint64_t wgmma_desc(const void *p, unsigned lbo_bytes, unsigned sbo_bytes)
{
    // sm_90 shared-memory matrix descriptor: start address, leading (K direction) and stride (M / N direction) byte
    // offsets between core matrices, all in 16-byte units; base offset 0, layout type 0 = no swizzle
    const uint64_t a = (uint64_t)(((unsigned)__cvta_generic_to_shared(p) >> 4) & 0x3fffu);
    return a | ((uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32);
}

// the accumulator registers pass through here: nothing that reads or writes them moves across a wgmma fence or wait
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ void warpgroup_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// D[64 x N] (+)= A[64 x 8] * B[8 x N], TF32 in, fp32 accumulate, A and B from shared memory (descriptors)
template <int N>
struct Wgmma;
#define PSB_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
template <> struct Wgmma<64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, int accumulate)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\nwgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
        "%30,%31"
        "}, %32, %33, p, 1, 1;\n}\n"
        : PSB_ACC8(0), PSB_ACC8(8), PSB_ACC8(16), PSB_ACC8(24)
        : "l"(a), "l"(b), "r"(accumulate));
    }
};
template <> struct Wgmma<128> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, int accumulate)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\nwgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
        "%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,"
        "%57,%58,%59,%60,%61,%62,%63"
        "}, %64, %65, p, 1, 1;\n}\n"
        : PSB_ACC8(0), PSB_ACC8(8), PSB_ACC8(16), PSB_ACC8(24), PSB_ACC8(32), PSB_ACC8(40), PSB_ACC8(48), PSB_ACC8(56)
        : "l"(a), "l"(b), "r"(accumulate));
    }
};
template <> struct Wgmma<256> {
    static __device__ __forceinline__ void mma(float (&d)[128], uint64_t a, uint64_t b, int accumulate)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\nwgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
        "%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,"
        "%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,"
        "%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,"
        "%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
        "}, %128, %129, p, 1, 1;\n}\n"
        : PSB_ACC8(0), PSB_ACC8(8), PSB_ACC8(16), PSB_ACC8(24), PSB_ACC8(32), PSB_ACC8(40), PSB_ACC8(48), PSB_ACC8(56),
          PSB_ACC8(64), PSB_ACC8(72), PSB_ACC8(80), PSB_ACC8(88), PSB_ACC8(96), PSB_ACC8(104), PSB_ACC8(112),
          PSB_ACC8(120)
        : "l"(a), "l"(b), "r"(accumulate));
    }
};
#undef PSB_ACC8

//   wumma   [K][2][8][ND][4] float   W halves (high, low) in the canonical K-major layout: chunk kc holds k = 4 kc .. 4 kc + 3
template <int FL, int ND, bool CHECK>
__global__ void __launch_bounds__(2 * 128, 1)
ptm_wgmma_kernel(const float *__restrict__ feats, long long total, int D, const int32_t *__restrict__ featoff,
                 const int32_t *__restrict__ klist, const float *__restrict__ wumma, const float *__restrict__ cen,
                 const float *__restrict__ bnd, const float *__restrict__ rec, const size_t *__restrict__ rec_off,
                 int4 *__restrict__ out, unsigned *__restrict__ flags, long long flag_words, int K, int n_feat,
                 int tiles_per_cta, uint4 *__restrict__ items, unsigned *__restrict__ n_items, unsigned item_cap,
                 float *__restrict__ check, unsigned long long *__restrict__ stats)
{
    constexpr int RF = (1 + 2 * FL + 3) / 4 * 4;
    constexpr int NTL = ND / 8;                          // 8-column n-tiles of the accumulator fragment
    constexpr int NPG = NTL / 8;                         // n-tiles per maximum group: 8 groups per row
    constexpr unsigned FULL = 0xffffffffu;
    static_assert(2 * FL + 1 <= TC_K && (ND == 64 || ND == 128 || ND == 256), "shape");
    extern __shared__ __align__(128) unsigned char wg_smem[];
    const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127, warp = t >> 5, lane = tid & 31;
    float *sW = reinterpret_cast<float *>(wg_smem);                                   // [2][8][ND][4]
    float *sX = sW + 2 * 8 * ND * 4 + wg * (2 * 8 * WG_ROWS * 4);                     // this warpgroup's [2][8][64][4]
    unsigned char *ex = wg_smem + (size_t)2 * 8 * ND * 16 + 2 * (2 * 8 * WG_ROWS * 16) + (size_t)wg * WG_EXTRA;
    float2 *Pv = reinterpret_cast<float2 *>(ex);                                      // [TC_CAP + 1][64][4] candidate column pairs
    unsigned *Pm = reinterpret_cast<unsigned *>(Pv + WG_SLOTS);                       // [64][4] n-tiles of the stored pairs
    float *thrs = reinterpret_cast<float *>(Pm + WG_ROWS * 4);                        // [64] candidate threshold per row
    float *epsr = thrs + WG_ROWS;                                                     // [2][64] error bound per row (two tiles)
    unsigned *Lc = reinterpret_cast<unsigned *>(epsr + 2 * WG_ROWS);                  // [64][5] candidate codewords (bytes)

    // grid: x = pair (fastest), y = group of tiles: CTAs that run together read the SAME frames for different pairs, so
    // the feature rows come out of L2 while the W blocks of all pairs stay L2-resident
    const int k = klist[blockIdx.x];
    const int f = k % n_feat;
    {
        const float4 *src = reinterpret_cast<const float4 *>(wumma + (size_t)k * 2 * 8 * ND * 4);
        float4 *dst = reinterpret_cast<float4 *>(sW);
        for (int i = tid; i < 2 * 8 * ND; i += 2 * 128) dst[i] = src[i];
    }
    __syncthreads();
    const float *m = cen + (size_t)k * 16, *bb = bnd + (size_t)k * 32;
    const float *rc = rec + rec_off[k];
    const int r = t & (WG_ROWS - 1), half = t >> 6;     // the frame whose X row this thread prepares (half of its chunks)
    const int g = lane >> 2, q4 = lane & 3;
    const int ra = warp * 16 + g, rb = ra + 8;           // the two accumulator rows this thread holds columns of

    // ---- a tile's frames: X rows (TF32 halves, canonical layout; two threads share the stores of a row) and error bounds ----
    float xn[FL];                                        // the feature row of the frame this thread prepares next
    auto fetch = [&](long long row) {
        const float *p = feats + (row < total ? row : 0) * D + featoff[f];
#pragma unroll
        for (int j = 0; j < FL; ++j) xn[j] = row < total ? p[j] : 0.f;
    };
    auto prepare = [&](float *eps) {
        float v[TC_K];
        float S = bb[2 * FL];
#pragma unroll
        for (int j = 0; j < FL; ++j) {
            const float y = __fsub_rn(xn[j], m[j]);
            const float y2 = __fmul_rn(y, y);
            v[j] = y2;
            v[FL + j] = y;
            if (half == 0) {                                      // the thread that stores the bound (warp-uniform)
                S = __fadd_ru(S, __fmul_ru(bb[j], y2));           // no FMA anywhere in these kernels: tests/test_abi.py greps for it
                S = __fadd_ru(S, __fmul_ru(bb[FL + j], fabsf(y)));
            }
        }
        v[2 * FL] = 1.0f;
#pragma unroll
        for (int j = 2 * FL + 1; j < TC_K; ++j) v[j] = 0.f;
#pragma unroll
        for (int kc = 0; kc < 8; ++kc) {
            if ((kc & 1) != half) continue;
            float4 h, l;
            h.x = to_tf32(v[4 * kc]); h.y = to_tf32(v[4 * kc + 1]); h.z = to_tf32(v[4 * kc + 2]); h.w = to_tf32(v[4 * kc + 3]);
            l.x = to_tf32(__fsub_rn(v[4 * kc], h.x)); l.y = to_tf32(__fsub_rn(v[4 * kc + 1], h.y));
            l.z = to_tf32(__fsub_rn(v[4 * kc + 2], h.z)); l.w = to_tf32(__fsub_rn(v[4 * kc + 3], h.w));
            reinterpret_cast<float4 *>(sX)[kc * WG_ROWS + r] = h;
            reinterpret_cast<float4 *>(sX)[(8 + kc) * WG_ROWS + r] = l;
        }
        if (half == 0) eps[r] = __fadd_ru(__fmul_ru(S, TC_ERR), 2.0f);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> visible to the tensor core
        warpgroup_bar(1 + wg);
    };
    // ---- 3 x TF32 GEMM of the warpgroup's 64 rows against all ND codewords, issued asynchronously ----
    float acc[ND / 2];
    auto gemm = [&]() {
#pragma unroll
        for (int i = 0; i < ND / 2; ++i) acc[i] = 0.f;
        wgmma_fence_regs(acc);
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
        // chunk kc of A at sX + kc * 1024 B (64 rows x 16 B), of B at sW + kc * ND * 16 B; core matrices 128 B apart
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {           // lo*hi, hi*lo, hi*hi
            const int ha = pass == 0 ? 1 : 0, hb = pass == 1 ? 1 : 0;
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const uint64_t ad = wgmma_desc(sX + (size_t)(ha * 8 + 2 * ks) * WG_ROWS * 4, WG_ROWS * 16, 128);
                const uint64_t bd = wgmma_desc(sW + (size_t)(hb * 8 + 2 * ks) * ND * 4, ND * 16, 128);
                Wgmma<ND>::mma(acc, ad, bd, (pass | ks) ? 1 : 0);
            }
        }
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    };

    // ---- the rows of a tile whose candidates are stored: two threads per row; thread h takes the pairs of quad lanes 2 h
    // and 2 h + 1, keeps its five largest candidates and writes its candidate codewords to the row's byte list (h = 0 from
    // the front, h = 1 from byte TC_CAP - 1 down: they meet only if the row has more than TC_CAP candidates); the halves
    // meet by shuffles ----
    auto resolve = [&](const long long row0, const float *eps) {
        const int rr = t >> 1, h = t & 1;
        const long long row = row0 + rr;
        const bool valid = row < total;
        unsigned char *lb = reinterpret_cast<unsigned char *>(Lc + rr * 5);
        float a[5] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY, -INFINITY};
        int c[5] = {0, 0, 0, 0, 0};
        int nl = 0;
        bool over = false;                               // a lane of the row kept more than TC_CAP pairs
        {
            const float thr = thrs[rr];
            auto cand = [&](float v, int col) {
                const bool p = v >= thr;
                if (p && nl < TC_CAP) lb[h ? TC_CAP - 1 - nl : nl] = (unsigned char)col;
                nl += p ? 1 : 0;
                v = p ? v : -INFINITY;
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    const bool s = v > a[j];
                    const float tv = a[j];
                    const int tc = c[j];
                    a[j] = s ? v : tv; c[j] = s ? col : tc;
                    v = s ? tv : v; col = s ? tc : col;
                }
            };
            // one loop over the stored pairs of both lanes (the first TC_CAP of each): a warp runs as many iterations as
            // its busiest thread has pairs
            unsigned m0 = Pm[rr * 4 + 2 * h], m1 = Pm[rr * 4 + 2 * h + 1];
            over = __popc(m0) > TC_CAP || __popc(m1) > TC_CAP;
            int j0 = 0, j1 = 0;
            while ((m0 | m1) != 0u) {
                const bool first = m0 != 0u;
                const unsigned msk = first ? m0 : m1;
                const int i = __ffs(msk) - 1, q = 2 * h + (first ? 0 : 1), j = first ? j0 : j1;
                const float2 v = Pv[j * WG_ROWS * 4 + rr * 4 + q];
                cand(v.x, 8 * i + 2 * q);
                cand(v.y, 8 * i + 2 * q + 1);
                if (first) { m0 = ++j0 < TC_CAP ? m0 & (m0 - 1u) : 0u; }
                else { m1 = ++j1 < TC_CAP ? m1 & (m1 - 1u) : 0u; }
            }
        }
        const int n1 = __shfl_xor_sync(FULL, nl, 1), n = nl + n1;
        over = __shfl_xor_sync(FULL, (int)over, 1) != 0 || over;
        {
            // the five largest of the row: max(a[j], b[4 - j]) over the two sorted halves, then a sorting network
            float b[5];
            int bc[5];
#pragma unroll
            for (int j = 0; j < 5; ++j) { b[j] = __shfl_xor_sync(FULL, a[j], 1); bc[j] = __shfl_xor_sync(FULL, c[j], 1); }
#pragma unroll
            for (int j = 0; j < 5; ++j)
                if (b[4 - j] > a[j]) { a[j] = b[4 - j]; c[j] = bc[4 - j]; }
            auto cmpx = [&](int i, int j) {
                if (a[j] > a[i]) { const float tv = a[i]; const int tc = c[i]; a[i] = a[j]; c[i] = c[j]; a[j] = tv; c[j] = tc; }
            };
            cmpx(0, 1); cmpx(3, 4); cmpx(2, 4); cmpx(2, 3); cmpx(1, 4); cmpx(0, 3); cmpx(0, 2); cmpx(1, 3); cmpx(1, 2);
        }
        const bool listed = n >= 5 && n <= TC_CAP && !over;
        const float ee = eps[rr];

        // ---- the record straight from the filter values when they leave no doubt ----
        bool certain = listed;
        {
            // order and distinctness of the truncated scores: neighbours more than 2 eps + 1 apart, everything safely
            // negative (truncation is towards zero); s >> 10 of the four best: the same at both ends of [a - eps, a + eps]
            const float gap = __fadd_ru(__fadd_ru(ee, ee), 1.0f);
            int qv[4];
            bool gap_ok = true, straddle_ok = true;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                gap_ok &= __fsub_rd(a[j], a[j + 1]) > gap;
                const int lo = __float2int_ru(__fsub_rd(a[j], ee)), hi = __float2int_ru(__fadd_ru(a[j], ee));
                straddle_ok &= (lo >> PSB_SENSCR_SHIFT) == (hi >> PSB_SENSCR_SHIFT);
                qv[j] = lo >> PSB_SENSCR_SHIFT;
            }
            const bool sign_ok = __fadd_ru(a[0], ee) < -2.0f, sat_ok = a[4] > -2.0e9f;
            certain &= gap_ok && straddle_ok && sign_ok && sat_ok;
            if (valid && h == 0) {
                if (CHECK) {
                    atomicMax(reinterpret_cast<int *>(check) + 1, n);
                    if (n > TC_CAP) atomicAdd(stats + ST_OVER_CAP, 1ull);
                    if (over) atomicAdd(stats + ST_LANE_OVER, 1ull);
                    if (listed) {
                        if (!gap_ok) atomicAdd(stats + ST_FAIL_GAP, 1ull);
                        if (!straddle_ok) atomicAdd(stats + ST_FAIL_STRADDLE, 1ull);
                        if (!sign_ok) atomicAdd(stats + ST_FAIL_SIGN, 1ull);
                        if (!sat_ok) atomicAdd(stats + ST_FAIL_SAT, 1ull);
                    }
                }
                if (certain) {
                    unsigned cb = 0, eb = 0;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        int ev = qv[0] - qv[j];
                        ev = ev > 255 ? 255 : ev;
                        cb |= (unsigned)c[j] << (8 * j);
                        eb |= (unsigned)ev << (8 * j);
                    }
                    out[row * K + k] = make_int4(qv[0], (int)cb, (int)eb, 0);
                    if (CHECK) { atomicAdd(stats, 1ull); atomicAdd(stats + 1, 1ull); }
                }
            }
        }
        // ---- doubt: the row goes to ptm_tc_exact_kernel's work list (one atomic per warp); only when that list is full
        // is the exact arithmetic done here ----
        __syncwarp();                                    // the partner's codeword bytes are in the row's list
        const bool doubt = valid && h == 0 && !certain;
        const int n0 = listed ? nl : 255, nb = listed ? n1 : 0;   // n0 = 255: all codewords
        if (CHECK && doubt && listed && nl > 0 && n1 > 0) atomicAdd(stats + ST_SPLIT, 1ull);
        bool handled = false;
        if (items) {
            const unsigned need = __ballot_sync(FULL, doubt);
            if (need) {
                const int leader = __ffs(need) - 1;
                unsigned base = 0;
                if (lane == leader) base = atomicAdd(n_items, (unsigned)__popc(need));
                base = __shfl_sync(FULL, base, leader);
                const unsigned slot = base + (unsigned)__popc(need & ((1u << lane) - 1u));
                if (doubt && slot < item_cap) {
                    const unsigned *w = Lc + rr * 5;
                    items[2 * (size_t)slot] = make_uint4((unsigned)row, (unsigned)k | ((unsigned)n0 << 16) | ((unsigned)nb << 24), w[0], w[1]);
                    items[2 * (size_t)slot + 1] = make_uint4(w[2], w[3], w[4], (unsigned)(row >> 32));
                    handled = true;
                    if (CHECK) atomicAdd(stats, 1ull);
                }
            }
        }
        if (doubt && !handled) {
            // the reference's exact arithmetic for this row's candidates (all codewords if the list overflowed)
            float x[FL];
            const float *px = feats + row * D + featoff[f];
#pragma unroll
            for (int j = 0; j < FL; ++j) x[j] = px[j];
            Top5 top;
            top.n = 0; top.c = 0u; top.c4 = 0;
#pragma unroll
            for (int j = 0; j < 5; ++j) top.s[j] = INT_MIN;
            const int cnt_l = listed ? n : ND;
            if (CHECK) atomicAdd(stats + (listed ? ST_FALLBACK_LISTED : ST_FALLBACK_ALL), 1ull);
            for (int i = 0; i < cnt_l; ++i) {
                const int cw = listed ? (int)lb[i < n0 ? i : i - n0 + TC_CAP - nb] : i;
                const float d = gau_dist<FL>(reinterpret_cast<const float4 *>(rc + (size_t)cw * RF), x);
                top5_insert(top, f2i_clamped(d), cw);
            }
            const bool distinct = top.n >= 5 && top.s[0] > top.s[1] && top.s[1] > top.s[2] && top.s[2] > top.s[3] && top.s[3] > top.s[4];
            const int tp = top.s[0] >> PSB_SENSCR_SHIFT;
            unsigned eb = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int ev = tp - (top.s[j] >> PSB_SENSCR_SHIFT);
                ev = ev > 255 ? 255 : ev;
                eb |= (unsigned)ev << (8 * j);
            }
            out[row * K + k] = make_int4(tp, (int)top.c, (int)eb, 0);
            if (!distinct) atomicOr(&flags[(size_t)k * flag_words + (row >> 5)], 1u << (row & 31));
            if (CHECK) { atomicAdd(stats, 1ull); atomicAdd(stats + 2, (unsigned long long)cnt_l); if (!distinct) atomicAdd(stats + 3, 1ull); }
        }
    };

    // the next tile's GEMM runs on the tensor core while this tile's rows are resolved: X and its bounds are written as
    // soon as this tile's candidates are stored (its GEMM is complete then), the bounds alternate between two buffers
    long long row0 = (long long)blockIdx.y * tiles_per_cta * TC_ROWS + wg * WG_ROWS;
    if (row0 >= total) return;                           // uniform in the warpgroup: its rows lie past the end
    fetch(row0 + r);
    prepare(epsr);
    int buf = 0;                                         // the bounds buffer of the current tile
    for (int tile = 0;; ++tile, buf ^= 1, row0 += TC_ROWS) {
        gemm();
        const bool more = tile + 1 < tiles_per_cta && row0 + TC_ROWS < total;
        if (more) fetch(row0 + TC_ROWS + r);
        if (tile > 0) {
            resolve(row0 - TC_ROWS, epsr + (buf ^ 1) * WG_ROWS);
            warpgroup_bar(1 + wg);                       // lists consumed: this tile may overwrite pairs and lists
        }
        const float *eps = epsr + buf * WG_ROWS;
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        wgmma_fence_regs(acc);

        // ---- rows ra / rb: group maxima (the quad's four lanes hold a row between them), threshold, the columns above it ----
        float gma[8], gmb[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            float a = -INFINITY, b = -INFINITY;
#pragma unroll
            for (int i = q * NPG; i < (q + 1) * NPG; ++i) {     // a chain: the pair maxima below are not kept live
                a = fmaxf(fmaxf(a, acc[4 * i]), acc[4 * i + 1]);
                b = fmaxf(fmaxf(b, acc[4 * i + 2]), acc[4 * i + 3]);
            }
            a = fmaxf(a, __shfl_xor_sync(FULL, a, 1)); a = fmaxf(a, __shfl_xor_sync(FULL, a, 2));
            b = fmaxf(b, __shfl_xor_sync(FULL, b, 1)); b = fmaxf(b, __shfl_xor_sync(FULL, b, 2));
            gma[q] = a; gmb[q] = b;
        }
        // five distinct columns >= L0: the fifth largest of the eight group maxima.  With both halves sorted (descending)
        // it is max_i min(first[i], second[3 - i])
        auto fifth = [](float (&gm)[8]) {
            auto cmpx = [&](int i, int j) { const float hi = fmaxf(gm[i], gm[j]); gm[j] = fminf(gm[i], gm[j]); gm[i] = hi; };
#pragma unroll
            for (int o = 0; o < 8; o += 4) { cmpx(o, o + 1); cmpx(o + 2, o + 3); cmpx(o, o + 2); cmpx(o + 1, o + 3); cmpx(o + 1, o + 2); }
            return fmaxf(fmaxf(fminf(gm[0], gm[7]), fminf(gm[1], gm[6])), fmaxf(fminf(gm[2], gm[5]), fminf(gm[3], gm[4])));
        };
        const float e_a = eps[ra], e_b = eps[rb];
        // L' = floor(L0 - eps) - 1, candidates: a_c >= L' - eps; every step rounded towards -inf
        const float thra = __fsub_rd(__fsub_rd(floorf(__fsub_rd(fifth(gma), e_a)), 1.0f), e_a);
        const float thrb = __fsub_rd(__fsub_rd(floorf(__fsub_rd(fifth(gmb), e_b)), 1.0f), e_b);
        {
            // the lane's pair (8 i + 2 q4, + 1) of a row is kept when its larger value passes: predicated stores to the
            // lane's next slot and a mask bit, no branch; past TC_CAP pairs the lane writes the overflow slot again (the row
            // then has more than TC_CAP candidates, and its mask says so)
            constexpr int SS = WG_ROWS * 4;                  // slot stride in pairs
            int oa = ra * 4 + q4, ob = rb * 4 + q4;
            const int lim_a = oa + TC_CAP * SS, lim_b = ob + TC_CAP * SS;
            unsigned ma = 0u, mb = 0u;
#pragma unroll
            for (int i = 0; i < NTL; ++i) {
                const bool pa = fmaxf(acc[4 * i], acc[4 * i + 1]) >= thra;
                const bool pb = fmaxf(acc[4 * i + 2], acc[4 * i + 3]) >= thrb;
                if (pa) Pv[oa] = make_float2(acc[4 * i], acc[4 * i + 1]);
                if (pb) Pv[ob] = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
                oa = pa ? min(oa + SS, lim_a) : oa;
                ob = pb ? min(ob + SS, lim_b) : ob;
                ma |= pa ? 1u << i : 0u;
                mb |= pb ? 1u << i : 0u;
            }
            Pm[ra * 4 + q4] = ma;
            Pm[rb * 4 + q4] = mb;
            if (q4 == 0) { thrs[ra] = thra; thrs[rb] = thrb; }
        }
        if (CHECK) {
            // exact distances of every column this lane holds (debug only): |a - d| / eps
            float worst = 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int rr = h ? rb : ra;
                if (row0 + rr >= total) continue;
                const float *px = feats + (row0 + rr) * D + featoff[f];
                const float er = eps[rr];
#pragma unroll
                for (int i = 0; i < NTL; ++i)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float *rp = rc + (size_t)(8 * i + 2 * q4 + e) * RF;
                        float d = rp[0];
                        for (int j = 0; j < FL; ++j) {
                            const float df = __fsub_rn(px[j], rp[1 + 2 * j]);
                            d = __fsub_rn(d, __fmul_rn(__fmul_rn(df, df), rp[2 + 2 * j]));
                        }
                        worst = fmaxf(worst, __fdividef(fabsf(acc[4 * i + 2 * h + e] - d), er));
                    }
            }
            atomicMax(reinterpret_cast<int *>(check), __float_as_int(worst));     // non-negative floats order like ints
        }
        warpgroup_bar(1 + wg);                           // every row's pairs are stored, the GEMM's X may be overwritten
        if (!more) break;
        prepare(epsr + (buf ^ 1) * WG_ROWS);
    }
    resolve(row0, epsr + buf * WG_ROWS);
}

// Rows the filter values left in doubt (work list of ptm_wgmma_kernel): one thread per row, the reference's exact
// arithmetic for its candidate codewords (all codewords when its list had overflowed), the five best, the record;
// exact ties go on to the fix-up.  Item: {row low, pair | n0 << 16 | n1 << 24, 18 codeword bytes, row high}: the
// candidates are bytes 0 .. n0 - 1 and TC_CAP - n1 .. TC_CAP - 1 (n0 = 255: all codewords).
template <int FL>
__global__ void __launch_bounds__(128)
ptm_tc_exact_kernel(const float *__restrict__ feats, int D, const int32_t *__restrict__ featoff, const uint4 *__restrict__ items,
                    const unsigned *__restrict__ n_items, unsigned item_cap, const float *__restrict__ rec,
                    const size_t *__restrict__ rec_off, int4 *__restrict__ out, unsigned *__restrict__ flags, long long flag_words,
                    int K, int n_feat, int nd, unsigned long long *__restrict__ stats)
{
    constexpr int RF = (1 + 2 * FL + 3) / 4 * 4;
    const unsigned count = min(*n_items, item_cap);
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        const uint4 a = items[2 * (size_t)i], b = items[2 * (size_t)i + 1];
        const long long row = (long long)a.x | ((long long)b.w << 32);
        const int k = (int)(a.y & 0xffffu), n0 = (int)((a.y >> 16) & 0xffu), n1 = (int)(a.y >> 24);
        const unsigned wv[5] = {a.z, a.w, b.x, b.y, b.z};
        const float *px = feats + row * D + featoff[k % n_feat];
        const float *rc = rec + rec_off[k];
        float x[FL];
#pragma unroll
        for (int j = 0; j < FL; ++j) x[j] = px[j];
        Top5 top;
        top.n = 0; top.c = 0u; top.c4 = 0;
#pragma unroll
        for (int j = 0; j < 5; ++j) top.s[j] = INT_MIN;
        const int cnt = n0 == 255 ? nd : n0 + n1;
        for (int q = 0; q < cnt; ++q) {
            const int pos = q < n0 ? q : q - n0 + TC_CAP - n1;
            const int cw = n0 == 255 ? q : (int)((wv[pos >> 2] >> (8 * (pos & 3))) & 0xffu);
            const float d = gau_dist<FL>(reinterpret_cast<const float4 *>(rc + (size_t)cw * RF), x);
            top5_insert(top, f2i_clamped(d), cw);
        }
        const bool distinct = top.n >= 5 && top.s[0] > top.s[1] && top.s[1] > top.s[2] && top.s[2] > top.s[3] && top.s[3] > top.s[4];
        const int tp = top.s[0] >> PSB_SENSCR_SHIFT;
        unsigned eb = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int ev = tp - (top.s[j] >> PSB_SENSCR_SHIFT);
            ev = ev > 255 ? 255 : ev;
            eb |= (unsigned)ev << (8 * j);
        }
        out[row * K + k] = make_int4(tp, (int)top.c, (int)eb, 0);
        if (!distinct) atomicOr(&flags[(size_t)k * flag_words + (row >> 5)], 1u << (row & 31));
        if (stats) { atomicAdd(stats + 2, (unsigned long long)cnt); if (!distinct) atomicAdd(stats + 3, 1ull); }
    }
}

// Frames whose five best scores tie: the reference's loop, literally (eval_topn ptm_mgau.c:88-136, eval_cb :152-226),
// seeded with the previous frame's list -- the record the filter kernel (or this warp, one frame earlier) wrote -- or
// with codewords 0..3 at the start of an utterance (:791-792).  One WARP per (utterance, pair) chain: lanes = codewords
// (ND / 32 each), the flagged frames of the chain in order.  All distances of a frame in parallel, the four seeds
// fetched by shuffle, then the scan only visits -- in ascending codeword order -- the codewords whose distance reaches
// the seeds' worst score (ballots), each re-tested against the list as it stands: eval_topn + eval_cb literally, like
// semi_scan_kernel does for semi-continuous models.
template <int FL, int NDW>
__global__ void __launch_bounds__(128)
ptm_fixup_warp_kernel(const float *__restrict__ feats, int D, const int32_t *__restrict__ featoff, const int32_t *__restrict__ utt_off,
                      int n_utt, const float *__restrict__ rec, const size_t *__restrict__ rec_off, int4 *__restrict__ out,
                      const unsigned *__restrict__ flags, long long flag_words, int K, int n_feat)
{
    constexpr int RF = (1 + 2 * FL + 3) / 4 * 4;
    constexpr unsigned FULL = 0xffffffffu;
    const long long id = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (id >= (long long)n_utt * K) return;
    const int u = (int)(id / K), k = (int)(id % K);
    const int f = k % n_feat;
    const long long f0 = utt_off[u], f1 = utt_off[u + 1];
    if (f1 <= f0) return;
    const unsigned *fl = flags + (size_t)k * flag_words;
    const float *rc = rec + rec_off[k];
    for (long long w0 = f0 >> 5; w0 <= (f1 - 1) >> 5; w0 += 32) {
        const long long wd_l = w0 + lane;
        unsigned mine = wd_l <= ((f1 - 1) >> 5) ? fl[wd_l] : 0u;
        unsigned any = __ballot_sync(FULL, mine != 0u);
        while (any) {
            const int wl = __ffs(any) - 1;
            any &= any - 1;
            unsigned bits = __shfl_sync(FULL, mine, wl);
            while (bits) {
                const int b = __ffs(bits) - 1;
                bits &= bits - 1;
                const long long row = (w0 + wl) * 32 + b;
                if (row < f0 || row >= f1) continue;
                const float *px = feats + row * D + featoff[f];
                float x[FL];
#pragma unroll
                for (int j = 0; j < FL; ++j) x[j] = px[j];
                float d[NDW];
#pragma unroll
                for (int q = 0; q < NDW; ++q) d[q] = gau_dist<FL>(reinterpret_cast<const float4 *>(rc + (size_t)(lane + 32 * q) * RF), x);
                auto dist_of = [&](int c) {                            // uniform c: the owner lane's value
                    float v = d[0];
#pragma unroll
                    for (int q = 1; q < NDW; ++q) v = (c >> 5) == q ? d[q] : v;
                    return __shfl_sync(FULL, v, c & 31);
                };
                const unsigned seeds = row == f0 ? 0x03020100u : (unsigned)out[(row - 1) * K + k].y;
                int cw[4], sc[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {                          // eval_topn: stable, strict >
                    const int c = (seeds >> (8 * i)) & 0xff;
                    const int s = f2i_clamped(dist_of(c));
                    int p = 0;
#pragma unroll
                    for (int j = 0; j < i; ++j) p += (s > sc[j]) ? 0 : 1;
#pragma unroll
                    for (int j = 2; j >= 0; --j)
                        if (j < i && j >= p) { sc[j + 1] = sc[j]; cw[j + 1] = cw[j]; }
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (j == p) { sc[j] = s; cw[j] = c; }
                }
                const float th0 = (float)sc[3];                        // the scan's threshold only rises from here
#pragma unroll
                for (int q = 0; q < NDW; ++q) {
                    unsigned cand = __ballot_sync(FULL, d[q] >= th0);
                    while (cand) {
                        const int l = __ffs(cand) - 1;
                        cand &= cand - 1;
                        const int c = l + 32 * q;
                        const float dv = __shfl_sync(FULL, d[q], l);
                        if (!(dv >= (float)sc[3])) continue;            // eval_cb :207
                        if (cw[0] == c || cw[1] == c || cw[2] == c || cw[3] == c) continue;   // :209-215
                        const int s = f2i_clamped(dv);
                        int p = 0;
#pragma unroll
                        for (int j = 0; j < 3; ++j) p += (s >= sc[j]) ? 0 : 1;     // insertion_sort_cb :140-149
#pragma unroll
                        for (int j = 2; j >= 0; --j)
                            if (j >= p) { sc[j + 1] = sc[j]; cw[j + 1] = cw[j]; }
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            if (j == p) { sc[j] = s; cw[j] = c; }
                    }
                }
                if (lane == 0) {
                    const int tp = sc[0] >> PSB_SENSCR_SHIFT;
                    unsigned cb = 0, eb = 0;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        int ev = tp - (sc[j] >> PSB_SENSCR_SHIFT);
                        ev = ev > 255 ? 255 : ev;
                        cb |= (unsigned)cw[j] << (8 * j);
                        eb |= (unsigned)ev << (8 * j);
                    }
                    out[row * K + k] = make_int4(tp, (int)cb, (int)eb, 0);
                }
                __syncwarp();
            }
        }
    }
}

float round_tf32_host(float x)
{
    // cvt.rna.tf32.f32: round to nearest, ties away from zero, 10 explicit mantissa bits
    uint32_t u;
    memcpy(&u, &x, 4);
    if ((u & 0x7f800000u) == 0x7f800000u) return x;
    u = (u + 0x1000u) & ~0x1fffu;
    float r;
    memcpy(&r, &u, 4);
    return r;
}

template <int FL, int ND>
int launch_wgmma(psb_batch_t *b, const float *d_feats, long long total, const int32_t *d_klist, int n_k, const int32_t *d_featoff,
               bool check)
{
    psb_model_t *m = b->m;
    const size_t smem = (size_t)2 * 8 * ND * 16 + 2 * ((size_t)2 * 8 * WG_ROWS * 16 + WG_EXTRA);
    const long long tiles = (total + TC_ROWS - 1) / TC_ROWS;
    const int n_sm = psb_sm_count(m->device);
    int per_sm = 1;                                      // sm_90: 151-255 registers x 256 threads, one CTA per SM
    PSB_CUDA(cudaFuncSetAttribute(ptm_wgmma_kernel<FL, ND, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PSB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ptm_wgmma_kernel<FL, ND, false>, TC_ROWS * 2, smem));
    // W (64 KB at 256 densities) is staged once per CTA, and a CTA's first GEMM and last rows do not overlap: many tiles
    // per CTA, but still >= 4 waves of the resident CTAs
    int tpc = 1;
    while (tpc < 32 && (tiles / (tpc * 2)) * n_k >= (long long)n_sm * std::max(per_sm, 1) * 4) tpc *= 2;
    PSB_REQUIRE((tiles + tpc - 1) / tpc <= 65535, "too many frames for one launch of the tensor-core filter");
    const dim3 grid((unsigned)n_k, (unsigned)((tiles + tpc - 1) / tpc));
    b->tc_last_tpc = tpc;
    b->tc_last_ctas = grid.y;
    float *chk = b->d_tc_check;
    unsigned long long *stats = reinterpret_cast<unsigned long long *>(b->d_tc_check + 4);
    if (check) {
        auto kern = ptm_wgmma_kernel<FL, ND, true>;
        PSB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, TC_ROWS * 2, smem, b->stream>>>(d_feats, total, m->sumlen, d_featoff, d_klist, m->d_tc_wumma, m->d_tc_cen, m->d_tc_bnd,
                                                m->d_rec, m->d_rec_off, b->d_topn, b->d_tc_flags, (long long)b->tc_flag_words, m->K,
                                                m->n_feat, tpc, b->d_tc_items, b->d_tc_nitems, b->tc_item_cap, chk, stats);
    }
    else {
        auto kern = ptm_wgmma_kernel<FL, ND, false>;
        PSB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, TC_ROWS * 2, smem, b->stream>>>(d_feats, total, m->sumlen, d_featoff, d_klist, m->d_tc_wumma, m->d_tc_cen, m->d_tc_bnd,
                                                m->d_rec, m->d_rec_off, b->d_topn, b->d_tc_flags, (long long)b->tc_flag_words, m->K,
                                                m->n_feat, tpc, b->d_tc_items, b->d_tc_nitems, b->tc_item_cap, nullptr, nullptr);
    }
    PSB_LAUNCH_CHECK();
    if (b->d_tc_items) {
        // the rows in doubt: the count lives on the device, so the grid covers the list's capacity (grid-stride loop, idle
        // blocks leave at once)
        const unsigned blocks = (unsigned)std::min<size_t>(((size_t)b->tc_item_cap + 127) / 128, (size_t)n_sm * 64);
        ptm_tc_exact_kernel<FL><<<blocks, 128, 0, b->stream>>>(d_feats, m->sumlen, d_featoff, b->d_tc_items, b->d_tc_nitems, b->tc_item_cap,
                                                              m->d_rec, m->d_rec_off, b->d_topn, b->d_tc_flags, (long long)b->tc_flag_words,
                                                              m->K, m->n_feat, ND, check ? stats : nullptr);
        PSB_LAUNCH_CHECK();
    }
    return PSB_OK;
}

}  // namespace

// Host side: the GEMM operand W, the centre and the error-bound coefficients of every pair.
// hm / hv / hd: the model's means, variance terms and determinants on the host (build_records).
int psb_tc_prepare(psb_model_t *m, const float *hm, const float *hv, const float *hd)
{
    m->tc_ok = false;
    if (m->kind != PSB_KIND_PTM || m->fixed_point || m->topn != 4) return PSB_OK;
    if (m->n_density != 64 && m->n_density != 128 && m->n_density != 256) return PSB_OK;
    for (int f = 0; f < m->n_feat; ++f)
        if (m->featlen[f] != 13) return PSB_OK;              // the kernels are instantiated for 13-dimensional streams
    const int nd = m->n_density, FL = 13, K = m->K;
    std::vector<float> cen((size_t)K * 16, 0.f), bnd((size_t)K * 32, 0.f);
    std::vector<float> wu((size_t)K * 2 * 8 * nd * 4, 0.f);     // canonical K-major layout of wgmma's B operand: [half][chunk][n][4]
    std::vector<double> W((size_t)TC_K * nd);
    for (int cb = 0; cb < m->n_mgau; ++cb)
        for (int f = 0; f < m->n_feat; ++f) {
            const int k = cb * m->n_feat + f;
            const size_t src = ((size_t)cb * m->sumlen + m->featoff[f]) * nd;
            const float *mu = hm + src, *vv = hv + src, *dt = hd + (size_t)k * nd;
            float *c = cen.data() + (size_t)k * 16, *bb = bnd.data() + (size_t)k * 32;
            for (int j = 0; j < FL; ++j) {
                double s = 0;
                for (int q = 0; q < nd; ++q) s += mu[(size_t)q * FL + j];
                c[j] = (float)(s / nd);
            }
            std::fill(W.begin(), W.end(), 0.0);
            double cmax = 0;
            for (int q = 0; q < nd; ++q) {
                double c0 = dt[q], quad = 0;
                for (int j = 0; j < FL; ++j) {
                    const double v = vv[(size_t)q * FL + j], mp = (double)mu[(size_t)q * FL + j] - (double)c[j];
                    W[(size_t)j * nd + q] = -v;
                    W[(size_t)(FL + j) * nd + q] = 2.0 * v * mp;
                    quad += std::fabs(v) * mp * mp;
                    c0 -= v * mp * mp;
                    bb[j] = std::max(bb[j], (float)std::fabs(v));
                    bb[FL + j] = std::max(bb[FL + j], (float)std::fabs(2.0 * v * mp));
                }
                W[(size_t)(2 * FL) * nd + q] = c0;
                cmax = std::max(cmax, std::fabs((double)dt[q]) + quad);
            }
            bb[2 * FL] = (float)(cmax * 1.0001);
            for (int j = 0; j < 2 * FL; ++j) bb[j] = std::nextafter(bb[j] * 1.0001f, INFINITY);
            // high and low TF32 halves of the fp32 value of every W entry: w = hi + lo + O(2^-22 w)
            float *u = wu.data() + (size_t)k * 2 * 8 * nd * 4;
            for (int kk = 0; kk < TC_K; ++kk)
                for (int q = 0; q < nd; ++q) {
                    const float v = (float)W[(size_t)kk * nd + q], h = round_tf32_host(v);
                    u[((size_t)(kk >> 2) * nd + q) * 4 + (kk & 3)] = h;
                    u[((size_t)(8 + (kk >> 2)) * nd + q) * 4 + (kk & 3)] = round_tf32_host(v - h);
                }
            for (int i = 0; i < 32; ++i)
                if (!std::isfinite(bb[i])) return PSB_OK;    // degenerate model: keep the scan kernels
        }
    int rc = m->d_tc_wumma.reserve(wu.size());
    if (!rc) rc = m->d_tc_cen.reserve(cen.size());
    if (!rc) rc = m->d_tc_bnd.reserve(bnd.size());
    if (rc) return rc;
    PSB_CUDA(cudaMemcpy(m->d_tc_wumma, wu.data(), wu.size() * sizeof(float), cudaMemcpyHostToDevice));
    PSB_CUDA(cudaMemcpy(m->d_tc_cen, cen.data(), cen.size() * sizeof(float), cudaMemcpyHostToDevice));
    PSB_CUDA(cudaMemcpy(m->d_tc_bnd, bnd.data(), bnd.size() * sizeof(float), cudaMemcpyHostToDevice));
    m->tc_ok = true;
    return PSB_OK;
}

bool psb_tc_usable(const psb_model_t *m)
{
    return m->tc_ok && m->ds_ratio == 1;
}

// Top-N records of a whole batch into b->d_topn (same format as the scan kernels write).
int psb_launch_ptm_tc(psb_batch_t *b, const float *d_feats, const int32_t *utt_off, int32_t n_utt, const int32_t *d_klist,
                      const int32_t *d_featoff)
{
    psb_model_t *m = b->m;
    const long long total = utt_off[n_utt];
    const size_t fw = (size_t)((total + 31) / 32) + 1;
    int rc = b->d_tc_flags.reserve(fw * m->K, fw * m->K / 8);
    if (!rc) rc = b->d_uttoff.reserve((size_t)n_utt + 1, 64);
    if (!rc && !b->d_tc_check) {                              // float[2] check values, then (16-byte offset) ST_N 64-bit counters
        rc = b->d_tc_check.reserve(TC_CHECK_BYTES / sizeof(float));
        if (!rc) PSB_CUDA(cudaMemsetAsync(b->d_tc_check, 0, TC_CHECK_BYTES, b->stream));
    }
    if (!rc) rc = b->d_tc_nitems.reserve(1);
    if (rc) return rc;
    {
        // work list of the rows the filter leaves in doubt: room for a quarter of all (frame, pair) rows, 32 bytes each
        const size_t want = std::max<size_t>(4096, (size_t)total * m->K / 4);
        if (want > b->tc_item_cap) {
            const unsigned cap = (unsigned)std::min<size_t>(want + want / 8, 0x7fffffffu);
            b->tc_item_cap = 0;
            if ((rc = b->d_tc_items.reserve(2 * (size_t)cap))) return rc;     // two uint4 per item
            b->tc_item_cap = cap;
        }
        PSB_CUDA(cudaMemsetAsync(b->d_tc_nitems, 0, 4, b->stream));
    }
    b->tc_flag_words = fw;
    PSB_CUDA(cudaMemsetAsync(b->d_tc_flags, 0, fw * m->K * 4, b->stream));
    PSB_CUDA(cudaMemcpyAsync(b->d_uttoff, utt_off, ((size_t)n_utt + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, b->stream));
    static const bool check = [] { const char *v = getenv("PSB_TC_CHECK"); return v && atoi(v) != 0; }();
    switch (m->n_density) {
    case 256: rc = launch_wgmma<13, 256>(b, d_feats, total, d_klist, m->K, d_featoff, check); break;
    case 128: rc = launch_wgmma<13, 128>(b, d_feats, total, d_klist, m->K, d_featoff, check); break;
    default: rc = launch_wgmma<13, 64>(b, d_feats, total, d_klist, m->K, d_featoff, check); break;
    }
    if (rc) return rc;
    const long long chains = (long long)n_utt * m->K;
    const unsigned blocks = (unsigned)((chains * 32 + 127) / 128);
#define PSB_FIXW(NDW) ptm_fixup_warp_kernel<13, NDW><<<blocks, 128, 0, b->stream>>>(d_feats, m->sumlen, d_featoff, b->d_uttoff, n_utt, \
        m->d_rec, m->d_rec_off, b->d_topn, b->d_tc_flags, (long long)fw, m->K, m->n_feat)
    if (m->n_density == 256) PSB_FIXW(8);
    else if (m->n_density == 128) PSB_FIXW(4);
    else PSB_FIXW(2);
#undef PSB_FIXW
    PSB_LAUNCH_CHECK();
    return PSB_OK;
}

// debug (PSB_TC_CHECK=1): max |a - d| / eps and max candidate count seen by the filter kernels of this batch;
// stats4 = rows, rows resolved from the filter values alone, exact distances computed, rows handed to the tie fix-up
extern "C" int psb_batch_tc_check(psb_batch_t *b, float *ratio, int32_t *max_candidates, int64_t *stats4)
{
    PSB_REQUIRE(b && ratio && max_candidates, "psb_batch_tc_check: null argument");
    *ratio = 0.f; *max_candidates = 0;
    if (stats4) stats4[0] = stats4[1] = stats4[2] = stats4[3] = 0;
    if (!b->d_tc_check) return PSB_OK;
    PSB_CUDA(cudaSetDevice(b->m->device));
    PSB_CUDA(cudaStreamSynchronize(b->stream));
    unsigned char h[64];
    PSB_CUDA(cudaMemcpy(h, b->d_tc_check, sizeof(h), cudaMemcpyDeviceToHost));
    memcpy(ratio, h, 4);
    memcpy(max_candidates, h + 4, 4);
    if (stats4) memcpy(stats4, h + 16, 32);
    return PSB_OK;
}

// debug (PSB_TC_CHECK=1): the filter's decision-path counters (include/psb200.h lists them), then the last launch's
// tiles per CTA and CTAs per pair; the first min(n, PSB_TC_N_COUNTERS) values go to out
extern "C" int psb_batch_tc_counters(psb_batch_t *b, int64_t *out, int32_t n)
{
    PSB_REQUIRE(b && (out || n == 0) && n >= 0, "psb_batch_tc_counters: bad argument");
    static_assert(ST_N + 2 == PSB_TC_N_COUNTERS, "psb200.h lists every counter");
    int64_t v[PSB_TC_N_COUNTERS] = {0};
    if (b->d_tc_check) {
        PSB_CUDA(cudaSetDevice(b->m->device));
        PSB_CUDA(cudaStreamSynchronize(b->stream));
        PSB_CUDA(cudaMemcpy(v, reinterpret_cast<unsigned char *>(b->d_tc_check.get()) + 16, 8 * ST_N, cudaMemcpyDeviceToHost));
    }
    v[ST_N] = b->tc_last_tpc;
    v[ST_N + 1] = b->tc_last_ctas;
    memcpy(out, v, sizeof(int64_t) * (size_t)std::min<int32_t>(n, PSB_TC_N_COUNTERS));
    return PSB_OK;
}
