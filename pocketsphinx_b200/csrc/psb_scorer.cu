// psb_scorer.cu -- the per-frame drop-in behind ps_mgaufuncs_t.frame_eval (acmod.h:101-107)
// for one stream: host buffers in, int16 senone scores out, top-N history ring on the device.
//
// Latency path (one frame per call), so the mapping differs from the batch kernels: one CTA
// per (codebook, stream) pair with one *thread per codeword* computing the full distance, then
// a single thread replays the reference's insertion scan over the staged distances.
#include "psb_gau.cuh"
#include "psb_internal.cuh"
#include "psb_tm.cuh"

#include <string.h>

#include <vector>

struct psb_scorer_s {
    psb_model_t *m;
    Stream stream;                // declared first: destroyed after the buffers below
    int n_hist, frame_idx;
    DevBuf<int32_t> d_cw;         // [n_hist][K][topn]
    DevBuf<int32_t> d_sc;         // [n_hist][K][topn]  raw after the top-N pass, normalised after the norm pass
    DevBuf<uint8_t> d_active;     // [n_hist][n_mgau]
    DevBuf<uint8_t> d_cnt;        // semi: [n_hist][n_feat] entries inside topn_beam (s2_semi_mgau.h:81)
    DevBuf<unsigned char> d_msdist;   // ms: top-N distance lists of the current frame
    DevBuf<int32_t> d_msbest;
    DevBuf<float> d_feat;         // [sumlen]
    DevBuf<int32_t> d_list;       // [n_sen] absolute senone ids of the active list
    DevBuf<int16_t> d_senscr;     // [n_sen]
    HostBuf<float> h_feat; HostBuf<int32_t> h_list; HostBuf<int16_t> h_senscr;
};

namespace {

// eval_topn + eval_cb for every (codebook, stream) pair of one frame (ptm_mgau.c:232-254;
// SEMI: mgau_dist, s2_semi_mgau.c:172-183, whose scan also needs the partial sum before the last
// dimension, :137-155).
template <bool SEMI>
__global__ void __launch_bounds__(256)
scorer_topn_kernel(const float *__restrict__ rec, const size_t *__restrict__ rec_off, const float *__restrict__ feat,
                   const int32_t *__restrict__ prev_cw, int32_t *__restrict__ cur_cw, int32_t *__restrict__ cur_sc,
                   const uint8_t *__restrict__ active, int nd, int n_feat, int topn,
                   const int *__restrict__ featlen, const int *__restrict__ featoff, int do_scan, int fx)
{
    extern __shared__ float sd[];          // [nd] distances (+ [nd] penultimate partial sums when SEMI)
    __shared__ float sx[64];
    const int k = blockIdx.x, cb = k / n_feat, f = k % n_feat;
    const int fl = featlen[f], fo = featoff[f];
    const int rf = (1 + 2 * fl + 3) / 4 * 4;
    if (threadIdx.x < fl) sx[threadIdx.x] = feat[fo + threadIdx.x];
    __syncthreads();
    // FIXED_POINT arithmetic (fx): Q12 integers, fx_mul / fx_gmmsub, and because the scan's early exits are
    // observable there, the minimum of d over the reference's test points next to the final value
    // (see gau_dist_fx in psb_ptm.cu); sd[] then carries int32 bit patterns.
    if (fx) {
        for (int c = threadIdx.x; c < nd; c += blockDim.x) {
            const float *r = rec + rec_off[k] + (size_t)c * rf;
            int d = __float_as_int(r[0]), mn = d;
            for (int j = 0; j < fl; ++j) {
                if (SEMI || j < fl % 4 || (j - fl % 4) % 4 == 0) mn = min(mn, d);
                const int diff = (int)((unsigned)__float_as_int(sx[j]) - (unsigned)__float_as_int(r[1 + 2 * j]));
                d = fx_gmmsub(d, fx_mul(fx_mul(diff, diff), __float_as_int(r[2 + 2 * j])));
            }
            sd[c] = __int_as_float(d);
            sd[nd + c] = __int_as_float(min(mn, d));
        }
    }
    else
    for (int c = threadIdx.x; c < nd; c += blockDim.x) {
        const float *r = rec + rec_off[k] + (size_t)c * rf;
        float d = r[0], dpen = r[0];
        for (int j = 0; j < fl; ++j) {
            float diff = __fsub_rn(sx[j], r[1 + 2 * j]);
            float sq = __fmul_rn(diff, diff);
            dpen = d;
            d = __fsub_rn(d, __fmul_rn(sq, r[2 + 2 * j]));
        }
        sd[c] = d;
        if (SEMI) sd[nd + c] = dpen;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    int cw[PSB_MAX_TOPN], sc[PSB_MAX_TOPN];
    // eval_topn (ptm_mgau.c:88-136 / s2_semi_mgau.c:70-109)
    for (int i = 0; i < topn; ++i) {
        const int c = prev_cw[k * topn + i];
        const int s = fx ? __float_as_int(sd[c]) : __float2int_rz(sd[c]);
        int j = i - 1;
        while (j >= 0 && s > sc[j]) { sc[j + 1] = sc[j]; cw[j + 1] = cw[j]; --j; }
        sc[j + 1] = s; cw[j + 1] = c;
    }
    // eval_cb (ptm_mgau.c:152-226 / s2_semi_mgau.c:112-170) for active codebooks on non-skipped frames
    if (do_scan && active[cb]) {
        for (int c = 0; c < nd; ++c) {
            const float d = sd[c];
            const float th = (float)sc[topn - 1];
            if (fx) {
                if (__float_as_int(sd[nd + c]) < sc[topn - 1]) continue;
            }
            else if (SEMI) {
                if (!(sd[nd + c] >= th)) continue;
                if (__float2int_rz(d) < sc[topn - 1]) continue;
            }
            else if (!(d >= th)) continue;
            bool listed = false;
            for (int i = 0; i < topn; ++i) listed |= cw[i] == c;
            if (listed) continue;
            const int s = fx ? __float_as_int(d) : __float2int_rz(d);
            int kk = topn - 1;
            while (kk > 0 && s >= sc[kk - 1]) { sc[kk] = sc[kk - 1]; cw[kk] = cw[kk - 1]; --kk; }
            sc[kk] = s; cw[kk] = c;
        }
    }
    for (int i = 0; i < topn; ++i) { cur_cw[k * topn + i] = cw[i]; cur_sc[k * topn + i] = sc[i]; }
}

// ptm_mgau_calc_cb_active (:298-321) for a new frame
__global__ void scorer_active_kernel(uint8_t *active, const int32_t *__restrict__ list, int n_list,
                                     const uint16_t *__restrict__ sen2cb, int n_mgau, int compall)
{
    for (int i = threadIdx.x; i < n_mgau; i += blockDim.x) active[i] = compall ? 1 : 0;
    __syncthreads();
    if (!compall)
        for (int i = threadIdx.x; i < n_list; i += blockDim.x) active[sen2cb[list[i]]] = 1;
}

// ptm_mgau_codebook_norm (new frames only) + ptm_mgau_senone_eval (ptm_mgau.c:266-403).
template <bool FOURBIT>
__global__ void __launch_bounds__(1024)
scorer_senone_kernel(int32_t *__restrict__ slot_cw, int32_t *__restrict__ slot_sc, const uint8_t *__restrict__ active,
                     const int32_t *__restrict__ list, int n_list, int compall, int is_new,
                     const uint8_t *__restrict__ mixw, const uint8_t *__restrict__ mixw_cb,
                     const uint16_t *__restrict__ sen2cb, const uint8_t *__restrict__ logadd_tab,
                     int16_t *__restrict__ senscr, int n_sen, int n_mgau, int n_feat, int nd, int topn, int mixw_stride)
{
    extern __shared__ int sm[];
    const int K = n_mgau * n_feat, tid = threadIdx.x;
    int *sc = sm;                                       // [K*topn]
    int *cw = sc + K * topn;                            // [K*topn]
    int *norm = cw + K * topn;                          // [8]
    int *red = norm + 8;                                // [32]
    uint8_t *tab = reinterpret_cast<uint8_t *>(red + 32);   // [PSB_LOGADD8_N]
    uint8_t *cb16 = tab + PSB_LOGADD8_N;                // [16]
    uint8_t *act = cb16 + 16;                           // [n_mgau]
    int16_t *asc = reinterpret_cast<int16_t *>(act + ((n_mgau + 15) & ~15));   // [n_sen]

    for (int i = tid; i < K * topn; i += blockDim.x) { sc[i] = slot_sc[i]; cw[i] = slot_cw[i]; }
    for (int i = tid; i < n_mgau; i += blockDim.x) act[i] = active[i];
    for (int i = tid; i < PSB_LOGADD8_N; i += blockDim.x) tab[i] = logadd_tab[i];
    if (FOURBIT && tid < 16) cb16[tid] = mixw_cb[tid];
    if (tid < n_feat) norm[tid] = PSB_WORST_SCORE;
    for (int i = tid; i < n_sen; i += blockDim.x) asc[i] = 0;            // memset (:333)
    __syncthreads();
    if (is_new) {
        for (int i = tid; i < K; i += blockDim.x)
            if (act[i / n_feat]) atomicMax(&norm[i % n_feat], sc[i * topn] >> PSB_SENSCR_SHIFT);
        __syncthreads();
        for (int i = tid; i < K * topn; i += blockDim.x) {
            const int k = i / topn;
            if (!act[k / n_feat]) continue;
            int v = -((sc[i] >> PSB_SENSCR_SHIFT) - norm[k % n_feat]);
            sc[i] = v > PSB_MAX_NEG_ASCR ? PSB_MAX_NEG_ASCR : v;
        }
        __syncthreads();
    }
    // senones of pruned codebooks see the floor, and the slot keeps it (:353-364)
    const int n = compall ? n_sen : n_list;
    for (int i = tid; i < n; i += blockDim.x) {
        const int cb = sen2cb[compall ? i : list[i]];
        if (!act[cb])
            for (int j = 0; j < n_feat * topn; ++j) sc[cb * n_feat * topn + j] = PSB_MAX_NEG_ASCR;
    }
    __syncthreads();
    int best = 0x7fffffff;
    for (int i = tid; i < n; i += blockDim.x) {
        const int s = compall ? i : list[i];
        const int cb = sen2cb[s];
        int ascore = 0;
        for (int f = 0; f < n_feat; ++f) {
            const int base = (cb * n_feat + f) * topn;
            const uint8_t *row = mixw + (size_t)f * nd * mixw_stride;
            int fden = 0;
            for (int j = 0; j < topn; ++j) {
                const int w = FOURBIT ? ptm_weight4(cb16, row[(size_t)cw[base + j] * mixw_stride + (s >> 1)])
                                      : row[(size_t)cw[base + j] * mixw_stride + s];
                const int v = w + sc[base + j];
                fden = j == 0 ? v : logadd8(tab, fden, v);
            }
            ascore += fden;
        }
        best = min(best, ascore);
        asc[s] = (int16_t)ascore;     // duplicate ids in a bridged list recompute the same value
    }
    store_relative_to_best(best, red, asc, senscr, n_sen);
    for (int i = tid; i < K * topn; i += blockDim.x) slot_sc[i] = sc[i];
}

// s2_semi_mgau_frame_eval's per-frame tail (s2_semi_mgau.c:837-883): mgau_norm for new frames
// (:186-203, keeps the count inside topn_beam per history slot) and get_scores_{8b,4b}_feat*
// (:206-831).  4-bit quirks reproduced: the unrolled active-list variants for 1..6 entries add
// mixw_cb + score in uint8 (:453-463), _any and _all use int; _all stops at n_sen & ~1 (:809).
template <bool FOURBIT>
__global__ void __launch_bounds__(1024)
scorer_semi_senone_kernel(int32_t *__restrict__ slot_cw, int32_t *__restrict__ slot_sc, uint8_t *__restrict__ slot_n,
                          const int32_t *__restrict__ list, int n_list, int compall, int is_new,
                          const uint8_t *__restrict__ mixw, const uint8_t *__restrict__ mixw_cb,
                          const uint8_t *__restrict__ logadd_tab, const int32_t *__restrict__ topn_beam,
                          int16_t *__restrict__ senscr, int n_sen, int n_feat, int nd, int topn, int mixw_stride)
{
    __shared__ int sc[PSB_MAX_FEAT * PSB_MAX_TOPN], cw[PSB_MAX_FEAT * PSB_MAX_TOPN], cnt[PSB_MAX_FEAT];
    __shared__ uint8_t tab[PSB_LOGADD8_N], cb16[16];
    const int tid = threadIdx.x;
    for (int i = tid; i < PSB_LOGADD8_N; i += blockDim.x) tab[i] = logadd_tab[i];
    if (FOURBIT && tid < 16) cb16[tid] = mixw_cb[tid];
    if (tid < n_feat * topn) { sc[tid] = slot_sc[tid]; cw[tid] = slot_cw[tid]; }
    __syncthreads();
    if (tid < n_feat) {
        if (is_new) {
            const int norm = sc[tid * topn] >> PSB_SENSCR_SHIFT;
            const int beam = topn_beam[tid];
            int j;
            for (j = 0; j < topn; ++j) {
                int v = -((sc[tid * topn + j] >> PSB_SENSCR_SHIFT) - norm);
                if (v > PSB_MAX_NEG_ASCR) v = PSB_MAX_NEG_ASCR;
                sc[tid * topn + j] = v;
                if (beam && v > beam) break;
            }
            cnt[tid] = j;
            slot_n[tid] = (uint8_t)j;
            for (int q = 0; q < topn; ++q) slot_sc[tid * topn + q] = sc[tid * topn + q];
        }
        else
            cnt[tid] = slot_n[tid];
    }
    __syncthreads();
    for (int i = tid; i < n_sen; i += blockDim.x) senscr[i] = 0;      // memset (:847)
    __syncthreads();
    const int n = compall ? (FOURBIT ? (n_sen & ~1) : n_sen) : n_list;
    for (int i = tid; i < n; i += blockDim.x) {
        const int s = compall ? i : list[i];
        int16_t acc = 0;
        for (int f = 0; f < n_feat; ++f) {
            const int tn = cnt[f];
            const bool wrap8 = FOURBIT && !compall && tn >= 1 && tn <= 6;
            const uint8_t *row = mixw + (size_t)f * nd * mixw_stride;
            int tmp = 0;
            for (int k = 0; k == 0 || k < tn; ++k) {
                const int w = FOURBIT ? semi_weight4(cb16, row[(size_t)cw[f * topn + k] * mixw_stride + (s >> 1)], s)
                                      : row[(size_t)cw[f * topn + k] * mixw_stride + s];
                int v = w + sc[f * topn + k];
                if (wrap8) v &= 0xff;
                tmp = k == 0 ? v : logadd8(tab, tmp, v);
            }
            acc = (int16_t)(acc + tmp);
        }
        // a bridged active list can name a senone twice; the reference then accumulates twice
        // (senone_scores[sen] += tmp runs per list entry).  Lists from acmod_flags2list never
        // repeat an id, so plain stores are equivalent.
        senscr[s] = acc;
    }
}

}  // namespace

extern "C" int psb_scorer_create(psb_model_t *m, int32_t n_hist, psb_scorer_t **out)
{
    PSB_REQUIRE(m && out && n_hist >= 1, "psb_scorer_create: bad argument");
    PSB_REQUIRE(m->n_density <= 1024 && m->sumlen <= 4096, "model too large for the scorer kernels");
    for (int f = 0; f < m->n_feat; ++f) PSB_REQUIRE(m->featlen[f] <= 64, "stream longer than 64 dims");
    PSB_CUDA(cudaSetDevice(m->device));
    std::unique_ptr<psb_scorer_t> s(new psb_scorer_t());
    s->m = m; s->n_hist = n_hist;
    const size_t per = (size_t)m->K * m->topn;
    const cudaError_t e = s->stream.create();
    if (e != cudaSuccess) {
        psb_set_error("psb_scorer_create: %s", cudaGetErrorString(e));
        return PSB_ERR_CUDA;
    }
    int rc = s->d_cw.reserve(n_hist * per);
    if (!rc) rc = s->d_sc.reserve(n_hist * per);
    if (!rc) rc = s->d_active.reserve((size_t)n_hist * m->n_mgau);
    if (!rc) rc = s->d_cnt.reserve((size_t)n_hist * PSB_MAX_FEAT);
    if (!rc && m->kind == PSB_KIND_MS) rc = s->d_msdist.reserve(psb_ms_dist_bytes(m));
    if (!rc) rc = s->d_msbest.reserve(1);
    if (!rc) rc = s->d_feat.reserve((size_t)m->sumlen);
    if (!rc) rc = s->d_list.reserve((size_t)m->n_sen);
    if (!rc) rc = s->d_senscr.reserve((size_t)m->n_sen);
    if (!rc) rc = s->h_feat.reserve((size_t)m->sumlen);
    if (!rc) rc = s->h_list.reserve((size_t)m->n_sen);
    if (!rc) rc = s->h_senscr.reserve((size_t)m->n_sen);
    if (!rc) rc = psb_scorer_reset(s.get());
    if (rc) return rc;
    *out = s.release();
    return PSB_OK;
}

extern "C" void psb_scorer_free(psb_scorer_t *s)
{
    if (!s) return;
    cudaSetDevice(s->m->device);
    cudaStreamSynchronize(s->stream);
    delete s;
}

extern "C" int psb_scorer_reset(psb_scorer_t *s)
{
    PSB_REQUIRE(s, "psb_scorer_reset: null");
    psb_model_t *m = s->m;
    PSB_CUDA(cudaSetDevice(m->device));
    const size_t per = (size_t)m->K * m->topn;
    std::vector<int32_t> cw(s->n_hist * per), sc(s->n_hist * per, INT32_MIN);
    for (size_t i = 0; i < cw.size(); ++i) cw[i] = (int32_t)(i % m->topn);     // ptm_mgau.c:791-792
    PSB_CUDA(cudaStreamSynchronize(s->stream));
    PSB_CUDA(cudaMemcpy(s->d_cw, cw.data(), cw.size() * 4, cudaMemcpyHostToDevice));
    PSB_CUDA(cudaMemcpy(s->d_sc, sc.data(), sc.size() * 4, cudaMemcpyHostToDevice));
    PSB_CUDA(cudaMemset(s->d_active, 1, (size_t)s->n_hist * m->n_mgau));
    PSB_CUDA(cudaMemset(s->d_cnt, 0, (size_t)s->n_hist * PSB_MAX_FEAT));
    s->frame_idx = 0;
    return PSB_OK;
}

extern "C" int psb_scorer_set_frame_idx(psb_scorer_t *s, int32_t frame_idx)
{
    PSB_REQUIRE(s && frame_idx >= 0, "psb_scorer_set_frame_idx: bad argument");
    s->frame_idx = frame_idx;
    return PSB_OK;
}

extern "C" int32_t psb_scorer_get_frame_idx(const psb_scorer_t *s) { return s ? s->frame_idx : -1; }

extern "C" int psb_scorer_frame_eval(psb_scorer_t *s, int16_t *senscr, const uint8_t *senone_active,
                                     int32_t n_senone_active, const float *const *feat, int32_t frame,
                                     int32_t compallsen)
{
    PSB_REQUIRE(s && senscr && feat && frame >= 0, "psb_scorer_frame_eval: bad argument");
    psb_model_t *m = s->m;
    PSB_REQUIRE(compallsen || n_senone_active == 0 || senone_active, "senone_active missing");
    PSB_CUDA(cudaSetDevice(m->device));
    const size_t per = (size_t)m->K * m->topn;
    const int idx = frame % s->n_hist;                       // ptm_mgau.c:425
    const bool is_new = frame >= s->frame_idx;               // :430
    int n_list = 0;
    if (!compallsen) {
        // decode the delta list (acmod.c:1224-1275 coding; ptm_mgau.c:342-350 decoding)
        int last = 0;
        for (int i = 0; i < n_senone_active; ++i) {
            last += senone_active[i];
            PSB_REQUIRE(last < m->n_sen, "active list runs past n_sen");
            s->h_list[n_list++] = last;
        }
        PSB_CUDA(cudaMemcpyAsync(s->d_list, s->h_list, (size_t)n_list * 4, cudaMemcpyHostToDevice, s->stream));
    }
    int32_t *cur_cw = s->d_cw + per * idx, *cur_sc = s->d_sc + per * idx;
    uint8_t *cur_act = s->d_active + (size_t)idx * m->n_mgau;
    if (is_new || m->kind == PSB_KIND_MS) {
        for (int f = 0; f < m->n_feat; ++f)
            memcpy(s->h_feat + m->featoff[f], feat[f], m->featlen[f] * sizeof(float));
        PSB_CUDA(cudaMemcpyAsync(s->d_feat, s->h_feat, m->sumlen * 4, cudaMemcpyHostToDevice, s->stream));
    }
    if (m->kind == PSB_KIND_MS) {
        // ms_cont_mgau_frame_eval has no history: every call recomputes (ms_mgau.c:192-282)
        if (!compallsen)        // unlisted entries keep the caller's values: start from them
            PSB_CUDA(cudaMemsetAsync(s->d_senscr, 0, (size_t)m->n_sen * 2, s->stream));
        int rc = psb_ms_score_one(m, s->stream, s->d_feat, s->d_msdist, s->d_msbest, s->d_senscr,
                                  compallsen ? nullptr : s->d_list.get(), compallsen ? m->n_sen : n_list);
        if (rc) return rc;
    }
    else {
        const bool semi = m->kind == PSB_KIND_SEMI;
        if (is_new) {
            const int prev = idx == 0 ? s->n_hist - 1 : idx - 1;
            scorer_active_kernel<<<1, 256, 0, s->stream>>>(cur_act, s->d_list, n_list, m->d_sen2cb, m->n_mgau,
                                                           compallsen || semi);
            PSB_LAUNCH_CHECK();
            const int threads = m->n_density < 256 ? roundup(m->n_density, 32) : 256;
            if (semi)
                scorer_topn_kernel<true><<<m->K, threads, 2 * m->n_density * sizeof(float), s->stream>>>(
                    m->d_rec, m->d_rec_off, s->d_feat, s->d_cw + per * prev, cur_cw, cur_sc, cur_act, m->n_density,
                    m->n_feat, m->topn, m->d_featlen, m->d_featoff, frame % m->ds_ratio == 0, m->fixed_point);
            else
                scorer_topn_kernel<false><<<m->K, threads, (m->fixed_point ? 2 : 1) * m->n_density * sizeof(float), s->stream>>>(
                    m->d_rec, m->d_rec_off, s->d_feat, s->d_cw + per * prev, cur_cw, cur_sc, cur_act, m->n_density,
                    m->n_feat, m->topn, m->d_featlen, m->d_featoff, frame % m->ds_ratio == 0, m->fixed_point);
            PSB_LAUNCH_CHECK();
        }
        if (semi) {
            uint8_t *cur_cnt = s->d_cnt + (size_t)idx * PSB_MAX_FEAT;
            if (m->mixw_4bit)
                scorer_semi_senone_kernel<true><<<1, 1024, 0, s->stream>>>(
                    cur_cw, cur_sc, cur_cnt, s->d_list, n_list, compallsen, is_new, m->d_mixw, m->d_mixw_cb, m->d_logadd8,
                    m->d_topn_beam, s->d_senscr, m->n_sen, m->n_feat, m->n_density, m->topn, m->mixw_stride);
            else
                scorer_semi_senone_kernel<false><<<1, 1024, 0, s->stream>>>(
                    cur_cw, cur_sc, cur_cnt, s->d_list, n_list, compallsen, is_new, m->d_mixw, m->d_mixw_cb, m->d_logadd8,
                    m->d_topn_beam, s->d_senscr, m->n_sen, m->n_feat, m->n_density, m->topn, m->mixw_stride);
            PSB_LAUNCH_CHECK();
        }
        else {
            const int K = m->K;
            size_t smem = ((size_t)2 * K * m->topn + 8 + 32) * 4 + PSB_LOGADD8_N + 16 + ((m->n_mgau + 15) & ~15) + (size_t)m->n_sen * 2;
            PSB_REQUIRE(smem <= 227 * 1024, "model too large for scorer_senone_kernel (%zu bytes of shared memory)", smem);
            if (m->mixw_4bit) {
                PSB_CUDA(cudaFuncSetAttribute(scorer_senone_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                scorer_senone_kernel<true><<<1, 1024, smem, s->stream>>>(
                    cur_cw, cur_sc, cur_act, s->d_list, n_list, compallsen, is_new, m->d_mixw, m->d_mixw_cb, m->d_sen2cb,
                    m->d_logadd8, s->d_senscr, m->n_sen, m->n_mgau, m->n_feat, m->n_density, m->topn, m->mixw_stride);
            }
            else {
                PSB_CUDA(cudaFuncSetAttribute(scorer_senone_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                scorer_senone_kernel<false><<<1, 1024, smem, s->stream>>>(
                    cur_cw, cur_sc, cur_act, s->d_list, n_list, compallsen, is_new, m->d_mixw, m->d_mixw_cb, m->d_sen2cb,
                    m->d_logadd8, s->d_senscr, m->n_sen, m->n_mgau, m->n_feat, m->n_density, m->topn, m->mixw_stride);
            }
            PSB_LAUNCH_CHECK();
        }
    }
    PSB_CUDA(cudaMemcpyAsync(s->h_senscr, s->d_senscr, (size_t)m->n_sen * 2, cudaMemcpyDeviceToHost, s->stream));
    PSB_CUDA(cudaStreamSynchronize(s->stream));
    if (m->kind == PSB_KIND_MS && !compallsen) {
        // the ms back-end writes only the listed senones (ms_mgau.c:254-276)
        for (int i = 0; i < n_list; ++i) senscr[s->h_list[i]] = s->h_senscr[s->h_list[i]];
    }
    else
        memcpy(senscr, s->h_senscr, (size_t)m->n_sen * 2);
    return PSB_OK;
}
