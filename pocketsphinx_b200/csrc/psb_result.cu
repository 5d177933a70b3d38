// psb_result.cu -- reading a hypothesis out of the tables the search kernels return: the exit the
// reference would pick and the word segments along its predecessor chain.  Host code (the reference
// does this on the host too, once per utterance, over a few thousand rows); no device work, so these
// entry points also run where there is no GPU.
#include "psb_internal.cuh"
#include "psb_ngs_host.h"

#include <limits.h>

// fsg_search_find_exit (fsg_search.c:883-954): *entry = the exit, 0 / -1 when there is none (no word
// exit yet / the final state was not reached).  hist rows as psb_fsg_batch_device returns them
// ({link, frame, score, pred, lc, rc.bv[8]}), links [n_link][5].
extern "C" int psb_fsg_find_exit(const int32_t *hist, int32_t n_hist, const int32_t *links, int32_t n_link,
                                 int32_t frame_idx, int32_t final_state, int32_t final, int32_t *entry, int32_t *out_score)
{
    PSB_REQUIRE(hist && links && entry && n_hist >= 0 && n_link >= 0, "psb_fsg_find_exit: bad arguments");
    *entry = -1;
    int bp = n_hist - 1;
    int frm = frame_idx, last = frame_idx;
    while (bp > 0) {                                   // last word exit at or before frame_idx
        if (hist[(size_t)bp * 13 + 1] <= frame_idx) {
            frm = last = hist[(size_t)bp * 13 + 1];
            break;
        }
        --bp;
    }
    if (bp <= 0) {                                     // no hypothesis (yet): only the start entry, or nothing
        *entry = bp < 0 ? -1 : 0;
        return PSB_OK;
    }
    int32_t best = INT_MIN;
    int besthist = -1;
    while (frm == last) {
        const int32_t l = hist[(size_t)bp * 13], score = hist[(size_t)bp * 13 + 2];
        if (l < 0) break;                              // the start entry has no link
        PSB_REQUIRE(l < n_link, "psb_fsg_find_exit: entry %d names link %d of %d", bp, l, n_link);
        const int32_t to = links[(size_t)l * 5 + 1];
        if (score == best && to == final_state)        // equal scores: prefer the final state
            besthist = bp;
        else if (score > best && (!final || to == final_state)) {
            best = score;
            besthist = bp;
        }
        if (--bp < 0) break;
        frm = hist[(size_t)bp * 13 + 1];
    }
    if (besthist == -1) return PSB_OK;                 // the final state was not reached: *entry stays -1
    if (out_score) *out_score = best;
    *entry = besthist;
    return PSB_OK;
}

// The segments of fsg_search_seg_iter (fsg_search.c:1122-1180) with fsg_seg_bp2itor's fields
// (:1062-1091), in time order: seg [cap][7] = {entry, link, wid (-1: null transition), sf, ef, ascr,
// lscr}.  Returns the number of segments on the chain (rows past cap are not written).
extern "C" int32_t psb_fsg_backtrace(const int32_t *hist, int32_t n_hist, const int32_t *links, int32_t n_link,
                                     int32_t exit_entry, int32_t *seg, int32_t cap)
{
    PSB_REQUIRE(hist && links && n_hist >= 0 && (seg || cap == 0) && cap >= 0, "psb_fsg_backtrace: bad arguments");
    PSB_REQUIRE(exit_entry >= 0 && exit_entry < (n_hist > 0 ? n_hist : 1), "psb_fsg_backtrace: entry %d of %d", exit_entry, n_hist);
    int n = 0;
    for (int bp = exit_entry; bp > 0;) {               // predecessors always precede (fsg_history.c:200-240)
        const int32_t pred = hist[(size_t)bp * 13 + 3], l = hist[(size_t)bp * 13];
        PSB_REQUIRE(pred >= -1 && pred < bp && l >= 0 && l < n_link, "psb_fsg_backtrace: entry %d is not a history row", bp);
        bp = pred;
        ++n;
    }
    int cur = n - 1;
    for (int bp = exit_entry; bp > 0; --cur) {
        const int32_t *h = hist + (size_t)bp * 13;
        const int32_t *fl = links + (size_t)h[0] * 5;
        const int32_t *ph = h[3] >= 0 ? hist + (size_t)h[3] * 13 : nullptr;
        if (cur < cap) {
            int32_t *s = seg + (size_t)cur * 7;
            s[0] = bp; s[1] = h[0]; s[2] = fl[2];
            s[4] = h[1];
            s[3] = ph ? ph[1] + 1 : 0;
            if (s[3] > s[4]) s[3] = s[4];              // null transitions
            s[6] = fl[3] >> 10;                        // SENSCR_SHIFT
            s[5] = h[2] - (ph ? ph[2] : 0) - s[6];
        }
        bp = h[3];
    }
    return n;
}

// ngram_search_find_exit with frame_idx = -1 (ngram_search.c:498-541): </s> in the last frame that has
// exits, else that frame's best entry.  bp rows [n][10] and bp_idx [n_frame + 1] as the n-gram entry
// points return them.
extern "C" int psb_ngram_find_exit(const int32_t *bp, int32_t n_bp, const int32_t *bp_idx, int32_t n_frame,
                                   int32_t finish_wid, int32_t *entry, int32_t *out_score)
{
    PSB_REQUIRE(bp && bp_idx && entry && n_bp >= 0 && n_frame >= 0, "psb_ngram_find_exit: bad arguments");
    *entry = -1;
    if (n_frame == 0) return PSB_OK;
    int f = n_frame - 1;
    const int32_t end = bp_idx[f];
    while (f >= 0 && bp_idx[f] == end) --f;            // frames without exits
    if (f < 0) return PSB_OK;
    PSB_REQUIRE(bp_idx[f] >= 0 && end <= n_bp && bp_idx[f] <= end, "psb_ngram_find_exit: bp_idx does not index the table");
    int32_t best = (int32_t)0xE0000000;                // WORST_SCORE
    int best_exit = -1;
    for (int b = bp_idx[f]; b < end; ++b) {
        const int32_t *e = bp + (size_t)b * 10;
        if (e[2] == finish_wid || e[4] > best) {
            best = e[4];
            best_exit = b;
        }
        if (e[2] == finish_wid) break;
    }
    if (out_score) *out_score = best;
    *entry = best_exit;
    return PSB_OK;
}

// The backpointer chain of ngram_search_bp_iter (ngram_search.c:958-997) in time order:
// seg [cap][5] = {entry, wid, sf, ef, path score at the exit}.  Returns the chain's length.
extern "C" int32_t psb_ngram_backtrace(const int32_t *bp, int32_t n_bp, int32_t exit_entry, int32_t *seg, int32_t cap)
{
    PSB_REQUIRE(bp && n_bp >= 0 && (seg || cap == 0) && cap >= 0, "psb_ngram_backtrace: bad arguments");
    if (exit_entry == -1) return 0;
    PSB_REQUIRE(exit_entry >= 0 && exit_entry < n_bp, "psb_ngram_backtrace: entry %d of %d", exit_entry, n_bp);
    int n = 0;
    for (int b = exit_entry; b != -1; ++n) {
        const int32_t p = bp[(size_t)b * 10 + 3];
        PSB_REQUIRE(p >= -1 && p < b, "psb_ngram_backtrace: entry %d does not point backwards", b);
        b = p;
    }
    int cur = n - 1;
    for (int b = exit_entry; b != -1; --cur) {
        const int32_t *e = bp + (size_t)b * 10;
        if (cur < cap) {
            int32_t *s = seg + (size_t)cur * 5;
            s[0] = b; s[1] = e[2]; s[2] = e[3] >= 0 ? bp[(size_t)e[3] * 10] + 1 : 0; s[3] = e[0]; s[4] = e[4];
        }
        b = e[3];
    }
    return n;
}

// The phone LM's dense tables of allphone_search (allphone_search.c:420-441, 497-513), scored through the
// same restatement of ngram_tg_score the n-gram kernels use: the block's "dictionary" is the CI phones, its
// widmap allphone_search_init's ci2lmwid (:552-577).  Everything is checked before the first write.
extern "C" int psb_allphone_lm_tables(const int32_t *lm_block, int32_t n_ci, int32_t *bg, int32_t *tg)
{
    PSB_REQUIRE(lm_block && bg && tg, "psb_allphone_lm_tables: bad arguments");
    PSB_REQUIRE(n_ci > 0 && n_ci <= 64, "psb_allphone_lm_tables: %d CI phones (1 to 64: the phone net's context sets are 64-bit masks)", n_ci);
    PSB_REQUIRE(lm_block[7] == n_ci, "psb_allphone_lm_tables: the block maps %d words, not the %d CI phones", lm_block[7], n_ci);
    std::string err;
    if (lm_arr_check(lm_block, (long long)lm_arr_words(lm_block), n_ci, err) != 0)
        PSB_REQUIRE(false, "psb_allphone_lm_tables: %s", err.c_str());
    LmArr L;
    lm_arr_bind(L, lm_block, lm_block);
    for (int a = 0; a < n_ci; ++a)
        PSB_REQUIRE(L.widmap[a] >= 0 && L.widmap[a] < L.V, "psb_allphone_lm_tables: CI phone %d maps to LM word %d, outside the LM's %d words",
                    a, L.widmap[a], L.V);
    for (int a = 0; a < n_ci; ++a)
        for (int b = 0; b < n_ci; ++b) {
            bg[a * n_ci + b] = lm_tg_score(L, a, b, -1) >> PSB_SENSCR_SHIFT;       // ngram_bg_score(lm, wid[a], wid[b])
            for (int c = 0; c < n_ci; ++c)
                tg[((size_t)a * n_ci + b) * n_ci + c] = lm_tg_score(L, a, b, c) >> PSB_SENSCR_SHIFT;
        }
    return PSB_OK;
}

// ngram_search_bp2itor (ngram_search.c:886-928) for every entry of the chain: what ps_seg_iter reports
// without -bestpath.  seg [cap][7] = {entry, wid, sf, ef, path score, ascr, lscr}; the right-context
// exit score of the predecessor comes from the score stack (ngram_search_exit_score :655-676), the LM
// score from the search description (dense table or LM arrays), scaled by lwf (the float32
// fwdflat_fwdtree_lw_ratio after a second pass, 1.0 after the first alone: ngram_search_seg_iter :1033-1036).
extern "C" int32_t psb_ngram_segments(const psb_ngram_desc_t *g, const int32_t *bp, int32_t n_bp, const int32_t *bss,
                                      int32_t n_bss, int32_t exit_entry, float lwf, int32_t *seg, int32_t cap)
{
    PSB_REQUIRE(g && g->info && g->model && bp && bss && n_bp >= 0 && n_bss >= 0 && (seg || cap == 0) && cap >= 0,
                "psb_ngram_segments: bad arguments");
    const int32_t *info = g->info;
    NgsGraph G;
    memset(&G, 0, sizeof(G));
    G.n_words = info[1]; G.n_ci = info[6]; G.n_lm = info[26];
    const long long n_root = info[2], n_nonroot = info[3], n_1ph = info[4], nc = G.n_ci, nl = G.n_lm;
    G.use_lma = g->lm_arrays != nullptr;
    PSB_REQUIRE(G.n_words > 0 && nc > 0 && nc <= 256 && n_root >= 0 && n_nonroot >= 0 && n_1ph >= 0 && nl >= 0 && nl <= 512 &&
                (nl > 0 || G.use_lma), "psb_ngram_segments: sizes in info out of range");
    const long long o_words = n_root * 5 + n_nonroot * 6, o_cimap = o_words + (long long)G.n_words * 8 + n_1ph * 5 + nc * nc + nc * nc * nc,
                    o_lm = o_cimap + 2 * nc * nc * nc, need = o_lm + (G.use_lma ? 0 : nl * (nl + 1) * (nl + 1));
    PSB_REQUIRE(g->model_len >= need, "psb_ngram_segments: model block holds %lld words, the sizes in info need %lld",
                (long long)g->model_len, need);
    G.words = g->model + o_words; G.rs_cimap = g->model + o_cimap; G.lm = g->model + o_lm;
    if (G.use_lma) {
        std::string err;
        if (lm_arr_check(g->lm_arrays, g->lm_arrays_len, G.n_words, err) != 0) PSB_REQUIRE(false, "psb_ngram_segments: %s", err.c_str());
        lm_arr_bind(G.lma, g->lm_arrays, g->lm_arrays);
    }
    const int silence_wid = info[21];
    const int silpen = info[17], fillpen = info[18];
    if (exit_entry == -1) return 0;
    PSB_REQUIRE(exit_entry >= 0 && exit_entry < n_bp, "psb_ngram_segments: entry %d of %d", exit_entry, n_bp);
    auto lm_ok = [&](int w, bool hist) {                // a dictionary id the LM lookup may be given
        if (hist && w == -1) return true;
        if (w < 0 || w >= G.n_words) return false;
        return G.use_lma || (NGS_W(G, w, 7) >= 0 && NGS_W(G, w, 7) < G.n_lm);
    };
    int n = 0;
    for (int b = exit_entry; b != -1; ++n) {
        const int32_t *e = bp + (size_t)b * 10;
        PSB_REQUIRE(e[3] >= -1 && e[3] < b && e[2] >= 0 && e[2] < G.n_words, "psb_ngram_segments: entry %d is not a backpointer row", b);
        b = e[3];
    }
    int cur = n - 1;
    for (int b = exit_entry; b != -1; --cur) {
        const int32_t *e = bp + (size_t)b * 10;
        const int32_t *pe = e[3] >= 0 ? bp + (size_t)e[3] * 10 : nullptr;
        int32_t ascr = e[4], lscr = 0;
        if (pe) {
            int32_t start_score = pe[4];
            if (pe[9] != -1) {                          // multi-phone predecessor: its exit into this word's first phone
                PSB_REQUIRE(pe[8] >= 0 && pe[8] < nc && pe[9] >= 0 && pe[9] < nc, "psb_ngram_segments: entry %d: phones out of range", e[3]);
                const int rc = G.rs_cimap[((size_t)pe[8] * nc + pe[9]) * nc + NGS_W(G, e[2], 0)];
                PSB_REQUIRE(pe[5] >= 0 && rc >= 0 && (long long)pe[5] + rc < n_bss, "psb_ngram_segments: entry %d: score stack index out of range", e[3]);
                start_score = bss[pe[5] + rc];
            }
            if (e[2] == silence_wid) lscr = silpen;
            else if (NGS_W(G, e[2], 4)) lscr = fillpen;
            else {
                PSB_REQUIRE(lm_ok(e[6], false) && lm_ok(pe[6], true) && lm_ok(pe[7], true), "psb_ngram_segments: entry %d: LM word ids out of range", b);
                lscr = ngs_tg(G, e[6], pe[6], pe[7]);
                lscr = (int32_t)((float)lscr * lwf);
            }
            ascr = (int32_t)((uint32_t)e[4] - (uint32_t)start_score - (uint32_t)lscr);
        }
        if (cur < cap) {
            int32_t *s = seg + (size_t)cur * 7;
            s[0] = b; s[1] = e[2]; s[2] = pe ? pe[0] + 1 : 0; s[3] = e[0]; s[4] = e[4]; s[5] = ascr; s[6] = lscr;
        }
        b = e[3];
    }
    return n;
}
