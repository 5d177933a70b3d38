"""GPU (-m gpu): score renormalisation in the device searches that have it, and the phone loop at every shape it
accepts.  Every case is compared bit for bit with the oracle's C restatements (oracle/ps_oracle.c).

Renormalisation subtracts the best score from every HMM once the best score comes close to the int32 floor,
WORST_SCORE = -536 870 912.  The conditions are the reference's:
- phone loop (phone_loop_search.c:177-191) and both n-gram passes: best_score + 2 * beam < WORST_SCORE;
- forced alignment (state_align_search.c:199-203): best_score - 0x300000 < WORST_SCORE.
A frame lowers the best score by at most one senone score (32 767) plus one transition, so the branch is reached
either by tens of thousands of frames of heavy scores (the "natural crossing" cases below, ~17 800 frames at
>= 30 000 per frame) or by a beam below WORST_SCORE / 2, which makes the condition true in every frame.  Each case
asserts from the oracle's own outputs that the branch was taken, so none passes because the bound was out of reach."""
import ctypes as C

import numpy as np
import pytest

from conftest import assert_hmm_equal, golden

pytestmark = pytest.mark.gpu

WORST = -0x20000000
INT_MAX = 2**31 - 1
SMEM_MAX = 227 * 1024                    # psb_phoneloop_launch: the kernel's dynamic shared memory ceiling
JUMP = 400_000_000                       # a renormalisation moves the best score up by > 5.3e8, nothing else by > 3.3e4


@pytest.fixture(scope="module")
def api():
    from pocketsphinx_b200 import api
    assert api.device_count() > 0, "no CUDA device visible"
    return api


def _topology(n_emit, n_sen, H, seed):
    """A synthetic Bakis topology (skip arcs for 5 states) and H phones with their own senone sequences."""
    from pocketsphinx_b200 import s3io
    from pocketsphinx_b200.model import synth_tmat_float
    rng = np.random.default_rng(seed)
    tp = s3io.quantize_tmat(synth_tmat_float(rng, 8, n_emit, n_emit == 5))
    sseq = rng.integers(0, n_sen, (H, n_emit)).astype(np.uint16)
    return tp, sseq, np.arange(H, dtype=np.int32), rng.integers(0, len(tp), H).astype(np.int32)


def _oracle_pl(tp, sseq, ssid, tmat, scr, window, beam, pbeam, pip, weight):
    # the oracle's penalty ring needs window >= 1; the search itself never reads the penalties
    from oracle import oracle
    return oracle.phoneloop_run(tp, sseq, ssid, tmat, scr, max(window, 1), beam, pbeam, pip, weight)


def _phoneloop_vs_oracle(api, tp, sseq, n_sen, ssid, tmat, parts, params, trace, ctx=None):
    """One batch of utterances (parts: [T][n_sen] each, any T >= 0) through run_host, every utterance against the
    oracle.  Returns the oracle's outputs per utterance."""
    own = ctx is None
    ctx = api.HmmContext(tp, sseq, n_sen) if own else ctx
    pl = api.PhoneLoop(ctx, ssid, tmat, *params)
    off = api.Batch.offsets([len(p) for p in parts])
    got = pl.run_host(np.concatenate(parts), off, trace=trace)
    n_emit, window = tp.shape[1], params[0]
    wants = []
    for u, p in enumerate(parts):
        a, b = off[u], off[u + 1]
        want = _oracle_pl(tp, sseq, ssid, tmat, p, *params)
        assert np.array_equal(got["best"][a:b], want["best"]), "utt %d (%d frames): best scores differ" % (u, len(p))
        if window:
            assert np.array_equal(got["pen"][a:b], want["pen"]), "utt %d (%d frames): penalties differ" % (u, len(p))
        if trace:
            assert_hmm_equal(got["hmm"][a:b], want["hmm"], n_emit, "utt %d (%d frames)" % (u, len(p)))
        wants.append(want)
    pl.close()
    if own:
        ctx.close()
    return wants


# ---------------------------------------------------------------------------------------------------------------
# phone loop: renormalisation

@pytest.mark.parametrize("n_emit", [3, 5])
def test_phoneloop_renormalises_where_the_best_score_reaches_the_floor(api, n_emit):
    """40 000 frames at 30 000 - 32 767 per frame with beam -40 000: the best score reaches the 80 000-wide window
    above the floor (it cannot jump over it in one frame) by frame 17 895 and again before frame 40 000; around it
    a ragged batch of 0, 1 and 17 000 frames, which stays short of the bound."""
    n_sen, H = 64, 64
    tp, sseq, ssid, tmat = _topology(n_emit, n_sen, H, 7 + n_emit)
    rng = np.random.default_rng(70 + n_emit)
    lens = [40000, 0, 1, 17000]
    parts = [rng.integers(30000, 32768, (t, n_sen)).astype(np.int16) for t in lens]
    wants = _phoneloop_vs_oracle(api, tp, sseq, n_sen, ssid, tmat, parts, (5, -40000, -30000, 0, 3.0), trace=False)
    best = wants[0]["best"].astype(np.int64)
    jumps = np.flatnonzero(np.diff(best) > JUMP)
    assert len(jumps) >= 2, "the best score never renormalised: minimum %d" % best.min()
    assert (best[jumps] < WORST + 80000).all() and (best[jumps + 1] > -40000).all()
    assert not (np.diff(wants[3]["best"].astype(np.int64)) > JUMP).any()


def _every_frame_case(n_emit):
    n_sen, H = 300, 64
    tp, sseq, ssid, tmat = _topology(n_emit, n_sen, H, 90 + n_emit)
    rng = np.random.default_rng(900 + n_emit)
    parts = [rng.integers(1000, 4000, (t, n_sen)).astype(np.int16) for t in (120, 0, 1, 57)]
    return tp, sseq, n_sen, ssid, tmat, parts


@pytest.mark.parametrize("n_emit", [3, 5])
def test_phoneloop_renormalising_in_every_frame(api, n_emit):
    """beam = -300 000 000 makes best_score + 2 * beam < WORST_SCORE hold in every frame (and prunes nothing):
    every frame starts from scores relative to the last best one.  Full trace, best scores and penalties."""
    tp, sseq, n_sen, ssid, tmat, parts = _every_frame_case(n_emit)
    wants = _phoneloop_vs_oracle(api, tp, sseq, n_sen, ssid, tmat, parts, (5, -300000000, -250, -7, 2.5), trace=True)
    # pulled back every frame: no best score below one frame's cost (<= 4 000 + transitions), where the same
    # search without renormalisation sinks by >= 1 000 per frame
    base = _oracle_pl(tp, sseq, ssid, tmat, parts[0], 5, -300, -250, -7, 2.5)["best"]
    for u in (0, 3):
        assert wants[u]["best"].min() > -5000, u
    assert base.min() < -100000


@pytest.mark.parametrize("n_emit", [3, 5])
def test_phoneloop_penalties_past_the_int32_range(api, n_emit):
    """With a normal beam phones get pruned and carry bestscore = WORST_SCORE, and with weight 6
    (WORST_SCORE - best) * 6 lies below INT_MIN.  The double-to-int conversion saturates to INT_MIN on both sides
    (x86 cvttsd2si in the oracle, cvt.rzi.s32.f64 on the device); the window's maximum then floors the penalty at
    WORST_SCORE.  A conversion that wrapped would give a positive penalty instead."""
    tp, sseq, n_sen, ssid, tmat, parts = _every_frame_case(n_emit)
    wants = _phoneloop_vs_oracle(api, tp, sseq, n_sen, ssid, tmat, parts, (5, -300, -250, -7, 6.0), trace=True)
    for u in (0, 3):
        w = wants[u]
        assert ((WORST - w["best"].astype(np.int64)) * 6 < -2**31).all()
        assert (w["hmm"]["bestscore"] == WORST).any() and (w["pen"] == WORST).any(), u
        assert (w["pen"] > WORST).any() and (w["pen"] <= 0).all(), u


@pytest.mark.parametrize("H", [64, 1500])
def test_phoneloop_transition_where_the_entry_threshold_is_below_the_floor(api, H):
    """pip = +5 and pbeam = -600 000 000: best_score + pbeam < WORST_SCORE + pip in every frame, so the reference's
    sequential phone_transition also takes the phones that an earlier source just entered (idle or just pruned,
    exit score WORST_SCORE) as sources.  Their candidate, WORST_SCORE + 5, never beats what the entering source
    left, so the kernel's max over the survivors gives the same HMMs.  Full trace."""
    n_sen = 300
    tp, sseq, ssid, tmat = _topology(3, n_sen, H, 11)
    rng = np.random.default_rng(12)
    parts = [rng.integers(0, 3000, (t, n_sen)).astype(np.int16) for t in (90, 0, 1, 33)]
    for p in parts:
        p[:, rng.integers(0, n_sen, 20)] = rng.integers(0, 50)
    pbeam, pip = -600000000, 5
    wants = _phoneloop_vs_oracle(api, tp, sseq, n_sen, ssid, tmat, parts, (5, -300, pbeam, pip, 2.5), trace=True)
    extra = 0
    for w in (wants[0], wants[3]):
        assert (w["best"].astype(np.int64) + pbeam < WORST + pip).all()
        h = w["hmm"]
        nxt = h["frame"] == np.arange(1, len(h) + 1)[:, None]          # active in the next frame
        surv = h["bestscore"] != WORST                                 # survived pruning (an entry leaves bestscore alone)
        first = np.argmax(surv, axis=1)
        later = np.arange(H)[None, :] > first[:, None]
        extra += int((nxt & ~surv & later).sum())                      # entered from idle or pruned, after a source
    assert extra > 0


# ---------------------------------------------------------------------------------------------------------------
# phone loop: shapes

SIZES = [1, 31, 33, 1024, 1025, 2049]


def _h_max(n_emit, window):
    return (SMEM_MAX // 4 - 64) // (2 * n_emit + 4 + window)


def _smem(n_emit, window, H):
    return ((2 * n_emit + 4 + window) * H + 64) * 4


@pytest.mark.parametrize("window", [0, 10])
@pytest.mark.parametrize("n_emit", [1, 3, 4, 5])
def test_phoneloop_shapes(api, n_emit, window):
    """1, 31, 33 HMMs (part of one warp, one HMM into a second warp), 1024 / 1025 (the CTA's 1024 threads, and one
    HMM that a thread takes on a second pass), 2049, and the largest set the shared memory holds; ragged batches
    with zero-frame utterances.  One HMM past the ceiling is an error naming the bytes, and the context stays
    usable."""
    g = golden("hmm_vit_eval.npz")
    tp, sseq = g["n%d_tp" % n_emit], g["n%d_sseq" % n_emit]
    n_sen = len(g["n%d_senscr" % n_emit])
    rng = np.random.default_rng(40 * n_emit + window)
    h_max = _h_max(n_emit, window)
    assert _smem(n_emit, window, h_max) <= SMEM_MAX < _smem(n_emit, window, h_max + 1)
    ctx = api.HmmContext(tp, sseq, n_sen)
    params = (window, -300, -250, -7, 2.5)
    for H in SIZES + [h_max]:
        ssid = (np.arange(H) % len(sseq)).astype(np.int32)               # repeated phones: ties in the arg-max
        tmat = rng.integers(0, len(tp), H).astype(np.int32)
        parts = [rng.integers(0, 600, (t, n_sen)).astype(np.int16) for t in (0, 23, 1, 0, 40)]
        for p in parts:
            p[:, rng.integers(0, n_sen, 8)] = 0
        _phoneloop_vs_oracle(api, tp, sseq, n_sen, ssid, tmat, parts, params, trace=True, ctx=ctx)
    H = h_max + 1
    pl = api.PhoneLoop(ctx, (np.arange(H) % len(sseq)).astype(np.int32), np.zeros(H, np.int32), *params)
    with pytest.raises(api.PsbError, match="%d HMMs needs %d bytes" % (H, _smem(n_emit, window, H))):
        pl.run_host(np.zeros((4, n_sen), np.int16), api.Batch.offsets([4]))
    pl.close()
    ssid, tmat = np.arange(40, dtype=np.int32), rng.integers(0, len(tp), 40).astype(np.int32)
    _phoneloop_vs_oracle(api, tp, sseq, n_sen, ssid, tmat, [rng.integers(0, 600, (30, n_sen)).astype(np.int16)], params,
                         trace=True, ctx=ctx)
    ctx.close()


@pytest.mark.parametrize("n_emit", [3, 5])
def test_phoneloop_run_device_and_final_hmms(api, n_emit):
    """psb_phoneloop_run_device on torch tensors: best scores and penalties in device memory equal run_host's,
    and final_hmms holds each utterance's HMMs after its last frame (the oracle's last trace row), or after
    phone_loop_search_start (hmm_clear + hmm_enter(0, -1, 0)) for an utterance of no frames."""
    import torch
    from oracle import oracle
    from pocketsphinx_b200.api import HMM_DTYPE
    from pocketsphinx_b200._lib import lib
    n_sen, H, window = 300, 100, 4
    tp, sseq, ssid, tmat = _topology(n_emit, n_sen, H, 50 + n_emit)
    rng = np.random.default_rng(500 + n_emit)
    lens = [0, 35, 1, 0, 60]
    scr = rng.integers(0, 800, (sum(lens), n_sen)).astype(np.int16)
    off = api.Batch.offsets(lens)
    params = (window, -300, -250, -7, 2.5)
    ctx = api.HmmContext(tp, sseq, n_sen)
    pl = api.PhoneLoop(ctx, ssid, tmat, *params)
    host = pl.run_host(scr, off)
    d_scr = torch.from_numpy(scr).cuda()
    d_best = torch.full((len(scr),), 7, dtype=torch.int32, device="cuda")
    d_pen = torch.full((len(scr), H), 7, dtype=torch.int32, device="cuda")
    final = np.zeros((len(lens), H), HMM_DTYPE)
    rc = lib().psb_phoneloop_run_device(pl.h, C.c_void_p(d_scr.data_ptr()), off.ctypes.data, len(lens),
                                        C.c_void_p(d_best.data_ptr()), C.c_void_p(d_pen.data_ptr()), final.ctypes.data, None)
    assert rc == 0, lib().psb_last_error().decode()
    assert np.array_equal(d_best.cpu().numpy(), host["best"]) and np.array_equal(d_pen.cpu().numpy(), host["pen"])
    start = oracle.OracleHmmCtx(tp, sseq).init(H, np.zeros(H, np.int32), ssid, tmat)
    for i in range(H):
        oracle.hmm_clear(start, i)
    start["score"][:, 0] = 0; start["history"][:, 0] = -1; start["frame"] = 0
    for u, T in enumerate(lens):
        if T == 0:
            want = start
        else:
            want = _oracle_pl(tp, sseq, ssid, tmat, scr[off[u]:off[u + 1]], *params)["hmm"][-1]
        assert_hmm_equal(final[u], want, n_emit, "utt %d (%d frames)" % (u, T))
    pl.close(); ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# forced alignment

def _align_case(n_emit):
    """40 000 frames at >= 30 000 per frame (the bound, best_score < -533 725 184, is certain by frame 17 792 and
    trips twice), phone k of the untimed chain's senones cheaper in the k-th of 60 stretches.  Three chains over the
    same scores: untimed (60 phones, the full-width token arena of 58 / 96 MB), windowed from word timings (a banded
    arena), and windowed with its last words past the end (cannot finish)."""
    from pocketsphinx_b200.align import phone_windows
    from pocketsphinx_b200.model import synth_ptm
    pm = synth_ptm(seed=31, n_density=32, n_sen=300, n_emit_state=n_emit, skip_arcs=(n_emit == 5))
    rng = np.random.default_rng(40 + n_emit)
    T, H = 40000, 60
    ssid = rng.integers(0, len(pm.sseq), H).astype(np.int32)
    tmat = rng.integers(0, pm.tp.shape[0], H).astype(np.int32)
    scr = rng.integers(31500, 32768, (T, pm.n_sen)).astype(np.int16)
    edge = np.linspace(0, T, H + 1).astype(int)
    for k in range(H):
        sen = np.unique(pm.sseq[ssid[k]])
        scr[edge[k]:edge[k + 1], sen] = rng.integers(30000, 30400, (edge[k + 1] - edge[k], len(sen)))
    chains = [(ssid, tmat, None, None)]
    n_words = 40
    n_ph = rng.integers(1, 4, n_words)
    dur = rng.multinomial(T - 20 * n_words, np.ones(n_words) / n_words) + 20
    word = np.repeat(np.arange(n_words), n_ph)
    w_ssid = rng.integers(0, len(pm.sseq), len(word)).astype(np.int32)
    w_tmat = rng.integers(0, pm.tp.shape[0], len(word)).astype(np.int32)
    for late in (0, 2500):                         # the last three words start 2 500 frames later: past the end
        start = np.concatenate([[0], np.cumsum(dur)[:-1]]) + late * (np.arange(n_words) >= n_words - 3)
        sf, ef = phone_windows(start[word], dur[word], n_emit)
        chains.append((w_ssid, w_tmat, sf, ef))
    return pm, scr, chains


@pytest.mark.parametrize("n_emit", [3, 5])
def test_align_renormalises_where_the_best_score_reaches_the_floor(api, n_emit):
    """Status, and start / duration / score of every state, against pso_align_run.  Without renormalisation every
    state scores <= 0 (token scores only fall along a path); a state whose frames span a renormalisation scores
    the difference of a normalised and a raw token score instead, > 0, as the reference's does.  That is the branch
    showing in the oracle's own output, and the device must agree on exactly those scores.  (Across a
    renormalisation the untimed chain's path degenerates: states left below the floor are not normalised.  The
    reference does the same.)"""
    import torch
    from oracle import oracle
    pm, scr, chains = _align_case(n_emit)
    T = len(scr)
    utt_off = (np.arange(len(chains) + 1) * T).astype(np.int32)
    ph_off = np.concatenate([[0], np.cumsum([len(c[0]) for c in chains])]).astype(np.int32)
    sf = np.concatenate([c[2] if c[2] is not None else np.zeros(len(c[0]), np.int32) for c in chains])
    ef = np.concatenate([c[3] if c[3] is not None else np.full(len(c[0]), INT_MAX, np.int32) for c in chains])
    ctx = api.HmmContext(pm.tp, pm.sseq, pm.n_sen)
    d_scr = torch.from_numpy(np.tile(scr, (len(chains), 1))).cuda()
    status, st, du, sc = ctx.align(None, utt_off, ph_off, np.concatenate([c[0] for c in chains]),
                                   np.concatenate([c[1] for c in chains]), sf=sf, ef=ef, device_ptr=d_scr.data_ptr())
    del d_scr
    for u, (ssid, tmat, usf, uef) in enumerate(chains):
        rc, wst, wdu, wsc = oracle.align_run(pm.tp, pm.sseq, ssid, tmat, scr, sf=usf, ef=uef)
        assert status[u] == rc, "chain %d: status %d, oracle %d" % (u, status[u], rc)
        sl = slice(ph_off[u] * n_emit, ph_off[u + 1] * n_emit)
        assert np.array_equal(st[sl], wst) and np.array_equal(du[sl], wdu) and np.array_equal(sc[sl], wsc), "chain %d" % u
        if u < 2:
            assert rc == 0 and (wsc > 0).any(), "chain %d: no state spans a renormalisation" % u
        else:
            assert rc != 0                     # the chain the two above show crossing the bound, cut short
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# n-gram search, both passes

def _ngram_case(tag, maxwpf):
    c = {k[len(tag) + 1:]: v for k, v in golden("en_us_fwdtree.npz").items() if k.startswith(tag + ".")}
    info = c["info"].copy()
    info[8] = -300000000                   # beam: best_score + 2 * beam < WORST_SCORE in every frame, both passes
    if maxwpf:
        info[14] = 3                       # -maxwpf keeps the first pass's tables small though the beam prunes nothing
    scr = golden("en_us_goforward.npz")["senscr"]
    parts = [scr[:60], scr[:0], scr[:1], scr[100:137], scr[200:260]]
    return c, info, parts


def _pulled_back(want, base):
    """Scores were pulled back towards 0: the renormalised table's largest score magnitude is below the plain one's."""
    return int(np.abs(want[0][:, 4]).max()) < int(np.abs(base[0][:, 4]).max())


def _same(got, want, what):
    assert len(got[0]) == len(want[0]) and np.array_equal(got[0], want[0]), what + ": bp"
    assert np.array_equal(got[1], want[1]), what + ": bscore stack"
    assert np.array_equal(got[2], want[2]), what + ": bp_table_idx"


def _device_scores(parts):
    import torch
    utt_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int32)
    return utt_off, torch.from_numpy(np.ascontiguousarray(np.concatenate(parts))).cuda()


def test_ngram_first_pass_renormalises_on_the_device(api, en_us):
    from oracle import oracle
    c, info, parts = _ngram_case("default", True)
    cit = en_us.phone_tmat[:int(info[6])]
    want = [oracle.fwdtree_run(en_us.tp, en_us.sseq, cit, info, c["model"], p) for p in parts]
    for u in (0, 3, 4):
        assert _pulled_back(want[u], oracle.fwdtree_run(en_us.tp, en_us.sseq, cit, c["info"], c["model"], parts[u])), u
    utt_off, d_scr = _device_scores(parts)
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    out = ctx.ngram_fwdtree(d_scr.data_ptr(), utt_off, info, c["model"], cit, max(len(w[0]) for w in want) + 64,
                            max(len(w[1]) for w in want) + 4096)
    for u in range(len(parts)):
        _same(out[u], want[u], "utt %d (%d frames)" % (u, len(parts[u])))
    ctx.close()


def test_ngram_second_pass_renormalises_on_the_device(api, en_us):
    """The second pass alone, behind a plain first pass (the second pass tests the same beam field,
    ngram_search_fwdflat.c:830)."""
    from oracle import oracle
    c, info, parts = _ngram_case("flat_wide", False)
    n_ci = int(info[6])
    cit, cis = en_us.phone_tmat[:n_ci], en_us.phone_ssid[:n_ci]
    first = [oracle.fwdtree_run(en_us.tp, en_us.sseq, cit, c["info"], c["model"], p)[0] for p in parts]
    want = [oracle.fwdflat_run(en_us.tp, en_us.sseq, cit, cis, info, c["model"], b, p) for b, p in zip(first, parts)]
    for u in (0, 3, 4):
        base = oracle.fwdflat_run(en_us.tp, en_us.sseq, cit, cis, c["info"], c["model"], first[u], parts[u])
        assert _pulled_back(want[u], base), u
    utt_off, d_scr = _device_scores(parts)
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    out = ctx.ngram_fwdflat(d_scr.data_ptr(), utt_off, info, c["model"], cit, cis, first, max(len(w[0]) for w in want) + 64,
                            max(len(w[1]) for w in want) + 4096)
    for u in range(len(parts)):
        _same(out[u], want[u], "utt %d (%d frames)" % (u, len(parts[u])))
    ctx.close()


def test_ngram_two_pass_renormalises_on_the_device(api, en_us):
    """Both passes back to back on the device, both renormalising in every frame."""
    from oracle import oracle
    c, info, parts = _ngram_case("flat_wide", True)
    n_ci = int(info[6])
    cit, cis = en_us.phone_tmat[:n_ci], en_us.phone_ssid[:n_ci]
    first = [oracle.fwdtree_run(en_us.tp, en_us.sseq, cit, info, c["model"], p)[0] for p in parts]
    want = [oracle.fwdflat_run(en_us.tp, en_us.sseq, cit, cis, info, c["model"], b, p) for b, p in zip(first, parts)]
    for u in (0, 3, 4):
        base1 = oracle.fwdtree_run(en_us.tp, en_us.sseq, cit, c["info"], c["model"], parts[u])[0]
        base = oracle.fwdflat_run(en_us.tp, en_us.sseq, cit, cis, c["info"], c["model"], base1, parts[u])
        assert _pulled_back(want[u], base), u
    utt_off, d_scr = _device_scores(parts)
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    out, n_first = ctx.ngram_two_pass(d_scr.data_ptr(), utt_off, info, c["model"], cit, cis, max(len(w[0]) for w in want) + 64,
                                      max(len(w[1]) for w in want) + 4096, first_cap=max(len(b) for b in first) + 64,
                                      first_bss_cap=1 << 18)
    assert n_first.tolist() == [len(b) for b in first]
    for u in range(len(parts)):
        _same(out[u], want[u], "utt %d (%d frames)" % (u, len(parts[u])))
    ctx.close()
