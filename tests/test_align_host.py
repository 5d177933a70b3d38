"""CPU: the host side of forced alignment (pocketsphinx_b200.align) -- word lookup, phone chains, the per-phone
windows of the second pass, ps_alignment_propagate -- against the compiled reference (oracle/_ref/libpsref.so), and
the token band align_kernel keeps (the C restatement tests/emul/align_banded.c: no token outside the band, the same
alignments as pso_align_run)."""
import os

import numpy as np
import pytest

from conftest import ROOT

REF = os.path.join(ROOT, "oracle", "_ref")
M = os.path.join(REF, "model")
HD, DIC, LM = os.path.join(M, "en-us"), os.path.join(M, "cmudict-en-us.dict"), os.path.join(M, "en-us.lm.bin")
GO = os.path.join(REF, "data", "goforward.raw")
TI_HD, TI_DIC, TI_LM = (os.path.join(M, "tidigits_hmm"), os.path.join(M, "tidigits_lm", "tidigits.dic"),
                        os.path.join(M, "tidigits_lm", "tidigits.lm.bin"))
TI_AUDIO = os.path.join(REF, "data", "dhd.2934z.raw")
INT_MAX = 2**31 - 1


def _needs_ref():
    from oracle import refdrv
    if not (refdrv.available() and os.path.exists(HD) and os.path.exists(GO)):
        pytest.skip("compiled reference and its model files not present")


def _tables(hd=HD, dic=DIC, cache={}):
    from pocketsphinx_b200.align import AlignTables
    if (hd, dic) not in cache:
        cache[(hd, dic)] = AlignTables(hd, dic)
    return cache[(hd, dic)]


def _levels(al):
    return [np.array([[e.start, e.duration, e.score, e.parent] for e in lv], np.int64)
            for lv in (al.words, al.phones, al.states)]


def _host_align(hd, tb, scr, wids, w_start, w_dur, windows):
    """What align_batch does for one utterance, with the C restatement in place of the kernel."""
    from oracle import oracle
    from pocketsphinx_b200 import align
    s, t, ci, word = tb.chain(wids)
    if windows:
        sf, ef = align.phone_windows(np.asarray(w_start)[word], np.asarray(w_dur)[word], tb.n_emit)
    else:
        sf, ef = np.zeros(len(s), np.int32), np.full(len(s), INT_MAX, np.int32)
    pm = _packed(hd)
    rc, st, du, sc = oracle.align_run(pm["tp"], pm["sseq"], s, t, scr, sf=sf, ef=ef)
    if rc:
        return None, align.failure_reason(rc)
    return align.propagate([tb.words[w] for w in wids], w_start, w_dur, [tb.md["ciname"][c] for c in ci], word,
                           [str(int(x)) for x in tb.md["sseq"][s].reshape(-1)], tb.n_emit, st, du, sc), None


_PACKED = {}


def _packed(hd):
    from oracle import refdrv
    if hd not in _PACKED:
        _PACKED[hd] = refdrv.RefModel(hd).packed()
    return _PACKED[hd]


def _ref_scores(hd, pcm, second, **kv):
    """The reference's senone scores of one decode of pcm on a fresh decoder, or of the second decode of it (the front
    end's state carried from the first, as decode_single's second pass sees it)."""
    from oracle import refdrv
    m = refdrv.RefModel(hd, **kv)
    f = m.featurize_fresh(pcm)
    if second:
        f = m.featurize(pcm)
    s = m.score(f)
    m.close()
    return s


# ---------------------------------------------------------------------------------------------------------------
# words and chains

def test_lookup_words_fillers_and_unknown():
    _needs_ref()
    tb = _tables()
    w = tb.lookup("  <s> go\\tforward  <sil> the(2) ten meters </s>\n".replace("\\t", "\t"))
    assert [tb.words[i] for i in w] == ["<s>", "go", "forward", "<sil>", "the(2)", "ten", "meters", "</s>"]
    with pytest.raises(ValueError, match="'zzyzxq'"):
        tb.lookup("go zzyzxq forward")
    assert tb.lookup("") == []


@pytest.mark.parametrize("text", ["<s> go forward ten meters </s>", "go forward the(2) ten meters",
                                  "<s> go <sil> forward ten meters </s> <s> go forward </s>"])
def test_transcript_alignment_matches_reference(text):
    """Chains with alternates and fillers equal ps_alignment_populate's, and the states of the restated search over the
    reference's scores equal its own alignment (refdrv_align: ps_alignment_add_word with no timing)."""
    _needs_ref()
    from oracle import refdrv
    tb = _tables()
    pcm = np.fromfile(GO, np.int16)
    r = refdrv.align(HD, DIC, text, pcm)
    wids = tb.lookup(text)
    s, t, _, _ = tb.chain(wids)
    assert np.array_equal(s, r["ssid"]) and np.array_equal(t, r["tmatid"])
    al, why = _host_align(HD, tb, _ref_scores(HD, pcm, False, compallsen="yes"), wids, np.zeros(len(wids)),
                          np.zeros(len(wids)), False)
    assert why is None
    st = _levels(al)[2]
    assert np.array_equal(st[:, 0], r["start"]) and np.array_equal(st[:, 1], r["dur"])
    assert np.array_equal(st[:, 2], r["score"])


def _second_pass_case(hd, dic, lm, audio, **kv):
    import align_cases
    from oracle import refdrv
    pcm = np.fromfile(audio, np.int16)
    kv = dict(compallsen="yes", bestpath="no", **kv)
    r = align_cases.phone_align(hd, lm, dic, pcm, **kv)
    d = refdrv.decode(hd, lm, dic, pcm, **kv)
    tb = _tables(hd, dic)
    seg = [l.split() for l in d["seg"].strip().split("\n") if l]
    wids = [tb.wid[x[0]] for x in seg]
    sf = np.array([int(x[1]) for x in seg]); ef = np.array([int(x[2]) for x in seg])
    al, why = _host_align(hd, tb, _ref_scores(hd, pcm, True, **kv), wids, sf, ef - sf + 1, True)
    return r, tb, wids, al, why


@pytest.mark.parametrize("case", ["en_us", "tidigits"])
def test_second_pass_matches_reference(case):
    """-state_align yes: the words of ps_seg_iter with their timing, phones confined to their word's window
    (state_align_search_init, min_nframes included), searched over the second decode's scores, propagated: all three
    levels equal the reference's (its public API: decode, ps_set_alignment(ps, NULL), decode again)."""
    _needs_ref()
    if case == "tidigits":
        if not os.path.exists(TI_LM):
            pytest.skip("tidigits files not present")
        r, tb, wids, al, why = _second_pass_case(TI_HD, TI_DIC, TI_LM, TI_AUDIO)
    else:
        r, tb, wids, al, why = _second_pass_case(HD, DIC, LM, GO)
    assert r["end_utt"] >= 0 and why is None
    assert [e[0] for e in r["words"]] == [tb.words[w] for w in wids]
    for got, want in zip(_levels(al), (r["words"], r["phones"], r["states"])):
        assert np.array_equal(got, np.array([e[1:] for e in want], np.int64))
    assert [e[0] for e in r["phones"]] == [e.name for e in al.phones]
    assert [e[0] for e in r["states"]] == [e.name for e in al.states]
    # the phones of each word are its children, the states of each phone theirs
    assert [e.name for e in al.children("word", 1)] == [tb.md["ciname"][c] for c in tb.prons[wids[1]]]
    assert len(al.children("phone", 0)) == tb.n_emit


def test_first_pass_scores_would_differ():
    """The second decode's scores differ from the first's (the front end carries its noise tracker), and so does the
    alignment: the Decoder scores the second pass as the utterance's own repeat."""
    _needs_ref()
    r, tb, wids, al, why = _second_pass_case(HD, DIC, LM, GO)
    pcm = np.fromfile(GO, np.int16)
    assert not np.array_equal(_ref_scores(HD, pcm, False, compallsen="yes"), _ref_scores(HD, pcm, True, compallsen="yes"))


def test_phone_windows_rules():
    from pocketsphinx_b200.align import phone_windows
    sf, ef = phone_windows([0, 10, 20, 23, 30], [10, 2, 3, 7, 0], 3)
    assert sf.tolist() == [0, 0, 20, 23, 0]                 # start 0, or a window shorter than 3 states: always active
    assert ef.tolist() == [10, INT_MAX, 23, 30, INT_MAX]


def test_propagate_keeps_populate_values_for_unvisited_states():
    """A state the backtrace skips keeps its word's start and duration and score 0, and its phone sums them anyway
    (ps_alignment_propagate sums every state)."""
    from pocketsphinx_b200.align import propagate
    al = propagate(["a", "b"], [0, 5], [5, 4], ["x", "y"], np.array([0, 1]), ["1", "2", "3", "4"], 2,
                   [0, 3, 5, -1], [3, 2, 4, -1], [0, -7, -9, -1])
    assert [(e.start, e.duration, e.score) for e in al.states] == [(0, 3, 0), (3, 2, -7), (5, 4, -9), (5, 4, 0)]
    assert [(e.start, e.duration, e.score) for e in al.phones] == [(0, 5, -7), (5, 8, -9)]
    assert [(e.start, e.duration, e.score, e.parent) for e in al.words] == [(0, 5, -7, -1), (5, 8, -9, -1)]


# ---------------------------------------------------------------------------------------------------------------
# the token band

def _band_cases(n_emit):
    from pocketsphinx_b200.model import synth_ptm
    pm = synth_ptm(seed=31, n_density=32, n_sen=300, n_emit_state=n_emit, skip_arcs=(n_emit == 5))
    rng = np.random.default_rng(5 + n_emit)
    cases = []
    for k in range(14):
        n_words = int(rng.integers(1, 25))
        n_ph = rng.integers(1, 5, n_words)
        dur = rng.integers(1, 30, n_words)                   # some words shorter than a phone's states
        if k % 3 == 0:
            dur[rng.integers(0, n_words)] = 0
        start = np.concatenate([[0], np.cumsum(dur)[:-1]])
        T = int(dur.sum()) + int(rng.integers(-3, 4))
        if k == 5:
            T = max(1, T // 4)                               # too short: fails
        word = np.repeat(np.arange(n_words), n_ph)
        from pocketsphinx_b200.align import phone_windows
        sf, ef = phone_windows(start[word], dur[word], n_emit)
        if k == 7:                                           # a closed window ahead: alignment fails in a frame
            ef[len(ef) // 2] = 1
        H = len(word)
        ssid = rng.integers(0, len(pm.sseq), H).astype(np.int32)
        tmat = rng.integers(0, pm.tp.shape[0], H).astype(np.int32)
        hi_scr = k in (3, 9)                                 # large scores, far from the floor in so few frames
        scr = rng.integers(20000, 32000, (max(T, 1), pm.n_sen)) if hi_scr else rng.integers(0, 400, (max(T, 1), pm.n_sen))
        cases.append((ssid, tmat, sf, ef, scr[:max(T, 1)].astype(np.int16)))
    # untimed chains: the full width
    H = 30
    cases.append((rng.integers(0, len(pm.sseq), H).astype(np.int32), rng.integers(0, pm.tp.shape[0], H).astype(np.int32),
                  None, None, rng.integers(0, 400, (150, pm.n_sen)).astype(np.int16)))
    cases.append(_renorm_case(pm, n_emit))
    return pm, cases


RENORM_T = 20000


def _renorm_case(pm, n_emit):
    """A windowed chain over RENORM_T frames at >= 30 000 per frame: the best score falls below the alignment's
    bound (best_score - 0x300000 < WORST_SCORE, -533 725 184) by frame 17 792, and the search renormalises."""
    from pocketsphinx_b200.align import phone_windows
    rng = np.random.default_rng(50 + n_emit)
    n_words = 30
    dur = rng.multinomial(RENORM_T - 20 * n_words, np.ones(n_words) / n_words) + 20
    start = np.concatenate([[0], np.cumsum(dur)[:-1]])
    word = np.repeat(np.arange(n_words), rng.integers(1, 4, n_words))
    sf, ef = phone_windows(start[word], dur[word], n_emit)
    H = len(word)
    return (rng.integers(0, len(pm.sseq), H).astype(np.int32), rng.integers(0, pm.tp.shape[0], H).astype(np.int32), sf, ef,
            rng.integers(30000, 32768, (RENORM_T, pm.n_sen)).astype(np.int16))


@pytest.mark.parametrize("n_emit", [3, 5])
def test_band_restatement_keeps_every_token_and_result(n_emit):
    import align_cases
    from oracle import oracle
    from pocketsphinx_b200.align import band_tokens, token_band
    pm, cases = _band_cases(n_emit)
    kinds = set()
    narrower = 0
    for k, (ssid, tmat, sf, ef, scr) in enumerate(cases):
        T, H = len(scr), len(ssid)
        lo, hi = align_cases.band(H, T, sf, ef)
        plo, phi = token_band(sf, ef, T, H)
        assert np.array_equal(lo, plo) and np.array_equal(hi, phi)
        want = oracle.align_run(pm.tp, pm.sseq, ssid, tmat, scr, sf=sf, ef=ef)
        got = align_cases.align_run_banded(pm.tp, pm.sseq, ssid, tmat, scr, sf=sf, ef=ef)
        assert got[4] == 0, "%d tokens outside the band" % got[4]
        assert got[0] == want[0]
        for a, b in zip(got[1:4], want[1:4]):
            assert np.array_equal(a, b)
        kinds.add(0 if want[0] == 0 else (-1 if want[0] == -1 else -2))
        if k == len(cases) - 1:
            # the bound was crossed: without renormalisation no state scores above 0 (token scores only fall along a
            # path), while a state that spans it scores a normalised minus a raw token score
            assert T == RENORM_T and want[0] == 0 and (want[3] > 0).any()
        n = band_tokens(sf, ef, T, H, n_emit)
        assert n <= T * H * n_emit
        narrower += n < T * H * n_emit
        if sf is None:
            assert n == T * H * n_emit
    assert kinds == {0, -1, -2} and narrower >= 10


def test_band_is_tight_at_its_edges():
    """The band's edges are reached: with every phone entered as early as its window allows, lo_f and hi_f phones
    hold tokens (pinned against the restatement: a band one phone narrower on either side loses tokens)."""
    import align_cases
    from pocketsphinx_b200.align import token_band
    from pocketsphinx_b200.model import synth_ptm
    pm = synth_ptm(seed=3, n_density=32, n_sen=300, n_emit_state=3)
    H, w = 20, 6
    sf = np.array([0] + [w * i for i in range(1, H)], np.int32)
    ef = np.array([w * (i + 1) for i in range(H)], np.int32)
    T = w * H
    scr = np.full((T, pm.n_sen), 10, np.int16)
    ssid = np.zeros(H, np.int32); tmat = np.zeros(H, np.int32)
    lo, hi = token_band(sf, ef, T, H)
    lo, hi = np.asarray(lo, np.int32), np.asarray(hi, np.int32)
    # shrink the band by one phone at one end in a frame where it is wider than one phone, and tokens fall outside
    f = int(np.argmax(hi - lo >= 1))
    for dlo, dhi in ((1, 0), (0, -1)):
        l2, h2 = lo.copy(), hi.copy()
        l2[f] += dlo; h2[f] += dhi
        n_out = align_cases.align_run_banded(pm.tp, pm.sseq, ssid, tmat, scr, sf, ef, l2, h2)[4]
        assert n_out > 0
    assert align_cases.align_run_banded(pm.tp, pm.sseq, ssid, tmat, scr, sf, ef, lo, hi)[4] == 0


def test_band_widths_of_reference_segments():
    """The band of the second pass over the reference's own segments of goforward (DESIGN 4.7 states these counts)."""
    _needs_ref()
    from oracle import refdrv
    from pocketsphinx_b200.align import band_tokens, phone_windows
    tb = _tables()
    pcm = np.fromfile(GO, np.int16)
    d = refdrv.decode(HD, LM, DIC, pcm, compallsen="yes", bestpath="no")
    seg = [l.split() for l in d["seg"].strip().split("\n") if l]
    wids = [tb.wid[x[0]] for x in seg]
    sf = np.array([int(x[1]) for x in seg]); ef = np.array([int(x[2]) for x in seg])
    _, _, _, word = tb.chain(wids)
    psf, pef = phone_windows(sf[word], (ef - sf + 1)[word], 3)
    T, H = d["n_frames"], len(word)
    n = band_tokens(psf, pef, T, H, 3)
    assert n < T * H * 3 / 3                                  # at least three times smaller than the dense table
