"""GPU: forced alignment from audio -- pocketsphinx_b200.align.Aligner (transcripts) and the Decoder's
-phone_align / -state_align second pass -- against the reference's own alignments, and align_kernel's banded token
arena on windowed and long utterances against the C restatement."""
import os

import numpy as np
import pytest

from conftest import ROOT, golden

pytestmark = [pytest.mark.gpu]
REF = os.path.join(ROOT, "oracle", "_ref")
M = os.path.join(REF, "model")
HD, DIC, LM = os.path.join(M, "en-us"), os.path.join(M, "cmudict-en-us.dict"), os.path.join(M, "en-us.lm.bin")
GO = os.path.join(REF, "data", "goforward.raw")
TI_HD, TI_DIC, TI_LM = (os.path.join(M, "tidigits_hmm"), os.path.join(M, "tidigits_lm", "tidigits.dic"),
                        os.path.join(M, "tidigits_lm", "tidigits.lm.bin"))
TI_AUDIO = os.path.join(REF, "data", "dhd.2934z.raw")
TEXTS = {"a": "<s> go forward ten meters </s>", "b": "go forward ten meters",
         "c": "<s> go forward ten meters </s> <s> go forward </s>"}       # tests/golden/en_us_align.npz


def _needs_files(*paths):
    for p in paths or (HD, GO):
        if not os.path.exists(p):
            pytest.skip("reference model and data files not present")


def _states(al):
    return np.array([[e.start, e.duration, e.score] for e in al.states], np.int64)


def _check_levels(al):
    """Words and phones are ps_alignment_propagate over the states."""
    n = len(al.states) // len(al.phones)
    s = _states(al)
    for i, p in enumerate(al.phones):
        assert p.start == s[i * n, 0] and p.duration == s[i * n:(i + 1) * n, 1].sum() and p.score == s[i * n:(i + 1) * n, 2].sum()
    for w, e in enumerate(al.words):
        mine = al.children("word", w)
        assert e.start == mine[0].start and e.duration == sum(p.duration for p in mine)
        assert e.score == sum(p.score for p in mine)


@pytest.mark.timeout(600)
def test_aligner_on_reference_scores_is_exact():
    """On the reference's own senone scores the Aligner's states are its alignments, bit for bit."""
    _needs_files()
    import torch
    from pocketsphinx_b200.align import Aligner
    g, ga = golden("en_us_goforward.npz"), golden("en_us_align.npz")
    al = Aligner(HD, DIC, max_utts=8, max_frames=4096)
    scr = torch.from_numpy(np.concatenate([g["senscr"]] * 3)).cuda()
    T = len(g["senscr"])
    out = al.align_senscr(scr.data_ptr(), np.arange(4, dtype=np.int32) * T, [TEXTS[t] for t in "abc"])
    for t, a in zip("abc", out):
        s = _states(a)
        assert np.array_equal(s[:, 0], ga[t + "_start"]) and np.array_equal(s[:, 1], ga[t + "_dur"]), t
        assert np.array_equal(s[:, 2], ga[t + "_score"]), t
        _check_levels(a)
        assert [w.name for w in a.words] == TEXTS[t].split()
    al.close()


@pytest.mark.timeout(600)
def test_aligner_from_audio_mixed_batch():
    """From audio: the three transcripts (states equal to the reference's own alignments), a
    shorter utterance, a transcript too long for its frames (fails to reach the final state), the same utterance
    twice (identical), an unknown word refused before any launch."""
    _needs_files()
    from pocketsphinx_b200.align import Aligner, band_tokens
    ga = golden("en_us_align.npz")
    go = np.fromfile(GO, np.int16)
    al = Aligner(HD, DIC, max_utts=8, max_frames=8192)
    with pytest.raises(ValueError, match="'qqzx'"):
        al.align_raw_batch([go], ["go qqzx"])
    texts = [TEXTS["a"], TEXTS["b"], TEXTS["c"], "go forward", " ".join(["go forward ten meters"] * 12), TEXTS["a"]]
    utts = [go, go, go, go[:20000], go[:8000], go]
    out = al.align_raw_batch(utts, texts)
    assert out[4] is None and al.reasons[4] == "Failed to reach final state in alignment"
    assert all(a is not None for k, a in enumerate(out) if k != 4)
    assert np.array_equal(_states(out[0]), _states(out[5]))
    n_equal, n_all, worst = 0, 0, 0
    for k, t in enumerate("abc"):
        s = _states(out[k])
        d = np.abs(s[:, 0] - ga[t + "_start"])
        n_equal += int((d == 0).sum()); n_all += len(d); worst = max(worst, int(d.max()))
        _check_levels(out[k])
    print("state starts equal to the reference's: %d of %d, largest difference %d frames" % (n_equal, n_all, worst))
    assert worst == 0 and n_equal == n_all
    # untimed chains: the arena is the dense table, frames x phones x states
    frames = [al.fe.n_frames(len(u)) for u in utts]
    n_ph = [len(al.tables.chain(al.tables.lookup(t))[0]) for t in texts]
    assert al.last_token_bytes == 8 * sum(band_tokens(None, None, T, H, 3) for T, H in zip(frames, n_ph))
    al.close()


def _second_pass_vs_reference(hd, dic, lm, audio):
    import align_cases
    from pocketsphinx_b200.decoder import Decoder
    pcm = np.fromfile(audio, np.int16)
    r = align_cases.phone_align(hd, lm, dic, pcm, compallsen="yes", bestpath="no")
    dec = Decoder(hd, dic, lm, max_utts=4, max_frames=4096, state_align="yes")
    out = dec.decode_raw_batch([pcm, pcm])
    a = out[0]["alignment"]
    assert a is not None and out[0]["alignment_error"] is None
    assert np.array_equal(_states(a), _states(out[1]["alignment"]))
    _check_levels(a)
    assert [w.name for w in a.words] == [dec.search["words"][w] for w in out[0]["seg"][:, 1]]
    got = {lv: np.array([[e.start, e.duration, e.score] for e in getattr(a, lv)]) for lv in ("words", "phones", "states")}
    want = {lv: np.array([e[1:4] for e in r[lv]]) for lv in ("words", "phones", "states")}
    same_words = [w.name for w in a.words] == [e[0] for e in r["words"]]
    report = {}
    if same_words:
        for lv in got:
            d = np.abs(got[lv][:, 0] - want[lv][:, 0])
            report[lv] = (int((got[lv] == want[lv]).all(1).sum()), len(d), int(d.max()))
    print("%s: same words %s; entries equal / total / largest start difference: %s" % (os.path.basename(audio), same_words, report))
    dec.close()
    return same_words, report


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", ["en_us", "tidigits"])
def test_decoder_state_align_matches_reference(case):
    """-state_align yes from audio against the reference's run (decode, ps_set_alignment(ps, NULL), decode again) at
    -compallsen yes: the same words, and start / duration / score equal at all three levels."""
    from oracle import refdrv
    if not refdrv.available():
        pytest.skip("compiled reference not present")
    if case == "en_us":
        _needs_files(HD, GO, LM)
        same, rep = _second_pass_vs_reference(HD, DIC, LM, GO)
    else:
        _needs_files(TI_HD, TI_AUDIO, TI_LM)
        same, rep = _second_pass_vs_reference(TI_HD, TI_DIC, TI_LM, TI_AUDIO)
    assert same
    for lv, (n_eq, n, worst) in rep.items():
        assert worst == 0 and n_eq == n, (lv, n_eq, n, worst)


@pytest.mark.timeout(900)
def test_decoder_without_align_unchanged_and_stream_carries_alignment():
    _needs_files(HD, GO, LM)
    from pocketsphinx_b200.decoder import Decoder
    go = np.fromfile(GO, np.int16)
    plain = Decoder(HD, DIC, LM, max_utts=8, max_frames=8192)
    dec = Decoder(HD, DIC, LM, max_utts=8, max_frames=8192, phone_align="yes")
    a, b = plain.decode_raw_batch([go]), dec.decode_raw_batch([go])
    assert "alignment" not in a[0] and a[0]["hyp"] == b[0]["hyp"] and np.array_equal(a[0]["seg"], b[0]["seg"])
    sil = np.zeros(16000, np.int16)
    stream = np.concatenate([sil, go, sil, sil, go, sil])
    res = dec.decode_stream_batch([stream, go], start_stream="session")
    n = 0
    for row in res:
        for d in row:
            al = d["alignment"]
            if len(d["seg"]) == 0:
                assert al is None and d["alignment_error"] is not None
                continue
            assert al is not None, d["alignment_error"]
            assert [w.name for w in al.words] == d["words"]
            assert sum(w.duration for w in al.words) == d["n_frames"]
            n += 1
    assert n >= 2
    plain.close(); dec.close()


@pytest.mark.timeout(900)
def test_windowed_and_long_utterances_arena_is_the_band():
    """A batch of windowed chains (the second pass's shape) and one long utterance of 3 000 phones whose dense table
    would be 2.2 GB: the results equal the C restatement's, and the arena is exactly the band sum."""
    import torch
    import align_cases
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.align import band_tokens, phone_windows
    from pocketsphinx_b200.model import synth_ptm
    pm = synth_ptm(seed=11, n_density=32, n_sen=300, n_emit_state=3)
    rng = np.random.default_rng(23)
    cases = []
    for n_words, T_long in ((30, None), (200, None), (1000, 30000)):
        dur = rng.integers(2, 40, n_words) if T_long is None else np.full(n_words, T_long // n_words)
        n_ph = rng.integers(1, 5, n_words) if T_long is None else np.full(n_words, 3)
        start = np.concatenate([[0], np.cumsum(dur)[:-1]])
        word = np.repeat(np.arange(n_words), n_ph)
        sf, ef = phone_windows(start[word], dur[word], 3)
        T = int(dur.sum())
        H = len(word)
        scr = rng.integers(0, 400, (T, pm.n_sen)).astype(np.int16)
        cases.append((rng.integers(0, len(pm.sseq), H).astype(np.int32), rng.integers(0, pm.tp.shape[0], H).astype(np.int32),
                      sf, ef, scr))
    utt_off = np.concatenate([[0], np.cumsum([len(c[4]) for c in cases])]).astype(np.int32)
    ph_off = np.concatenate([[0], np.cumsum([len(c[0]) for c in cases])]).astype(np.int32)
    ctx = api.HmmContext(pm.tp, pm.sseq, pm.n_sen)
    d = torch.from_numpy(np.concatenate([c[4] for c in cases])).cuda()
    cat = lambda k: np.concatenate([c[k] for c in cases])
    status, st, du, sc = ctx.align(None, utt_off, ph_off, cat(0), cat(1), cat(2), cat(3), device_ptr=d.data_ptr())
    want_bytes = 8 * sum(band_tokens(c[2], c[3], len(c[4]), len(c[0]), 3) for c in cases)
    got_bytes = int(api.lib().psb_align_last_token_bytes(ctx.h))
    dense = 8 * sum(len(c[4]) * len(c[0]) * 3 for c in cases)
    print("token arena %d bytes, dense table %d bytes" % (got_bytes, dense))
    assert got_bytes == want_bytes and dense > 50 * got_bytes
    for u, c in enumerate(cases):
        rc, wst, wdu, wsc, n_out = align_cases.align_run_banded(pm.tp, pm.sseq, c[0], c[1], c[4], sf=c[2], ef=c[3])
        assert n_out == 0 and status[u] == rc
        sl = slice(ph_off[u] * 3, ph_off[u + 1] * 3)
        assert np.array_equal(st[sl], wst) and np.array_equal(du[sl], wdu) and np.array_equal(sc[sl], wsc), u
    ctx.close()
