"""GPU (-m gpu): per-utterance VTLN filter banks on the device (psb_fe_set_filterbanks, FrontEnd.set_warps).
Batches whose utterances carry different warps against the compiled reference under each warp, and bit for bit
against the same utterances processed one warp per call; with sessions, live CMN, carried noise trackers, dither,
s2_4x and LDA; empty filters; the refusals; and Decoder with -warp_params."""
import os

import numpy as np
import pytest

from oracle import refdrv

import fe_noise_cases as N
import fe_warp_cases as wc
import vad_cases as V

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not refdrv.available(), reason="compiled reference not built")]
REF = os.path.dirname(refdrv.LIB_PATH)
TIDIGITS = dict(wlen=0.025, nfilt=20, lowerf=1, upperf=4000, round_filters=False, remove_dc=True, remove_noise=False,
                lifter=0, transform="dct")
FACTORS = ["%.2f" % (0.88 + 0.02 * i) for i in range(13)]          # 0.88 .. 1.12


def _close(got, want, what):
    """The front end's tolerance (tests/test_gpu_fe.py), NaN where the reference has NaN."""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    if got.size and not nan.all():
        g, w = got[~nan].astype(np.float64), want[~nan].astype(np.float64)
        assert np.abs(g - w).max() <= 1e-4 * max(1.0, float(np.abs(w).max())), what


def _utterances():
    a = V.audio()
    rng = np.random.default_rng(11)
    return [a["goforward"], a["numbers"]] + [N.pcm(int(n), int(s)) for n, s in zip((411, 1200, 7777, 16000, 30000),
                                                                                  rng.integers(0, 1 << 30, 5))]


def _run(fe, utts, warps=None, sess_off=None, starts=None, want_mfcc=False):
    off = fe.sample_offsets([len(u) for u in utts])
    pcm = np.concatenate(utts) if utts else np.zeros(0, np.int16)
    if sess_off is None:
        if warps is not None:
            fe.set_warps(warps)
        return fe.process_host(pcm, off, want_mfcc)
    return fe.process_sessions(pcm, off, sess_off, starts=starts, warp=warps, want_mfcc=want_mfcc)


def _split(feats, foff):
    return [feats[foff[u]:foff[u + 1]] for u in range(len(foff) - 1)]


def _single_warp_calls(make_fe, utts, warps):
    """Each distinct warp's utterances through a front end built with that warp, in one call each."""
    out = [None] * len(utts)
    for w in dict.fromkeys(warps):
        idx = [i for i, x in enumerate(warps) if x == w]
        fe = make_fe(w)
        feats, foff = _run(fe, [utts[i] for i in idx])[:2]
        for i, f in zip(idx, _split(feats, foff)):
            out[i] = f
        fe.close()
    return out


def test_mixed_warps_match_reference_and_single_warp_calls():
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.fe_tables import make_fe_desc
    utts = _utterances()
    warps = ["0.8", None, "1.12", "0.88", "1.2", "0.8", None]
    fe = api.FrontEnd(make_fe_desc())
    got = _split(*_run(fe, utts, warps))
    single = _single_warp_calls(lambda w: api.FrontEnd(make_fe_desc(warp_params=w)), utts, warps)
    for u, (g, s) in enumerate(zip(got, single)):
        assert g.tobytes() == s.tobytes(), "utterance %d" % u
    for w in dict.fromkeys(warps):
        r = wc.ref_model("en-us", "inverse_linear", w)
        for u in [i for i, x in enumerate(warps) if x == w]:
            _close(got[u], r.featurize_fresh(utts[u]), "utterance %d, warp %s" % (u, w))
        r.close()
    # the setting is for one call: the next one reads the handle's own bank again
    plain = _split(*_run(fe, utts))
    assert plain[1].tobytes() == got[1].tobytes() and plain[0].tobytes() != got[0].tobytes()
    fe.close()


@pytest.mark.parametrize("case", ["live_cmn", "noise_sessions", "tidigits_s2_4x_dither", "lda"])
def test_mixed_warps_with_sessions_and_feature_options(case):
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.fe_tables import make_fe_desc, make_fe_opts
    utts = _utterances() + [N.pcm(5000, 3), np.zeros(0, np.int16), N.pcm(300, 4)]
    sess_off = [0, 3, 4, 7, 10]
    warps = ["0.9", None, "1.1", "0.9"]
    starts = None
    desc_kw, opts = {}, make_fe_opts(cmn="live")
    if case == "noise_sessions":
        starts = np.zeros(len(utts), bool)
        starts[sess_off[:-1]] = True                                   # ps_start_stream once per session
    elif case == "tidigits_s2_4x_dither":
        desc_kw, opts = TIDIGITS, make_fe_opts(feat="s2_4x", cmn="live", dither=True, seed=5)
    elif case == "lda":
        lda = np.random.default_rng(2).standard_normal((29, 39)).astype(np.float32)
        opts = make_fe_opts(cmn="batch", lda=lda)
    fe = api.FrontEnd(make_fe_desc(**desc_kw), 0, opts)
    r = _run(fe, utts, warps, sess_off, starts)
    got, states = _split(r[0], r[1]), r[2]
    # one front end per warp, over that warp's sessions only
    for w in dict.fromkeys(warps):
        ss = [s for s in range(len(warps)) if warps[s] == w]
        sub = [utts[u] for s in ss for u in range(sess_off[s], sess_off[s + 1])]
        off = np.cumsum([0] + [sess_off[s + 1] - sess_off[s] for s in ss])
        st = None if starts is None else np.concatenate([starts[sess_off[s]:sess_off[s + 1]] for s in ss])
        one = api.FrontEnd(make_fe_desc(warp_params=w, **desc_kw), 0, opts)
        r1 = _run(one, sub, None, off, st)
        want = _split(r1[0], r1[1])
        k = 0
        for s_i, s in enumerate(ss):
            for u in range(sess_off[s], sess_off[s + 1]):
                assert got[u].tobytes() == want[k].tobytes(), (case, u)
                k += 1
            assert bytes(states[s]) == bytes(r1[2][s_i]), (case, "state", s)
        one.close()
    fe.close()


def test_one_utterance_under_13_factors():
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.fe_tables import make_fe_desc
    go = V.audio()["goforward"]
    fe = api.FrontEnd(make_fe_desc())
    got = _split(*_run(fe, [go] * 13, FACTORS))
    single = _single_warp_calls(lambda w: api.FrontEnd(make_fe_desc(warp_params=w)), [go] * 13, FACTORS)
    assert all(g.tobytes() == s.tobytes() for g, s in zip(got, single))
    assert len({g.tobytes() for g in got}) == 13
    fe.close()


def test_empty_filters():
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.fe_tables import make_fe_desc, make_fe_opts
    utts = _utterances()[:4]
    # doublebw on tidigits' band: the reference's bank is all empty filters at spec_start 0 (fe_init ignores the
    # builder's range error); banks with them run on the device and match the reference
    kv = dict(TIDIGITS, samprate=8000)
    with pytest.warns(UserWarning):
        empty = make_fe_desc(doublebw=True, warp_params="0.9", **kv)
    with pytest.warns(UserWarning):
        empty_neutral = make_fe_desc(doublebw=True, **kv)
    # psb_fe_create wants coefficients, so the handle has the ordinary bank and every utterance names an empty one
    # (CMN off: with every mel energy 0, batch CMN finds no frame with c0 >= 0 and gives NaN on both sides)
    fe = api.FrontEnd(make_fe_desc(**kv), 0, make_fe_opts(feat="s2_4x", cmn="none"))
    got = _split(*_run(fe, utts, [empty, empty_neutral, empty, empty_neutral]))
    for w, us in (("0.9", (0, 2)), (None, (1, 3))):
        r = wc.ref_model("tidigits", "inverse_linear", w, samprate="8000", doublebw="yes", dither="no", cmn="none")
        for u in us:
            refdrv.lib().refdrv_fe_reset(r.h)
            want = r.featurize(utts[u], max_frames=len(utts[u]) // 80 + 16)       # 8 kHz: 80 samples a frame
            assert np.isfinite(want).all()
            _close(got[u], want, "utterance %d" % u)
        r.close()
    fe.close()
    # the calloc form of an empty filter (spec_start -1, filt_start 0) gives what a width-0 filter at the running
    # coefficient count gives: a mel energy of 0
    d = make_fe_desc()
    n = int(d["filt_width"][:-1].sum())
    a = dict(spec_start=d["spec_start"].copy(), filt_start=d["filt_start"].copy(), filt_width=d["filt_width"].copy(),
             filt_coeffs=d["filt_coeffs"][:n].copy())
    a["filt_width"][-1] = 0
    b = {k: v.copy() for k, v in a.items()}
    a["spec_start"][-1], a["filt_start"][-1] = -1, 0
    fe = api.FrontEnd(d)
    fa = _split(*_run(fe, utts, [a] * 4))
    fb = _split(*_run(fe, utts, [b] * 4))
    full = _split(*_run(fe, utts))
    for x, y, z in zip(fa, fb, full):
        assert x.tobytes() == y.tobytes() and x.tobytes() != z.tobytes()
    fe.close()


def test_refusals_change_nothing():
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.fe_tables import make_fe_desc
    utts = _utterances()[:3]
    d = make_fe_desc()
    fe = api.FrontEnd(d)
    plain = _run(fe, utts)[0]
    warped = make_fe_desc(warp_params="0.8")
    bad_width = dict(warped, filt_width=warped["filt_width"].copy())
    bad_width["filt_width"][-1] = 300                                   # past fft_size / 2 + 1
    bad_start = dict(warped, filt_start=warped["filt_start"].copy())
    bad_start["filt_start"][3] += 1
    bad_calloc = dict(warped, spec_start=warped["spec_start"].copy())
    bad_calloc["spec_start"][0] = -1                                   # -1 with a width is not an empty filter
    for banks, which in (([warped], [0, 1, 0]), ([warped], [0, -1, 0]), ([bad_width], [0, 0, 0]),
                         ([bad_start], [0, 0, 0]), ([bad_calloc], [0, 0, 0])):
        with pytest.raises(api.PsbError, match="psb_fe_set_filterbanks"):
            fe.set_filterbanks(banks, which)
        assert _run(fe, utts)[0].tobytes() == plain.tobytes()
    with pytest.raises(ValueError, match="filters"):
        fe.set_filterbanks([dict(warped, spec_start=warped["spec_start"][:-1])], [0, 0, 0])
    # a refused call keeps what an earlier call set
    fe.set_warps(["0.8"] * 3)
    with pytest.raises(api.PsbError):
        fe.set_filterbanks([warped], [2, 0, 0])
    assert _run(fe, utts)[0].tobytes() == _run(fe, utts, ["0.8"] * 3)[0].tobytes() != plain.tobytes()
    # a count that does not match the call refuses the call, and the next call reads the handle's bank
    fe.set_warps(["0.8"] * 2)
    with pytest.raises(api.PsbError, match="filter banks name 2 utterances, the call has 3"):
        _run(fe, utts)
    assert _run(fe, utts)[0].tobytes() == plain.tobytes()
    fe.close()


@pytest.mark.timeout(900)
def test_decoder_with_warp_params():
    from pocketsphinx_b200.decoder import Decoder
    hd, dic, lm = os.path.join(REF, "model", "en-us"), os.path.join(REF, "data", "turtle.dic"), os.path.join(REF, "data", "turtle.lm.bin")
    if not os.path.exists(lm):
        pytest.skip("reference data files not present")
    a = V.audio()
    utts = [a["goforward"], a["numbers"]]
    dec = Decoder(hd, dic, lm, max_utts=16, max_frames=1 << 14, warp_params="0.9")
    out = dec.decode_raw_batch(utts)
    for u, d in enumerate(utts):
        wc.fresh("inverse_linear", "0.9")
        r = N.ref_decoder(hd, lm, dic, [d], [1], warp_params="0.9")[0]
        assert out[u]["words"] == [w for w, _, _ in r["seg"]], (out[u]["words"], r["seg"])
        assert np.abs(out[u]["seg"][:, 2] - np.array([sf for _, sf, _ in r["seg"]])).max() <= 2
        assert np.abs(out[u]["seg"][:, 3] - np.array([ef for _, _, ef in r["seg"]])).max() <= 2
    # a mixed-warp batch is one single-warp Decoder per warp; None is the decoder's own -warp_params
    warps = ["1.1", None, "0.9", "1.1"]
    mixed = dec.decode_raw_batch(utts + utts, warp=warps)
    plain = Decoder(hd, dic, lm, max_utts=16, max_frames=1 << 14)
    dec11 = Decoder(hd, dic, lm, max_utts=16, max_frames=1 << 14, warp_params="1.1")
    want = [dec11.decode_raw_batch([utts[0]])[0], out[1], out[0], dec11.decode_raw_batch([utts[1]])[0]]
    for m, w in zip(mixed, want):
        assert (m["hyp"], m["score"], m["seg"].tobytes()) == (w["hyp"], w["score"], w["seg"].tobytes())
    # the default is today's result
    assert [d["seg"].tobytes() for d in plain.decode_raw_batch(utts)] == \
        [d["seg"].tobytes() for d in plain.decode_raw_batch(utts, warp=[None, None])]
    # sessions: one warp per session
    with pytest.raises(ValueError, match="names two warps"):
        dec.decode_raw_batch(utts, sessions=[0, 0], warp=["0.9", "1.1"])
    s = dec.decode_raw_batch(utts + utts, sessions=[0, 1, 0, 1], warp=["1.1", "0.9", "1.1", "0.9"])
    assert s[0]["hyp"] == mixed[0]["hyp"]
    # None is the decoder's own warp (0.9 here), so a session may mix the two spellings
    s2 = dec.decode_raw_batch(utts + utts, sessions=[0, 1, 0, 1], warp=["1.1", None, "1.1", "0.9"])
    assert [(d["hyp"], d["score"], d["seg"].tobytes()) for d in s2] == [(d["hyp"], d["score"], d["seg"].tobytes()) for d in s]
    # decode_stream_batch: one warp per stream, each stream as a Decoder of that warp decodes it alone
    sil = np.zeros(16000, np.int16)
    s1 = np.concatenate([sil, a["goforward"], sil, a["numbers"], sil])
    st2 = np.concatenate([sil[:4000], a["goforward"], sil])
    got = dec.decode_stream_batch([s1, st2], warp=["1.1", None])
    want = [dec11.decode_stream_batch([s1])[0], dec.decode_stream_batch([st2])[0]]
    key = lambda row: [(d["start_sample"], d["end_sample"], d["hyp"], d["score"], d["seg"].tobytes()) for d in row]
    assert len(got[0]) >= 2 and [key(r) for r in got] == [key(r) for r in want]
    assert key(got[0]) != key(dec.decode_stream_batch([s1])[0])                  # the warp is applied
    for o in (dec, plain, dec11):
        o.close()


def test_refused_warp_names_nothing_for_the_next_call():
    """A warp refused while sessions and stream starts are being named leaves none of them for the next call."""
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.fe_tables import make_fe_desc, make_fe_opts
    utts = _utterances()[:4]
    d = make_fe_desc()
    opts = make_fe_opts(cmn="live")
    fe, fresh = api.FrontEnd(d, 0, opts), api.FrontEnd(d, 0, opts)
    off = fe.sample_offsets([len(u) for u in utts])
    pcm = np.concatenate(utts)
    want = fresh.process_host(pcm, off)[0]
    starts = np.array([1, 0, 0, 0], bool)
    # refused on the host (the reference's process ends under this warp) ...
    with pytest.raises(ValueError):
        fe.process_sessions(pcm, off, [0, 4], starts=starts, warp=[("affine", "1 -1e6")])
    assert fe.process_host(pcm, off)[0].tobytes() == want.tobytes()
    # ... and by psb_fe_set_filterbanks, after the sessions and stream starts were named
    bad = dict(d, filt_width=d["filt_width"].copy())
    bad["filt_width"][-1] = 300
    with pytest.raises(api.PsbError, match="psb_fe_set_filterbanks"):
        fe.process_sessions(pcm, off, [0, 4], starts=starts, warp=[bad])
    assert fe.process_host(pcm, off)[0].tobytes() == want.tobytes()
    with pytest.raises(api.PsbError, match="the last call had"):
        fe.get_states(1)                                  # the last call named no sessions
    # cancel_settings drops named settings directly
    fe.set_sessions([0, 4])
    fe.set_warps(["0.8"] * 4)
    fe.cancel_settings()
    assert fe.process_host(pcm, off)[0].tobytes() == want.tobytes()
    fe.close(); fresh.close()
