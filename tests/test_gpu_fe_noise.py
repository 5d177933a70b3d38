"""GPU: the -remove_noise tracker carried across a session's utterances (psb_fe_set_stream_starts,
fe_noise_kernel) against the compiled reference fed the same utterances with ps_start_stream at exactly the
same positions (tests/fe_noise_cases.py): en-us, tidigits-style 20 filters with dither and -remove_noise forced
on, and live CMN.  The carried features are far from fresh-stream ones; all-ones flags are the default's bytes;
a session cut into calls with the trackers passed through is one call's bytes; Decoder.decode_stream_batch with
start_stream="session" against a reference decoder that calls ps_start_stream once per recording."""
import os

import numpy as np
import pytest

import fe_noise_cases as N
import fe_sessions as fs
import vad_cases as V
from conftest import ROOT
from oracle import fe_golden, refdrv
from pocketsphinx_b200.fe_tables import make_fe_desc, make_fe_opts

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not refdrv.available(), reason="compiled reference not built")]
REF = os.path.join(ROOT, "oracle", "_ref")
TIDIGITS_NOISE = dict(wlen=0.025, nfilt=20, lowerf=1, upperf=4000, round_filters=False, remove_dc=True, remove_noise=True,
                      lifter=0, transform="dct")
SEED = 11


def _sessions():
    """(utterances, stream-start flags) of sessions of 1 to 5 utterances: sub-frame and empty utterances, speech and
    noise at changing levels, stream starts first, inside and at the end.  Noise that goes on at the level of the
    utterance before it is where a carried tracker differs most from a fresh one."""
    go = fe_golden.goforward()
    return [([go[:20000]], [1]),
            ([N.pcm(9000, 1, 300), N.pcm(9000, 2, 300), go[15000:], N.pcm(250, 3, 4000)], [1, 0, 0, 0]),
            ([N.pcm(12000, 4, 2000), N.pcm(12000, 5, 2000), np.zeros(0, np.int16), N.pcm(8000, 6, 500), N.pcm(9000, 7, 500)],
             [1, 0, 0, 1, 0]),
            ([N.pcm(7000, 8, 2000), go[5000:30000]], [1, 1]),
            ([go[:16000], N.pcm(300, 9, 100), N.pcm(11000, 10, 3000), N.pcm(11000, 11, 3000), go[20000:]], [1, 0, 1, 0, 0])]


def _flat(sessions):
    utts = [u for us, _ in sessions for u in us]
    starts = [s for _, ss in sessions for s in ss]
    sess_off = np.cumsum([0] + [len(us) for us, _ in sessions])
    return utts, starts, sess_off


def _run(fe, utts, sess_off, starts=None, states=None, noise=None):
    off = fe.sample_offsets([len(u) for u in utts])
    pcm = np.concatenate(utts) if utts else np.zeros(0, np.int16)
    return fe.process_sessions(pcm, off, sess_off, states, want_mfcc=True, starts=starts, noise=noise)


def _ref_features(name, kv, sessions):
    out = []
    for us, ss in sessions:
        r = refdrv.RefModel(fs.ref_model_dir(name), **kv)      # one decoder per session: fe_init seeds the dither
        out += N.ref_stream_features(r, us, ss)
        r.close()
    return out


def _ref_live_cmn_features(sessions, opts):
    hmm = fs.ref_model_dir("en-us")
    lm, dic = os.path.join(REF, "data", "turtle.lm.bin"), os.path.join(REF, "data", "turtle.dic")
    out = []
    for us, ss in sessions:
        cep = [d["cep"] for d in N.ref_decoder(hmm, lm, dic, us, ss, cmn="live")]
        st = fs.CmnState(opts["cmn_init"])
        out += [fs.dyn_features(st.utterance(c), 0) for c in cep]
    return out


def _check(feats, foff, ref, sessions, fresh):
    utts, starts, sess_off = _flat(sessions)
    for s in range(len(sessions)):
        u0, u1 = sess_off[s], sess_off[s + 1]
        for u in range(u0, u1):
            N.close_enough(feats[foff[u]:foff[u + 1]], ref[u], 0)
        N.close_enough(feats[foff[u0]:foff[u1]], np.concatenate(ref[u0:u1]))
    # the test discriminates: carried utterances of some length are far from the same utterances as fresh streams,
    # and a session's first utterance is a fresh stream either way
    n_far = 0
    for u in range(len(utts)):
        a, b = feats[foff[u]:foff[u + 1]], fresh[foff[u]:foff[u + 1]]
        if u in sess_off[:-1]:
            assert a.tobytes() == b.tobytes(), u
        elif not starts[u] and len(a) > 40:
            n_far += np.abs(a - b).max() > 100 * 1e-4 * max(1.0, float(np.abs(ref[u]).max()))
    assert n_far >= 5, n_far


@pytest.mark.parametrize("config", ["en-us", "tidigits dither", "en-us live CMN"])
def test_carried_tracker_matches_reference(config):
    from pocketsphinx_b200 import api
    sessions = _sessions()
    utts, starts, sess_off = _flat(sessions)
    if config == "en-us":
        fe = api.FrontEnd(make_fe_desc(), 0)
    elif config == "tidigits dither":
        fe = api.FrontEnd(make_fe_desc(**TIDIGITS_NOISE), 0, make_fe_opts(feat="s2_4x", cmn="batch", dither=True, seed=SEED))
    else:
        opts = make_fe_opts(cmn="live")
        fe = api.FrontEnd(make_fe_desc(), 0, opts)
    feats, foff, _, _, noise = _run(fe, utts, sess_off, starts)
    fresh, foff2, _, _ = _run(fe, utts, sess_off)
    assert np.array_equal(foff, foff2) and len(noise) == len(sessions)
    if config == "en-us":
        ref = _ref_features("en-us", {}, sessions)
    elif config == "tidigits dither":
        ref = _ref_features("tidigits", dict(dither="yes", seed=str(SEED), remove_noise="yes"), sessions)
    else:
        ref = _ref_live_cmn_features(sessions, opts)
    _check(feats, foff, ref, sessions, fresh)
    # every session ends on a defined tracker; filters past n_filt read 0
    nf = fe.desc["n_filt"]
    for z in noise:
        assert z.undefined == 0 and z.reserved == 0
        assert all(v > 0 for v in z.power[:nf]) and not any(z.power[nf:]) and not any(z.peak[nf:])
    fe.close()


@pytest.mark.parametrize("desc,opts", [({}, None),
                                       (TIDIGITS_NOISE, dict(feat="s2_4x", cmn="live", dither=True, seed=SEED)),
                                       (dict(TIDIGITS_NOISE, remove_noise=False), dict(feat="s2_4x", cmn="batch"))])
def test_default_bytes_unchanged(desc, opts):
    """All-ones flags, and a first utterance that continues a tracker nobody defined, give the bytes of a call that
    never names stream starts; without -remove_noise any flags do."""
    from pocketsphinx_b200 import api
    fe = api.FrontEnd(make_fe_desc(**desc), 0, None if opts is None else make_fe_opts(**opts))
    utts, starts, sess_off = _flat(_sessions())
    plain = _run(fe, utts, sess_off)
    ones = _run(fe, utts, sess_off, [1] * len(utts))
    first_zero = [0 if u in sess_off[:-1] else 1 for u in range(len(utts))]
    z = _run(fe, utts, sess_off, first_zero)
    for r in (ones, z):
        assert r[0].tobytes() == plain[0].tobytes() and r[3].tobytes() == plain[3].tobytes()
        assert [bytes(s) for s in r[2]] == [bytes(s) for s in plain[2]]
    assert [bytes(s) for s in ones[4]] == [bytes(s) for s in z[4]]
    if not desc.get("remove_noise", True):
        carried = _run(fe, utts, sess_off, starts)
        assert carried[0].tobytes() == plain[0].tobytes()
    # the flags were for the call after them only
    again = _run(fe, utts, sess_off)
    assert again[0].tobytes() == plain[0].tobytes()
    fe.close()


def test_split_calls_are_one_call():
    """One session cut into two calls at every utterance boundary, the trackers (and the dither and live-CMN
    states) passed through, gives one call's bytes; so do two sessions and an empty one in one call."""
    from pocketsphinx_b200 import api
    go = fe_golden.goforward()
    utts = [go[:20000], N.pcm(250, 8, 3000), np.zeros(0, np.int16), N.pcm(9000, 9, 400), go[15000:], N.pcm(250, 10, 50),
            np.zeros(0, np.int16), N.pcm(6000, 11, 2500)]
    starts = [1, 0, 0, 0, 1, 0, 1, 0]
    fe = api.FrontEnd(make_fe_desc(**TIDIGITS_NOISE), 0, make_fe_opts(feat="s2_4x", cmn="live", dither=True, seed=SEED))
    whole, foff, st_w, mf_w, nz_w = _run(fe, utts, [0, len(utts)], starts)
    for k in range(1, len(utts)):
        a, fa, st_a, mf_a, nz_a = _run(fe, utts[:k], [0, k], starts[:k])
        b, fb, st_b, mf_b, nz_b = _run(fe, utts[k:], [0, len(utts) - k], starts[k:], st_a, nz_a)
        assert np.concatenate([a, b]).tobytes() == whole.tobytes(), k
        assert np.concatenate([mf_a, mf_b]).tobytes() == mf_w.tobytes(), k
        assert bytes(st_b[0]) == bytes(st_w[0]) and bytes(nz_b[0]) == bytes(nz_w[0]), k
    # the tracker after a stream start with no frame behind it is undefined, whatever came in
    _, _, _, _, nz = _run(fe, utts[6:7], [0, 1], [1], None, nz_w)
    assert nz[0].undefined == 1 and not any(nz[0].power)
    _, _, _, _, nz = _run(fe, utts[6:7], [0, 1], [0], None, nz_w)
    assert bytes(nz[0]) == bytes(nz_w[0])
    # sessions side by side, one of them empty: the empty one hands its tracker through
    k = 4
    two, ft, st_t, mf_t, nz_t = _run(fe, utts, [0, k, k, len(utts)], starts, None, [nz_w[0]] * 3)
    a, fa, st_a, mf_a, nz_a = _run(fe, utts[:k], [0, k], starts[:k], None, [nz_w[0]])
    assert two[:fa[-1]].tobytes() == a.tobytes() and bytes(nz_t[0]) == bytes(nz_a[0]) and bytes(nz_t[1]) == bytes(nz_w[0])
    fe.close()


def test_refusals():
    from pocketsphinx_b200 import api
    from pocketsphinx_b200._lib import FeNoise
    fe = api.FrontEnd(make_fe_desc(), 0)
    utts = [N.pcm(4000, 1), N.pcm(5000, 2)]
    off = fe.sample_offsets([len(u) for u in utts])
    pcm = np.concatenate(utts)
    fe.process_host(pcm, off)
    with pytest.raises(api.PsbError, match="set no stream starts"):
        fe.get_noise_states(2)
    fe.set_stream_starts([1, 0, 1])
    with pytest.raises(api.PsbError, match="stream starts cover 3 utterances"):
        fe.process_host(pcm, off)
    fe.set_stream_starts([1, 0], [FeNoise(undefined=1)] * 3)
    with pytest.raises(api.PsbError, match="3 noise trackers for 2 sessions"):
        fe.process_host(pcm, off)
    bad = np.array([1, 2], np.uint8)
    assert api.lib().psb_fe_set_stream_starts(fe.h, bad.ctypes.data, 2, None, 0) != 0
    assert "not 0 or 1" in api.lib().psb_last_error().decode()
    with pytest.raises(api.PsbError, match="not a noise tracker"):
        fe.set_stream_starts([0, 0], [FeNoise(undefined=2), FeNoise(undefined=1)])
    # a refused call consumed its settings: the next one is the default
    fe.process_host(pcm, off)
    fe.set_stream_starts([1, 0])
    fe.process_host(pcm, off)
    with pytest.raises(api.PsbError, match="the last call had 2 sessions"):
        fe.get_noise_states(1)
    assert len(fe.get_noise_states(2)) == 2
    fe.close()


@pytest.mark.timeout(900)
def test_decode_stream_batch_session_starts_match_reference():
    from pocketsphinx_b200.decoder import Decoder
    hd, dic, lm = os.path.join(REF, "model", "en-us"), os.path.join(REF, "data", "turtle.dic"), os.path.join(REF, "data", "turtle.lm.bin")
    if not (os.path.exists(lm) and V.ref_available()):
        pytest.skip("reference data files not present")
    a = V.audio()
    sil = np.zeros(16000, np.int16)
    s1 = np.concatenate([sil, a["goforward"], sil, a["numbers"], sil, a["libri_0880"], sil])
    s2 = np.concatenate([sil[:4000], a["goforward"], sil])
    dec = Decoder(hd, dic, lm, max_utts=64, max_frames=1 << 15)
    out = dec.decode_stream_batch([s1, s2], start_stream="session")
    for stream, got in zip((s1, s2), out):
        want = V.ref_segments(stream, 0, 16000, 0.03, 0.3, 0.9)
        assert [(d["start_time"], d["end_time"], d["start_sample"], d["end_sample"]) for d in got] == want
        segs = [stream[w[2]:w[3]] for w in want]
        ref = N.ref_decoder(hd, lm, dic, segs, [1] + [0] * (len(segs) - 1))
        for d, r in zip(got, ref):
            print("segment %d..%d: %d frames, score %d (reference %d), %s" % (d["start_sample"], d["end_sample"], d["n_frames"],
                                                                          d["score"], r["score"], d["hyp"]))
        assert [d["hyp"] for d in got] == [r["hyp"] for r in ref]
        for d, r in zip(got, ref):
            assert d["words"] == [w for w, _, _ in r["seg"]], (d["words"], r["seg"])
            assert np.abs(d["seg"][:, 2] - np.array([sf for _, sf, _ in r["seg"]])).max() <= 2
            assert np.abs(d["seg"][:, 3] - np.array([ef for _, _, ef in r["seg"]])).max() <= 2
    # start_stream="utterance" is the default's result, score and segmentation included
    base = dec.decode_stream_batch([s1, s2])
    per_utt = dec.decode_stream_batch([s1, s2], start_stream="utterance")
    for x, y in zip(base, per_utt):
        assert [(d["hyp"], d["score"], d["seg"].tobytes()) for d in x] == [(d["hyp"], d["score"], d["seg"].tobytes()) for d in y]
    # the first segment of a stream starts the stream either way
    assert [d["score"] for d in (out[0][0], out[1][0])] == [d["score"] for d in (base[0][0], base[1][0])]
    with pytest.raises(ValueError):
        dec.decode_raw_batch([s2], start_stream="recording")
    dec.close()
