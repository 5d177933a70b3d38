"""GPU: the device front end's s2_4x / s3_1x39 features, live CMN over sessions and dither (psb_fe_create_ex)
against the compiled reference run live and against tests/fe_sessions.py applied to the device's own cepstra;
sessions split over calls and reordered; Decoder with the tidigits model's own feat.params and an en-us session
with live CMN."""
import os

import numpy as np
import pytest

import fe_sessions as fs
from conftest import ROOT
from oracle import fe_golden, refdrv
from pocketsphinx_b200.fe_tables import make_fe_desc, make_fe_opts

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not refdrv.available(), reason="compiled reference not built")]
REF = os.path.join(ROOT, "oracle", "_ref")
TIDIGITS = dict(wlen=0.025, nfilt=20, lowerf=1, upperf=4000, round_filters=False, remove_dc=True, remove_noise=False,
                lifter=0, transform="dct")
AN4 = dict(nfilt=40, lowerf=133.3334, upperf=6855.4976, transform="legacy", lifter=0, remove_noise=False)


def _pcm(n, seed, amp=3000):
    return (np.random.default_rng(seed).standard_normal(n) * amp).astype(np.int16)


def _close_enough(got, ref, bit_share=0.99):
    assert got.shape == ref.shape
    if not got.size:
        return
    assert np.abs(got - ref).max() <= 1e-4 * max(1.0, float(np.abs(ref).max()))
    if bit_share:
        assert (got == ref).mean() > bit_share


def _run(fe, utts, sess_off=None, states=None, want_mfcc=True):
    off = fe.sample_offsets([len(u) for u in utts])
    pcm = np.concatenate(utts) if utts else np.zeros(0, np.int16)
    if sess_off is None:
        sess_off = list(range(len(utts) + 1))
    feats, foff, st, mfcc = fe.process_sessions(pcm, off, sess_off, states, want_mfcc=want_mfcc)
    return feats, foff, st, mfcc


@pytest.mark.parametrize("name,kv,desc,opts", [
    ("tidigits", dict(dither="no"), TIDIGITS, dict(feat="s2_4x", cmn="batch")),
    ("an4", dict(feat="s3_1x39"), AN4, dict(feat="s3_1x39", cmn="batch")),
    ("an4", dict(feat="s3_1x39", cmn="none"), AN4, dict(feat="s3_1x39", cmn="none")),
])
def test_feature_types_match_reference(name, kv, desc, opts):
    from pocketsphinx_b200 import api
    fe = api.FrontEnd(make_fe_desc(**desc), 0, make_fe_opts(**opts))
    utts = [fe_golden.goforward(), _pcm(7000, 1), _pcm(300, 2), np.zeros(0, np.int16)]
    feats, foff, _, _ = _run(fe, utts)
    assert feats.shape[1] == fs.FEAT_DIM[make_fe_opts(**opts)["feat"]]
    r = refdrv.RefModel(fs.ref_model_dir(name), **kv)
    for u, pcm in enumerate(utts):
        _close_enough(feats[foff[u]:foff[u + 1]], r.featurize_fresh(pcm) if len(pcm) else np.zeros((0, feats.shape[1]), np.float32),
                      0.99 if len(pcm) else 0)
    r.close()
    fe.close()


def _long_session():
    go = fe_golden.goforward()
    # one utterance of more than 800 frames, an all-silent one (every c0 < 0), and 800 frames crossed across utterances
    return [go, np.zeros(4000, np.int16), np.tile(go, 3)[:90000], _pcm(1, 3), go[:30000], go, np.zeros(0, np.int16), go[5000:40000]]


@pytest.mark.parametrize("feat", ["1s_c_d_dd", "s2_4x", "s3_1x39"])
def test_live_cmn_is_fe_port_on_device_cepstra(feat):
    from pocketsphinx_b200 import api
    d = make_fe_desc()
    utts = _long_session()
    sess_off = [0, 3, 3, len(utts)]                      # an empty session in the middle
    live = api.FrontEnd(d, 0, make_fe_opts(feat=feat, cmn="live"))
    raw = api.FrontEnd(d, 0, make_fe_opts(feat=feat, cmn="none"))
    feats, foff, states, mfcc = _run(live, utts, sess_off)
    _, foff2, _, cep = _run(raw, utts, sess_off)
    assert np.array_equal(foff, foff2)
    opts = make_fe_opts(feat=feat, cmn="live")
    for s in range(len(sess_off) - 1):
        st = fs.CmnState(opts["cmn_init"])
        for u in range(sess_off[s], sess_off[s + 1]):
            c = st.utterance(cep[foff[u]:foff[u + 1]])
            assert c.tobytes() == mfcc[foff[u]:foff[u + 1]].tobytes(), (s, u)
            assert fs.dyn_features(c, opts["feat"]).tobytes() == feats[foff[u]:foff[u + 1]].tobytes(), (s, u)
        got = states[s]
        assert np.array(got.cmn_mean[:13], np.float32).tobytes() == st.mean.tobytes()
        assert np.array(got.cmn_sum[:13], np.float32).tobytes() == st.sum.tobytes() and got.cmn_nframe == st.nframe
    # against the reference run live, the first utterance of a session (nothing carried in yet)
    r = refdrv.RefModel(fs.ref_model_dir("en-us"), cmn="live")
    if feat == "1s_c_d_dd":
        _close_enough(feats[foff[0]:foff[1]], r.featurize_fresh(utts[0]), 0)
    r.close()
    live.close(); raw.close()


@pytest.mark.parametrize("name,desc,seed", [("tidigits", TIDIGITS, -1), ("en-us", {}, 77)])
def test_dither_draws(name, desc, seed):
    from pocketsphinx_b200 import api
    d = make_fe_desc(**desc)
    fsz, sh = d["frame_size"], d["frame_shift"]
    lens = [0, 1, fsz - 1, fsz, fsz + 1, fsz + sh - 1, fsz + sh, fsz + sh + 1, 20000]
    utts = [np.zeros(n, np.int16) if i % 3 == 0 else _pcm(n, i, amp=3) for i, n in enumerate(lens)]
    fe = api.FrontEnd(d, 0, make_fe_opts(cmn="none", dither=True, seed=seed))
    feats, foff, states, mfcc = _run(fe, utts, [0, len(utts)])
    rng = fs.MT19937(seed)
    r = refdrv.RefModel(fs.ref_model_dir(name), dither="yes", seed=str(seed), cmn="none")
    for u, pcm in enumerate(utts):
        ours = fe_port_cepstra(d, fs.mfspec_dithered(d, pcm, rng))
        ref = r.mfcc(pcm)
        _close_enough(mfcc[foff[u]:foff[u + 1]], ours, 0)
        _close_enough(mfcc[foff[u]:foff[u + 1]], ref, 0)
    r.close()
    # the generator's state after the session is exactly the numpy one's
    assert states[0].mt_index == rng.mti and list(states[0].mt) == rng.mt
    fe.close()


def fe_port_cepstra(d, mf):
    from oracle import fe_port
    return fe_port.cepstra(d, mf)


def test_sessions_split_and_reordered():
    from pocketsphinx_b200 import api
    d = make_fe_desc(**TIDIGITS)
    fe = api.FrontEnd(d, 0, make_fe_opts(feat="s2_4x", cmn="live", dither=True, seed=5))
    utts = _long_session()
    whole, foff, st_whole, _ = _run(fe, utts, [0, len(utts)])
    k = 4
    a, fa, st_a, _ = _run(fe, utts[:k], [0, k])
    b, fb, st_b, _ = _run(fe, utts[k:], [0, len(utts) - k], st_a)
    assert np.concatenate([a, b]).tobytes() == whole.tobytes()
    assert bytes(st_b[0]) == bytes(st_whole[0])
    # two sessions, in either order in the batch
    s1, s2 = utts[:3], utts[3:]
    x, fx, stx, _ = _run(fe, s1 + s2, [0, 3, len(utts)])
    y, fy, sty, _ = _run(fe, s2 + s1, [0, len(s2), len(utts)])
    n1 = fx[3]
    assert x[:n1].tobytes() == y[fy[len(s2)]:].tobytes() and x[n1:].tobytes() == y[:fy[len(s2)]].tobytes()
    assert bytes(stx[0]) == bytes(sty[1]) and bytes(stx[1]) == bytes(sty[0])
    # the initial state is the one psb_fe_state_init reports, and one session of everything = the first run
    assert bytes(fe.initial_state()) == bytes(_run(fe, [], [0, 0])[2][0])
    fe.close()


@pytest.mark.timeout(900)
def test_decoder_tidigits_own_feat_params():
    from pocketsphinx_b200.decoder import Decoder
    hd = os.path.join(REF, "model", "tidigits_hmm")
    lm, dic = os.path.join(REF, "model", "tidigits_lm", "tidigits.lm.bin"), os.path.join(REF, "model", "tidigits_lm", "tidigits.dic")
    utts = [np.fromfile(os.path.join(REF, "data", "dhd.2934z.raw"), np.int16), fe_golden.goforward()]
    dec = Decoder(hd, dic, lm, max_utts=4, max_frames=4096)
    assert dec.fe.feat_dim == 51
    out = dec.decode_raw_batch(utts)
    for u, pcm in enumerate(utts):
        # a fresh reference decoder per utterance: the dither generator starts from -seed each time, as here
        want = fs.ref_session_decode(hd, lm, dic, [pcm], bestpath="no")[0]
        assert out[u]["hyp"] == want, (u, out[u]["hyp"], want)
    dec.close()


@pytest.mark.timeout(900)
def test_decoder_en_us_live_cmn_session():
    from pocketsphinx_b200.decoder import Decoder
    hd, dic, lm = os.path.join(REF, "model", "en-us"), os.path.join(REF, "data", "turtle.dic"), os.path.join(REF, "data", "turtle.lm.bin")
    go = fe_golden.goforward()
    utts = [go, go[:30000], go]
    want = fs.ref_session_decode(hd, lm, dic, utts, cmn="live", bestpath="no")
    dec = Decoder(hd, dic, lm, max_utts=8, max_frames=4096, cmn="live")
    # the session interleaved with a one-utterance session: ids, not positions, name the decoders
    out = dec.decode_raw_batch([utts[0], go, utts[1], utts[2]], sessions=["a", "b", "a", "a"])
    got = [out[0], out[2], out[3]]
    assert [o["hyp"] for o in got] == want
    single = dec.decode_raw_batch([go])[0]
    assert out[1]["hyp"] == single["hyp"] and np.array_equal(out[1]["seg"], single["seg"])
    dec.close()
