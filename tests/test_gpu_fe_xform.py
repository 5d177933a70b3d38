"""GPU: the device front end's -varnorm, -agc max / emax / noise and LDA transforms (psb_fe_create_ex) against the
compiled reference run live and against tests/fe_xform.py applied to the device's own cepstra; emax sessions split
over calls and reordered; senone scores on LDA features; Decoder with a model's feature_transform, -agc emax over a
session and -varnorm yes against reference decoders."""
import os

import numpy as np
import pytest

import fe_sessions as fs
import fe_xform as fx
from conftest import ROOT
from oracle import fe_golden, refdrv
from pocketsphinx_b200 import s3io
from pocketsphinx_b200.fe_tables import make_fe_desc, make_fe_opts

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not refdrv.available(), reason="compiled reference not built")]
REF = os.path.join(ROOT, "oracle", "_ref")
AN4 = dict(nfilt=40, lowerf=133.3334, upperf=6855.4976, transform="legacy", lifter=0, remove_noise=False)
DESC = {"an4": AN4, "en-us": {}}
DIC, LM = os.path.join(REF, "data", "turtle.dic"), os.path.join(REF, "data", "turtle.lm.bin")


def _pcm(n, seed, amp=3000):
    return (np.random.default_rng(seed).standard_normal(n) * amp).astype(np.int16)


def _ragged():
    go = fe_golden.goforward()
    # speech, noise, a sub-frame utterance, an empty one, an all-silent one (every c0 < 0), a short one
    return [go, _pcm(7000, 1), _pcm(300, 2), np.zeros(0, np.int16), np.zeros(4000, np.int16), go[20000:32000]]


def _close_enough(got, ref, bit_share=0.99):
    assert got.shape == ref.shape
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan)          # batch CMN of an all-silent utterance divides 0 by 0
    got, ref = got[~nan], ref[~nan]
    if not got.size:
        return
    assert np.abs(got - ref).max() <= 1e-4 * max(1.0, float(np.abs(ref).max()))
    if bit_share:
        assert (got == ref).mean() > bit_share


def _same(got, want):
    # bit for bit, except that a NaN's sign and payload are the platform's
    nan = np.isnan(want)
    assert got.shape == want.shape and np.array_equal(np.isnan(got), nan)
    assert got[~nan].tobytes() == want[~nan].tobytes()


def _run(fe, utts, sess_off=None, states=None):
    off = fe.sample_offsets([len(u) for u in utts])
    pcm = np.concatenate(utts) if utts else np.zeros(0, np.int16)
    return fe.process_sessions(pcm, off, sess_off if sess_off is not None else list(range(len(utts) + 1)), states, want_mfcc=True)


@pytest.fixture(scope="module")
def an4_lda(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("an4_lda")
    a29, a39 = fx.orthonormal(29, 39, 7), fx.block_rotation(11)
    return dict(a29=a29, d29=fx.derive_lda_model(fs.ref_model_dir("an4"), str(tmp / "an4_29"), a29),
                a39=a39, d39=fx.derive_lda_model(fs.ref_model_dir("an4"), str(tmp / "an4_39"), a39),
                d29_plain=fx.derive_lda_model(fs.ref_model_dir("an4"), str(tmp / "an4_29_plain"), a29, False))


CASES = [
    ("an4", dict(varnorm="yes"), dict(cmn="batch", varnorm=True)),
    ("en-us", dict(varnorm="yes"), dict(cmn="batch", varnorm=True)),
    ("en-us", dict(agc="max"), dict(cmn="batch", agc="max")),
    ("en-us", dict(agc="max", cmn="none"), dict(cmn="none", agc="max")),
    ("an4", dict(agc="noise"), dict(cmn="batch", agc="noise")),
    ("an4", dict(agc="noise", agcthresh=0.0), dict(cmn="batch", agc="noise", agcthresh=0.0)),
    ("en-us", dict(agc="emax"), dict(cmn="batch", agc="emax")),
    ("en-us", dict(agc="emax", cmn="none"), dict(cmn="none", agc="emax")),
]


@pytest.mark.parametrize("name,kv,opts", CASES)
def test_matches_reference_live(name, kv, opts):
    from pocketsphinx_b200 import api
    fe = api.FrontEnd(make_fe_desc(**DESC[name]), 0, make_fe_opts(**opts))
    utts = _ragged()
    # one session: emax carries its estimate from utterance to utterance, as successive reference calls do
    feats, foff, _, _ = _run(fe, utts, [0, len(utts)])
    r = refdrv.RefModel(fs.ref_model_dir(name), **kv)
    for u, pcm in enumerate(utts):
        want = r.featurize_fresh(pcm)
        _close_enough(feats[foff[u]:foff[u + 1]], want, 0.99 if len(pcm) else 0)
    r.close()
    fe.close()


@pytest.mark.parametrize("which,ldadim", [("d29", 0), ("d29", 20), ("d29", 40), ("d39", 0)])
def test_lda_matches_reference_live(an4_lda, which, ldadim):
    from pocketsphinx_b200 import api
    a = s3io.read_lda(os.path.join(an4_lda[which], "feature_transform"))[0]
    fe = api.FrontEnd(make_fe_desc(**AN4), 0, make_fe_opts(cmn="batch", lda=a, ldadim=ldadim))
    assert fe.feat_dim == (20 if ldadim == 20 else a.shape[0])
    utts = _ragged()
    feats, foff, _, _ = _run(fe, utts)
    # no model has 20-dimensional streams to open the reference with: its cepstra through fe_xform instead
    r = refdrv.RefModel(fs.ref_model_dir("an4") if ldadim == 20 else an4_lda[which], ldadim=ldadim)
    for u, pcm in enumerate(utts):
        want = fx.features(r.mfcc(pcm), a=a, ldadim=20)[0] if ldadim == 20 else r.featurize_fresh(pcm)
        _close_enough(feats[foff[u]:foff[u + 1]], want, 0.99 if len(pcm) else 0)
    r.close()
    fe.close()


XFORMS = [
    dict(cmn="batch", varnorm=True),
    dict(cmn="batch", agc="max"),
    dict(cmn="none", agc="max"),
    dict(cmn="batch", agc="noise"),
    dict(cmn="none", agc="noise", agcthresh=0.5),
    dict(cmn="batch", agc="emax"),
    dict(cmn="none", agc="emax"),
    dict(cmn="batch", lda="a29"),
    dict(cmn="batch", lda="a29", ldadim=12),
    dict(cmn="batch", varnorm=True, agc="noise", lda="a39"),
    dict(cmn="none", agc="emax", lda="a29", feat="s3_1x39"),
]


@pytest.mark.parametrize("opts", XFORMS, ids=lambda o: "-".join("%s=%s" % kv for kv in o.items()))
def test_is_fe_xform_on_device_cepstra(an4_lda, opts):
    """Given the device's own cepstra before CMN, the device's cepstra after CMN and AGC and its features are the
    numpy restatement's, bit for bit, over a session that crosses 16 utterances."""
    from pocketsphinx_b200 import api
    opts = dict(opts)
    a = an4_lda[opts.pop("lda")] if "lda" in opts else None
    feat = opts.pop("feat", "1s_c_d_dd")
    d = make_fe_desc(**AN4)
    utts = _session()
    sess_off = [0, 5, 5, len(utts)]                      # an empty session in the middle
    fe = api.FrontEnd(d, 0, make_fe_opts(feat=feat, lda=a, **opts))
    raw = api.FrontEnd(d, 0, make_fe_opts(feat=feat, cmn="none"))
    feats, foff, states, mfcc = _run(fe, utts, sess_off)
    _, foff2, _, cep = _run(raw, utts, sess_off)
    assert np.array_equal(foff, foff2)
    ff = make_fe_opts(feat=feat)["feat"]
    for s in range(len(sess_off) - 1):
        agc = fx.Agc(opts["agc"], opts["cmn"] == "none", opts.get("agcthresh", 2.0)) if "agc" in opts else None
        for u in range(sess_off[s], sess_off[s + 1]):
            f, c = fx.features(cep[foff[u]:foff[u + 1]], cmn=opts["cmn"], varnorm=opts.get("varnorm", False), agc=agc, a=a,
                               ldadim=opts.get("ldadim", 0), feat=ff)
            _same(mfcc[foff[u]:foff[u + 1]], c)
            _same(feats[foff[u]:foff[u + 1]], f)
        if opts.get("agc") == "emax":
            st = states[s]
            assert (np.float32(st.agc_max), np.float32(st.agc_obs_max), np.float32(st.agc_obs_max_sum), st.agc_obs_frame,
                    st.agc_obs_utt) == agc.state()
    fe.close(); raw.close()


def _session():
    go = fe_golden.goforward()
    u = fx.emax_session()                                # 21 utterances: empty, silent, speech, sub-frame, ...
    return u[:5] + [go[5000:40000], np.zeros(0, np.int16)] + u[5:]


def test_emax_sessions_split_and_reordered():
    from pocketsphinx_b200 import api
    fe = api.FrontEnd(make_fe_desc(), 0, make_fe_opts(cmn="none", agc="emax"))
    utts = _session()
    whole, foff, st_whole, _ = _run(fe, utts, [0, len(utts)])
    for k in (1, 9, 17):
        a, _, st_a, _ = _run(fe, utts[:k], [0, k])
        b, _, st_b, _ = _run(fe, utts[k:], [0, len(utts) - k], st_a)
        assert np.concatenate([a, b]).tobytes() == whole.tobytes()
        assert bytes(st_b[0]) == bytes(st_whole[0])
    s1, s2 = utts[:6], utts[6:]
    x, fx_, stx, _ = _run(fe, s1 + s2, [0, 6, len(utts)])
    y, fy, sty, _ = _run(fe, s2 + s1, [0, len(s2), len(utts)])
    n1 = fx_[6]
    assert x[:n1].tobytes() == y[fy[len(s2)]:].tobytes() and x[n1:].tobytes() == y[:fy[len(s2)]].tobytes()
    assert bytes(stx[0]) == bytes(sty[1]) and bytes(stx[1]) == bytes(sty[0])
    # the initial state is agc_init + agc_emax_set's (10 without CMN), and a fresh front end starts from it
    init = fe.initial_state()
    assert (init.agc_max, init.agc_obs_max, init.agc_obs_max_sum, init.agc_obs_frame, init.agc_obs_utt) == (10.0, 0.0, 0.0, 0, 0)
    assert bytes(init) == bytes(_run(fe, [], [0, 0])[2][0])
    fe.close()


def test_states_untouched_without_emax():
    from pocketsphinx_b200 import api
    fe = api.FrontEnd(make_fe_desc(), 0, make_fe_opts(cmn="live", agc="max", dither=True))
    st = fe.initial_state()
    st.agc_max, st.agc_obs_max, st.agc_obs_max_sum, st.agc_obs_frame, st.agc_obs_utt = 1.5, -3.0, 7.0, 1, 3
    out = _run(fe, _ragged(), [0, 6], [st])[2][0]
    assert (out.agc_max, out.agc_obs_max, out.agc_obs_max_sum, out.agc_obs_frame, out.agc_obs_utt) == (1.5, -3.0, 7.0, 1, 3)
    fe.close()


def test_senone_scores_on_lda_features(an4_lda):
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.model import PackedModel
    a = an4_lda["a29"]
    fe = api.FrontEnd(make_fe_desc(**AN4), 0, make_fe_opts(cmn="batch", lda=a))
    utts = [fe_golden.goforward(), _pcm(9000, 4)]
    feats, foff, _, _ = _run(fe, utts)
    pm = PackedModel.from_dir(an4_lda["d29"])
    assert pm.sumlen == 29
    m = api.Model(pm)
    b = api.Batch(m, 4, 2048)
    scr = b.score_host(feats, foff)
    ref = refdrv.RefModel(an4_lda["d29"])
    assert ref.sumlen == 29
    assert np.array_equal(scr, ref.score(feats))              # the reference's GMM on the device's features
    b.close(); m.close(); fe.close(); ref.close()


def _decode(hd, utts, sessions=None, **cfg):
    from pocketsphinx_b200.decoder import Decoder
    dec = Decoder(hd, DIC, LM, max_utts=8, max_frames=4096, **cfg)
    try:
        out = dec.decode_raw_batch(utts, sessions)
        return [o["hyp"] for o in out], dec.fe.feat_dim
    finally:
        dec.close()


@pytest.mark.timeout(900)
def test_decoder_picks_up_feature_transform(an4_lda):
    go = fe_golden.goforward()
    utts = [go, go[:30000], go[8000:]]
    for which, dim in (("d29", 29), ("d39", 39)):
        hyps, fd = _decode(an4_lda[which], utts)
        assert fd == dim
        assert hyps == [fs.ref_session_decode(an4_lda[which], LM, DIC, [u], bestpath="no")[0] for u in utts]
    # the same model without its feature_transform: the front end's 39 dimensions do not fit, and it says so
    from pocketsphinx_b200.decoder import Decoder
    with pytest.raises(ValueError, match="39-dimensional.*wants 29"):
        Decoder(an4_lda["d29_plain"], DIC, LM, max_utts=2, max_frames=1024)


@pytest.mark.timeout(900)
def test_decoder_agc_emax_session():
    hd = fs.ref_model_dir("en-us")
    go = fe_golden.goforward()
    utts = [go, go[:30000], go, go[10000:]]
    want = fs.ref_session_decode(hd, LM, DIC, utts, agc="emax", bestpath="no")
    hyps, _ = _decode(hd, [utts[0], go, utts[1], utts[2], utts[3]], ["a", "b", "a", "a", "a"], agc="emax")
    assert [hyps[0]] + hyps[2:] == want
    assert hyps[1] == fs.ref_session_decode(hd, LM, DIC, [go], agc="emax", bestpath="no")[0]


@pytest.mark.parametrize("name", ["an4", "en-us"])
def test_decoder_varnorm_front_end(name):
    # the shipped models were not trained with -varnorm: the reference's search finds no word on them, so the
    # front end Decoder builds is checked against the reference's features instead of hypotheses
    from pocketsphinx_b200.decoder import Decoder
    hd = fs.ref_model_dir(name)
    dec = Decoder(hd, DIC, LM, max_utts=2, max_frames=2048, varnorm="yes", cmn="batch")
    utts = [fe_golden.goforward(), _pcm(7000, 1)]
    feats, foff, _, _ = _run(dec.fe, utts)
    dec.close()
    r = refdrv.RefModel(hd, varnorm="yes", cmn="batch")
    for u, pcm in enumerate(utts):
        _close_enough(feats[foff[u]:foff[u + 1]], r.featurize_fresh(pcm))
    r.close()
