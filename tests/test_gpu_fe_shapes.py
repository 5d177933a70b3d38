"""GPU (-m gpu): the device front end at every shape of tests/fe_shape_cases.GRID -- 8 to 32 kHz, odd frame sizes
(205, 283, 565 samples: the middle sample is not windowed), 256- to 1024-point FFTs (8 and 10 butterfly stages,
up to 513 power-spectrum bins), frame shifts of 80 to 320 samples, -remove_dc at 1024 points, pre-emphasis off,
64 filters (every thread of the per-utterance kernel a filter), 1, 20 and 32 cepstra -- against the compiled
reference run live and against oracle/fe_port.py; the feature options on those shapes (dither at an 80-sample shift,
live CMN and -varnorm at 32 cepstra, -agc max and LDA at 20, the carried noise tracker at 64 filters, two VTLN warps
at 22 kHz); the shapes psb_fe_create refuses; and one decode of 8 kHz audio.

Tolerance as in tests/test_gpu_fe.py: device log() and glibc log() can differ in the last bit of a float64, so
features are compared at 1e-4 of the largest value, and more than 99 % of them must be bit-identical.  Given the
device's own cepstra, CMN, -varnorm, AGC, deltas and LDA are float32 operations in a fixed order, so those are
compared bit for bit."""
import os

import numpy as np
import pytest

import fe_noise_cases as N
import fe_sessions as fs
import fe_shape_cases as sc
import fe_warp_cases as wc
import fe_xform as fx
from oracle import fe_port, refdrv
from pocketsphinx_b200.fe_tables import make_fe_desc, make_fe_opts

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not refdrv.available(), reason="compiled reference not built")]
IDS = [e["id"] for e in sc.GRID]


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    return tmp_path_factory.mktemp("models")


def _nan_bits_equal(got, want):
    """Bit for bit, except that a NaN matches any NaN (the device's 0/0 and x86's have different bits)."""
    nan = np.isnan(want)
    return got.shape == want.shape and np.array_equal(np.isnan(got), nan) and \
        np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


def _compare(got, want, what):
    """test_gpu_fe._close's rule; returns (bit-identical values, values compared, max error / scale)."""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    if nan.all():
        return 0, 0, 0.0
    g, w = got[~nan], want[~nan]
    scale = max(1.0, float(np.abs(w.astype(np.float64)).max()))
    err = float(np.abs(g.astype(np.float64) - w.astype(np.float64)).max()) / scale
    assert err <= 1e-4, "%s: max abs err %g of scale %g" % (what, err * scale, scale)
    return int((g.view(np.uint32) == w.view(np.uint32)).sum()), g.size, err


def _split(a, off):
    return [a[off[u]:off[u + 1]] for u in range(len(off) - 1)]


def _process(fe, utts, want_mfcc=False):
    off = fe.sample_offsets([len(u) for u in utts])
    return fe.process_host(np.concatenate(utts), off, want_mfcc)


@pytest.mark.parametrize("entry", sc.GRID, ids=IDS)
def test_shape_matches_reference_and_fe_port(entry, models):
    from pocketsphinx_b200 import api
    ref = sc.ref_model(entry, models)
    rd, mk = ref.fe_desc(), make_fe_desc(**entry["mk"])
    assert (rd["frame_size"], rd["frame_shift"], rd["fft_size"]) == entry["shape"]
    nc = rd["n_cep"]
    utts = sc.utterances(entry)
    fe = api.FrontEnd(mk)
    feats, foff, mfcc = _process(fe, utts, want_mfcc=True)
    assert feats.shape == (foff[-1], 3 * nc)
    # (a) the reference's own tables and the Python mirror's give the same bytes
    fe_ref = api.FrontEnd(rd)
    feats_r, foff_r = _process(fe_ref, utts)
    assert np.array_equal(foff, foff_r) and feats.tobytes() == feats_r.tobytes()
    fe_ref.close()
    # (b) against the reference run live: frame counts, 1e-4 of scale, the share of bit-identical values
    same = n = 0
    worst = 0.0
    for u, pcm in enumerate(utts):
        want = ref.featurize_fresh(pcm) if len(pcm) else np.zeros((0, 3 * nc), np.float32)
        got = feats[foff[u]:foff[u + 1]]
        assert fe.n_frames(len(pcm)) == len(want) == len(got), (entry["id"], len(pcm))
        s, k, err = _compare(got, want, "%s, %d samples" % (entry["id"], len(pcm)))
        same, n, worst = same + s, n + k, max(worst, err)
    share = same / n
    print("\n%-15s frame %4d shift %3d fft %4d: %.4f of %d feature values bit-identical, worst error %.2e of scale"
          % ((entry["id"],) + entry["shape"] + (share, n, worst)))
    assert share > 0.99, "%s: share of bit-identical feature values %.4f" % (entry["id"], share)
    # (c) against fe_port: the device cepstra before CMN at the same tolerance, and the CMN and deltas fe_port
    # computes from them bit for bit
    raw = api.FrontEnd(make_fe_desc(**dict(entry["mk"], cmn="none")))
    _, foff_c, cep = _process(raw, utts, want_mfcc=True)
    raw.close()
    assert np.array_equal(foff_c, foff)
    for u, pcm in enumerate(utts):
        c = cep[foff[u]:foff[u + 1]]
        what = "%s, %d samples" % (entry["id"], len(pcm))
        _compare(c, fe_port.cepstra(rd, fe_port.mfspec(rd, pcm)), "cepstra, " + what)
        f, c_cmn = fe_port.features(mk, c)
        assert _nan_bits_equal(feats[foff[u]:foff[u + 1]], f), "features from the device cepstra, " + what
        assert _nan_bits_equal(mfcc[foff[u]:foff[u + 1]], c_cmn), "cepstra after CMN, " + what
    # (d) the batch's order does not matter
    rev, foff_v = _process(fe, utts[::-1])
    for u in range(len(utts)):
        v = len(utts) - 1 - u
        assert rev[foff_v[v]:foff_v[v + 1]].tobytes() == feats[foff[u]:foff[u + 1]].tobytes(), (entry["id"], u)
    fe.close()
    ref.close()


# ---- feature options on the new shapes ----

def test_dither_s2_4x_sessions_at_8k():
    """tidigits' front end (s2_4x, -remove_dc, dither) at 8 kHz with 205-sample frames and an 80-sample shift:
    sessions of 3 utterances, each session one generator seeded with -seed."""
    from pocketsphinx_b200 import api
    kv = dict(samprate="8000", upperf="3500", wlen="0.025625", dither="yes", seed="13")
    desc = make_fe_desc(wlen=0.025625, nfilt=20, lowerf=1, upperf=3500, samprate=8000, round_filters=False,
                        remove_dc=True, remove_noise=False, lifter=0, transform="dct")
    assert (desc["frame_size"], desc["frame_shift"], desc["fft_size"]) == (205, 80, 256)
    opts = make_fe_opts(feat="s2_4x", cmn="batch", dither=True, seed=13)
    fe = api.FrontEnd(desc, 0, opts)
    go = sc.goforward()
    fsz, sh = 205, 80
    utts = [go[:fsz + sh + 1], go[3000:3001], go[5000:11000], go[:fsz - 1], go[9000:9000 + fsz], go[20000:24000]]
    sess_off = [0, 3, 6]
    off = fe.sample_offsets([len(u) for u in utts])
    feats, foff, states = fe.process_sessions(np.concatenate(utts), off, sess_off)
    assert feats.shape[1] == 51
    same = n = 0
    for s in range(len(sess_off) - 1):
        r = refdrv.RefModel(fs.ref_model_dir("tidigits"), **kv)
        rng = fs.MT19937(13)
        for u in range(sess_off[s], sess_off[s + 1]):
            want = r.featurize(utts[u]) if len(utts[u]) else np.zeros((0, 51), np.float32)
            k = _compare(feats[foff[u]:foff[u + 1]], want, "session %d, %d samples" % (s, len(utts[u])))
            same, n = same + k[0], n + k[1]
            _, main, tail = fs.draw_plan(desc, len(utts[u]))
            rng.dither_bits(main + tail)
        r.close()
        assert states[s].mt_index == rng.mti and list(states[s].mt) == rng.mt, "session %d" % s
    assert same / n > 0.99, same / n
    fe.close()


def _raw_cepstra(desc, utts):
    from pocketsphinx_b200 import api
    raw = api.FrontEnd(dict(desc, cmn=0))
    _, foff, cep = _process(raw, utts, want_mfcc=True)
    raw.close()
    return _split(cep, foff)


def _long_session():
    go = sc.goforward()
    return [go, np.tile(go, 6), np.zeros(3000, np.int16), go[:15000]]        # one utterance of more than 800 frames


def test_live_cmn_32_cepstra(models):
    from pocketsphinx_b200 import api
    e = sc.BY_ID["ncep32"]
    desc = make_fe_desc(**e["mk"])
    opts = make_fe_opts(cmn="live", ncep=32)
    utts = _long_session()
    fe = api.FrontEnd(desc, 0, opts)
    off = fe.sample_offsets([len(u) for u in utts])
    feats, foff, states, mfcc = fe.process_sessions(np.concatenate(utts), off, [0, len(utts)], want_mfcc=True)
    fe.close()
    assert foff[-1] > 800 and feats.shape[1] == 96
    # the reference's own cmn_live over the device's cepstra, utterance by utterance
    rc = fs.RefCmn("40,3,-1", 32)
    for u, c in enumerate(_raw_cepstra(desc, utts)):
        want = rc.utterance(c)
        assert want.tobytes() == mfcc[foff[u]:foff[u + 1]].tobytes(), u
        assert _nan_bits_equal(feats[foff[u]:foff[u + 1]], fs.dyn_features(want, 0)), u
    mean, s, nframe = rc.state()
    rc.close()
    assert np.array(states[0].cmn_mean[:32], np.float32).tobytes() == mean.tobytes()
    assert np.array(states[0].cmn_sum[:32], np.float32).tobytes() == s.tobytes() and states[0].cmn_nframe == nframe
    # and the first utterance against the reference front end run live
    r = sc.ref_model(e, models, cmn="live")
    N.close_enough(feats[foff[0]:foff[1]], r.featurize_fresh(utts[0]))
    r.close()


@pytest.mark.parametrize("which,extra,opts", [
    ("ncep32", dict(varnorm="yes"), dict(cmn="batch", varnorm=True)),
    ("ncep20", dict(agc="max"), dict(cmn="batch", agc="max")),
])
def test_varnorm_and_agc_at_other_cepstra(models, which, extra, opts):
    from pocketsphinx_b200 import api
    e = sc.BY_ID[which]
    desc = make_fe_desc(**e["mk"])
    fe = api.FrontEnd(desc, 0, make_fe_opts(ncep=e["ncep"], **opts))
    utts = sc.utterances(e)
    feats, foff = _process(fe, utts)
    fe.close()
    r = sc.ref_model(e, models, **extra)
    for u, (pcm, c) in enumerate(zip(utts, _raw_cepstra(desc, utts))):
        got = feats[foff[u]:foff[u + 1]]
        if not len(pcm):
            assert got.shape == (0, 3 * e["ncep"])
            continue
        want, _ = fx.features(c, "batch", opts.get("varnorm", False), fx.Agc(opts["agc"]) if "agc" in opts else None)
        assert _nan_bits_equal(got, want), (which, u)
        _compare(got, r.featurize_fresh(pcm), "%s, %d samples" % (which, len(pcm)))
    r.close()


def test_lda_60_dimensions(models, tmp_path):
    from pocketsphinx_b200 import api, s3io
    e = sc.BY_ID["ncep20"]
    path = str(tmp_path / "feature_transform")
    s3io.write_lda(path, fx.orthonormal(60, 60, 5)[None])
    a = s3io.read_lda(path)[0]
    desc = make_fe_desc(**e["mk"])
    fe = api.FrontEnd(desc, 0, make_fe_opts(cmn="batch", ncep=20, lda=a))
    assert fe.feat_dim == 60
    utts = sc.utterances(e)
    feats, foff = _process(fe, utts)
    fe.close()
    r = sc.ref_model(e, models, lda=path)
    for u, (pcm, c) in enumerate(zip(utts, _raw_cepstra(desc, utts))):
        got = feats[foff[u]:foff[u + 1]]
        if not len(pcm):
            assert got.shape == (0, 60)
            continue
        assert _nan_bits_equal(got, fx.features(c, a=a)[0]), u
        _compare(got, r.featurize_fresh(pcm), "lda, %d samples" % len(pcm))
    r.close()


def test_noise_tracker_carried_at_64_filters():
    """-remove_noise over a session with ps_start_stream once, 64 filters."""
    from pocketsphinx_b200 import api
    e = sc.BY_ID["nfilt64"]
    fe = api.FrontEnd(make_fe_desc(**e["mk"]))
    utts = [N.pcm(6000, 1, 300), sc.goforward()[:20000], np.zeros(0, np.int16), N.pcm(3000, 2, 3000), sc.goforward()]
    starts = np.zeros(len(utts), bool)
    starts[0] = True
    off = fe.sample_offsets([len(u) for u in utts])
    feats, foff, _, noise = fe.process_sessions(np.concatenate(utts), off, [0, len(utts)], starts=starts)
    fe.close()
    assert not noise[0].undefined
    r = sc.ref_model(e, None)
    want = N.ref_stream_features(r, utts, starts)
    r.close()
    for u, w in enumerate(want):
        N.close_enough(feats[foff[u]:foff[u + 1]], w)
    # without the carried tracker the later utterances differ: the test sees the carry
    r = sc.ref_model(e, None)
    fresh = N.ref_stream_features(r, utts[3:4], [True])[0]
    r.close()
    assert fresh.tobytes() != want[3].tobytes()


def test_two_warps_in_one_batch_at_22k():
    from pocketsphinx_b200 import api
    e = sc.BY_ID["22k"]
    fe = api.FrontEnd(make_fe_desc(**e["mk"]))
    utts = sc.utterances(e)
    warps = [("inverse_linear", "0.9"), ("inverse_linear", "1.1")]
    which = [u % 2 for u in range(len(utts))]
    fe.set_filterbanks(warps, which)
    feats, foff = _process(fe, utts)
    fe.close()
    for b, (wt, wp) in enumerate(warps):
        r = wc.ref_model("en-us", wt, wp, **e["kv"])
        for u in [i for i in range(len(utts)) if which[i] == b and len(utts[i])]:
            _compare(feats[foff[u]:foff[u + 1]], r.featurize_fresh(utts[u]), "warp %s, %d samples" % (wp, len(utts[u])))
        r.close()


# ---- what psb_fe_create refuses ----

@pytest.mark.parametrize("mk,limit", [
    (dict(samprate=44100), "1024] (got 2048)"),
    (dict(samprate=48000), "1024] (got 2048)"),
    (dict(nfilt=65), "n_filt <= 64"),
    (dict(ncep=33, nfilt=40), "n_cep <= 32"),
    (dict(ncep=20, nfilt=16), "n_cep <= n_filt"),
], ids=["44k", "48k", "nfilt65", "ncep33", "ncep_gt_nfilt"])
def test_refused_shapes(mk, limit):
    import ctypes as C
    from pocketsphinx_b200 import api
    from pocketsphinx_b200._lib import FeDesc
    desc = make_fe_desc(**mk)
    launches = api.lib().psb_kernel_launch_count()
    with pytest.raises(api.PsbError, match="psb_fe_create"):
        api.FrontEnd(desc)
    assert limit in api.lib().psb_last_error().decode()
    # through the C entry point: refused, and no handle comes back
    fd = FeDesc()
    for k in ("frame_size", "frame_shift", "fft_size", "fft_order", "n_filt", "n_cep", "remove_dc", "remove_noise",
              "transform", "lifter_val", "window", "cmn"):
        setattr(fd, k, int(desc[k]))
    fd.pre_emphasis_alpha, fd.sqrt_inv_n, fd.sqrt_inv_2n = float(desc["alpha"]), float(desc["sqrt_inv_n"]), float(desc["sqrt_inv_2n"])
    keep = {k: np.ascontiguousarray(desc[k]) for k in ("hamming", "ccc", "sss", "spec_start", "filt_start",
                                                       "filt_width", "filt_coeffs", "mel_cosine", "lifter")}
    for k, a in keep.items():
        setattr(fd, k, a.ctypes.data if a.size else None)
    fd.n_coeffs = int(keep["filt_coeffs"].size)
    h = C.c_void_p()
    assert api.lib().psb_fe_create(C.byref(fd), 0, C.byref(h)) != 0 and not h.value
    assert limit in api.lib().psb_last_error().decode()
    assert api.lib().psb_kernel_launch_count() == launches


def test_decoder_refuses_44k():
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.decoder import Decoder
    hd, dic, lm = sc.EN_US, os.path.join(sc.REF, "data", "turtle.dic"), os.path.join(sc.REF, "data", "turtle.lm.bin")
    launches = api.lib().psb_kernel_launch_count()
    with pytest.raises(api.PsbError, match="fft_size"):
        Decoder(hd, dic, lm, max_utts=2, max_frames=1024, samprate="44100")
    assert api.lib().psb_kernel_launch_count() == launches


# ---- downstream of another sample rate ----

@pytest.mark.timeout(900)
def test_decode_8k_audio(tmp_path):
    """goforward decimated to 8 kHz and decoded with -samprate 8000 -upperf 3500: the downstream kernels on features
    of another sample rate.  Compared as tests/test_gpu_zz_decoder.py compares the 16 kHz decode: words, segment end
    frames and path score against the reference's own two-pass backpointer table (refdrv.fwdtree), here run on a
    copy of en-us whose feat.params names the 8 kHz settings (they must be in that file: the reference reads it
    after the caller's settings); and the hypothesis against the reference's full decode."""
    from scipy.signal import resample_poly
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.decoder import Decoder
    hd, dic, lm = sc.EN_US, os.path.join(sc.REF, "data", "turtle.dic"), os.path.join(sc.REF, "data", "turtle.lm.bin")
    go = np.fromfile(os.path.join(sc.REF, "data", "goforward.raw"), np.int16)
    pcm = np.clip(np.round(resample_poly(go.astype(np.float64), 1, 2)), -32768, 32767).astype(np.int16)
    dec = Decoder(hd, dic, lm, max_utts=2, max_frames=4096, samprate="8000", upperf="3500")
    out = dec.decode_raw_batch([pcm])[0]
    dec.close()
    hd8 = fx.copy_model(hd, str(tmp_path / "en-us-8k"))
    with open(os.path.join(hd8, "feat.params"), "a") as f:
        f.write("-samprate 8000\n-upperf 3500\n")
    r = refdrv.fwdtree(hd8, lm, dic, pcm, fwdflat="yes", pl_window="5")
    assert out["n_frames"] == r["n_frame"] == fe_port.n_frames(make_fe_desc(samprate=8000, upperf=3500), len(pcm))
    _, score, chain = api.ngram_hyp(r["bp"], r["bp_idx"], len(r["bp_idx"]) - 1, int(r["info"][20]))
    print("\n8 kHz decode: %r, score %d (reference %d)" % (out["hyp"], out["score"], score))
    assert [int(w) for w in out["seg"][:, 1]] == [int(w) for w in chain[:, 1]]
    assert np.abs(out["seg"][:, 3] - chain[:, 3]).max() <= 2 and abs(out["score"] - score) < 200
    assert out["hyp"] == refdrv.decode(hd8, lm, dic, pcm, bestpath="no")["hyp"] != ""
