"""CPU: the numpy restatement of s2_4x / s3_1x39, live CMN over sessions and dither (tests/fe_sessions.py)
against the compiled reference, bit for bit; make_fe_desc / make_fe_opts for the shipped models' feat.params;
psb_fe_create_ex argument checks (no device needed)."""
import ctypes as C

import numpy as np
import pytest

import fe_sessions as fs
from oracle import fe_golden, refdrv
from pocketsphinx_b200.fe_tables import make_fe_desc, make_fe_opts

needs_ref = pytest.mark.skipif(not refdrv.available(), reason="compiled reference not built")

TIDIGITS = dict(wlen=0.025, nfilt=20, lowerf=1, upperf=4000, round_filters=False, remove_dc=True, remove_noise=False,
                lifter=0, transform="dct")
AN4 = dict(nfilt=40, lowerf=133.3334, upperf=6855.4976, transform="legacy", lifter=0, remove_noise=False)


def _pcm(n, seed, amp=3000):
    return (np.random.default_rng(seed).standard_normal(n) * amp).astype(np.int16)


@needs_ref
@pytest.mark.parametrize("name,kw", [("tidigits", TIDIGITS), ("an4", AN4)])
def test_make_fe_desc_matches_reference_tables(name, kw):
    r = refdrv.RefModel(fs.ref_model_dir(name))
    ref, ours = r.fe_desc(), make_fe_desc(**kw)
    r.close()
    for k in ("frame_size", "frame_shift", "fft_size", "fft_order", "n_filt", "n_cep", "remove_dc", "remove_noise",
              "transform", "lifter_val"):
        assert ours[k] == ref[k], k
    for k in ("alpha", "sqrt_inv_n", "sqrt_inv_2n"):
        assert np.float32(ours[k]).tobytes() == np.float32(ref[k]).tobytes(), k
    for k in ("hamming", "ccc", "sss", "spec_start", "filt_start", "filt_width", "filt_coeffs", "mel_cosine", "lifter"):
        assert ours[k].dtype == ref[k].dtype and ours[k].tobytes() == ref[k].tobytes(), k


def test_make_fe_opts_parses_like_cmn_set_repr():
    o = make_fe_opts(feat="1s_12c_12d_3p_12dd", cmn="current", cmninit="63,-1,1", dither=True, seed=7)
    assert (o["feat"], o["cmn"], o["dither"], o["seed"]) == (2, 1, 1, 7)
    assert o["cmn_init"][:4].tolist() == [63.0, -1.0, 1.0, 0.0]
    assert make_fe_opts(cmninit="1,2,3,4", ncep=2)["cmn_init"][:3].tolist() == [1.0, 2.0, 0.0]
    with pytest.raises(KeyError):
        make_fe_opts(feat="1s_c_d_ld_dd")


@needs_ref
@pytest.mark.parametrize("name,kv,desc,opts", [
    ("tidigits", dict(dither="no"), TIDIGITS, dict(feat="s2_4x", cmn="batch")),
    ("an4", dict(feat="s3_1x39"), AN4, dict(feat="s3_1x39", cmn="batch")),
    ("an4", dict(feat="1s_12c_12d_3p_12dd", cmn="none"), AN4, dict(feat="s3_1x39", cmn="none")),
])
def test_feature_types_match_reference(name, kv, desc, opts):
    r = refdrv.RefModel(fs.ref_model_dir(name), **kv)
    d, o = make_fe_desc(**desc), make_fe_opts(**opts)
    for pcm in (fe_golden.goforward(), _pcm(5000, 1), _pcm(300, 2)):
        ref = r.featurize_fresh(pcm)
        assert fs.session(d, o, [pcm])[0][0].tobytes() == ref.tobytes()
    r.close()


@needs_ref
def test_mt19937_matches_reference_genrand():
    L = fs.ref_lib()
    for seed in (-1, 12345):
        L.genrand_seed(seed & 0xffffffffffffffff)
        ours = fs.MT19937(seed)
        assert [ours.int31() for _ in range(1500)] == [L.genrand_int31() for _ in range(1500)]


def _cep_session(seed):
    rng = np.random.default_rng(seed)
    utts = []
    for T, silent in ((30, False), (12, True), (900, False), (0, False), (500, False), (350, False), (1, False)):
        c = (rng.standard_normal((T, 13)) * 4).astype(np.float32)
        c[:, 0] = -1.5 if silent else np.abs(c[:, 0]) + 5
        c[::7, 0] = -0.25 if T else c[::7, 0]              # some frames with c0 < 0 in every utterance
        utts.append(c)
    return utts


@needs_ref
def test_live_cmn_session_matches_reference_cmn_live():
    # one utterance longer than 800 frames, and 500 + 350 frames crossing 800 over two utterances
    ref, ours = fs.RefCmn("40,3,-1"), fs.CmnState(make_fe_opts(cmninit="40,3,-1")["cmn_init"])
    for cep in _cep_session(3):
        assert ours.utterance(cep).tobytes() == ref.utterance(cep).tobytes()
        mean, s, n = ref.state()
        assert (ours.mean.tobytes(), ours.sum.tobytes(), ours.nframe) == (mean.tobytes(), s.tobytes(), n)
    ref.close()


@needs_ref
@pytest.mark.parametrize("name,desc", [("tidigits", TIDIGITS), ("en-us", {})])
def test_dither_session_matches_reference(name, desc):
    d = make_fe_desc(**desc)
    fsz, sh = d["frame_size"], d["frame_shift"]
    lens = [0, 1, fsz - 1, fsz, fsz + 1, fsz + sh - 1, fsz + sh, fsz + sh + 1, 3000]
    for seed in (-1, 4242):
        # refdrv.mfcc: a fresh noise tracker per utterance, the generator seeded once when the reference opens
        r = refdrv.RefModel(fs.ref_model_dir(name), dither="yes", seed=str(seed), cmn="none")
        rng = fs.MT19937(seed)
        for i, n in enumerate(lens):
            pcm = _pcm(n, 10 + i, amp=2 if i % 2 else 3000)
            if i == 2:
                pcm[:] = 32767                               # the int16 wrap of a dithered sample
            ref = r.mfcc(pcm)
            ours = fe_port_cepstra(d, fs.mfspec_dithered(d, pcm, rng))
            assert ours.tobytes() == ref.tobytes(), (seed, n)
        r.close()


def fe_port_cepstra(d, mf):
    from oracle import fe_port
    return fe_port.cepstra(d, mf)


def test_fe_create_ex_checks_arguments():
    from pocketsphinx_b200 import _lib
    L = _lib.lib()
    d = make_fe_desc()
    x = _lib.FeDesc()
    for k in ("frame_size", "frame_shift", "fft_size", "fft_order", "n_filt", "n_cep", "remove_dc", "remove_noise",
              "transform", "lifter_val", "window", "cmn"):
        setattr(x, k, int(d[k]))
    x.pre_emphasis_alpha, x.sqrt_inv_n, x.sqrt_inv_2n = float(d["alpha"]), float(d["sqrt_inv_n"]), float(d["sqrt_inv_2n"])
    for k in ("hamming", "ccc", "sss", "spec_start", "filt_start", "filt_width", "filt_coeffs", "mel_cosine", "lifter"):
        setattr(x, k, d[k].ctypes.data)
    x.n_coeffs = int(d["filt_coeffs"].size)
    h = C.c_void_p()
    for over, word in ((dict(feat=3), "feat"), (dict(cmn=3), "cmn"), (dict(cmn=2, varnorm=1), "live mode"),
                       (dict(varnorm=1), "variance"), (dict(dither=2), "dither")):
        o = _lib.FeOpts()
        for k, v in over.items():
            setattr(o, k, v)
        rc = L.psb_fe_create_ex(C.byref(x), C.byref(o), 0, C.byref(h))
        assert rc < 0 and word in L.psb_last_error().decode(), (over, L.psb_last_error())
    x.n_cep = 12
    o = _lib.FeOpts()
    o.feat = 1
    assert L.psb_fe_create_ex(C.byref(x), C.byref(o), 0, C.byref(h)) < 0 and "n_cep 13" in L.psb_last_error().decode()
