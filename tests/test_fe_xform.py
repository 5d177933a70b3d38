"""CPU: tests/fe_xform.py (varnorm, the three AGC modes and LDA) applied to the compiled reference's own
cepstra equals the reference's features bit for bit; s3io.read_lda reads what the reference reads and
refuses malformed files; Decoder refuses what the reference cannot load."""
import os
import struct

import numpy as np
import pytest

import fe_sessions as fs
import fe_xform as fx
from oracle import fe_golden, refdrv
from pocketsphinx_b200 import s3io

pytestmark = pytest.mark.skipif(not refdrv.available(), reason="compiled reference not built")


def _pcm(n, seed, amp=3000):
    return (np.random.default_rng(seed).standard_normal(n) * amp).astype(np.int16)


def _utts():
    go = fe_golden.goforward()
    return [go, _pcm(7000, 1), go[:300], go[20000:52000]]


def _same(got, want):
    assert got.shape == want.shape and got.tobytes() == want.tobytes()


def _check(r, utts, **kw):
    for pcm in utts:
        want = r.featurize_fresh(pcm)
        got, _ = fx.features(r.mfcc(pcm), **kw)
        _same(got, want)


@pytest.fixture(scope="module")
def an4_lda(tmp_path_factory):
    """an4_ci_cont mapped through an orthonormal 29 x 39 transform, and through a full-rank 39 x 39 rotation."""
    tmp = tmp_path_factory.mktemp("an4_lda")
    a29 = fx.orthonormal(29, 39, 7)
    a39 = fx.block_rotation(11)
    d29 = fx.derive_lda_model(fs.ref_model_dir("an4"), str(tmp / "an4_29"), a29)
    d39 = fx.derive_lda_model(fs.ref_model_dir("an4"), str(tmp / "an4_39"), a39)
    return dict(a29=a29, d29=d29, a39=a39, d39=d39)


@pytest.mark.parametrize("ldadim", [0, 29, 40])
def test_lda_29_an4(an4_lda, ldadim):
    # the model directory's feature_transform is picked up by ps_expand_model_config; ldadim 40 > m means m
    r = refdrv.RefModel(an4_lda["d29"], ldadim=ldadim)
    assert r.sumlen == 29
    _check(r, _utts(), a=s3io.read_lda(os.path.join(an4_lda["d29"], "feature_transform"))[0], ldadim=ldadim)
    r.close()


def test_lda_full_rank_an4_with_varnorm_and_agc(an4_lda):
    a = an4_lda["a39"]
    for kv, kw in ((dict(), dict()), (dict(varnorm="yes"), dict(varnorm=True)), (dict(agc="max"), dict(agc="max"))):
        r = refdrv.RefModel(an4_lda["d39"], **kv)
        assert r.sumlen == 39
        for pcm in _utts():
            agc = fx.Agc(kw["agc"]) if "agc" in kw else None
            got, _ = fx.features(r.mfcc(pcm), varnorm=kw.get("varnorm", False), agc=agc, a=a)
            _same(got, r.featurize_fresh(pcm))
        r.close()


@pytest.mark.parametrize("model", ["an4", "en-us"])
def test_varnorm(model):
    r = refdrv.RefModel(fs.ref_model_dir(model), varnorm="yes", cmn="batch")
    _check(r, _utts() + [_pcm(400, 5), np.full(3000, 7, np.int16)], varnorm=True)
    r.close()


@pytest.mark.parametrize("cmn", ["batch", "none"])
def test_agc_max(cmn):
    r = refdrv.RefModel(fs.ref_model_dir("en-us"), agc="max", cmn=cmn)
    for pcm in _utts() + [np.zeros(3000, np.int16)] * (cmn == "none"):
        got, _ = fx.features(r.mfcc(pcm), cmn=cmn, agc=fx.Agc("max"))
        _same(got, r.featurize_fresh(pcm))
    r.close()


@pytest.mark.parametrize("thresh", [2.0, 0.5, 0.0])
def test_agc_noise_with_and_without_qualifying_frames(thresh):
    # agcthresh 0: no frame is below the minimum, so nothing is subtracted
    r = refdrv.RefModel(fs.ref_model_dir("an4"), agc="noise", agcthresh=thresh)
    for pcm in _utts():
        cep = r.mfcc(pcm)
        got, _ = fx.features(cep, agc=fx.Agc("noise", thresh=thresh))
        _same(got, r.featurize_fresh(pcm))
        if thresh == 0.0:
            _same(got, fx.features(cep)[0])
    r.close()


@pytest.mark.parametrize("cmn,empty_first", [("none", True), ("none", False), ("batch", True)])
def test_agc_emax_session(cmn, empty_first):
    utts = fx.emax_session() if empty_first else fx.emax_session()[1:]
    r = refdrv.RefModel(fs.ref_model_dir("en-us"), agc="emax", cmn=cmn)
    agc = fx.Agc("emax", cmn_none=cmn == "none")
    decayed = False
    for pcm in utts:
        want = r.featurize_fresh(pcm)        # the reference's agc_t carries over from call to call
        prev = agc.obs_utt
        got, _ = fx.features(r.mfcc(pcm), cmn=cmn, agc=agc)
        _same(got, want)
        decayed |= prev == 15 and agc.obs_utt == 8
    r.close()
    assert decayed


def test_agc_emax_empty_utterance_lowers_obs_max():
    # on a fresh decoder obs_max is 0 (calloc); an utterance without frames resets it to -1000, after which an
    # all-silent utterance counts
    a, b = fx.Agc("emax", cmn_none=True), fx.Agc("emax", cmn_none=True)
    r = refdrv.RefModel(fs.ref_model_dir("en-us"), agc="emax", cmn="none")
    sil = r.mfcc(np.zeros(4000, np.int16))
    a.utterance(sil)
    b.utterance(np.zeros((0, 13), np.float32))
    b.utterance(sil)
    assert a.obs_utt == 0 and b.obs_utt == 1 and b.max < 0
    r.close()


def _write_raw_lda(path, a, order="<", tail=b"", chksum=None):
    a = np.ascontiguousarray(a, order + "f4")
    payload = struct.pack(order + "4I", *a.shape, a.size) + a.tobytes()
    hdr = b"s3\nversion 0.1\nchksum0 yes\nendhdr\n" + struct.pack(order + "I", 0x11223344)
    with open(path, "wb") as f:
        f.write(hdr + payload + struct.pack(order + "I", chksum or 0) + tail)


def test_read_lda_big_endian_and_unchecked_checksum(an4_lda, tmp_path):
    # feat_read_lda accepts either byte order and never compares the checksum: the features through the
    # matrix read_lda returns equal the reference's
    a = an4_lda["a29"]
    r0 = refdrv.RefModel(an4_lda["d29"])
    for order in ("<", ">"):
        p = str(tmp_path / ("lda" + order))
        _write_raw_lda(p, a[None], order, chksum=0xdeadbeef)
        got = s3io.read_lda(p)
        assert got.shape == (1, 29, 39) and got.tobytes() == a[None].tobytes()
        r = refdrv.RefModel(an4_lda["d29"], lda=p)
        pcm = _utts()[0]
        _same(r.featurize_fresh(pcm), r0.featurize_fresh(pcm))
        _same(fx.features(r.mfcc(pcm), a=got[0])[0], r.featurize_fresh(pcm))
        r.close()
    r0.close()


def test_read_lda_refuses_malformed(tmp_path):
    a = fx.orthonormal(29, 39, 1)[None]
    p = str(tmp_path / "lda")
    s3io.write_lda(p, a)
    raw = open(p, "rb").read()
    start = raw.find(b"endhdr\n") + 11
    for name, data in (("truncated data", raw[:start + 16 + 4 * a.size - 8]), ("no dimensions", raw[:start + 8]),
                       ("not s3", b"s4" + raw[2:]), ("no endhdr", raw[:20])):
        with open(p, "wb") as f:
            f.write(data)
        with pytest.raises(ValueError):
            s3io.read_lda(p)
    bad = bytearray(raw)
    bad[start + 12:start + 16] = struct.pack("<I", a.size + 1)        # count != d1 * d2 * d3
    with open(p, "wb") as f:
        f.write(bytes(bad))
    with pytest.raises(ValueError, match="dimensions"):
        s3io.read_lda(p)


def test_decoder_refuses_lda_with_subvectors(tmp_path):
    # en-us splits its 39 dimensions into three streams (-svspec); with a transform, feat_dimension2 is the LDA
    # output for every stream and the reference's acmod_init fails, so Decoder refuses the model too
    from pocketsphinx_b200.decoder import Decoder
    d = fx.copy_model(fs.ref_model_dir("en-us"), str(tmp_path / "en-us"))
    s3io.write_lda(os.path.join(d, "feature_transform"), fx.block_rotation(3)[None])
    with pytest.raises(RuntimeError):
        refdrv.RefModel(d)
    ref = os.path.join(os.path.dirname(refdrv.LIB_PATH), "data")
    with pytest.raises(ValueError, match="svspec"):
        Decoder(d, os.path.join(ref, "turtle.dic"), os.path.join(ref, "turtle.lm.bin"))


def test_fe_create_ex_refuses_bad_transforms():
    import ctypes as C
    from pocketsphinx_b200 import _lib
    from pocketsphinx_b200.fe_tables import make_fe_desc
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
    a = fx.orthonormal(29, 39, 2)
    h = C.c_void_p()
    for over, word in ((dict(agc=4), "agc"), (dict(agc=-1), "agc"), (dict(feat=1, lda_cols=51), "s2_4x"),
                       (dict(lda_cols=38), "columns"), (dict(lda_rows=0), "rows"), (dict(lda_rows=40, lda_cols=39), "outputs"),
                       (dict(cmn=1, varnorm=2), "varnorm")):
        o = _lib.FeOpts()
        o.lda, o.lda_rows, o.lda_cols = a.ctypes.data, 29, 39
        for k, v in over.items():
            setattr(o, k, v)
        rc = L.psb_fe_create_ex(C.byref(x), C.byref(o), 0, C.byref(h))
        assert rc < 0 and word in L.psb_last_error().decode(), (over, L.psb_last_error())
