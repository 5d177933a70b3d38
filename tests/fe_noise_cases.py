"""TEST INFRASTRUCTURE: the compiled reference run over several utterances with ps_start_stream at chosen
utterances only, so the -remove_noise tracker (fe_noise.c) carries across the others.  Shared by
tests/test_fe_noise_oracle.py (CPU: the two drivers below agree) and tests/test_gpu_fe_noise.py (the device
against them).

  ref_stream_features  one reference acmod_t (oracle/refdrv.RefModel): refdrv_fe_reset, which is what
                       ps_start_stream does (pocketsphinx.c:1073-1083), before the utterances that start a
                       stream, and refdrv_featurize -- which never resets the tracker -- on each.  refdrv_featurize
                       restores the CMN state after init first, so live CMN does not carry here.
  ref_decoder          a plain ps_decoder_t through the public API only: ps_start_stream where a stream starts,
                       then ps_start_utt, ps_process_raw(full_utt), ps_end_utt.  Returns each utterance's
                       hypothesis, score and word segments, and its cepstra before CMN from the decoder's own
                       -mfclogdir files (acmod_log_mfc, big-endian float32 after a 4-byte count)."""
import ctypes as C
import os
import tempfile

import numpy as np

import fe_sessions as fs


def ref_stream_features(r, utterances, starts):
    """Features of utterances through RefModel r in order, the noise tracker reset before utterance u iff starts[u]."""
    from oracle import refdrv
    out = []
    for pcm, st in zip(utterances, starts):
        if st:
            refdrv.lib().refdrv_fe_reset(r.h)
        # no samples: fe_process_frames and fe_end_utt make no frame and leave the tracker alone
        out.append(r.featurize(pcm) if len(pcm) else np.zeros((0, r.sumlen), np.float32))
    return out


def _ps_lib():
    L = fs.ref_lib()
    L.ps_config_init.restype = C.c_void_p
    L.ps_config_init.argtypes = [C.c_void_p]
    L.ps_config_set_str.restype = C.c_void_p
    L.ps_config_set_str.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    L.ps_init.restype = C.c_void_p
    L.ps_init.argtypes = [C.c_void_p]
    for f in ("ps_start_stream", "ps_start_utt", "ps_end_utt", "ps_free", "ps_config_free"):
        getattr(L, f).argtypes = [C.c_void_p]
    L.ps_process_raw.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int]
    L.ps_get_hyp.restype = C.c_char_p
    L.ps_get_hyp.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
    L.ps_seg_iter.restype = L.ps_seg_next.restype = C.c_void_p
    L.ps_seg_iter.argtypes = L.ps_seg_next.argtypes = [C.c_void_p]
    L.ps_seg_word.restype = C.c_char_p
    L.ps_seg_word.argtypes = [C.c_void_p]
    L.ps_seg_frames.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    return L


def read_mfc(path, n_cep):
    """An -mfclogdir file: int32 count of the values, then the cepstra, both big-endian."""
    raw = open(path, "rb").read()
    n = int(np.frombuffer(raw[:4], ">i4")[0])
    return np.frombuffer(raw[4:4 + 4 * n], ">f4").astype(np.float32).reshape(-1, n_cep)


def ref_decoder(hmm, lm, dic, utterances, starts, **feat_params):
    """One reference ps_decoder_t (-bestpath no) over utterances in order, ps_start_stream before utterance u iff
    starts[u].  feat_params replace keys of the model's feat.params (ps_init parses that file after the caller's
    settings, so the overrides go into a copy of it).  Returns per utterance dict(hyp, score, seg [(word, sf, ef)],
    cep [T][ncep] before CMN)."""
    L = _ps_lib()
    params = {}
    for line in open(os.path.join(hmm, "feat.params")):
        parts = line.split()
        if len(parts) == 2:
            params[parts[0].lstrip("-")] = parts[1]
    params["bestpath"] = "no"
    params.update({k: str(v) for k, v in feat_params.items()})
    n_cep = int(params.get("ncep", 13))
    out = []
    with tempfile.TemporaryDirectory() as tmp:
        fp = os.path.join(tmp, "feat.params")
        with open(fp, "w") as f:
            f.write("".join("-%s %s\n" % kv for kv in params.items()))
        logdir = os.path.join(tmp, "mfc")
        os.mkdir(logdir)
        cfg = L.ps_config_init(None)
        for k, v in (("hmm", hmm), ("lm", lm), ("dict", dic), ("featparams", fp), ("mfclogdir", logdir)):
            L.ps_config_set_str(cfg, k.encode(), v.encode())
        ps = L.ps_init(cfg)
        assert ps, "ps_init failed"
        for u, (pcm, st) in enumerate(zip(utterances, starts)):
            pcm = np.ascontiguousarray(pcm, np.int16)
            if st:
                L.ps_start_stream(ps)
            L.ps_start_utt(ps)
            L.ps_process_raw(ps, pcm.ctypes.data if len(pcm) else None, len(pcm), 0, 1)
            L.ps_end_utt(ps)
            score = C.c_int32()
            h = L.ps_get_hyp(ps, C.byref(score))
            segs, it = [], L.ps_seg_iter(ps)
            while it:
                sf, ef = C.c_int(), C.c_int()
                L.ps_seg_frames(it, C.byref(sf), C.byref(ef))
                segs.append((L.ps_seg_word(it).decode(), sf.value, ef.value))
                it = L.ps_seg_next(it)
            out.append(dict(hyp=h.decode() if h else "", score=score.value, seg=segs,
                            cep=read_mfc(os.path.join(logdir, "%09d.mfc" % u), n_cep)))
        L.ps_free(ps)
        L.ps_config_free(cfg)
    return out


def pcm(n, seed, amp=3000):
    """Seeded white noise; the amplitude changes the noise floor the tracker follows."""
    return (np.random.default_rng(seed).standard_normal(n) * amp).astype(np.int16)


def close_enough(got, ref, bit_share=0.99):
    """The front end's tolerance (tests/test_gpu_fe.py): 1e-4 relative to the largest value, and more than
    bit_share of the values bit-identical (device log() and glibc log() differ in the last bit now and then)."""
    assert got.shape == ref.shape, (got.shape, ref.shape)
    if not got.size:
        return
    assert np.abs(got - ref).max() <= 1e-4 * max(1.0, float(np.abs(ref).max()))
    if bit_share:
        assert (got == ref).mean() > bit_share, (got == ref).mean()
