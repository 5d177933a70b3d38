"""CPU: the VAD and endpointer arithmetic of pocketsphinx_b200/csrc/psb_vad_core.h (built for the host by
tests/emul/vad_emul.cpp) against the compiled reference (ps_vad_* / ps_endpointer_* looped by
tests/emul/vad_refdrv.c): per-frame decisions and the whole VadInstT after every frame, the chunked
feature computation with its boundary repairs, and the endpointer's segments and float64 times."""
import ctypes as C

import numpy as np
import pytest

import vad_cases as V

pytestmark = pytest.mark.skipif(not V.ref_available(), reason="compiled reference (oracle/_ref) not built")


def _emul_run(mode, rate, fl, pcm):
    fs, _ = V.ref_params(mode, rate, fl)
    closest = V.closest_rate(rate)
    nf = len(pcm) // fs
    flags = np.zeros(max(nf, 1), np.int8)
    st = np.zeros((max(nf, 1), V.STATE_BYTES), np.uint8)
    V.emul().vad_emul_run(mode, closest, fs, V._p(np.ascontiguousarray(pcm, np.int16)), nf, V._p(flags), V._p(st))
    return flags[:nf], st[:nf]


def _cases():
    a = V.audio()
    out = [("test_audio_8k", 8000, a["test_audio_8k"]), ("leak_test_8k", 8000, a["leak_test"]),
           ("goforward", 16000, a["goforward"]), ("numbers", 16000, a["numbers"]), ("libri", 16000, a["libri_0870"]),
           ("goforward_32k", 32000, V.upsample2(a["goforward"])), ("numbers_11025", 11025, a["test_audio_8k"]),
           ("numbers_22050", 22050, a["numbers"])]
    for r in (8000, 16000, 32000):
        out.append(("synthetic_%d" % r, r, V.synthetic(r, seed=r)))
    return out


@pytest.mark.parametrize("fl", [0.01, 0.02, 0.03])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_flags_and_state_after_every_frame(mode, fl):
    for name, rate, pcm in _cases():
        want_f, want_s = V.ref_flags(mode, rate, fl, pcm, states=True)
        got_f, got_s = _emul_run(mode, rate, fl, pcm)
        assert np.array_equal(got_f, want_f), (name, mode, fl)
        bad = np.nonzero((got_s != want_s).any(axis=1))[0]
        assert len(bad) == 0, (name, mode, fl, "first differing frame", bad[:1])
        assert want_f.any() or name.startswith("synthetic"), name


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_initial_state_and_thresholds(mode):
    """ps_vad_init's struct before any frame: the emulation's initial state, byte for byte (the reference's
    state is read after one frame of digital silence, which changes only what a below-energy frame changes)."""
    want_f, want_s = V.ref_flags(mode, 8000, 0.01, np.zeros(80, np.int16), states=True)
    init = np.zeros(V.STATE_BYTES, np.uint8)
    V.emul().vad_emul_init_state(mode, V._p(init))
    assert want_f[0] == 0
    # a silent frame leaves everything but `vad` (now 0) where ps_vad_init put it
    got = init.copy()
    got[0:4] = 0
    assert np.array_equal(got, want_s[0])


@pytest.mark.parametrize("rate,fl", [(8000, 0.01), (16000, 0.01), (16000, 0.03), (32000, 0.02)])
def test_chunked_features_with_repairs_equal_sequential(rate, fl):
    a = V.audio()
    pcm = {8000: a["leak_test"], 16000: np.concatenate([a["numbers"], a["goforward"]]),
           32000: V.upsample2(a["libri_0880"])}[rate]
    fs, _ = V.ref_params(0, rate, fl)
    nf = len(pcm) // fs
    L = V.emul()
    ref = np.zeros((nf, 8), np.int16)
    passes = C.c_int()
    L.vad_emul_features(rate, fs, V._p(pcm), nf, nf + 1, 0, V._p(ref), C.byref(passes))   # one chunk: the sequential run
    default = int(np.ceil(0.5 / (fs / rate) - 1e-9))       # psb_vad_create's default warm-up: 0.5 s of audio
    for chunk in (7, 16, 64):
        assert nf % chunk != 0 or chunk == 16
        for warmup in (0, 1, 2, default):
            got = np.zeros((nf, 8), np.int16)
            rep = L.vad_emul_features(rate, fs, V._p(pcm), nf, chunk, warmup, V._p(got), C.byref(passes))
            assert np.array_equal(got, ref), (chunk, warmup, rep)
            assert passes.value >= 1 and (rep == 0) == (passes.value == 1), (rep, passes.value)
            if warmup == 0:
                assert rep > 0, chunk
            print("rate %d frame %.2f chunk %d warmup %d: %d recomputations in %d passes (%d chunks)"
                  % (rate, fl, chunk, warmup, rep, passes.value, -(-nf // chunk)))


def _emul_segments(pcm, mode, rate, fl, window, ratio):
    fs, sr = V.ref_params(mode, rate, fl)
    closest = V.closest_rate(rate)
    maxlen, sf, ef = V.ep_params(window, ratio, fs, sr)
    nf = len(pcm) // fs
    feat = np.zeros((max(nf, 1), 8), np.int16)
    L = V.emul()
    L.vad_emul_features(closest, fs, V._p(pcm), nf, max(nf, 1), 0, V._p(feat), C.byref(C.c_int()))
    flags = np.zeros(max(nf, 1), np.int8)
    segs = np.zeros((nf + 1, 2), np.int64)
    times = np.zeros((nf + 1, 2), np.float64)
    n = L.vad_emul_segments(mode, closest, fs, sr, maxlen, sf, ef, V._p(feat), nf, len(pcm) - nf * fs, V._p(flags),
                            V._p(segs), V._p(times))
    return [(float(times[i, 0]), float(times[i, 1]), int(segs[i, 0]), int(segs[i, 1])) for i in range(n)]


def _speech_stream(rate):
    a = V.audio()
    sil = np.zeros(rate // 2, np.int16)
    if rate == 8000:
        return np.concatenate([sil, a["test_audio_8k"], sil, a["leak_test"]])
    s = np.concatenate([sil, a["goforward"], sil, a["numbers"], sil, a["libri_0880"]])
    return V.upsample2(s) if rate == 32000 else s


@pytest.mark.parametrize("mode,rate,fl,window,ratio", [
    (0, 16000, 0.03, 0.3, 0.9), (3, 16000, 0.01, 0.3, 0.9), (1, 8000, 0.02, 0.5, 0.7), (2, 32000, 0.03, 0.3, 0.9),
    (0, 16000, 0.03, 0.3, 0.3), (0, 16000, 0.01, 0.3, 0.3), (0, 22050, 0.03, 0.3, 0.9)])
def test_endpointer_segments_and_times(mode, rate, fl, window, ratio):
    pcm = _speech_stream(V.closest_rate(rate))
    fs, _ = V.ref_params(mode, rate, fl)
    cuts = [0, 1, fs - 1, fs, 5 * fs, 37 * fs + 11, len(pcm) // 2, len(pcm) // fs * fs, len(pcm)]
    for n in cuts:
        want = V.ref_segments(pcm[:n], mode, rate, fl, window, ratio)
        assert want is not None
        got = _emul_segments(pcm[:n], mode, rate, fl, window, ratio)
        assert got == want, (n, got[:3], want[:3])
    assert len(V.ref_segments(pcm, mode, rate, fl, window, ratio)) > 0


def test_stream_that_ends_in_speech_keeps_its_trailing_samples():
    a = V.audio()
    pcm = np.concatenate([np.zeros(8000, np.int16), a["numbers"][:40000]])
    pcm = pcm[:len(pcm) // 480 * 480 + 123]
    want = V.ref_segments(pcm)
    assert want[-1][3] == len(pcm)                    # the last segment runs to the end, partial frame included
    assert _emul_segments(pcm, 0, 16000, 0.03, 0.3, 0.9) == want


@pytest.mark.parametrize("rate,fl,window,ratio", [(42, 0.03, 0.3, 0.9), (96000, 0.03, 0.3, 0.9), (16000, 0.03, 0.3, 0.99),
                                                  (16000, 0.03, 0.03, 0.1), (16000, 0.025, 0.3, 0.9),
                                                  (16000, 0.04, 0.3, 0.9)])
def test_refused_settings(rate, fl, window, ratio):
    """What ps_endpointer_init refuses (test/unit/test_endpointer.c) the device API refuses too (tests/test_gpu_vad.py
    checks the device side); here the reference's own refusals are pinned."""
    assert V.ref_segments(np.zeros(1000, np.int16), 0, rate, fl, window, ratio) is None
