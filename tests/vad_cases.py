"""Shared by the VAD tests: the audio fixtures (tests/golden/vad_audio.npz: the reference's test
recordings, data only), synthetic signals, and two small libraries built on first use --
tests/emul/vad_emul.cpp (psb_vad_core.h for the host) and tests/emul/vad_refdrv.c (whole-stream
loops over the compiled reference's ps_vad_* / ps_endpointer_*, linked against oracle/_ref/libpsref.so)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
STATE_BYTES = 736                                   # sizeof(VadInstT)
_libs = {}


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _build(name, cmd_tail, src, compiler):
    if name not in _libs:
        out = os.path.join(tempfile.mkdtemp(prefix="psbvad"), "lib%s.so" % name)
        subprocess.check_call([compiler, "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-o", out,
                               os.path.join(ROOT, "tests", "emul", src)] + cmd_tail)
        _libs[name] = C.CDLL(out)
    return _libs[name]


def emul():
    L = _build("vademul", [], "vad_emul.cpp", "g++")
    L.vad_emul_run.restype = L.vad_emul_features.restype = L.vad_emul_segments.restype = C.c_long
    L.vad_emul_run.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_long, C.c_void_p, C.c_void_p]
    L.vad_emul_features.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.vad_emul_segments.argtypes = [C.c_int] * 7 + [C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.vad_emul_init_state.argtypes = [C.c_int, C.c_void_p]
    return L


def ref_available():
    return os.path.exists(os.path.join(REF_DIR, "libpsref.so"))


def ref():
    L = _build("vadref", ["-L" + REF_DIR, "-lpsref", "-Wl,-rpath," + REF_DIR], "vad_refdrv.c", "gcc")
    L.refdrv_vad_params.argtypes = [C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
    L.refdrv_vad_run.restype = C.c_long
    L.refdrv_vad_run.argtypes = [C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_long, C.c_void_p, C.c_void_p, C.c_long]
    L.refdrv_endpoint_run.restype = C.c_long
    L.refdrv_endpoint_run.argtypes = [C.c_double, C.c_double, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_long,
                                      C.c_void_p, C.c_void_p, C.c_long]
    return L


def audio():
    from conftest import golden
    return golden("vad_audio.npz")


def upsample2(x):
    """Any int16 signal is a valid input: a 2x linear interpolation, to make 32 kHz audio of the 16 kHz fixtures."""
    x = x.astype(np.int32)
    y = np.empty(2 * len(x), np.int32)
    y[0::2] = x
    y[1::2] = (x + np.concatenate([x[1:], x[-1:]])) // 2
    return y.astype(np.int16)


def synthetic(rate, seconds=3.0, seed=0):
    """Digital silence, DC, full-scale square waves, clipped and wrapped sine, white noise at several levels."""
    rng = np.random.default_rng(seed)
    n = int(rate * seconds / 6)
    t = np.arange(n)
    sq = np.where((t // max(1, rate // 440)) % 2 == 0, 32767, -32768)
    sine = 60000.0 * np.sin(2 * np.pi * 300.0 * t / rate)
    parts = [np.zeros(n), np.full(n, 12000.0), sq, np.clip(sine, -32768, 32767),
             (sine.astype(np.int64) & 0xFFFF).astype(np.uint16).view(np.int16).astype(np.float64),
             np.concatenate([rng.normal(0, s, n // 4) for s in (3, 100, 3000, 30000)])]
    return np.concatenate([np.clip(p, -32768, 32767).astype(np.int16) for p in parts])


def ref_params(mode, rate, fl):
    fs, sr = C.c_int(), C.c_int()
    if ref().refdrv_vad_params(mode, rate, fl, C.byref(fs), C.byref(sr)) < 0:
        return None
    return fs.value, sr.value


def ref_flags(mode, rate, fl, pcm, states=False):
    pcm = np.ascontiguousarray(pcm, np.int16)
    fs, _ = ref_params(mode, rate, fl)
    nf = len(pcm) // fs
    flags = np.zeros(max(nf, 1), np.int8)
    st = np.zeros((max(nf, 1), STATE_BYTES), np.uint8) if states else None
    n = ref().refdrv_vad_run(mode, rate, fl, _p(pcm), len(pcm), _p(flags), _p(st) if states else None, STATE_BYTES)
    assert n == nf
    return (flags[:nf], st[:nf]) if states else flags[:nf]


def ref_segments(pcm, mode=0, rate=16000, fl=0.03, window=0.3, ratio=0.9):
    """[(start_time, end_time, start_sample, end_sample)] of the reference endpointer, or None if it refuses."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    cap = len(pcm) // 80 + 2
    segs = np.zeros((cap, 2), np.int64)
    times = np.zeros((cap, 2), np.float64)
    n = ref().refdrv_endpoint_run(window, ratio, mode, rate, fl, _p(pcm), len(pcm), _p(segs), _p(times), cap)
    if n == -1:
        return None
    assert n >= 0, "reference endpointer driver error %d" % n
    return [(float(times[i, 0]), float(times[i, 1]), int(segs[i, 0]), int(segs[i, 1])) for i in range(n)]


def closest_rate(rate):
    best, out = 0.5, 0
    for r in (8000, 16000, 32000, 48000):
        d = abs(1.0 - r / rate)
        if d < best:
            best, out = d, r
    return out


def ep_params(window, ratio, frame_size, rate):
    fl = frame_size / rate
    maxlen = int(window / fl + 0.5)
    return maxlen, int(ratio * maxlen), int((1.0 - ratio) * maxlen + 0.5)


def ref_session_segments(hmm, lm, dic, utterances):
    """One reference ps_decoder_t (-bestpath no) over several utterances in order, as fe_sessions.ref_session_decode
    runs it, with each utterance's hypothesis, best score and ps_seg_iter word segments [(word, sf, ef)]."""
    import fe_sessions
    L = fe_sessions.ref_lib()
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
    params = {}
    for line in open(os.path.join(hmm, "feat.params")):
        parts = line.split()
        if len(parts) == 2:
            params[parts[0].lstrip("-")] = parts[1]
    params["bestpath"] = "no"                    # ps_init parses feat.params after the caller's settings
    out = []
    with tempfile.TemporaryDirectory() as tmp:
        fp = os.path.join(tmp, "feat.params")
        with open(fp, "w") as f:
            f.write("".join("-%s %s\n" % kv for kv in params.items()))
        cfg = L.ps_config_init(None)
        for k, v in (("hmm", hmm), ("lm", lm), ("dict", dic), ("featparams", fp)):
            L.ps_config_set_str(cfg, k.encode(), v.encode())
        ps = L.ps_init(cfg)
        assert ps, "ps_init failed"
        for pcm in utterances:
            pcm = np.ascontiguousarray(pcm, np.int16)
            L.ps_start_stream(ps)
            L.ps_start_utt(ps)
            L.ps_process_raw(ps, pcm.ctypes.data, len(pcm), 0, 1)
            L.ps_end_utt(ps)
            score = C.c_int32()
            h = L.ps_get_hyp(ps, C.byref(score))
            segs, it = [], L.ps_seg_iter(ps)
            while it:
                sf, ef = C.c_int(), C.c_int()
                L.ps_seg_frames(it, C.byref(sf), C.byref(ef))
                segs.append((L.ps_seg_word(it).decode(), sf.value, ef.value))
                it = L.ps_seg_next(it)
            out.append(dict(hyp=h.decode() if h else "", score=score.value, seg=segs))
        L.ps_free(ps)
        L.ps_config_free(cfg)
    return out
