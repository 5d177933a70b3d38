"""Shared by the pitch tests: signals, the options grid, and two small libraries built on first use --
tests/emul/pitch_emul.cpp (psb_pitch_core.h for the host) and tests/emul/pitch_refdrv.c (extract_pitch's loop over
the compiled reference's yin_*, linked against oracle/_ref/libpsref.so) -- and a runner for the compiled
reference program oracle/_ref/pocketsphinx_pitch."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
PITCH_BIN = os.path.join(REF_DIR, "pocketsphinx_pitch")
RATES = (8000, 16000, 44100, 48000)
SMOOTH = (0, 1, 2, 5, 127)
THRESH = (0.0, 0.1, 1.0, 1.5)
_libs = {}


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _build(name, cmd_tail, src, compiler):
    if name not in _libs:
        out = os.path.join(tempfile.mkdtemp(prefix="psbpitch"), "lib%s.so" % name)
        subprocess.check_call([compiler, "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-o", out,
                               os.path.join(ROOT, "tests", "emul", src)] + cmd_tail)
        _libs[name] = C.CDLL(out)
    return _libs[name]


def ref_available():
    return os.path.exists(os.path.join(REF_DIR, "libpsref.so")) and os.path.exists(PITCH_BIN)


def samples(rate, seconds):
    return int(0.5 + rate * seconds)          # (size_t)(0.5 + sps * seconds), as the program sizes flen / fshift


def q15(v):
    return int(np.uint16(np.float32(v) * np.float32(32768)))


def emul_run(pcm, rate, flen=0.025, fshift=0.01, smooth_window=2, voice_thresh=0.1, search_range=0.2):
    """(period, bestdiff, main-loop reads) of the host restatement."""
    L = _build("pitchemul", [], "pitch_emul.cpp", "g++")
    L.pitch_emul_run.restype = C.c_long
    L.pitch_emul_run.argtypes = [C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                 C.c_void_p, C.c_void_p]
    pcm = np.ascontiguousarray(pcm, np.int16)
    fl, fs = samples(rate, flen), samples(rate, fshift)
    cap = max(len(pcm), 1)
    period, bestdiff, n_main = np.zeros(cap, np.uint16), np.zeros(cap, np.uint16), C.c_long()
    k = L.pitch_emul_run(_p(pcm), len(pcm), fl, fs, q15(voice_thresh), q15(search_range), smooth_window, _p(period),
                         _p(bestdiff), C.byref(n_main))
    return period[:k], bestdiff[:k], n_main.value


def ref_run(pcm, rate, flen=0.025, fshift=0.01, smooth_window=2, voice_thresh=0.1, search_range=0.2):
    """(period, bestdiff, main-loop reads) of the compiled reference's yin_* in extract_pitch's loop."""
    L = _build("pitchref", ["-L" + REF_DIR, "-lpsref", "-Wl,-rpath," + REF_DIR], "pitch_refdrv.c", "gcc")
    L.refdrv_pitch_run.restype = C.c_long
    L.refdrv_pitch_run.argtypes = [C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_void_p,
                                   C.c_void_p, C.c_void_p]
    pcm = np.ascontiguousarray(pcm, np.int16)
    fl, fs = samples(rate, flen), samples(rate, fshift)
    cap = max(len(pcm), 1)
    period, bestdiff, n_main = np.zeros(cap, np.uint16), np.zeros(cap, np.uint16), C.c_long()
    k = L.refdrv_pitch_run(_p(pcm), len(pcm), fl, fs, voice_thresh, search_range, smooth_window, _p(period),
                           _p(bestdiff), C.byref(n_main))
    return period[:k], bestdiff[:k], n_main.value


def program_output(pcm, rate, flen=0.025, fshift=0.01, smooth_window=2, voice_thresh=0.1, search_range=0.2):
    """The bytes `pocketsphinx_pitch -raw yes` writes for pcm (little-endian int16)."""
    d = tempfile.mkdtemp(prefix="psbpitchrun")
    src, out = os.path.join(d, "in.raw"), os.path.join(d, "out.txt")
    np.ascontiguousarray(pcm, "<i2").tofile(src)
    subprocess.run([PITCH_BIN, "-raw", "yes", "-samprate", str(rate), "-flen", repr(float(flen)),
                    "-fshift", repr(float(fshift)), "-smooth_window", str(smooth_window),
                    "-voice_thresh", repr(float(voice_thresh)), "-search_range", repr(float(search_range)),
                    "-i", src, "-o", out], check=True, capture_output=True)
    with open(out, "rb") as f:
        return f.read()


def recording(name):
    return np.fromfile(os.path.join(REF_DIR, "data", name), "<i2")


def signals(rate, seconds=0.3, seed=0):
    """Synthetic signals at `rate`: silence, DC, full-scale and alternating squares and clipped sines (their squared
    differences wrap in int), noise, a 60 -> 500 Hz chirp."""
    n = samples(rate, seconds)
    t = np.arange(n) / rate
    rng = np.random.default_rng(seed + rate)
    sq = np.where(np.sin(2 * np.pi * 110 * t) >= 0, 32767, -32768)
    alt = np.where(np.arange(n) % 2 == 0, 32767, -32768)
    clip = np.clip(4 * 32767 * np.sin(2 * np.pi * 180 * t), -32768, 32767)
    noise = np.clip(rng.normal(0, 6000, n), -32768, 32767)
    phase = 2 * np.pi * (60 * t + (500 - 60) / (2 * seconds) * t * t)
    chirp = 12000 * np.sin(phase)
    out = dict(silence=np.zeros(n), dc=np.full(n, 1234.0), square=sq, alternating=alt, clipped_sine=clip,
               noise=noise, chirp=chirp)
    return {k: np.asarray(v).astype(np.int16) for k, v in out.items()}


def length_cases(rate, flen=0.025, fshift=0.01):
    """Stream lengths around the framing edges: 0, flen - 1, flen, flen + k * fshift - 1 / + 1."""
    fl, fs = samples(rate, flen), samples(rate, fshift)
    out = [0, fl - 1, fl]
    for k in (1, 2, 3, 7):
        out += [fl + k * fs - 1, fl + k * fs, fl + k * fs + 1]
    return out


# flen 8 and fshift 1 at 16 kHz: every sample starts a frame, so the uint16 frame counter wraps cheaply
WRAP_OPTS = dict(flen=0.0005, fshift=0.0000625)
