"""Shared by the live endpointing tests: the compiled reference fed in chunks (tests/emul/vad_live_refdrv.c), the host
emulation of one live slot (tests/emul/vad_live_emul.cpp), random chunkings of a stream, and the per-call result
comparison.  Each feed returns the dict api.LiveEndpointer.feed gives for one slot."""
import ctypes as C

import numpy as np

import vad_cases as V


def _ref_lib():
    L = V._build("vadliveref", ["-L" + V.REF_DIR, "-lpsref", "-Wl,-rpath," + V.REF_DIR], "vad_live_refdrv.c", "gcc")
    L.refdrv_live_open.restype = C.c_void_p
    L.refdrv_live_open.argtypes = [C.c_double, C.c_double, C.c_int, C.c_int, C.c_double, C.c_int]
    L.refdrv_live_free.argtypes = L.refdrv_live_reset.argtypes = [C.c_void_p]
    L.refdrv_live_feed.restype = C.c_long
    L.refdrv_live_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long,
                                   C.c_void_p, C.c_void_p]
    return L


def _emul_lib():
    L = V._build("vadliveemul", [], "vad_live_emul.cpp", "g++")
    L.vad_live_emul_open.restype = C.c_void_p
    L.vad_live_emul_open.argtypes = [C.c_int] * 8
    L.vad_live_emul_free.argtypes = L.vad_live_emul_reset.argtypes = [C.c_void_p]
    L.vad_live_emul_feed.restype = C.c_long
    L.vad_live_emul_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p]
    return L


class _Stream:
    def __init__(self, mode, rate, fl, window, ratio):
        self.fs, self.sr = V.ref_params(mode, rate, fl)
        self.maxlen, self.sf, self.ef = V.ep_params(window, ratio, self.fs, self.sr)
        self.frames = 0

    def feed(self, chunk, final=False):
        chunk = np.ascontiguousarray(chunk, np.int16)
        cap = (len(chunk) + self.fs - 1) // self.fs + 1
        flags = np.zeros(cap, np.int8)
        segs = np.zeros((cap, 2), np.int64)
        times = np.zeros((cap, 2), np.float64)
        status = np.zeros(3, np.int64)
        st_times = np.zeros(2, np.float64)
        k = self._feed(chunk, int(bool(final)), flags, segs, times, cap, status, st_times)
        assert k >= 0, "live driver error %d" % k
        nf = int(status[2]) - self.frames
        self.frames = int(status[2])
        return dict(flags=flags[:nf].copy(),
                    segments=[(float(times[i, 0]), float(times[i, 1]), int(segs[i, 0]), int(segs[i, 1])) for i in range(k)],
                    in_speech=bool(status[0]), speech_start=float(st_times[0]), speech_end=float(st_times[1]),
                    start_sample=int(status[1]), frames=int(status[2]))


class RefStream(_Stream):
    """One reference ps_endpointer_t fed live."""

    def __init__(self, mode=0, rate=16000, fl=0.03, window=0.3, ratio=0.9):
        super().__init__(mode, rate, fl, window, ratio)
        self.L = _ref_lib()
        self.h = self.L.refdrv_live_open(window, ratio, mode, rate, fl, self.maxlen)
        assert self.h

    def _feed(self, chunk, final, flags, segs, times, cap, status, st_times):
        return self.L.refdrv_live_feed(self.h, V._p(chunk), len(chunk), final, V._p(flags), V._p(segs), V._p(times), cap,
                                       V._p(status), V._p(st_times))

    def reset(self):
        assert self.L.refdrv_live_reset(self.h) == 0
        self.frames = 0

    def close(self):
        self.L.refdrv_live_free(self.h)


class EmulStream(_Stream):
    """One live slot of psb_vad_feed_* restated on the host, saved and restored between calls."""

    def __init__(self, mode=0, rate=16000, fl=0.03, window=0.3, ratio=0.9, warmup=0):
        super().__init__(mode, rate, fl, window, ratio)
        self.L = _emul_lib()
        self.h = self.L.vad_live_emul_open(mode, V.closest_rate(rate), self.fs, self.sr, self.maxlen, self.sf, self.ef, warmup)

    def _feed(self, chunk, final, flags, segs, times, cap, status, st_times):
        return self.L.vad_live_emul_feed(self.h, V._p(chunk), len(chunk), final, V._p(flags), V._p(segs), V._p(times),
                                         V._p(status), V._p(st_times))

    def reset(self):
        self.L.vad_live_emul_reset(self.h)
        self.frames = 0

    def close(self):
        self.L.vad_live_emul_free(self.h)


def same(a, b):
    """Two per-call results equal, flags element for element and times bit for bit."""
    return (np.array_equal(a["flags"], b["flags"]) and a["segments"] == b["segments"]
            and all(a[k] == b[k] for k in ("in_speech", "speech_start", "speech_end", "start_sample", "frames")))


def chunking(rng, total, fs, rate, finals=0.0):
    """[(length, final)] covering `total` samples: single samples, empty chunks, cuts inside a frame, exactly one frame,
    64 frames, 64 frames + 1 sample and + 1 frame, up to a minute; a chunk is final with probability `finals`, and the
    last chunk always is."""
    out, pos = [], 0
    while pos < total:
        kind = int(rng.integers(10))
        if kind == 0:
            run = [1] * int(rng.integers(1, 2 * fs))            # a burst of single samples across a frame boundary
        else:
            n = [0, int(rng.integers(1, fs)), fs, 64 * fs, 64 * fs + 1, 65 * fs, int(rng.integers(fs, 3 * rate)),
                 60 * rate, int(rng.integers(1, rate // 5))][kind - 1]
            run = [n]
        for n in run:
            n = min(n, total - pos)
            pos += n
            out.append((n, bool(rng.random() < finals)))
            if pos >= total:
                break
    if out:
        out[-1] = (out[-1][0], True)
    else:
        out.append((0, True))
    return out
