"""Shared by the live pitch tests: the compiled reference's yin_* fed in chunks (tests/emul/pitch_live_refdrv.c), the
host restatement of one live slot (tests/emul/pitch_live_emul.cpp), random chunkings of a stream, and the per-call
result comparison.  Each feed returns the dict api.LivePitchTracker.feed gives for one slot."""
import ctypes as C

import numpy as np

import pitch_cases as P
from pocketsphinx_b200 import api


def _ref_lib():
    L = P._build("pitchliveref", ["-L" + P.REF_DIR, "-lpsref", "-Wl,-rpath," + P.REF_DIR], "pitch_live_refdrv.c", "gcc")
    L.refdrv_pitch_live_open.restype = C.c_void_p
    L.refdrv_pitch_live_open.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_int]
    L.refdrv_pitch_live_free.argtypes = L.refdrv_pitch_live_reset.argtypes = [C.c_void_p]
    L.refdrv_pitch_live_feed.restype = C.c_long
    L.refdrv_pitch_live_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _emul_lib():
    L = P._build("pitchliveemul", [], "pitch_live_emul.cpp", "g++")
    L.pitch_live_emul_open.restype = C.c_void_p
    L.pitch_live_emul_open.argtypes = [C.c_int] * 5
    L.pitch_live_emul_free.argtypes = L.pitch_live_emul_reset.argtypes = [C.c_void_p]
    L.pitch_live_emul_feed.restype = C.c_long
    L.pitch_live_emul_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


class _Stream:
    def __init__(self, rate, flen, fshift, smooth_window):
        self.rate, self.sw = rate, smooth_window
        self.fl, self.fs = P.samples(rate, flen), P.samples(rate, fshift)

    def feed(self, chunk, final=False):
        chunk = np.ascontiguousarray(chunk, np.int16)
        cap = -(-len(chunk) // self.fs) + 2 * self.sw + 1
        period, bestdiff = np.zeros(cap, np.uint16), np.zeros(cap, np.uint16)
        status = np.zeros(1, api.PITCH_LIVE_STATUS)
        k = self._feed(chunk, int(bool(final)), period, bestdiff, status)
        assert k >= 0, "live driver refused the feed"
        assert k <= cap - 1
        return api.pitch_live_result(period[:k].copy(), bestdiff[:k].copy(), status[0], self.fs, self.rate)


class RefStream(_Stream):
    """One reference yin_t fed live."""

    def __init__(self, rate=16000, flen=0.025, fshift=0.01, smooth_window=2, voice_thresh=0.1, search_range=0.2):
        super().__init__(rate, flen, fshift, smooth_window)
        self.L = _ref_lib()
        self.h = self.L.refdrv_pitch_live_open(self.fl, self.fs, voice_thresh, search_range, smooth_window)

    def _feed(self, chunk, final, period, bestdiff, status):
        return self.L.refdrv_pitch_live_feed(self.h, P._p(chunk), len(chunk), final, P._p(period), P._p(bestdiff),
                                             P._p(status))

    def reset(self):
        self.L.refdrv_pitch_live_reset(self.h)

    def close(self):
        self.L.refdrv_pitch_live_free(self.h)


class EmulStream(_Stream):
    """One live slot of psb_pitch_feed_* restated on the host, saved and restored between calls."""

    def __init__(self, rate=16000, flen=0.025, fshift=0.01, smooth_window=2, voice_thresh=0.1, search_range=0.2):
        super().__init__(rate, flen, fshift, smooth_window)
        self.L = _emul_lib()
        self.h = self.L.pitch_live_emul_open(self.fl, self.fs, P.q15(voice_thresh), P.q15(search_range), smooth_window)

    def _feed(self, chunk, final, period, bestdiff, status):
        return self.L.pitch_live_emul_feed(self.h, P._p(chunk), len(chunk), final, P._p(period), P._p(bestdiff),
                                           P._p(status))

    def reset(self):
        self.L.pitch_live_emul_reset(self.h)

    def close(self):
        self.L.pitch_live_emul_free(self.h)


KEYS = ("frames", "main_reads", "ended")


def same(a, b):
    """Two per-call results equal: period and bestdiff element for element, times bit for bit, the slot's counts."""
    return (np.array_equal(a["period"], b["period"]) and np.array_equal(a["bestdiff"], b["bestdiff"])
            and a["time"].tobytes() == b["time"].tobytes() and all(a[k] == b[k] for k in KEYS))


def join(results):
    """A slot's per-call results joined: the whole stream's period, bestdiff and time."""
    cat = lambda k, t: np.concatenate([r[k] for r in results]) if results else np.zeros(0, t)
    return cat("period", np.uint16), cat("bestdiff", np.uint16), cat("time", np.float64)


def lines(results, rate):
    """pitch_lines over a slot's calls, joined: the program's output file."""
    return "".join("".join(api.pitch_lines(r, rate)) for r in results).encode()


def chunking(rng, total, fl, fs, rate):
    """[lengths] covering `total` samples: single samples, empty chunks, cuts inside a frame, exactly fshift and flen,
    runs of chunks shorter than one frame, and chunks longer than a 255-frame window."""
    out, pos = [], 0
    while pos < total:
        kind = int(rng.integers(9))
        if kind == 0:
            run = [1] * int(rng.integers(1, 2 * fl))            # a burst of single samples across frame boundaries
        elif kind == 1:
            run = [int(rng.integers(1, fs + 1)) for _ in range(int(rng.integers(2, 40)))]   # short chunks, many calls
        else:
            run = [[0, int(rng.integers(1, fl)), fs, fl, fl + 1, 300 * fs + fl, int(rng.integers(fl, rate)),
                    ][kind - 2]]
        for n in run:
            n = min(n, total - pos)
            pos += n
            out.append(n)
            if pos >= total:
                break
    return out


def whole(pcm, rate, **opts):
    """The whole-stream restatement's result for pcm, as pitch_result gives it."""
    per, bd, main = P.emul_run(pcm, rate, **opts)
    return api.pitch_result(per, bd, main, P.samples(rate, opts.get("fshift", 0.01)), rate)
