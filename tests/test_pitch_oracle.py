"""CPU: the YIN pitch tracker's arithmetic and read schedule (pocketsphinx_b200/csrc/psb_pitch_core.h, built for the
host by tests/emul/pitch_emul.cpp) against the compiled reference: every (period, bestdiff) of extract_pitch's loop
over yin_* equal, and api.pitch_lines equal to the output file of the compiled pocketsphinx_pitch byte for byte."""
import numpy as np
import pytest

import pitch_cases as P
from pocketsphinx_b200 import api

pytestmark = pytest.mark.skipif(not P.ref_available(), reason="compiled reference (oracle/_ref) not built")


def _check(pcm, rate, lines=False, **opts):
    want = P.ref_run(pcm, rate, **opts)
    got = P.emul_run(pcm, rate, **opts)
    assert np.array_equal(got[0], want[0]), ("period", rate, opts)
    assert np.array_equal(got[1], want[1]), ("bestdiff", rate, opts)
    assert got[2] == want[2], ("main-loop reads", rate, opts)
    fl, fs = P.samples(rate, opts.get("flen", 0.025)), P.samples(rate, opts.get("fshift", 0.01))
    nf = 1 + (len(pcm) - fl) // fs if len(pcm) >= fl else 0
    assert api.pitch_main_reads(nf, opts.get("smooth_window", 2)) == want[2]
    if lines:
        res = api.pitch_result(got[0], got[1], got[2], fs, rate)
        text = "".join(api.pitch_lines(res, rate)).encode()
        assert text == P.program_output(pcm, rate, **opts), (rate, opts)
    return want


@pytest.mark.parametrize("rate", P.RATES)
def test_signals_at_every_rate(rate):
    for name, pcm in P.signals(rate).items():
        _check(pcm, rate, lines=True)
    for name in ("goforward.raw", "dhd.2934z.raw"):
        _check(P.recording(name), rate, lines=rate == 16000)


def test_square_waves_wrap_the_squared_difference():
    """Full-scale squares make diff * diff pass 2^31: the wrapped products must still match."""
    pcm = P.signals(16000)["alternating"]
    assert np.abs(pcm[1:].astype(np.int64) - pcm[:-1]).max() > 46340
    _check(pcm, 16000, lines=True)


@pytest.mark.parametrize("smooth_window", P.SMOOTH)
def test_smoothing_windows_and_thresholds(smooth_window):
    sig = P.signals(16000, seconds=0.6)
    cases = [sig["chirp"], sig["square"], sig["noise"], P.recording("goforward.raw")[:16000]]
    for thr in P.THRESH:
        for pcm in cases:
            _check(pcm, 16000, lines=True, smooth_window=smooth_window, voice_thresh=thr)
    _check(sig["chirp"], 16000, lines=True, smooth_window=smooth_window, search_range=0.9)


@pytest.mark.parametrize("smooth_window", [0, 1, 2, 5])
@pytest.mark.parametrize("rate", [8000, 44100])
def test_stream_lengths_at_the_framing_edges(rate, smooth_window):
    base = P.signals(rate, seconds=0.2)["chirp"]
    for n in P.length_cases(rate):
        _check(base[:n], rate, lines=True, smooth_window=smooth_window)


def test_one_and_two_frame_streams_read_never_written_slots():
    """A one-frame stream with smooth_window 2 prints period 0 and bestdiff 32768 (the unwritten slots' zeros)."""
    pcm = P.signals(16000)["chirp"]
    fl, fs = P.samples(16000, 0.025), P.samples(16000, 0.01)
    per, bd, main = _check(pcm[:fl], 16000, lines=True)
    assert main == 0 and list(per) == [0] and list(bd) == [32768]
    for sw in (1, 2, 5, 127):
        _check(pcm[:fl + fs], 16000, lines=True, smooth_window=sw)


@pytest.mark.parametrize("n,crossings", [(70000, 1), (140000, 2)])
def test_frame_counter_wrap(n, crossings):
    """The uint16 frame counter: 70 000 samples at flen 8 / fshift 1 are 69 993 frames but 69 988 reads."""
    pcm = P.signals(16000, seconds=n / 16000.0)["chirp"][:n]
    per, _, main = _check(pcm, 16000, lines=True, **P.WRAP_OPTS)
    nf = n - 8 + 1
    assert nf // 65536 == crossings
    if n == 70000:
        assert len(per) == 69988
    _check(pcm, 16000, smooth_window=5, **P.WRAP_OPTS)
    _check(pcm, 16000, smooth_window=0, **P.WRAP_OPTS)
