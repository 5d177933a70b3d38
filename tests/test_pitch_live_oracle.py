"""CPU: live pitch tracking.  The compiled reference's yin_t fed in chunks with extract_pitch's buffering
(tests/emul/pitch_live_refdrv.c) against the host restatement of one live slot (tests/emul/pitch_live_emul.cpp, the
save / restore psb_pitch_feed_* does): every call's reads and counts equal, and every slot's joined reads equal to the
whole-stream restatement (tests/emul/pitch_emul.cpp), over chunkings, smoothing windows, rates, the uint16 frame
counter's wrap, short and empty final calls and resets."""
import numpy as np
import pytest

import pitch_cases as P
import pitch_live_cases as L

pytestmark = pytest.mark.skipif(not P.ref_available(), reason="compiled reference (oracle/_ref) not built")


def _run(pcm, rate, cuts, program=False, **opts):
    """Feeds pcm cut into `cuts` (lengths summing to len(pcm)), the last call final, to both drivers."""
    assert sum(cuts) == len(pcm)
    ref, emu = L.RefStream(rate, **opts), L.EmulStream(rate, **opts)
    got = []
    try:
        pos = 0
        for i, n in enumerate(cuts):
            fin = i == len(cuts) - 1
            a, b = ref.feed(pcm[pos:pos + n], fin), emu.feed(pcm[pos:pos + n], fin)
            assert L.same(a, b), (rate, opts, i, n)
            got.append(b)
            pos += n
    finally:
        ref.close(), emu.close()
    per, bd, tm = L.join(got)
    want = L.whole(pcm, rate, **opts)
    assert np.array_equal(per, want["period"]) and np.array_equal(bd, want["bestdiff"]), (rate, opts)
    assert tm.tobytes() == want["time"].tobytes(), (rate, opts)
    if program:
        assert L.lines(got, rate) == P.program_output(pcm, rate, **opts), (rate, opts)
    return got


def _random_cuts(rng, n, rate, **opts):
    fl, fs = P.samples(rate, opts.get("flen", 0.025)), P.samples(rate, opts.get("fshift", 0.01))
    cuts = L.chunking(rng, n, fl, fs, rate)
    return cuts + [0] if not cuts else cuts


def test_chunkings_of_a_recording():
    rng = np.random.default_rng(1)
    pcm = P.recording("goforward.raw")
    fl, fs = 400, 160
    for cuts in ([len(pcm)], [1] * 5000 + [len(pcm) - 5000], [fs] * (len(pcm) // fs) + [len(pcm) % fs],
                 [fl] * (len(pcm) // fl) + [len(pcm) % fl], [0, 0, 399, 1, 0, 160, 241, len(pcm) - 801, 0]):
        _run(pcm, 16000, cuts, program=True)
    for _ in range(4):
        _run(pcm, 16000, _random_cuts(rng, len(pcm), 16000), program=True)


@pytest.mark.parametrize("smooth_window", [0, 1, 2, 127])
def test_smoothing_windows(smooth_window):
    """With 127 (wsize 255) most calls feed fewer frames than the window spans: the ring carries rows across calls."""
    rng = np.random.default_rng(10 + smooth_window)
    sig = P.signals(16000, seconds=2.0)
    for pcm in (sig["chirp"], sig["square"], P.recording("dhd.2934z.raw")):
        _run(pcm, 16000, _random_cuts(rng, len(pcm), 16000), smooth_window=smooth_window)
    pcm = P.recording("goforward.raw")
    _run(pcm, 16000, [1600] * (len(pcm) // 1600) + [len(pcm) % 1600], program=True, smooth_window=smooth_window)
    _run(pcm, 16000, [37] * (len(pcm) // 37) + [len(pcm) % 37], smooth_window=smooth_window, voice_thresh=1.0)


@pytest.mark.parametrize("rate", P.RATES)
def test_rates(rate):
    rng = np.random.default_rng(rate)
    for name, pcm in P.signals(rate, seconds=1.0).items():
        _run(pcm, rate, _random_cuts(rng, len(pcm), rate), program=True)
    _run(P.signals(rate, seconds=1.0)["noise"], rate, _random_cuts(rng, rate, rate), smooth_window=5)


@pytest.mark.parametrize("smooth_window", [0, 2, 127])
def test_frame_counter_wrap_inside_a_call_and_on_a_boundary(smooth_window):
    """flen 8 / fshift 1: frame count F after 7 + F samples.  The counter wraps when F reaches 65 536."""
    pcm = P.signals(16000, seconds=140000 / 16000.0)["chirp"]
    n = 70000
    opts = dict(P.WRAP_OPTS, smooth_window=smooth_window)
    on = 65536 + 7                                    # a call ends with exactly 65 536 frames written
    _run(pcm[:n], 16000, [on, n - on], **opts)
    _run(pcm[:n], 16000, [on - 1, 1, 0, n - on], **opts)
    _run(pcm[:n], 16000, [60000, 10000], **opts)      # crossed inside a call
    _run(pcm[:n], 16000, [on - 100] + [10] * 20 + [n - on - 100], **opts)
    _run(pcm, 16000, [70000, 61079, 1, 8920], **opts)  # twice: 131 079 samples, the second wrap on a boundary


def test_final_calls_without_samples_or_frames():
    pcm = P.signals(16000)["chirp"]
    for sw in (0, 2, 127):
        _run(pcm[:4000], 16000, [4000, 0], smooth_window=sw)          # the final call feeds nothing
        _run(pcm[:399], 16000, [399], smooth_window=sw)               # shorter than one frame: no read at all
        _run(pcm[:399], 16000, [200, 199], smooth_window=sw)
        _run(pcm[:0], 16000, [0], smooth_window=sw)
        got = _run(pcm[:400], 16000, [400, 0], program=True, smooth_window=sw)
        assert [len(g["period"]) for g in got] == ([1, 0] if sw == 0 else [0, 1])


def test_reset_in_mid_stream():
    """A slot reset after a final call, or in the middle of a stream, starts fresh: its window reads zeros again."""
    sig = P.signals(16000, seconds=1.0)
    for sw in (2, 127):
        ref, emu = L.RefStream(smooth_window=sw), L.EmulStream(smooth_window=sw)
        try:
            for pcm, cuts, end in ((sig["chirp"], [3000, 1234], True), (sig["noise"], [2000, 999], False),
                                   (sig["square"], [401, 1600, 5], True), (sig["chirp"][:400], [400], True)):
                got, pos = [], 0
                for i, n in enumerate(cuts):
                    fin = end and i == len(cuts) - 1
                    a, b = ref.feed(pcm[pos:pos + n], fin), emu.feed(pcm[pos:pos + n], fin)
                    assert L.same(a, b), (sw, i)
                    got.append(b)
                    pos += n
                if end:
                    per, bd, _ = L.join(got)
                    want = L.whole(pcm[:pos], 16000, smooth_window=sw)
                    assert np.array_equal(per, want["period"]) and np.array_equal(bd, want["bestdiff"])
                ref.reset(), emu.reset()
        finally:
            ref.close(), emu.close()
