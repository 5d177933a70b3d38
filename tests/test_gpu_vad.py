"""GPU: psb_vad_process_* (stage A: chunk-parallel filter bank with boundary repairs, stage B: one warp per stream
for the GMM and the endpointer) against the compiled reference run live (tests/emul/vad_refdrv.c over
ps_vad_classify / ps_endpointer_process + _end_stream): flags and segments equal, for ragged batches, every mode,
frame length and supported rate, one long stream, no warm-up (every boundary repaired), any stream order or split."""
import numpy as np
import pytest

import vad_cases as V

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not V.ref_available(), reason="compiled reference not built")]


def _ragged(rate, n=72, seed=0):
    """n streams: fixtures and synthetic signals cut at random lengths (0 samples to a minute), with silence gaps."""
    a = V.audio()
    rng = np.random.default_rng(seed)
    if rate == 8000:
        src = [a["test_audio_8k"], a["leak_test"], V.synthetic(8000, seed=seed)]
    else:
        src = [a["goforward"], a["numbers"], a["libri_0870"], a["libri_0880"], V.synthetic(16000, seed=seed)]
        if rate == 32000:
            src = [V.upsample2(x) for x in src]
    out = []
    for i in range(n):
        if i < 4:
            out.append(np.zeros(0, np.int16) if i == 0 else rng.integers(-300, 300, [1, rate // 100 - 1, rate // 100][i - 1]).astype(np.int16))
            continue
        parts, total = [], int(rng.integers(1, 60 if i % 17 == 0 else 8) * rate)
        while sum(len(p) for p in parts) < total:
            parts.append(np.zeros(int(rng.integers(0, rate)), np.int16))
            x = src[int(rng.integers(len(src)))]
            s = int(rng.integers(0, len(x)))
            parts.append(x[s:s + int(rng.integers(rate // 10, len(x)))])
        out.append(np.concatenate(parts)[:total + int(rng.integers(0, rate // 50))])
    return out


def _check(ep, streams, mode, rate, fl, window=0.3, ratio=0.9):
    flags = ep.classify_batch(streams)
    segs = ep.segment_batch(streams)
    for i, s in enumerate(streams):
        assert np.array_equal(flags[i], V.ref_flags(mode, rate, fl, s)), (i, len(s))
        assert segs[i] == V.ref_segments(s, mode, rate, fl, window, ratio), (i, len(s))
    return flags, segs


@pytest.mark.parametrize("rate", [8000, 16000, 32000, 11025, 22050])
@pytest.mark.parametrize("fl", [0.01, 0.02, 0.03])
def test_ragged_batch_every_rate_and_frame_length(rate, fl):
    from pocketsphinx_b200 import api
    mode = int(round(fl * 100)) % 4
    streams = _ragged(V.closest_rate(rate), n=64, seed=rate + int(fl * 1000))
    ep = api.Endpointer(0.3, 0.9, mode, rate, fl)
    _, segs = _check(ep, streams, mode, rate, fl)
    assert sum(len(s) for s in segs) > 0
    ep.close()


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_every_mode_and_endpointer_ratios(mode):
    from pocketsphinx_b200 import api
    streams = _ragged(16000, n=64, seed=100 + mode)
    for window, ratio in ((0.3, 0.9), (0.3, 0.3), (1.0, 0.5)):
        ep = api.Endpointer(window, ratio, mode, 16000, 0.01)
        _check(ep, streams, mode, 16000, 0.01, window, ratio)
        ep.close()


@pytest.mark.timeout(900)
def test_long_stream_and_no_warmup_repairs():
    """One 24-minute stream built from the fixtures with silence between them, with the default warm-up and with
    none (every chunk boundary then differs from the true state and is repaired): identical results."""
    from pocketsphinx_b200 import api
    a = V.audio()
    rng = np.random.default_rng(7)
    parts = []
    while sum(len(p) for p in parts) < 24 * 60 * 16000:
        parts.append(np.zeros(int(rng.integers(0, 3 * 16000)), np.int16))
        parts.append(a[["goforward", "numbers", "libri_0870", "libri_0880"][int(rng.integers(4))]])
    long = np.concatenate(parts)
    streams = [long] + _ragged(16000, n=63, seed=9)
    for fl in (0.01, 0.03):
        want_f = [V.ref_flags(0, 16000, fl, s) for s in streams]
        want_s = [V.ref_segments(s, 0, 16000, fl) for s in streams]
        for warmup in (None, 0):
            ep = api.Endpointer(0.3, 0.9, 0, 16000, fl, warmup=warmup)
            flags, segs = ep.classify_batch(streams), ep.segment_batch(streams)
            assert all(np.array_equal(f, w) for f, w in zip(flags, want_f)), (fl, warmup)
            assert segs == want_s, (fl, warmup)
            print("frame %.2f s, warmup %s (%d frames): %d chunk recomputations in %d passes, %d segments in the long stream"
                  % (fl, warmup, ep.warmup, ep.last_repairs, ep.last_passes, len(segs[0])))
            if warmup == 0:
                assert ep.last_repairs > 0
            ep.close()
    assert len(want_s[0]) > 50


def test_order_and_split_independence():
    from pocketsphinx_b200 import api
    streams = _ragged(16000, n=70, seed=3)
    ep = api.Endpointer(0.3, 0.9, 2, 16000, 0.02, warmup=3)
    whole = ep.segment_batch(streams)
    perm = np.random.default_rng(1).permutation(len(streams))
    shuffled = ep.segment_batch([streams[i] for i in perm])
    assert [shuffled[j] for j in np.argsort(perm)] == whole
    assert ep.segment_batch(streams[:10]) + ep.segment_batch(streams[10:]) == whole
    assert [ep.segment_batch([s])[0] for s in streams[:8]] == whole[:8]
    assert ep.segment_batch([]) == [] and ep.classify_batch([np.zeros(5, np.int16)])[0].size == 0
    ep.close()


def test_handles_with_different_windows_alternate():
    """Handles whose endpointer queues differ in size (10 / 30 ms frames, two windows) used in turn: each launch
    gets the shared memory its own queue needs, whichever handle was created or used last."""
    from pocketsphinx_b200 import api
    streams = _ragged(16000, n=16, seed=11)
    cfg = [(0.3, 0.01), (0.3, 0.03), (2.0, 0.01), (0.3, 0.02)]
    eps = [api.Endpointer(w, 0.9, 0, 16000, fl) for w, fl in cfg]
    want = [[V.ref_segments(s, 0, 16000, fl, w, 0.9) for s in streams] for w, fl in cfg]
    for _ in range(2):
        for ep, wv in zip(eps + eps[::-1], want + want[::-1]):
            assert ep.segment_batch(streams) == wv
    for ep in eps:
        ep.close()


@pytest.mark.parametrize("kw", [dict(sample_rate=42), dict(sample_rate=96000), dict(ratio=0.99), dict(window=0.03, ratio=0.1),
                                dict(frame_length=0.025), dict(vad_mode=4), dict(sample_rate=44100), dict(sample_rate=48000),
                                dict(window=1000.0, frame_length=0.01)])
def test_refusals(kw):
    from pocketsphinx_b200 import api
    with pytest.raises(api.PsbError):
        api.Endpointer(**kw)
    a = dict(window=0.3, ratio=0.9, mode=0, rate=16000, fl=0.03)
    a.update({dict(vad_mode="mode", sample_rate="rate", frame_length="fl").get(k, k): v for k, v in kw.items()})
    # the reference accepts 48 kHz and windows beyond the endpointer queue this port keeps in shared memory
    if a["rate"] not in (44100, 48000) and a["mode"] <= 3 and a["window"] < 500:
        assert V.ref_segments(np.zeros(100, np.int16), a["mode"], a["rate"], a["fl"], a["window"], a["ratio"]) is None


def test_endpointer_parameters_match_reference():
    from pocketsphinx_b200 import api
    for rate, fl in ((8000, 0.01), (11025, 0.03), (22050, 0.02), (32000, 0.03)):
        ep = api.Endpointer(0.5, 0.7, 1, rate, fl)
        fs, sr = V.ref_params(1, rate, fl)
        assert (ep.frame_size, ep.sample_rate, ep.frame_length) == (fs, sr, fs / sr)
        assert (ep.maxlen, ep.start_frames, ep.end_frames) == V.ep_params(0.5, 0.7, fs, sr)
        ep.close()
