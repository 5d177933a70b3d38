"""CPU: live endpointing as psb_vad_feed_* runs one slot (psb_vad_core.h's arithmetic with the slot saved and restored
between calls, built for the host by tests/emul/vad_live_emul.cpp) against the compiled reference fed the same chunks
(tests/emul/vad_live_refdrv.c): decisions, ended segments and the end-of-call status equal after every call, for random
chunkings, streams ended and fed on, and streams reset and reused."""
import numpy as np
import pytest

import vad_cases as V
import vad_live_cases as VL

pytestmark = pytest.mark.skipif(not V.ref_available(), reason="compiled reference (oracle/_ref) not built")


def _stream(rate, seed):
    a = V.audio()
    rng = np.random.default_rng(seed)
    closest = V.closest_rate(rate)
    src = [a["test_audio_8k"], a["leak_test"]] if closest == 8000 else [a["goforward"], a["numbers"], a["libri_0870"]]
    parts = []
    for _ in range(4):
        parts.append(np.zeros(int(rng.integers(0, closest)), np.int16))
        x = src[int(rng.integers(len(src)))]
        parts.append(V.upsample2(x) if closest == 32000 else x)
    parts.append(V.synthetic(closest, seconds=1.0, seed=seed))
    return np.concatenate(parts)


def _run(pcm, plan, a, b, reset_at=None):
    pos = 0
    for i, (n, fin) in enumerate(plan):
        if i == reset_at:
            a.reset(), b.reset()
        ra, rb = a.feed(pcm[pos:pos + n], fin), b.feed(pcm[pos:pos + n], fin)
        assert VL.same(ra, rb), (i, n, fin, pos, ra["segments"], rb["segments"], ra["frames"], rb["frames"])
        pos += n
    return pos


@pytest.mark.parametrize("rate", [8000, 16000, 32000, 11025, 22050])
@pytest.mark.parametrize("fl", [0.01, 0.02, 0.03])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_random_chunkings_equal_reference(mode, fl, rate):
    seed = mode * 1000 + int(fl * 100) * 10 + rate % 7
    pcm = _stream(rate, seed)
    rng = np.random.default_rng(seed)
    fs, sr = V.ref_params(mode, rate, fl)
    warmup = [0, 3, int(np.ceil(0.5 / (fs / sr) - 1e-9))][seed % 3]     # none, a little, psb_vad_create's default
    # one stream ended only at its end: the calls' flags and segments put together are the whole-stream result
    plan = VL.chunking(rng, len(pcm), fs, rate)
    ref, emu = VL.RefStream(mode, rate, fl), VL.EmulStream(mode, rate, fl, warmup=warmup)
    got = []
    pos = 0
    for n, fin in plan:
        r, e = ref.feed(pcm[pos:pos + n], fin), emu.feed(pcm[pos:pos + n], fin)
        assert VL.same(r, e), (n, fin, pos)
        got.append(r)
        pos += n
    assert np.array_equal(np.concatenate([g["flags"] for g in got]), V.ref_flags(mode, rate, fl, pcm))
    assert sum((g["segments"] for g in got), []) == V.ref_segments(pcm, mode, rate, fl)
    # ended now and then and fed on with the same endpointer, then reset half-way and reused
    ref.reset(), emu.reset()
    plan = VL.chunking(rng, len(pcm), fs, rate, finals=0.15)
    _run(pcm, plan, ref, emu, reset_at=len(plan) // 2)
    ref.close(), emu.close()


@pytest.mark.parametrize("window,ratio", [(0.3, 0.3), (1.0, 0.5)])
def test_end_then_continue_in_speech(window, ratio):
    """Streams ended in the middle of speech (the queue is dropped, the times lag) and fed on, each end 7 samples
    after a random cut."""
    a = V.audio()
    pcm = np.concatenate([np.zeros(8000, np.int16), a["numbers"], a["goforward"]])
    fs = 480
    ref, emu = VL.RefStream(0, 16000, 0.03, window, ratio), VL.EmulStream(0, 16000, 0.03, window, ratio, warmup=0)
    pos, speech_ends = 0, 0
    rng = np.random.default_rng(5)
    while pos < len(pcm):
        n = int(rng.integers(fs // 2, 40 * fs))
        fin = ref.feed(pcm[pos:pos + n], False)["in_speech"]
        emu.feed(pcm[pos:pos + n], False)
        pos += n
        r, e = ref.feed(pcm[pos:pos + 7], fin), emu.feed(pcm[pos:pos + 7], fin)
        assert VL.same(r, e), pos
        speech_ends += fin
        pos += 7
    assert speech_ends >= 3
    ref.close(), emu.close()


def test_reset_gives_fresh_stream():
    a = V.audio()
    pcm = a["goforward"]
    ref = VL.RefStream()
    first = [ref.feed(pcm[i:i + 4000], i + 4000 >= len(pcm)) for i in range(0, len(pcm), 4000)]
    ref.feed(a["numbers"][:30000])
    ref.reset()
    again = [ref.feed(pcm[i:i + 4000], i + 4000 >= len(pcm)) for i in range(0, len(pcm), 4000)]
    assert all(VL.same(x, y) for x, y in zip(first, again))
    ref.close()
