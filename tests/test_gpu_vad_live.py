"""GPU: live endpointing (psb_vad_feed_*, api.LiveEndpointer) against the compiled reference fed the same chunks
(tests/emul/vad_live_refdrv.c) and against the whole-stream results: ragged batches with every slot on its own random
chunking, changing subsets and orders of slots, streams ended and fed on, slots reset and reused, whole-stream calls
and a second handle between feeds, one 24-minute stream, the refusals, and the memory returned on close."""
import numpy as np
import pytest

import vad_cases as V
import vad_live_cases as VL
from test_gpu_vad import _ragged

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not V.ref_available(), reason="compiled reference not built")]


def _plans(streams, fs, rate, seed, finals=0.0):
    rng = np.random.default_rng(seed)
    return [VL.chunking(rng, len(s), fs, rate, finals) for s in streams]


def _drive(le, streams, plans, refs=None, rng=None, between=None):
    """Feeds every stream's plan, each call a random subset of the slots with work left, in random order.  Checks
    every per-call result against refs (one RefStream per slot) when given; returns each slot's results."""
    rng = rng or np.random.default_rng(0)
    nxt, pos = [0] * len(streams), [0] * len(streams)
    got = [[] for _ in streams]
    while True:
        todo = [i for i in range(len(streams)) if nxt[i] < len(plans[i])]
        if not todo:
            return got
        pick = [i for i in todo if rng.random() < 0.7] or todo[:1]
        pick = [pick[j] for j in rng.permutation(len(pick))]
        chunks, fins = [], []
        for i in pick:
            n, fin = plans[i][nxt[i]]
            chunks.append(streams[i][pos[i]:pos[i] + n])
            fins.append(fin)
            pos[i] += n
            nxt[i] += 1
        out = le.feed(chunks, slots=pick, final=fins)
        for i, c, f, r in zip(pick, chunks, fins, out):
            if refs is not None:
                want = refs[i].feed(c, f)
                assert VL.same(r, want), (i, len(c), f, r["segments"], want["segments"], r["frames"], want["frames"])
            got[i].append(r)
        if between is not None:
            between()


def _whole(got):
    return np.concatenate([g["flags"] for g in got]), sum((g["segments"] for g in got), [])


@pytest.mark.parametrize("rate", [8000, 16000, 32000, 11025, 22050])
@pytest.mark.parametrize("fl", [0.01, 0.02, 0.03])
def test_ragged_live_batch(rate, fl):
    from pocketsphinx_b200 import api
    mode = int(round(fl * 100) + rate) % 4
    streams = _ragged(V.closest_rate(rate), n=24, seed=rate + int(fl * 1000))
    le = api.LiveEndpointer(24, 0.3, 0.9, mode, rate, fl, warmup=[None, 0, 5][int(fl * 100) % 3])
    plans = _plans(streams, le.frame_size, rate, seed=rate)
    refs = [VL.RefStream(mode, rate, fl) for _ in streams]
    got = _drive(le, streams, plans, refs)
    for i, s in enumerate(streams):
        flags, segs = _whole(got[i])
        assert np.array_equal(flags, V.ref_flags(mode, rate, fl, s)), i
        assert segs == V.ref_segments(s, mode, rate, fl), i
    # ended now and then and fed on, per the reference fed the same way
    for r in refs:
        r.reset()
    le.reset(list(range(24)))
    _drive(le, streams, _plans(streams, le.frame_size, rate, seed=rate + 1, finals=0.2), refs, np.random.default_rng(1))
    for r in refs:
        r.close()
    le.close()


def test_reset_reuse_whole_stream_calls_and_two_handles():
    from pocketsphinx_b200 import api
    streams = _ragged(16000, n=12, seed=21)
    a = api.LiveEndpointer(12, 0.3, 0.9, 1, 16000, 0.01)
    b = api.LiveEndpointer(5, 1.0, 0.5, 2, 16000, 0.03)
    whole_a = a.segment_batch(streams)
    refs_a = [VL.RefStream(1, 16000, 0.01) for _ in streams]
    refs_b = [VL.RefStream(2, 16000, 0.03, 1.0, 0.5) for _ in streams[:5]]
    plans_b = _plans(streams[:5], b.frame_size, 16000, seed=3, finals=0.1)
    it_b = {"k": 0}
    pos_b, nxt_b = [0] * 5, [0] * 5

    def between():
        # a whole-stream call on the same handle and a live call on another handle, between every two feeds
        assert a.segment_batch(streams[:3]) == whole_a[:3]
        i = it_b["k"] % 5
        it_b["k"] += 1
        if nxt_b[i] < len(plans_b[i]):
            n, fin = plans_b[i][nxt_b[i]]
            c = streams[i][pos_b[i]:pos_b[i] + n]
            pos_b[i] += n
            nxt_b[i] += 1
            assert VL.same(b.feed([c], slots=[i], final=[fin])[0], refs_b[i].feed(c, fin))

    got = _drive(a, streams, _plans(streams, a.frame_size, 16000, seed=2), refs_a, between=between)
    assert [_whole(g)[1] for g in got] == whole_a
    # a slot reset after use gives the fresh stream's result
    a.feed([streams[0][:12345]], slots=[7])
    a.reset([7])
    r = a.feed([streams[3]], slots=[7], final=[True])[0]
    assert r["segments"] == whole_a[3] and r["frames"] == len(streams[3]) // a.frame_size
    for x in refs_a + refs_b:
        x.close()
    a.close()
    b.close()


@pytest.mark.timeout(1200)
def test_long_stream_live():
    """One 24-minute stream fed in 100 ms chunks, and in 10 s chunks with no warm-up (every chunk boundary inside a
    call repaired): both give the whole stream's flags and segments."""
    from pocketsphinx_b200 import api
    a = V.audio()
    rng = np.random.default_rng(7)
    parts = []
    while sum(len(p) for p in parts) < 24 * 60 * 16000:
        parts.append(np.zeros(int(rng.integers(0, 3 * 16000)), np.int16))
        parts.append(a[["goforward", "numbers", "libri_0870", "libri_0880"][int(rng.integers(4))]])
    long = np.concatenate(parts)
    for fl in (0.01, 0.03):
        want_f, want_s = V.ref_flags(0, 16000, fl, long), V.ref_segments(long, 0, 16000, fl)
        for step, warmup in ((1600, None), (160000, 0)):
            le = api.LiveEndpointer(1, 0.3, 0.9, 0, 16000, fl, warmup=warmup)
            got = [le.feed([long[p:p + step]], final=[p + step >= len(long)])[0] for p in range(0, len(long), step)]
            if warmup == 0:
                assert le.last_repairs > 0
            flags, segs = _whole(got)
            assert np.array_equal(flags, want_f), (fl, step)
            assert segs == want_s, (fl, step)
            le.close()
    assert len(want_s) > 50


def test_refusals_and_memory():
    from pocketsphinx_b200 import api
    L = api.lib()
    base = L.psb_device_bytes_live()
    ep = api.Endpointer()
    with pytest.raises(api.PsbError):                     # feeding before psb_vad_live_open
        api.LiveEndpointer.feed(ep, [np.zeros(10, np.int16)])
    with pytest.raises(api.PsbError):
        api.LiveEndpointer.reset(ep, [0])
    ep.close()
    le = api.LiveEndpointer(4)
    x = np.zeros(1000, np.int16)
    for slots in ([4], [-1], [1, 1]):
        with pytest.raises(api.PsbError):
            le.feed([x] * len(slots), slots=slots)
    with pytest.raises(api.PsbError):
        le.reset([4])
    with pytest.raises(api.PsbError):
        api.LiveEndpointer(0)
    # a refused call changes nothing: the slots go on as if it had not happened
    r = le.feed([x, x], slots=[2, 0])
    assert [d["frames"] for d in r] == [2, 2]
    assert le.feed([np.zeros(0, np.int16)], slots=[2])[0]["frames"] == 2
    le.close()
    assert L.psb_device_bytes_live() == base
