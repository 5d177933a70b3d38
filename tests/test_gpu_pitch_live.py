"""GPU: live pitch tracking (api.LivePitchTracker / psb_pitch_feed_*) against the compiled reference's yin_t fed in the
same chunks (tests/emul/pitch_live_refdrv.c): every call's reads equal, every slot's joined reads equal to track_batch
of its whole stream, the program's output byte for byte, across the uint16 frame-counter wrap of an hour-long stream,
and refusals that change no slot."""
import ctypes as C

import numpy as np
import pytest

import pitch_cases as P
import pitch_live_cases as L
from pocketsphinx_b200 import api
from pocketsphinx_b200._lib import PsbError, lib

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not P.ref_available(), reason="compiled reference (oracle/_ref) not built")]


def _rec():
    return np.concatenate([P.recording("goforward.raw"), P.recording("dhd.2934z.raw")])


def _streams(rng, n, max_len):
    rec = _rec()
    out = []
    for i in range(n):
        k = [0, 5, 399, 400, 401][i] if i < 5 else int(rng.integers(0, max_len))
        o = int(rng.integers(0, len(rec) - k))
        out.append(rec[o:o + k])
    return out


def _ragged(rng, total, fl, fs):
    """Chunk lengths covering `total` samples: empty, single samples, cuts inside a frame, fshift, flen, up to 0.5 s."""
    out, pos = [], 0
    while pos < total:
        n = min([0, 1, int(rng.integers(1, fl)), fs, fl, int(rng.integers(fl, 8000))][int(rng.integers(6))], total - pos)
        out.append(n)
        pos += n
    return out or [0]


def _drive(tracker, streams, rng, check_ref=True, **opts):
    """Feeds every stream through its slot in random chunks, random subsets and orders of slots per call, each slot's
    last chunk final; each call's result is checked against a reference yin_t per slot.  Returns per-slot results."""
    n = len(streams)
    fl, fs = tracker.frame_size, tracker.frame_shift
    cuts = [_ragged(rng, len(s), fl, fs) for s in streams]
    pos, step = [0] * n, [0] * n
    refs = [L.RefStream(tracker.sample_rate, **opts) for _ in range(n)] if check_ref else None
    got = [[] for _ in range(n)]
    try:
        while True:
            live = [i for i in range(n) if step[i] < len(cuts[i])]
            if not live:
                break
            pick = rng.permutation(live)[:int(rng.integers(1, len(live) + 1))]
            chunks, fin = [], []
            for i in pick:
                k = cuts[i][step[i]]
                chunks.append(streams[i][pos[i]:pos[i] + k])
                fin.append(step[i] == len(cuts[i]) - 1)
                pos[i] += k
                step[i] += 1
            res = tracker.feed(chunks, slots=pick, final=fin)
            for j, i in enumerate(pick):
                if check_ref:
                    want = refs[i].feed(chunks[j], fin[j])
                    assert L.same(res[j], want), (int(i), step[i])
                got[i].append(res[j])
    finally:
        for r in refs or ():
            r.close()
    return got


def _joined_equal_whole(tracker, streams, got, **opts):
    whole = api.PitchTracker(sample_rate=tracker.sample_rate, **opts)
    try:
        want = whole.track_batch(streams)
    finally:
        whole.close()
    for i in range(len(streams)):
        per, bd, tm = L.join(got[i])
        assert np.array_equal(per, want[i]["period"]) and np.array_equal(bd, want[i]["bestdiff"]), i
        assert tm.tobytes() == want[i]["time"].tobytes(), i


def test_1000_slots_in_random_chunks_subsets_and_orders():
    rng = np.random.default_rng(3)
    streams = _streams(rng, 1000, 24000)
    t = api.LivePitchTracker(1000)
    try:
        got = _drive(t, streams, rng)
    finally:
        t.close()
    _joined_equal_whole(t, streams, got)


@pytest.mark.parametrize("smooth_window", [0, 1, 127])
@pytest.mark.parametrize("rate", [8000, 44100])
def test_smoothing_windows_and_rates(smooth_window, rate):
    rng = np.random.default_rng(rate + smooth_window)
    streams = [np.resize(s, int(len(s) * rate / 16000)) for s in _streams(rng, 40, 40000)]
    t = api.LivePitchTracker(40, sample_rate=rate, smooth_window=smooth_window)
    try:
        got = _drive(t, streams, rng, smooth_window=smooth_window)
    finally:
        t.close()
    _joined_equal_whole(t, streams, got, smooth_window=smooth_window)


def test_program_output_of_two_recordings():
    recs = [P.recording("goforward.raw"), P.recording("dhd.2934z.raw")]
    t = api.LivePitchTracker(2)
    try:
        got = [[], []]
        for a in range(0, max(len(r) for r in recs), 1234):
            slots = [i for i in range(2) if a < len(recs[i])]
            res = t.feed([recs[i][a:a + 1234] for i in slots], slots=slots,
                         final=[a + 1234 >= len(recs[i]) for i in slots])
            for j, i in enumerate(slots):
                got[i].append(res[j])
        for i in range(2):
            assert got[i][-1]["ended"]
            assert L.lines(got[i], 16000) == P.program_output(recs[i], 16000)
    finally:
        t.close()


def test_two_handles_fed_in_turn():
    rng = np.random.default_rng(5)
    a, b = api.LivePitchTracker(3), api.LivePitchTracker(3, smooth_window=127)
    ra, rb = [L.RefStream() for _ in range(3)], [L.RefStream(smooth_window=127) for _ in range(3)]
    try:
        pcm = _rec()
        for c in range(40):
            n = int(rng.integers(0, 3000))
            chunks = [pcm[(c * 997 + 311 * i) % 30000:][:n] for i in range(3)]
            fin = [c == 39] * 3
            for t, refs in ((a, ra), (b, rb)):
                res = t.feed(chunks, final=fin)
                for i in range(3):
                    assert L.same(res[i], refs[i].feed(chunks[i], fin[i])), (c, i)
    finally:
        a.close(), b.close()
        for r in ra + rb:
            r.close()


def test_hour_long_stream_one_second_per_call():
    rec = _rec()
    n = 60 * 60 * 16000
    pcm = np.resize(rec, n)
    t = api.LivePitchTracker(1)
    try:
        got = [t.feed([pcm[a:a + 16000]], final=[a + 16000 >= n])[0] for a in range(0, n, 16000)]
        want = t.track_batch([pcm])[0]
    finally:
        t.close()
    assert got[-1]["frames"] // 65536 == 5
    per, bd, tm = L.join(got)
    assert np.array_equal(per, want["period"]) and np.array_equal(bd, want["bestdiff"])
    assert tm.tobytes() == want["time"].tobytes()
    rper, rbd, rmain = P.ref_run(pcm, 16000)
    assert np.array_equal(per, rper) and np.array_equal(bd, rbd) and got[-1]["main_reads"] == rmain


def test_device_call_equals_host_call():
    import torch
    rng = np.random.default_rng(9)
    streams = _streams(rng, 64, 20000)
    h, d = api.LivePitchTracker(64), api.LivePitchTracker(64)
    try:
        pos = [0] * 64
        for c in range(6):
            slots = rng.permutation(64)[:40].astype(np.int32)
            chunks = []
            for s in slots:
                k = int(rng.integers(0, 5000))
                chunks.append(streams[s][pos[s]:pos[s] + k])
                pos[s] += len(chunks[-1])
            fin = np.asarray([c == 5 or rng.random() < 0.1 for _ in slots], np.int8)
            want = h.feed(chunks, slots=slots, final=fin)
            samp_off = np.zeros(len(slots) + 1, np.int64)
            samp_off[1:] = np.cumsum([len(x) for x in chunks])
            pcm = torch.from_numpy(np.concatenate(chunks)).cuda()
            cap = int(sum(-(-len(x) // d.frame_shift) + 2 * d.smooth_window for x in chunks))
            d_per = torch.zeros(cap, dtype=torch.int16, device="cuda")
            d_bd = torch.zeros(cap, dtype=torch.int16, device="cuda")
            out_off = np.zeros(len(slots) + 1, np.int32)
            status = np.zeros(len(slots), api.PITCH_LIVE_STATUS)
            ms = C.c_float()
            api.check(lib().psb_pitch_feed_device(d.h, slots.ctypes.data, len(slots), pcm.data_ptr(), samp_off.ctypes.data,
                                                  fin.ctypes.data, out_off.ctypes.data, d_per.data_ptr(), d_bd.data_ptr(),
                                                  status.ctypes.data, C.byref(ms)))
            per = d_per.cpu().numpy().view(np.uint16)
            bd = d_bd.cpu().numpy().view(np.uint16)
            for i in range(len(slots)):
                assert per[out_off[i]:out_off[i + 1]].tobytes() == want[i]["period"].tobytes()
                assert bd[out_off[i]:out_off[i + 1]].tobytes() == want[i]["bestdiff"].tobytes()
                assert (status[i]["frames"], status[i]["main_reads"], bool(status[i]["ended"])) == \
                    (want[i]["frames"], want[i]["main_reads"], want[i]["ended"])
            ended = [int(s) for s, f in zip(slots, fin) if f]
            h.reset(ended), d.reset(ended)
            for s in ended:
                pos[s] = 0
            assert ms.value > 0.0
    finally:
        h.close(), d.close()


def test_refusals_change_no_slot():
    """Each refused call launches nothing and changes no slot: the slots then go on as if it had not happened."""
    L_ = lib()
    pcm = P.recording("goforward.raw")
    closed = api.PitchTracker()
    try:
        n = np.zeros(1, np.int32)
        so = np.zeros(2, np.int64)
        off = np.zeros(2, np.int32)
        st = np.zeros(1, api.PITCH_LIVE_STATUS)
        buf = np.zeros(8, np.uint16)
        rc = L_.psb_pitch_feed_host(closed.h, n.ctypes.data, 1, None, so.ctypes.data, None, off.ctypes.data,
                                    buf.ctypes.data, buf.ctypes.data, st.ctypes.data, None)
        assert rc != 0 and b"psb_pitch_live_open has not been called" in L_.psb_last_error()
        assert L_.psb_pitch_live_reset(closed.h, n.ctypes.data, 1) != 0
        assert b"psb_pitch_live_open has not been called" in L_.psb_last_error()
    finally:
        closed.close()
    t = api.LivePitchTracker(3)
    ref = [L.RefStream() for _ in range(3)]
    try:
        def ok(chunks, slots, final):
            res = t.feed(chunks, slots=slots, final=final)
            for j, s in enumerate(slots):
                assert L.same(res[j], ref[s].feed(chunks[j], final[j]))

        ok([pcm[:1000], pcm[:777]], [0, 1], [False, False])
        ok([pcm[:500]], [2], [True])
        before = L_.psb_kernel_launch_count()
        refusals = [
            (dict(chunks=[pcm[1000:1100]], slots=[3]), "out of range"),
            (dict(chunks=[pcm[1000:1100]], slots=[-1]), "out of range"),
            (dict(chunks=[pcm[1000:1100], pcm[777:800]], slots=[0, 0]), "fed twice"),
            (dict(chunks=[pcm[1000:1100], pcm[:10]], slots=[0, 2]), "has ended"),
        ]
        for kw, what in refusals:
            with pytest.raises(PsbError, match=what):
                t.feed(**kw)
        with pytest.raises(PsbError, match="out of range"):
            t.reset([0, 3])
        for off in ([1, 100], [0, 100, 50]):
            so = np.asarray(off, np.int64)
            k = len(off) - 1
            sl = np.arange(k, dtype=np.int32)
            outo = np.zeros(k + 1, np.int32)
            st = np.zeros(k, api.PITCH_LIVE_STATUS)
            rc = L_.psb_pitch_feed_host(t.h, sl.ctypes.data, k, pcm.ctypes.data, so.ctypes.data, None, outo.ctypes.data,
                                        buf.ctypes.data, buf.ctypes.data, st.ctypes.data, None)
            assert rc != 0 and b"samp_off" in L_.psb_last_error()
        assert L_.psb_kernel_launch_count() == before
        ok([pcm[1000:5000], pcm[777:9000]], [0, 1], [False, True])
        t.reset([2]), ref[2].reset()
        ok([pcm[:3000]], [2], [False])
        ok([pcm[5000:5000], pcm[3000:4000]], [0, 2], [True, True])
    finally:
        t.close()
        for r in ref:
            r.close()


def test_a_slot_past_2_31_frames_is_refused():
    """flen 2 / fshift 1 at 1 Hz: every sample after the first is a frame, so 32 calls of 2^26 samples take a slot to
    2^31 - 1 frames, the most it may have; one more sample is refused and the slot can still end."""
    import torch
    L_ = lib()
    t = api.LivePitchTracker(1, sample_rate=1, flen=2.0, fshift=1.0, smooth_window=0)
    try:
        n = 1 << 26
        pcm = torch.zeros(n, dtype=torch.int16, device="cuda")
        d_out = torch.zeros(2 * n, dtype=torch.int16, device="cuda")
        slots = np.zeros(1, np.int32)
        out_off = np.zeros(2, np.int32)
        status = np.zeros(1, api.PITCH_LIVE_STATUS)

        def feed(k, final=0):
            so = np.asarray([0, k], np.int64)
            fin = np.asarray([final], np.int8)
            return L_.psb_pitch_feed_device(t.h, slots.ctypes.data, 1, pcm.data_ptr(), so.ctypes.data, fin.ctypes.data,
                                            out_off.ctypes.data, d_out.data_ptr(), d_out.data_ptr() + 2 * n,
                                            status.ctypes.data, None)
        for _ in range(32):
            api.check(feed(n))
        assert status[0]["frames"] == (1 << 31) - 1 and status[0]["main_reads"] == (1 << 31) - 1
        assert feed(1) != 0 and b"would pass 2^31 - 1 frames" in L_.psb_last_error()
        api.check(feed(0, 1))
        assert status[0]["frames"] == (1 << 31) - 1 and status[0]["ended"] == 1 and out_off[1] == 0
    finally:
        t.close()


def test_closing_returns_memory_and_whole_stream_calls_are_unchanged():
    L_ = lib()
    before = L_.psb_device_bytes_live()
    sig = P.signals(16000, seconds=2.0)
    streams = [sig["chirp"], sig["noise"], P.recording("goforward.raw")]
    plain = api.PitchTracker()
    t = api.LivePitchTracker(8, smooth_window=2)
    try:
        want = plain.track_batch(streams)
        t.feed([s[:12345] for s in streams])
        mid = t.track_batch(streams)
        res = t.feed([s[12345:] for s in streams], final=[True] * 3)
        after = t.track_batch(streams)
        for i in range(3):
            for got in (mid[i], after[i]):
                assert got["period"].tobytes() == want[i]["period"].tobytes()
                assert got["bestdiff"].tobytes() == want[i]["bestdiff"].tobytes()
            assert res[i]["ended"]
        assert L_.psb_device_bytes_live() > before
    finally:
        t.close(), plain.close()
    assert L_.psb_device_bytes_live() == before
