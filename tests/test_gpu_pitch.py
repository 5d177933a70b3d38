"""GPU: api.PitchTracker / psb_pitch_process_* against the compiled reference (extract_pitch's loop over yin_* in
oracle/_ref/libpsref.so, and the pocketsphinx_pitch program): every period and bestdiff equal, on the signals, rates,
smoothing windows, thresholds and stream lengths of the CPU grid, in ragged batches of 1000 streams, and across the
uint16 frame-counter wrap of an hour-long stream."""
import ctypes as C

import numpy as np
import pytest

import pitch_cases as P
from pocketsphinx_b200 import api
from pocketsphinx_b200._lib import PitchOpts, PsbError, lib

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not P.ref_available(), reason="compiled reference (oracle/_ref) not built")]


@pytest.fixture(scope="module")
def tracker():
    t = api.PitchTracker()
    yield t
    t.close()


def _opts_key(rate, opts):
    return (rate, tuple(sorted(opts.items())))


def _batch_vs_ref(streams, rate, **opts):
    """One device call over all streams against the reference run stream by stream."""
    t = api.PitchTracker(sample_rate=rate, **opts)
    try:
        got = t.track_batch(streams)
    finally:
        t.close()
    for i, pcm in enumerate(streams):
        per, bd, main = P.ref_run(pcm, rate, **opts)
        assert np.array_equal(got[i]["period"], per), (i, _opts_key(rate, opts))
        assert np.array_equal(got[i]["bestdiff"], bd), (i, _opts_key(rate, opts))
        assert np.all(got[i]["time"][:main] == np.arange(main) * t.frame_shift / rate)
    return got


@pytest.mark.parametrize("rate", P.RATES)
def test_signals_at_every_rate(rate):
    streams = list(P.signals(rate).values()) + [P.recording("goforward.raw"), P.recording("dhd.2934z.raw")]
    got = _batch_vs_ref(streams, rate)
    if rate == 16000:
        for i in (3, 7):
            text = "".join(api.pitch_lines(got[i], rate)).encode()
            assert text == P.program_output(streams[i], rate)


@pytest.mark.parametrize("smooth_window", P.SMOOTH)
def test_smoothing_windows_and_thresholds(smooth_window):
    sig = P.signals(16000, seconds=0.6)
    streams = [sig["chirp"], sig["square"], sig["noise"], sig["alternating"], P.recording("goforward.raw")]
    for thr in P.THRESH:
        _batch_vs_ref(streams, 16000, smooth_window=smooth_window, voice_thresh=thr)
    _batch_vs_ref(streams, 16000, smooth_window=smooth_window, search_range=0.9)


@pytest.mark.parametrize("rate", [8000, 44100])
def test_stream_lengths_and_one_or_two_frames(rate):
    base = P.signals(rate, seconds=0.2)["chirp"]
    streams = [base[:n] for n in P.length_cases(rate)]
    for sw in (0, 1, 2, 5, 127):
        _batch_vs_ref(streams, rate, smooth_window=sw)


def test_frame_counter_wrap_once_and_twice():
    pcm = P.signals(16000, seconds=140000 / 16000.0)["chirp"]
    got = _batch_vs_ref([pcm[:70000], pcm[:140000]], 16000, **P.WRAP_OPTS)
    assert len(got[0]["period"]) == 69988
    _batch_vs_ref([pcm[:70000], pcm[:140000]], 16000, smooth_window=5, **P.WRAP_OPTS)


def test_ragged_batch_of_1000_streams():
    rng = np.random.default_rng(7)
    rec = np.concatenate([P.recording("goforward.raw"), P.recording("dhd.2934z.raw")])
    streams = []
    for i in range(1000):
        n = [0, 5, 399, 400, 401][i] if i < 5 else int(rng.integers(0, 24000))
        o = int(rng.integers(0, len(rec) - n))
        streams.append(rec[o:o + n])
    got = _batch_vs_ref(streams, 16000)
    assert [len(g["period"]) for g in got[:5]] == [0, 0, 0, 1, 1]


def test_hour_long_stream_crosses_the_wrap_five_times(tracker):
    rec = np.concatenate([P.recording("goforward.raw"), P.recording("dhd.2934z.raw")])
    n = 60 * 60 * 16000
    pcm = np.resize(rec, n)
    nf = tracker.n_frames(n)
    assert nf // 65536 == 5
    got = tracker.track_batch([pcm])[0]
    per, bd, main = P.ref_run(pcm, 16000)
    assert len(per) == nf - 5 * 3 and main == len(per) - 2
    assert np.array_equal(got["period"], per) and np.array_equal(got["bestdiff"], bd)


def test_host_and_device_calls_give_the_same_bytes(tracker):
    import torch
    sig = P.signals(16000, seconds=1.0)
    streams = [sig["chirp"], sig["noise"][:401], P.recording("goforward.raw"), sig["alternating"]]
    want = tracker.track_batch(streams)
    samp_off = np.zeros(len(streams) + 1, np.int64)
    samp_off[1:] = np.cumsum([len(s) for s in streams])
    pcm = torch.from_numpy(np.concatenate(streams)).cuda()
    cap = sum(tracker.n_frames(len(s)) for s in streams)
    d_per = torch.zeros(cap, dtype=torch.int16, device="cuda")
    d_bd = torch.zeros(cap, dtype=torch.int16, device="cuda")
    out_off = np.zeros(len(streams) + 1, np.int32)
    ms = C.c_float()
    api.check(lib().psb_pitch_process_device(tracker.h, pcm.data_ptr(), samp_off.ctypes.data, len(streams),
                                             out_off.ctypes.data, d_per.data_ptr(), d_bd.data_ptr(), C.byref(ms)))
    per = d_per.cpu().numpy().view(np.uint16)
    bd = d_bd.cpu().numpy().view(np.uint16)
    for i in range(len(streams)):
        assert per[out_off[i]:out_off[i + 1]].tobytes() == want[i]["period"].tobytes()
        assert bd[out_off[i]:out_off[i + 1]].tobytes() == want[i]["bestdiff"].tobytes()
    assert ms.value > 0.0


@pytest.mark.parametrize("opts,what", [
    (dict(fshift=0.0), "never advances"),
    (dict(fshift=0.03), "longer than"),
    (dict(flen=0.00005), "at least 2"),
    (dict(flen=1.1), "at most 16384"),
    (dict(smooth_window=128), "0..127"),
    (dict(smooth_window=-1), "0..127"),
    (dict(voice_thresh=2.0), "voice_thresh"),
    (dict(voice_thresh=-0.1), "voice_thresh"),
    (dict(search_range=2.5), "search_range"),
    (dict(sample_rate=0), "sample_rate"),
])
def test_refusals_launch_nothing(opts, what):
    L = lib()
    before = L.psb_kernel_launch_count()
    with pytest.raises(PsbError, match=what):
        api.PitchTracker(**opts)
    assert L.psb_kernel_launch_count() == before


def test_bad_offsets_are_refused_before_any_launch(tracker):
    L = lib()
    before = L.psb_kernel_launch_count()
    pcm = np.zeros(1000, np.int16)
    out_off = np.zeros(3, np.int32)
    per = np.zeros(8, np.uint16)
    for off in ([1, 500, 1000], [0, 600, 500]):
        so = np.asarray(off, np.int64)
        rc = L.psb_pitch_process_host(tracker.h, pcm.ctypes.data, so.ctypes.data, 2, out_off.ctypes.data,
                                      per.ctypes.data, per.ctypes.data, None)
        assert rc != 0 and b"samp_off" in L.psb_last_error()
    assert L.psb_kernel_launch_count() == before


def test_closing_a_handle_returns_its_memory():
    L = lib()
    before = L.psb_device_bytes_live()
    t = api.PitchTracker(sample_rate=48000, smooth_window=5)
    t.track_batch([P.signals(48000, seconds=2.0)["chirp"]] * 8)
    assert L.psb_device_bytes_live() > before
    t.close()
    assert L.psb_device_bytes_live() == before


def test_opts_struct_matches_the_header():
    assert C.sizeof(PitchOpts) == 40
