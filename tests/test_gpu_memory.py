"""GPU (-m gpu): handles reuse their grow-only workspaces, give their memory back when closed, and stay usable
after an allocation fails.  psb_device_bytes_live counts the library's own device and pinned bytes, so these
checks hold on a GPU that other processes share."""
import numpy as np
import pytest

from conftest import golden

pytestmark = pytest.mark.gpu

COUNTS = [3, 40, 7, 60]          # utterances per call: grow, shrink, grow again


@pytest.fixture(scope="module")
def api():
    from pocketsphinx_b200 import api
    assert api.device_count() > 0, "no CUDA device visible"
    return api


def live(api):
    return int(api.lib().psb_device_bytes_live())


def cut(rows, n, seed):
    """n utterances of 1 .. len(rows) rows cut from rows."""
    rng = np.random.default_rng(seed)
    lens = [int(x) for x in rng.integers(1, len(rows) + 1, n)]
    starts = [int(rng.integers(0, len(rows) - k + 1)) for k in lens]
    return np.concatenate([rows[s:s + k] for s, k in zip(starts, lens)]), np.cumsum([0] + lens).astype(np.int32)


def reuse_vs_fresh(api, make, run):
    """run(handle, n, seed) on one handle through COUNTS, each result equal to a fresh handle's; an identical
    repeat allocates nothing."""
    h = make()
    for i, n in enumerate(COUNTS):
        got = run(h, n, i)
        fresh = make()
        want = run(fresh, n, i)
        fresh.close()
        for a, b in zip(got, want):
            assert np.array_equal(a, b), "call %d (%d utterances)" % (i, n)
        held = live(api)
        again = run(h, n, i)
        assert live(api) == held, "an identical repeat grew the workspace"
        for a, b in zip(again, want):
            assert np.array_equal(a, b)
    h.close()


def test_ptm_decode_and_score_reuse(api, en_us):
    g = golden("en_us_goforward.npz")
    n_ph, beam, pbeam, pip, window = [int(x) for x in g["pl_params"]]
    start = live(api)
    m = api.Model(en_us)
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    pl = api.PhoneLoop(ctx, en_us.phone_ssid[:n_ph], en_us.phone_tmat[:n_ph], window, beam, pbeam, pip, float(g["pl_weight"]))

    def run(b, n, i):
        feats, off = cut(g["feats"], n, 10 + i)
        best, pen, scr = b.decode_host(pl, feats, off, want_senscr=True)       # pipelined sub-batches
        return best, pen, scr, b.score_host(feats, off)                         # one stream

    reuse_vs_fresh(api, lambda: api.Batch(m, 64, 16384), run)

    def run_pl(p, n, i):                                                        # per-call temporaries
        scr, off = cut(g["senscr"], n, 20 + i)
        r = p.run_host(scr, off, trace=True)
        return r["best"], r["pen"], r["hmm"]["score"], r["hmm"]["history"], r["hmm"]["bestscore"]

    reuse_vs_fresh(api, lambda: api.PhoneLoop(ctx, en_us.phone_ssid[:n_ph], en_us.phone_tmat[:n_ph], window, beam, pbeam, pip,
                                              float(g["pl_weight"])), run_pl)
    pl.close()
    ctx.close()
    m.close()
    assert live(api) == start


@pytest.mark.parametrize("name,golden_name", [("tidigits", "tidigits_goforward.npz"), ("an4", "an4_goforward.npz")])
def test_semi_and_ms_score_reuse(api, request, name, golden_name):
    pm = request.getfixturevalue(name)
    g = golden(golden_name)
    start = live(api)
    m = api.Model(pm)

    def run(b, n, i):
        feats, off = cut(g["feats"], n, 30 + i)
        return (b.score_host(feats, off),)

    reuse_vs_fresh(api, lambda: api.Batch(m, 64, 16384), run)
    m.close()
    assert live(api) == start


def test_alignment_reuse(api, en_us):
    g = golden("en_us_goforward.npz")
    start = live(api)
    n_ph = 3

    def run(c, n, i):
        scr, off = cut(g["senscr"], n, 40 + i)
        rng = np.random.default_rng(50 + i)
        ph = rng.integers(0, 40, n * n_ph)
        ph_off = np.arange(n + 1, dtype=np.int32) * n_ph
        status, *st = c.align(scr, off, ph_off, en_us.phone_ssid[ph], en_us.phone_tmat[ph])
        ok = np.repeat(status == 0, n_ph * c.n_emit)           # a failed utterance leaves its rows unwritten
        return [status] + [a[ok] for a in st]

    reuse_vs_fresh(api, lambda: api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen), run)
    assert live(api) == start


def test_front_end_and_vad_reuse(api):
    from pocketsphinx_b200.fe_tables import make_fe_desc
    start = live(api)

    def pcm(n, seed):
        rng = np.random.default_rng(seed)
        return [(rng.standard_normal(int(k)) * 800 * (1 + np.sin(np.arange(int(k)) / 3000.0))).astype(np.int16)
                for k in rng.integers(100, 40000, n)]

    def run_fe(fe, n, i):
        utts = pcm(n, 60 + i)
        off = api.FrontEnd.sample_offsets([len(u) for u in utts])
        feats, foff, mfcc = fe.process_host(np.concatenate(utts), off, want_mfcc=True)
        return feats.view(np.uint8), foff, mfcc.view(np.uint8)

    reuse_vs_fresh(api, lambda: api.FrontEnd(make_fe_desc()), run_fe)

    def run_vad(v, n, i):
        flags, frame_off, seg_n, segs, times = v.process(pcm(n, 70 + i))
        rows = np.concatenate([np.arange(frame_off[s], frame_off[s] + seg_n[s]) for s in range(n)]).astype(np.int64)
        return flags, frame_off, seg_n, segs[rows], times[rows]              # rows past seg_n are not written

    reuse_vs_fresh(api, lambda: api.Endpointer(), run_vad)
    assert live(api) == start


def test_batch_create_out_of_memory(api, en_us):
    """max_frames = 10 000 000 on en-us: the features (1.6 GB) fit, the senone scores (103 GB) do not."""
    g = golden("en_us_goforward.npz")
    m = api.Model(en_us)
    start = live(api)
    with pytest.raises(api.PsbError, match=r"\(-3\)"):
        api.Batch(m, 1, 10_000_000)
    assert live(api) == start
    # the failed allocation is not reported again by the next call
    n_ph, beam, pbeam, pip, window = [int(x) for x in g["pl_params"]]
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    pl = api.PhoneLoop(ctx, en_us.phone_ssid[:n_ph], en_us.phone_tmat[:n_ph], window, beam, pbeam, pip, float(g["pl_weight"]))
    b = api.Batch(m, 4, 1024)
    best, pen, scr = b.decode_host(pl, g["feats"], np.array([0, 278], np.int32), want_senscr=True)
    assert np.array_equal(scr, g["senscr"]) and np.array_equal(best, g["pl_best"])
    b.close(); pl.close(); ctx.close(); m.close()
