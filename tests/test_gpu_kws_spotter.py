"""GPU: keyword spotting for whole batches -- kws_kernel for keyphrase lists of any length against the C restatement
of kws_search.c (oracle.kws_run), pocketsphinx_b200.kws.KeywordSpotter on the reference's own senone scores (exact
detections) and from audio (the reference's live run, within the device front end's tolerance)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, golden

pytestmark = [pytest.mark.gpu]
REF = os.path.join(ROOT, "oracle", "_ref")
HD, DIC = os.path.join(REF, "model", "en-us"), os.path.join(REF, "model", "cmudict-en-us.dict")
GO, KWS_FILE = os.path.join(REF, "data", "goforward.raw"), os.path.join(GOLDEN, "goforward.kws")
KWS_MAX_HMMS = {3: 4834, 5: 3626}           # include/psb200.h, PSB_KWS_MAX_HMMS_3ST / _5ST (H100, 227 KB per block)


def _needs_ref_files():
    if not (os.path.exists(HD) and os.path.exists(GO)):
        pytest.skip("reference model and data files not present")


def _case(n_emit, n_pl, chains, seed):
    from pocketsphinx_b200.model import synth_ptm
    pm = synth_ptm(seed=seed, n_density=32, n_sen=300, n_emit_state=n_emit, skip_arcs=(n_emit == 5))
    rng = np.random.default_rng(seed)
    # the phone loop repeats a few phones: equal exit scores, so the smallest-index rule decides the best exit
    base = rng.integers(0, len(pm.sseq), max(1, n_pl // 3)).astype(np.int32)
    pl_ssid = np.resize(base, n_pl).astype(np.int32)
    pl_tmat = np.resize(rng.integers(0, pm.tp.shape[0], len(base)), n_pl).astype(np.int32)
    kp_off = np.concatenate([[0], np.cumsum(chains)]).astype(np.int32)
    kp_ssid = rng.integers(0, len(pm.sseq), kp_off[-1]).astype(np.int32)
    kp_tmat = rng.integers(0, pm.tp.shape[0], kp_off[-1]).astype(np.int32)
    kp_thresh = rng.choice(np.array([-50000, -3000, -200, 0], np.int32), len(chains)).astype(np.int32)
    return pm, (pl_ssid, pl_tmat, kp_off, kp_thresh, kp_ssid, kp_tmat)


def _chains(total, n_kp, seed):
    """n_kp chain lengths summing to total, with empty ones (a phrase whose words the dictionary lacks) among them."""
    rng = np.random.default_rng(seed)
    cut = np.sort(rng.integers(0, total + 1, n_kp - 1))
    c = np.diff(np.concatenate([[0], cut, [total]]))
    c[1] += c[0]; c[0] = 0
    return c.astype(np.int32)


@pytest.mark.parametrize("n_emit", [3, 5])
@pytest.mark.parametrize("H", [200, 512, 513, 3000])
def test_kws_kernel_any_length_matches_oracle(n_emit, H):
    """Below 512 HMMs, 512 and 513, and a few thousand in one CTA; a tight and a wide beam; ties in the phone-loop
    exit; empty keyphrases; the hit buffer at its default size (grown when a batch overflows it) and truncated at a
    set capacity."""
    import torch
    from oracle import oracle
    from pocketsphinx_b200 import api
    H = min(H, KWS_MAX_HMMS[n_emit])
    n_pl = 40
    n_kp = max(2, (H - n_pl) // 6)
    pm, cfg = _case(n_emit, n_pl, _chains(H - n_pl, n_kp, seed=H + n_emit), seed=7 * H + n_emit)
    assert n_pl + int(cfg[2][-1]) == H and (np.diff(cfg[2]) == 0).any()
    rng = np.random.default_rng(H)
    frames = [90, 1, 40]
    # coarse scores: many equal exit scores
    scr = [(rng.integers(0, 4, (t, pm.n_sen)) * 100).astype(np.int16) for t in frames]
    utt_off = np.concatenate([[0], np.cumsum(frames)]).astype(np.int32)
    ctx = api.HmmContext(pm.tp, pm.sseq, pm.n_sen)
    d_scr = torch.from_numpy(np.concatenate(scr)).cuda()
    total = 0
    for beam, plp in ((-1080, -23), (-60, -400)):
        want = [oracle.kws_run(pm.tp, pm.sseq, *cfg, beam, plp, s) for s in scr]
        hits, n = ctx.kws(d_scr.data_ptr(), utt_off, *cfg, beam, plp)
        for u in range(len(frames)):
            assert n[u] == len(want[u]) and np.array_equal(hits[u], want[u]), "H %d utterance %d beam %d" % (H, u, beam)
            total += len(want[u])
        h2, n2 = ctx.kws(d_scr.data_ptr(), utt_off, *cfg, beam, plp, cap=3)
        assert np.array_equal(n2, n) and all(np.array_equal(a, b[:3]) for a, b in zip(h2, hits))
    assert total > 0
    ctx.close()


@pytest.mark.parametrize("n_emit", [3, 5])
def test_kws_kernel_refuses_more_hmms_than_one_cta_holds(n_emit):
    """One HMM over the limit is refused with the count and the limit named; the context stays usable."""
    import torch
    from oracle import oracle
    from pocketsphinx_b200 import api
    lim = KWS_MAX_HMMS[n_emit]
    pm, cfg = _case(n_emit, 40, _chains(lim + 1 - 40, 300, seed=1), seed=3)
    rng = np.random.default_rng(5)
    scr = rng.integers(0, 300, (30, pm.n_sen)).astype(np.int16)
    ctx = api.HmmContext(pm.tp, pm.sseq, pm.n_sen)
    d_scr = torch.from_numpy(scr).cuda()
    with pytest.raises(api.PsbError, match=r"%d HMMs .* exceed the %d " % (lim + 1, lim)):
        ctx.kws(d_scr.data_ptr(), np.array([0, 30], np.int32), *cfg, -1080, -23)
    pm2, cfg2 = _case(n_emit, 40, _chains(lim - 40, 300, seed=1), seed=3)
    hits, n = ctx.kws(d_scr.data_ptr(), np.array([0, 30], np.int32), *cfg2, -1080, -23)
    assert np.array_equal(hits[0], oracle.kws_run(pm.tp, pm.sseq, *cfg2, -1080, -23, scr))
    ctx.close()


@pytest.fixture(scope="module")
def spotters(tmp_path_factory):
    _needs_ref_files()
    from pocketsphinx_b200.kws import KeywordSpotter
    f = tmp_path_factory.mktemp("kws") / "b.list"
    f.write_text("forward /1e-20/\nten meters /1e-30/\ngo /1e-10/\nbackward /1e-40/\n")
    s = dict(a=KeywordSpotter(HD, DIC, keyphrase="forward", kws_threshold="1e-20", max_utts=8, max_frames=4096),
             b=KeywordSpotter(HD, DIC, kws=str(f), max_utts=8, max_frames=4096),
             file=KeywordSpotter(HD, DIC, kws=KWS_FILE, max_utts=8, max_frames=4096))
    yield s
    for x in s.values():
        x.close()


def test_spot_senscr_equals_reference_detections(spotters):
    """On the reference's own senone scores of goforward.raw: exactly the reference's detection lists (tags a, b)."""
    import torch
    g = golden("en_us_kws.npz")
    scr = golden("en_us_goforward.npz")["senscr"]
    d = torch.from_numpy(np.concatenate([scr, scr])).cuda()
    for tag in ("a", "b"):
        s = spotters[tag]
        out = s.spot_senscr(d.data_ptr(), np.array([0, len(scr), 2 * len(scr)], np.int32))
        for o in out:
            got = np.array([(s.keyphrases.index(k), sf, ef, p, a) for k, sf, ef, p, a in o["detections"]], np.int32)
            assert np.array_equal(got.reshape(-1, 5), g[tag + "_det"]), tag
        assert out[0] == out[1]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("source", ["a", "file"])
def test_spot_raw_batch_matches_reference_live_run(spotters, source):
    """Audio in: goforward.raw whole, cut, and twice in one batch; the reference's live run's detections (same
    keyphrases in the same order, start and end frames within 2, as the device front end agrees with the
    reference's to 1e-4 relative), identical results for identical utterances."""
    from oracle import refdrv
    if not refdrv.available():
        pytest.skip("oracle/_ref/libpsref.so not built")
    from pocketsphinx_b200 import kws
    s = spotters[source]
    go = np.fromfile(GO, np.int16)
    utts = [go, go[:30000], go]
    out = s.spot_raw_batch(utts)
    assert out[0] == out[2]
    if source == "a":
        kv, listed = dict(keyphrase="forward", kws_threshold="1e-20"), ["forward"]
    else:
        kv, listed = dict(keyfile=KWS_FILE), [p for p, _ in kws.read_kws_list(KWS_FILE, s.def_threshold)]
    n_det = 0
    for pcm, o in zip(utts[:2], out[:2]):
        want = refdrv.kws(HD, DIC, pcm, **kv)
        assert abs(o["n_frames"] - want["n_frames"]) <= 1
        assert [d[0] for d in o["detections"]] == [listed[k] for k in want["det"][:, 0]]
        for d, w in zip(o["detections"], want["det"]):
            assert abs(d[1] - w[1]) <= 2 and abs(d[2] - w[2]) <= 2, (d, w)
        n_det += len(want["det"])
    assert n_det > 0


def test_refused_batch_leaves_the_spotter_usable(spotters):
    s = spotters["a"]
    go = np.fromfile(GO, np.int16)
    with pytest.raises(ValueError, match=r"max_frames \(4096\)"):
        s.spot_raw_batch([go, go, np.zeros(16000 * 40, np.int16)])
    with pytest.raises(ValueError, match=r"max_utts \(8\)"):
        s.spot_raw_batch([go[:2000]] * 9)
    assert s.spot_raw_batch([go])[0]["detections"]
