"""GPU (-m gpu): phones.PhoneDecoder against the reference's allphone search run through its public API
(ps_decode_raw / ps_decode_senscr, ps_get_hyp, ps_seg_iter; tests/phone_cases.py).

* decode_senscr on the reference's own senone scores: hyp, score and every segment equal, for the CI and the CD
  net, with and without the phone LM, at default and other settings, in ragged batches with 0- and 1-frame
  utterances.
* decode_raw_batch from audio (the device front end): the same phones and frames as the reference from the same
  PCM, and results that do not depend on batch order or batch size.
"""
import os

import numpy as np
import pytest

import phone_cases as P

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not P.have_ref(), reason="oracle/_ref not present")]

CONFIGS = {
    "ci": (None, {}),
    "ci_lm": (P.PHONE_LM, {}),
    "cd_lm": (P.PHONE_LM, dict(allphone_ci="no")),
    "cd": (None, dict(allphone_ci="no")),
    "ci_settings": (None, dict(beam="1e-30", pbeam="1e-20", pip="0.3", lw="3.7")),
    "ci_lm_settings": (P.PHONE_LM, dict(beam="1e-30", pbeam="1e-20", lw="3.7", wip="0.4")),
}


@pytest.fixture(scope="module")
def api():
    from pocketsphinx_b200 import api
    assert api.device_count() > 0, "no CUDA device visible"
    return api


@pytest.fixture(scope="module")
def goforward():
    return np.fromfile(P.GOFORWARD, np.int16)


@pytest.fixture(scope="module")
def go_scores(goforward, tmp_path_factory):
    return P.ref_senscr(P.EN_US, goforward, tmp_path_factory.mktemp("sen"))


def _ref_from_scores(scr, tmp_path, allphone, kv):
    """The reference's result from these senone scores (ps_decode_senscr on a dump of them)."""
    from pocketsphinx_b200 import api
    if len(scr) == 0:                                   # the dump format has no empty form: no audio is no frames
        return P.ref_phones(P.EN_US, allphone, pcm=np.zeros(0, np.int16), **kv)
    path = os.path.join(str(tmp_path), "u%d.sen" % len(scr))
    api.sendump_write(path, scr, mdef_file=os.path.join(P.EN_US, "mdef"))
    return P.ref_phones(P.EN_US, allphone, senfile=path, **kv)


def _same(got, want, what):
    assert got["status"] == 0 and got["reason"] is None, what
    assert got["hyp"] == want["hyp"], what
    assert got["score"] == want["score"], what
    assert got["seg"] == want["seg"], what


@pytest.mark.parametrize("name", list(CONFIGS))
def test_decode_senscr_equals_the_reference(api, goforward, go_scores, tmp_path, name):
    import torch
    from pocketsphinx_b200.phones import PhoneDecoder
    allphone, kv = CONFIGS[name]
    want = P.ref_phones(P.EN_US, allphone, pcm=goforward, **kv)
    utts = [go_scores, go_scores[:0], go_scores[:1], go_scores[:2], go_scores[:120]]
    d = torch.from_numpy(np.concatenate(utts)).cuda()
    off = np.concatenate([[0], np.cumsum([len(u) for u in utts])]).astype(np.int32)
    dec = PhoneDecoder(P.EN_US, allphone, max_utts=8, max_frames=4096, **kv)
    try:
        got = dec.decode_senscr(d.data_ptr(), off)
        assert [g["n_frames"] for g in got] == [len(u) for u in utts]
        _same(got[0], want, name)
        assert got[0]["hyp"] is not None and got[0]["seg"][-1][2] == len(go_scores) - 1
        for u in range(1, len(utts)):
            _same(got[u], _ref_from_scores(utts[u], tmp_path, allphone, kv), (name, u))
        # 0 frames: no history; 1 frame: only entry 0, which no segment reports; 2 frames: one SIL segment
        assert got[1]["hyp"] is None and got[2]["hyp"] is None and got[3]["hyp"] == "SIL"
        # the same utterances in the reverse order, and each alone
        d_rev = torch.from_numpy(np.concatenate(utts[::-1])).cuda()
        off_rev = np.concatenate([[0], np.cumsum([len(u) for u in utts[::-1]])]).astype(np.int32)
        assert dec.decode_senscr(d_rev.data_ptr(), off_rev)[::-1] == got
        for u in range(len(utts)):
            assert dec.decode_senscr(d.data_ptr() + int(off[u]) * go_scores.shape[1] * 2,
                                     np.array([0, len(utts[u])], np.int32)) == [got[u]]
        if name == "cd":
            assert dec.ctx.allphone_net(d.data_ptr(), off[:2], dec.search["net"], dec.search["beam"], dec.search["pbeam"],
                                        dec.search["inspen"])["n_hist"][0] == 7805547
    finally:
        dec.close()


def _from_audio(api, hmm, utts, allphone=None, **kv):
    from pocketsphinx_b200.phones import PhoneDecoder
    dec = PhoneDecoder(hmm, allphone, max_utts=16, max_frames=1 << 14, **kv)
    try:
        return dec.decode_raw_batch(utts)
    finally:
        dec.close()


@pytest.mark.parametrize("hmm,raw,allphone", [(P.EN_US, P.GOFORWARD, None), (P.EN_US, P.GOFORWARD, P.PHONE_LM),
                                              (P.TIDIGITS, P.DHD, None)])
def test_decode_raw_batch_matches_the_reference_from_audio(api, hmm, raw, allphone, capsys):
    pcm = np.fromfile(raw, np.int16)
    want = P.ref_phones(hmm, allphone, pcm=pcm)
    got = _from_audio(api, hmm, [pcm], allphone)[0]
    assert got["status"] == 0 and got["hyp"] == want["hyp"]
    assert [s[:3] for s in got["seg"]] == [s[:3] for s in want["seg"]]
    # scores: the device front end agrees with the reference's to 1e-4 relative (DESIGN 4.6), so a senone score
    # may differ by one unit in a few frames; the path scores move by as much
    d_seg = [(g[3] - w[3], g[4] - w[4]) for g, w in zip(got["seg"], want["seg"])]
    with capsys.disabled():
        print("\n%s %s: score %d (reference %d), segment score differences %s" % (
            os.path.basename(hmm), "phone LM" if allphone else "no LM", got["score"], want["score"],
            [d for d in d_seg if d != (0, 0)]))
    assert all(t == 0 for _, t in d_seg)                 # the LM scores depend on the phones alone
    assert abs(got["score"] - want["score"]) <= 1e-3 * abs(want["score"])


def test_from_audio_results_do_not_depend_on_batch_order_or_size(api, goforward):
    dhd = np.fromfile(P.DHD, np.int16)
    utts = [goforward, goforward[:16000], np.zeros(0, np.int16), goforward[:400], goforward[8000:]]
    for allphone in (None, P.PHONE_LM):
        whole = _from_audio(api, P.EN_US, utts, allphone)
        rev = _from_audio(api, P.EN_US, utts[::-1], allphone)[::-1]
        one = [_from_audio(api, P.EN_US, [u], allphone)[0] for u in utts]
        assert whole == rev == one
        assert whole[2]["hyp"] is None and whole[2]["n_frames"] == 0
    t = _from_audio(api, P.TIDIGITS, [dhd, dhd[:8000], dhd])
    assert t[0] == t[2] == _from_audio(api, P.TIDIGITS, [dhd])[0]


def test_batch_bounds_are_refused_with_the_spotter_messages(api, goforward):
    from pocketsphinx_b200.phones import PhoneDecoder
    dec = PhoneDecoder(P.EN_US, max_utts=2, max_frames=290)
    try:
        with pytest.raises(ValueError, match="more than this PhoneDecoder's max_utts"):
            dec.decode_raw_batch([goforward[:1600]] * 3)
        with pytest.raises(ValueError, match="more than this PhoneDecoder's max_frames"):
            dec.decode_raw_batch([goforward, goforward[:3200]])
        assert dec.decode_raw_batch([goforward])[0]["hyp"].startswith("SIL")
    finally:
        dec.close()
