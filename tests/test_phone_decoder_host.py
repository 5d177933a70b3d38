"""CPU: phone decoding's host side against the compiled reference.

* psb_allphone_lm_tables (through phones.phone_lm_tables) against the reference's own phone-LM tables, every cell,
  at three -lw / -wip settings, with the remap of phones the LM lacks and its refusals.
* The host rules of PhoneDecoder (phones.phone_result over the segments of the C restatement of the search, which
  stands in for allphone_net_kernel) against the reference's ps_get_hyp / ps_seg_iter, run from the same audio
  through its public API: hyp, score and every segment.
"""
import ctypes as C

import numpy as np
import pytest

import phone_cases as P

pytestmark = pytest.mark.skipif(not P.have_ref(), reason="oracle/_ref (compiled reference and its data) not present")


@pytest.fixture(scope="module")
def goforward():
    return np.fromfile(P.GOFORWARD, np.int16)


@pytest.fixture(scope="module")
def phone_lm():
    from pocketsphinx_b200 import lmio
    return lmio.read_lm_bin(P.PHONE_LM)


@pytest.fixture(scope="module")
def mdef():
    import os
    from pocketsphinx_b200 import s3io
    return s3io.read_mdef(os.path.join(P.EN_US, "mdef"))


@pytest.mark.parametrize("lw,wip", [(6.5, 0.65), (2.0, 0.65), (9.5, 0.2)])
def test_lm_tables_equal_the_reference_in_every_cell(goforward, phone_lm, mdef, lw, wip):
    from oracle import refdrv
    from pocketsphinx_b200 import phones
    want = refdrv.allphone(P.EN_US, goforward[:1600], allphone=P.PHONE_LM, lw=lw, wip=wip)
    bg, tg = phones.phone_lm_tables(phone_lm, mdef["ciname"], int(mdef["sil"]), lw, wip)
    assert bg.shape == (42, 42) and tg.shape == (42, 42, 42)
    assert np.array_equal(bg, want["bg"]) and np.array_equal(tg, want["tg"])
    assert len(np.unique(tg)) > 100                     # trigram, bigram and backed-off cells all occur


def test_phones_the_lm_lacks_score_as_sil(phone_lm, mdef):
    from pocketsphinx_b200 import phones
    names, sil = list(mdef["ciname"]), int(mdef["sil"])
    missing = [c for c, n in enumerate(names) if n not in set(phone_lm["words"])]
    fillers = [c for c in range(len(names)) if mdef["phone_filler"][c] and c != sil]
    assert fillers and set(fillers) <= set(missing)     # en-us's filler phones are not in en-us-phone.lm.bin
    bg, tg = phones.phone_lm_tables(phone_lm, names, sil)
    for c in missing:
        assert np.array_equal(bg[c], bg[sil]) and np.array_equal(bg[:, c], bg[:, sil])
        assert np.array_equal(tg[c], tg[sil]) and np.array_equal(tg[:, c], tg[:, sil]) and np.array_equal(tg[:, :, c], tg[:, :, sil])


def test_lm_without_sil_is_refused(phone_lm, mdef):
    from pocketsphinx_b200 import phones
    lm = dict(phone_lm, words=["SIL_" if w == "SIL" else w for w in phone_lm["words"]])
    with pytest.raises(ValueError, match="Phonetic LM does not have SIL phone in vocabulary"):
        phones.phone_lm_tables(lm, mdef["ciname"], int(mdef["sil"]))
    lm["words"] = lm["words"] + ["<UNK>"]               # with <UNK> in the LM, SIL's lookup gives <UNK>: refused alike
    lm["counts"] = [len(lm["words"])] + lm["counts"][1:]
    with pytest.raises(ValueError, match="does not have SIL"):
        phones.phone_lm_tables(lm, mdef["ciname"], int(mdef["sil"]))


def test_more_than_64_phones_and_bad_widmaps_are_refused_before_any_write(phone_lm, mdef):
    from pocketsphinx_b200 import _lib, lmio, phones
    names = ["P%d" % i for i in range(65)]
    with pytest.raises(ValueError, match="64"):
        phones.phone_lm_tables(dict(phone_lm, words=phone_lm["words"] + names), names, 0)
    L = _lib.lib()
    P_ = lambda a: a.ctypes.data_as(C.c_void_p)         # noqa: E731
    bg, tg = np.full((65, 65), 7, np.int32), np.full(65 ** 3, 7, np.int32)
    block = lmio.lm_arrays(phone_lm, names)
    assert L.psb_allphone_lm_tables(P_(block), 65, P_(bg), P_(tg)) < 0 and "64" in L.psb_last_error().decode()
    n = len(mdef["ciname"])
    for bad in (-1, phone_lm["counts"][0]):             # <UNK> / -1 is not a phone LM word; nor is one past the LM
        block = lmio.lm_arrays(phone_lm, list(mdef["ciname"]))
        block[10:10 + n] = 0
        block[10 + 5] = bad
        assert L.psb_allphone_lm_tables(P_(block), n, P_(bg), P_(tg)) < 0
        assert "outside the LM" in L.psb_last_error().decode() or "out of range" in L.psb_last_error().decode()
    assert L.psb_allphone_lm_tables(P_(block), n - 1, P_(bg), P_(tg)) < 0 and "words" in L.psb_last_error().decode()
    assert (bg == 7).all() and (tg == 7).all()


def _check(hmm, pcm, tmp_path, allphone=None, **kv):
    """PhoneDecoder's host rules on the search's segments against the reference's public API, from the same audio
    at the same settings."""
    from pocketsphinx_b200 import allphone_net, phones
    from pocketsphinx_b200.model import PackedModel
    search = phones.search_setup(hmm, allphone, **kv)
    pm = PackedModel.from_dir(hmm)
    scr = P.ref_senscr(hmm, pcm, tmp_path)
    segs = P.oracle_segs(pm.tp, pm.sseq, search, allphone_net.expand_links(search["net"]), scr)
    got = phones.phone_result(segs, 0, len(scr), search["ciname"])
    want = P.ref_phones(hmm, allphone, pcm=pcm, **kv)
    assert got["hyp"] == want["hyp"] and got["score"] == want["score"]
    assert got["seg"] == want["seg"]
    assert got["seg"][-1][2] == len(scr) - 1 and got["status"] == 0 and got["reason"] is None
    return got


def test_ci_net_without_lm(goforward, tmp_path):
    got = _check(P.EN_US, goforward, tmp_path)
    assert got["hyp"].startswith("SIL ") and got["score"] == sum(s[3] + s[4] for s in got["seg"])


def test_ci_net_with_phone_lm(goforward, tmp_path):
    got = _check(P.EN_US, goforward, tmp_path, P.PHONE_LM)
    assert any(s[4] != 0 for s in got["seg"])


def test_cd_net_with_phone_lm(goforward, tmp_path):
    _check(P.EN_US, goforward, tmp_path, P.PHONE_LM, allphone_ci="no")


@pytest.mark.parametrize("lm", [False, True])
def test_non_default_search_settings(goforward, tmp_path, lm):
    _check(P.EN_US, goforward, tmp_path, P.PHONE_LM if lm else None, beam="1e-30", pbeam="1e-20", pip="0.3", lw="3.7",
           wip="0.4")


def test_tidigits_ci_net(tmp_path):
    _check(P.TIDIGITS, np.fromfile(P.DHD, np.int16), tmp_path)


def test_status_rows_leave_the_other_utterances_alone():
    from pocketsphinx_b200 import phones
    names = ["SIL", "AA", "B"]
    segs = [np.array([[0, 0, 3, -50, 0], [2, 4, 9, -70, -5]], np.int32), np.zeros((0, 5), np.int32),
            np.array([[1, 0, 4, -10, -1]], np.int32), np.zeros((0, 5), np.int32)]
    out = [phones.phone_result(s, st, T, names) for s, st, T in zip(segs, [0, 1, 0, 0], [10, 7, 5, 0])]
    assert out[0]["hyp"] == "SIL B" and out[0]["score"] == -125 and out[0]["seg"] == [("SIL", 0, 3, -50, 0), ("B", 4, 9, -70, -5)]
    assert out[1]["hyp"] is None and out[1]["score"] is None and out[1]["status"] == 1 and "overflow" in out[1]["reason"]
    assert out[2]["hyp"] == "AA" and out[2]["score"] == -11 and out[2]["status"] == 0
    assert out[3]["hyp"] is None and out[3]["seg"] == [] and out[3]["reason"] is None and out[3]["n_frames"] == 0


def test_lms_read_lm_bin_refuses_stay_refused_before_the_device(tmp_path):
    from pocketsphinx_b200.phones import PhoneDecoder
    arpa = tmp_path / "phone.lm"
    arpa.write_text("\\data\\\nngram 1=2\n\n\\1-grams:\n-1.0 SIL\n-1.0 AA\n\n\\end\\\n")
    with pytest.raises(ValueError, match="not a binary trie LM"):
        PhoneDecoder(P.EN_US, str(arpa))
    with pytest.raises(ValueError, match="allphone_ci"):
        PhoneDecoder(P.EN_US, allphone_ci="maybe")
