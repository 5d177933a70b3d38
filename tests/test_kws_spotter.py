"""CPU (needs oracle/_ref/libpsref.so): pocketsphinx_b200.kws.KeywordSpotter's host code -- -kws list parsing, the
keyphrase chains and quantised settings, the detection list and the hyp / seg rules with -kws_delay -- against the
compiled reference's own kws search on goforward.raw.  The device stages are stubbed: the senone scores come from the
compiled reference's scorer and the search from the C restatement of kws_search.c (oracle.kws_run), which the GPU
tests hold the kernel equal to; the reference's answers come from its public API (ps_get_hyp, ps_seg_iter)."""
import ctypes as C
import os
import types

import numpy as np
import pytest

from conftest import GOLDEN, golden
from oracle import oracle, refdrv
from pocketsphinx_b200 import api as real_api, decoder, kws

pytestmark = pytest.mark.skipif(not refdrv.available(), reason="oracle/_ref/libpsref.so not built")
REF = os.path.dirname(refdrv.LIB_PATH)
HD, DIC = os.path.join(REF, "model", "en-us"), os.path.join(REF, "model", "cmudict-en-us.dict")
KWS_FILE = os.path.join(GOLDEN, "goforward.kws")                   # the reference's own test list (test/data)
GO = os.path.join(REF, "data", "goforward.raw")


def reference_run(pcm, keyphrase=None, keyfile=None, **kv):
    """The reference decoder with -keyphrase / -kws on one utterance (all senones, as the device scores them):
    ps_get_hyp and every ps_seg_iter segment (word, sf, ef, prob, ascr) after ps_end_utt."""
    L = C.CDLL(refdrv.LIB_PATH)
    L.ps_config_init.restype = C.c_void_p
    L.ps_config_set_str.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    L.ps_init.restype = C.c_void_p; L.ps_init.argtypes = [C.c_void_p]
    L.ps_start_utt.argtypes = [C.c_void_p]; L.ps_end_utt.argtypes = [C.c_void_p]
    L.ps_process_raw.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int]
    L.ps_get_hyp.restype = C.c_char_p; L.ps_get_hyp.argtypes = [C.c_void_p, C.c_void_p]
    L.ps_get_n_frames.argtypes = [C.c_void_p]
    L.ps_seg_iter.restype = C.c_void_p; L.ps_seg_iter.argtypes = [C.c_void_p]
    L.ps_seg_next.restype = C.c_void_p; L.ps_seg_next.argtypes = [C.c_void_p]
    L.ps_seg_word.restype = C.c_char_p; L.ps_seg_word.argtypes = [C.c_void_p]
    L.ps_seg_frames.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.ps_seg_prob.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.ps_free.argtypes = [C.c_void_p]; L.ps_config_free.argtypes = [C.c_void_p]
    L.err_set_loglevel(4)
    cfg = L.ps_config_init(None)
    settings = dict(hmm=HD, dict=DIC, dither="no", compallsen="yes", **kv)
    if keyfile:
        settings["kws"] = keyfile
    else:
        settings["keyphrase"] = keyphrase
    L.ps_config_set_str(cfg, b"lm", None)
    for k, v in settings.items():
        L.ps_config_set_str(cfg, k.encode(), str(v).encode())
    ps = L.ps_init(cfg)
    assert ps
    pcm = np.ascontiguousarray(pcm, np.int16)
    L.ps_start_utt(ps)
    L.ps_process_raw(ps, pcm.ctypes.data, len(pcm), 0, 1)
    L.ps_end_utt(ps)
    h = L.ps_get_hyp(ps, None)
    seg, it = [], L.ps_seg_iter(ps)
    while it:
        sf, ef, ascr, lscr, lback = C.c_int(), C.c_int(), C.c_int32(), C.c_int32(), C.c_int32()
        L.ps_seg_frames(it, C.byref(sf), C.byref(ef))
        prob = L.ps_seg_prob(it, C.byref(ascr), C.byref(lscr), C.byref(lback))
        seg.append((L.ps_seg_word(it).decode(), sf.value, ef.value, prob, ascr.value))
        it = L.ps_seg_next(it)
    n = L.ps_get_n_frames(ps)
    L.ps_free(ps); L.ps_config_free(cfg)
    return dict(hyp=None if h is None else h.decode(), seg=seg, n_frames=n)


class _FE:
    sample_offsets = staticmethod(real_api.FrontEnd.sample_offsets)
    def __init__(self, desc, device=0, opts=None): pass
    def n_frames(self, n): return n // 160 + 1
    def close(self): pass


class _Model:
    def __init__(self, pm, device=0): pass
    def close(self): pass


class _Batch:
    """Scores from the compiled reference's scorer (a fresh acmod per utterance, all senones)."""
    def __init__(self, model, max_utts, max_frames): pass
    def score_pcm(self, fe, pcm, off):
        scr = []
        for u in range(len(off) - 1):
            ref = refdrv.RefModel(HD)
            scr.append(np.ascontiguousarray(ref.score(ref.featurize_fresh(pcm[off[u]:off[u + 1]]))))
            ref.close()
        self.scr = np.ascontiguousarray(np.concatenate(scr))
        return np.cumsum([0] + [len(s) for s in scr]).astype(np.int32)
    def senscr_device_ptr(self): return self.scr.ctypes.data
    def close(self): pass


class _Ctx:
    """HmmContext.kws served by the C restatement of kws_search.c, one utterance at a time."""
    def __init__(self, tp, sseq, n_sen, device=0):
        self.tp, self.sseq, self.n_sen = tp, sseq, n_sen
    def kws(self, ptr, utt_off, pl_ssid, pl_tmat, kp_off, kp_thresh, kp_ssid, kp_tmat, beam, plp, cap=None):
        out = []
        for u in range(len(utt_off) - 1):
            T = int(utt_off[u + 1] - utt_off[u])
            a = (C.c_int16 * (T * self.n_sen)).from_address(ptr + int(utt_off[u]) * self.n_sen * 2)
            scr = np.frombuffer(a, np.int16).reshape(T, self.n_sen)
            out.append(oracle.kws_run(self.tp, self.sseq, pl_ssid, pl_tmat, kp_off, kp_thresh, kp_ssid, kp_tmat, beam, plp, scr))
        return out, np.array([len(h) for h in out], np.int32)
    def close(self): pass


@pytest.fixture
def stubbed(monkeypatch):
    ns = types.SimpleNamespace(FrontEnd=_FE, Model=_Model, Batch=_Batch, HmmContext=_Ctx)
    monkeypatch.setattr(decoder, "api", ns)
    monkeypatch.setattr(kws, "api", ns)


def _list_file(tmp_path, text):
    p = tmp_path / "phrases.list"
    p.write_bytes(text.encode())
    return str(p)


def test_keyphrase_and_list_settings_equal_the_references(stubbed, tmp_path):
    """-keyphrase: chain, threshold, beam and plp as tests/golden/en_us_kws.npz holds them (tag a); a -kws list with
    per-phrase thresholds (tag b): the same, in the reference's (reverse file) order."""
    g = golden("en_us_kws.npz")
    a = kws.KeywordSpotter(HD, DIC, keyphrase="forward", kws_threshold="1e-20")
    f = _list_file(tmp_path, "forward /1e-20/\nten meters /1e-30/\ngo /1e-10/\nbackward /1e-40/\n")
    b = kws.KeywordSpotter(HD, DIC, kws=f)
    assert b.keyphrases == ["backward ", "go ", "ten meters ", "forward "] and b.dropped == []
    for tag, s in (("a", a), ("b", b)):
        for k in ("pl_ssid", "pl_tmat", "kp_off", "kp_thresh", "kp_ssid", "kp_tmat"):
            assert np.array_equal(getattr(s, k), g[tag + "_" + k]), (tag, k)
        assert (s.beam, s.plp) == (int(g[tag + "_beam"]), int(g[tag + "_plp"]))


@pytest.mark.parametrize("text", [
    "# a comment first\n  forward  \n\n\t\ngo /1e-5/\n# another\n  ten meters/1e-25/  \nmeters\n",
    "forward /1e-20/\nforward\ngo forward /1e-40/\n/1e-3/\njust a line /\nx/0.5/\n",
    "forward\r\n  \r\n go \r\nbackward /abc/\n"])
def test_list_parsing_equals_the_references(text, tmp_path):
    """Comments, blank and whitespace-only lines, trimming, per-phrase thresholds with and without a space before
    the slash, unparsable thresholds, duplicate phrases, CRLF lines: thresholds and chain lengths in list order
    equal what the reference's kws search built from the same file."""
    f = _list_file(tmp_path, text)
    pcm = np.fromfile(GO, np.int16)[:4000]
    want = refdrv.kws(HD, DIC, pcm, keyfile=f)
    got = kws.read_kws_list(f, kws._logs(1e-30, 1.0001))
    assert [t for _, t in got] == want["kp_thresh"].tolist()
    assert len(got) == len(want["kp_off"]) - 1


@pytest.mark.parametrize("delay", [0, 10, 100000])
@pytest.mark.parametrize("source", ["keyphrase", "goforward.kws", "overlaps"])
def test_hyp_and_segments_equal_the_references(stubbed, tmp_path, source, delay):
    """goforward.raw with -keyphrase forward, with the reference's own goforward.kws (two phrases with words missing
    from the dictionary, one empty phrase), and with a list whose detections overlap -- the same phrase twice, and
    "go forward" over "forward" -- at a threshold low enough for many hits: ps_get_hyp and ps_seg_iter, -kws_delay 0,
    10 and longer than the utterance."""
    pcm = np.fromfile(GO, np.int16)
    kv = dict(kws_delay=delay)
    if source == "keyphrase":
        kv["keyphrase"] = "forward"
    elif source == "goforward.kws":
        kv["kws"] = KWS_FILE
    else:
        kv["kws"] = _list_file(tmp_path, "forward\ngo forward\nforward\nten\nmeters\nten meters\ngo\n")
        kv["kws_threshold"] = "1e-60"
    s = kws.KeywordSpotter(HD, DIC, **kv)
    out = s.spot_raw_batch([pcm])[0]
    want = reference_run(pcm, keyphrase=kv.get("keyphrase"), keyfile=kv.get("kws"),
                         **{k: v for k, v in kv.items() if k not in ("keyphrase", "kws")})
    assert out["n_frames"] == want["n_frames"] - 1                 # ps_get_n_frames: acmod->output_frame + 1
    assert out["hyp"] == want["hyp"]
    assert out["seg"] == want["seg"]
    if source == "goforward.kws":
        assert sorted(s.dropped) == ["bad line / here", "non_existign_word"] and "" in s.keyphrases
    if source == "overlaps":
        assert len(out["detections"]) >= 3 and len({d[0] for d in out["detections"]}) >= 2
    if delay == 0:
        assert out["seg"], "the utterance has detections to report"


@pytest.mark.parametrize("tag", ["a", "b"])
def test_detection_list_equals_the_oracle(tag):
    """kws.detections on the raw hits of the reference's own scores equals the test oracle's kws_detections_add and
    the reference's final detection list."""
    g, m = golden("en_us_kws.npz"), golden("en_us_ptm_model.npz")
    hits = oracle.kws_run(m["tp"], m["sseq"], g[tag + "_pl_ssid"], g[tag + "_pl_tmat"], g[tag + "_kp_off"],
                          g[tag + "_kp_thresh"], g[tag + "_kp_ssid"], g[tag + "_kp_tmat"], int(g[tag + "_beam"]),
                          int(g[tag + "_plp"]), golden("en_us_goforward.npz")["senscr"])
    names = ["kp%d" % k for k in range(len(g[tag + "_kp_off"]) - 1)]
    got = [(int(d[0][2:]),) + d[1:] for d in kws.detections(hits, names)]
    assert np.array_equal(np.array(got, np.int32).reshape(-1, 5), oracle.kws_detections(hits))
    assert np.array_equal(np.array(got, np.int32).reshape(-1, 5), g[tag + "_det"])


def test_detections_merge_by_keyphrase_text():
    """Two list entries with the same text are one keyphrase to kws_detections_add (strcmp): their overlapping hits
    merge; a different phrase overlapping them is kept apart."""
    hits = np.array([[10, 0, 2, -50, -1], [11, 1, 3, -40, -1], [12, 2, 4, -10, -1], [30, 0, 20, -70, -1]], np.int32)
    d = kws.detections(hits, ["forward", "forward", "go forward"])
    assert d == [("forward", 20, 30, -70, -1), ("go forward", 4, 12, -10, -1), ("forward", 3, 11, -40, -1)]
    hyp, seg = kws.hyp_and_segments(d, 35, 5)                      # ef == frame - delay: in seg, not in hyp
    assert hyp == "forward go forward" and seg == list(reversed(d))
    hyp, seg = kws.hyp_and_segments(d, 35, 6)
    assert hyp == "forward go forward" and seg == [d[2], d[1]]
    hyp, seg = kws.hyp_and_segments(d, 35, 24)
    assert hyp is None and seg == [d[2]]
    assert kws.hyp_and_segments(d, 35, 0) == ("forward go forward forward", list(reversed(d)))


def test_both_or_neither_phrase_source_is_refused(stubbed):
    for kv in (dict(), dict(keyphrase="forward", kws=KWS_FILE)):
        with pytest.raises(ValueError, match="exactly one of keyphrase and kws"):
            kws.KeywordSpotter(HD, DIC, **kv)


def test_batch_bounds_are_refused_and_the_spotter_stays_usable(stubbed):
    s = kws.KeywordSpotter(HD, DIC, keyphrase="forward", max_utts=2, max_frames=400)
    pcm = np.fromfile(GO, np.int16)
    with pytest.raises(ValueError, match=r"max_frames \(400\)"):
        s.spot_raw_batch([pcm, pcm])
    with pytest.raises(ValueError, match=r"max_utts \(2\)"):
        s.spot_raw_batch([pcm[:1000]] * 3)
    assert s.spot_raw_batch([pcm[:20000]])[0]["n_frames"] > 0
