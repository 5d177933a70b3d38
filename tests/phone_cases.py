"""Helpers of the phone-decoding tests (test_phone_decoder_host.py, test_gpu_phone_decoder.py).

* `ref_phones`: the reference's allphone search on one utterance through its public API (oracle/_ref/libpsref.so,
  bound with ctypes): ps_init with -allphone (or ps_add_allphone without an LM), -allphone_ci and -compallsen yes,
  then ps_decode_raw (audio) or ps_decode_senscr (a senone dump), ps_get_hyp and ps_seg_iter.
* `ref_senscr`: the reference's own senone scores for an utterance (its -senlogdir dump, read back).
* `oracle_segs`: the C restatement of the search (pso_allphone_run / pso_allphone_lm_run) and its backtrace, the
  CPU stand-in for allphone_net_kernel.
"""
import ctypes as C
import os
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
EN_US = os.path.join(REF, "model", "en-us")
# the phone LM the reference ships with its en-us model, kept as a test fixture
PHONE_LM = os.path.join(ROOT, "tests", "golden", "en-us-phone.lm.bin")
TIDIGITS = os.path.join(REF, "model", "tidigits_hmm")
GOFORWARD = os.path.join(REF, "data", "goforward.raw")
DHD = os.path.join(REF, "data", "dhd.2934z.raw")
# the n-gram setup ps_decode_senscr writes the senone dump under (the scores do not depend on it: -compallsen yes)
SENDUMP_ARGS = {EN_US: (os.path.join(REF, "model", "en-us.lm.bin"), os.path.join(REF, "model", "cmudict-en-us.dict")),
                TIDIGITS: (os.path.join(REF, "model", "tidigits_lm", "tidigits.lm.bin"),
                           os.path.join(REF, "model", "tidigits_lm", "tidigits.dic"))}


def have_ref():
    return os.path.exists(os.path.join(REF, "libpsref.so")) and os.path.exists(PHONE_LM) and os.path.isdir(TIDIGITS)


_REF = None


def _ref():
    global _REF
    if _REF is None:
        from oracle import refdrv
        L = refdrv.lib()
        V, I, P = C.c_void_p, C.c_int, C.POINTER(C.c_int32)
        for name, res, args in (("ps_config_init", V, [V]), ("ps_config_set_str", V, [V, C.c_char_p, C.c_char_p]),
                                ("ps_config_free", I, [V]), ("ps_init", V, [V]), ("ps_free", I, [V]),
                                ("ps_add_allphone", I, [V, C.c_char_p, V]), ("ps_activate_search", I, [V, C.c_char_p]),
                                ("ps_decode_raw", C.c_long, [V, V, C.c_long]), ("ps_decode_senscr", I, [V, V]),
                                ("ps_get_hyp", C.c_char_p, [V, P]),
                                ("ps_seg_iter", V, [V]), ("ps_seg_next", V, [V]), ("ps_seg_word", C.c_char_p, [V]),
                                ("ps_seg_frames", None, [V, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
                                ("ps_seg_prob", C.c_int32, [V, P, P, P]),
                                ("err_set_loglevel_str", C.c_char_p, [C.c_char_p])):
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        libc = C.CDLL(None)
        libc.fopen.restype, libc.fopen.argtypes = V, [C.c_char_p, C.c_char_p]
        libc.fclose.argtypes = [V]
        _REF = L, libc
    return _REF


def ref_phones(hmm, allphone=None, pcm=None, senfile=None, **kv):
    """The reference's phone decoding of one utterance, from audio (pcm, ps_decode_raw) or from a senone dump
    (senfile, ps_decode_senscr).  Returns dict(hyp, score (None with hyp), seg [(name, sf, ef, ascr, lscr)])."""
    L, libc = _ref()
    L.err_set_loglevel_str(b"ERROR")
    cfg = L.ps_config_init(None)
    settings = [("hmm", hmm), ("dither", "no"), ("compallsen", "yes"), ("lm", None), ("dict", None)]
    if allphone is not None:
        settings.append(("allphone", allphone))
    for k, v in settings + [(k, str(v)) for k, v in kv.items()]:
        L.ps_config_set_str(cfg, k.encode(), None if v is None else v.encode())
    ps = L.ps_init(cfg)
    if not ps:
        L.ps_config_free(cfg)
        raise RuntimeError("ps_init failed for " + hmm)
    tmp = None
    try:
        if allphone is None and (L.ps_add_allphone(ps, b"_ap", None) < 0 or L.ps_activate_search(ps, b"_ap") < 0):
            raise RuntimeError("ps_add_allphone failed")
        if pcm is not None:
            tmp = tempfile.NamedTemporaryFile(suffix=".raw", delete=False)
            tmp.write(np.ascontiguousarray(pcm, np.int16).tobytes())
            tmp.close()
            path = tmp.name
        else:
            path = senfile
        fh = libc.fopen(path.encode(), b"rb")
        assert fh, path
        try:
            rc = L.ps_decode_raw(ps, fh, -1) if pcm is not None else L.ps_decode_senscr(ps, fh)
        finally:
            libc.fclose(fh)
        assert rc >= 0, rc
        score = C.c_int32(0)
        hyp = L.ps_get_hyp(ps, C.byref(score))
        seg = []
        it = L.ps_seg_iter(ps)
        while it:
            sf, ef = C.c_int(), C.c_int()
            L.ps_seg_frames(it, C.byref(sf), C.byref(ef))
            a, l, b = C.c_int32(), C.c_int32(), C.c_int32()
            L.ps_seg_prob(it, C.byref(a), C.byref(l), C.byref(b))
            seg.append((L.ps_seg_word(it).decode(), sf.value, ef.value, a.value, l.value))
            it = L.ps_seg_next(it)
        return dict(hyp=None if hyp is None else hyp.decode(), score=None if hyp is None else score.value, seg=seg)
    finally:
        if tmp is not None:
            os.unlink(tmp.name)
        L.ps_free(ps)
        L.ps_config_free(cfg)


def ref_senscr(hmm, pcm, tmpdir):
    """The reference's own int16 senone scores of one utterance (every senone)."""
    from oracle import refdrv
    from pocketsphinx_b200 import api
    out = os.path.join(str(tmpdir), "ref_%d.sen" % len(pcm))
    refdrv.decode_senscr(hmm, *SENDUMP_ARGS[hmm], pcm=pcm, senout=out, pl_window=0)
    return api.sendump_read(out)


def oracle_segs(tp, sseq, search, links, scr):
    """The phone segments (ci, sf, ef, score, tscore) of one utterance by the C restatement of the search:
    search = phones.search_setup's result, links = allphone_net.expand_links(search["net"])."""
    from oracle import oracle
    net, T = search["net"], len(scr)
    if T == 0:
        return np.zeros((0, 5), np.int32)
    so, s = links
    if search["bg"] is None:
        hist, _ = oracle.allphone_run(tp, sseq, net["ssid"], net["tmatid"], so, s, net["start"], search["beam"],
                                      search["pbeam"], search["inspen"], scr)
        return oracle.allphone_backtrace(hist, net["ci"], T - 1, search["inspen"])
    hist, _ = oracle.allphone_lm_run(tp, sseq, net["ssid"], net["tmatid"], so, s, net["start"], search["beam"],
                                     search["pbeam"], net["ci"], search["bg"], search["tg"], scr)
    return oracle.allphone_backtrace_lm(hist, net["ci"], T - 1)
