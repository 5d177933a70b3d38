"""Helpers of the forced-alignment tests (test_align_host.py, test_gpu_align.py).

* `phone_align`: `pocketsphinx single -phone_align yes` on one utterance through the compiled reference's public API
  (oracle/_ref/libpsref.so, bound with ctypes): decode, ps_set_alignment(ps, NULL), decode the same audio again,
  and read the alignment's three levels with ps_alignment_iter_name / _seg / _children.
* `band` / `align_run_banded`: tests/emul/align_banded.c, the C restatement of state_align_search with the token
  table kept only in each frame's band (built here against libpsoracle.so, into a temporary directory).
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


_REF = None


def _ref():
    global _REF
    if _REF is None:
        from oracle import refdrv
        L = refdrv.lib()
        V = C.c_void_p
        for name, res, args in (("ps_config_init", V, [V]), ("ps_config_set_str", V, [V, C.c_char_p, C.c_char_p]),
                                ("ps_config_free", C.c_int, [V]), ("ps_init", V, [V]), ("ps_free", C.c_int, [V]),
                                ("ps_start_utt", C.c_int, [V]), ("ps_end_utt", C.c_int, [V]),
                                ("ps_process_raw", C.c_int, [V, V, C.c_size_t, C.c_int, C.c_int]),
                                ("ps_set_alignment", C.c_int, [V, V]), ("ps_get_alignment", V, [V]),
                                ("ps_get_n_frames", C.c_int, [V]), ("ps_alignment_words", V, [V]),
                                ("ps_alignment_iter_next", V, [V]), ("ps_alignment_iter_children", V, [V]),
                                ("ps_alignment_iter_name", C.c_char_p, [V]),
                                ("ps_alignment_iter_seg", C.c_int, [V, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
                                ("err_set_loglevel_str", C.c_char_p, [C.c_char_p])):
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _REF = L
    return _REF


def _entries(L, it, parent, out, below=None):
    """Walks one level of an alignment from iterator `it` (consumed), appending (name, start, duration, score,
    parent); with `below`, each entry's children go to below[0] with below[1:] under them."""
    while it:
        st, du = C.c_int(), C.c_int()
        sc = L.ps_alignment_iter_seg(it, C.byref(st), C.byref(du))
        out.append((L.ps_alignment_iter_name(it).decode(), st.value, du.value, sc, parent))
        if below:
            _entries(L, L.ps_alignment_iter_children(it), len(out) - 1, below[0], below[1:])
        it = L.ps_alignment_iter_next(it)


def phone_align(hmmdir, lm, dictfile, pcm, **kv):
    """The reference's `-phone_align yes` run on one utterance (decode_single, pocketsphinx_main.c:446-476).  Returns
    dict(n_frames, end_utt (the second ps_end_utt), words, phones, states: lists of (name, start, duration, score,
    parent), parent -1 for words); None where ps_set_alignment fails."""
    L = _ref()
    pcm = np.ascontiguousarray(pcm, np.int16)
    L.err_set_loglevel_str(b"ERROR")
    cfg = L.ps_config_init(None)
    for k, v in [("hmm", hmmdir), ("lm", lm), ("dict", dictfile), ("dither", "no")] + [(k, str(v)) for k, v in kv.items()]:
        L.ps_config_set_str(cfg, k.encode(), v.encode())
    ps = L.ps_init(cfg)
    if not ps:
        L.ps_config_free(cfg)
        raise RuntimeError("ps_init failed for " + hmmdir)
    try:
        L.ps_start_utt(ps)
        L.ps_process_raw(ps, _p(pcm), len(pcm), 0, 1)
        if L.ps_end_utt(ps) < 0:
            raise RuntimeError("the first decode failed")
        if L.ps_set_alignment(ps, None) < 0:
            return None
        L.ps_start_utt(ps)
        L.ps_process_raw(ps, _p(pcm), len(pcm), 0, 1)
        end = L.ps_end_utt(ps)
        al = L.ps_get_alignment(ps)
        if not al:
            raise RuntimeError("ps_get_alignment returned NULL")
        words, phones, states = [], [], []
        _entries(L, L.ps_alignment_words(al), -1, words, [phones, states])
        return dict(n_frames=L.ps_get_n_frames(ps), end_utt=end, words=words, phones=phones, states=states)
    finally:
        L.ps_free(ps)
        L.ps_config_free(cfg)


_BANDED = None


def _banded():
    global _BANDED
    if _BANDED is None:
        from oracle import oracle
        oracle.build()
        odir = os.path.dirname(oracle.LIB_PATH)
        out = os.path.join(tempfile.mkdtemp(prefix="align_banded"), "libalign_banded.so")
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-ffp-contract=off",
                               "-I" + os.path.join(ROOT, "oracle"), "-o", out,
                               os.path.join(ROOT, "tests", "emul", "align_banded.c"), "-L" + odir, "-lpsoracle",
                               "-Wl,-rpath," + odir])
        L = C.CDLL(out)
        L.emul_align_band.restype = None
        L.emul_align_band.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        L.emul_align_run_banded.restype = C.c_int32
        L.emul_align_run_banded.argtypes = ([C.c_int32, C.c_void_p, C.c_void_p, C.c_int32] + [C.c_void_p] * 5 +
                                            [C.c_int32, C.c_int32] + [C.c_void_p] * 6)
        _BANDED = L
    return _BANDED


def _i32(a):
    return None if a is None else np.ascontiguousarray(a, np.int32)


def band(n_phones, T, sf=None, ef=None):
    """The band rule restated in C: (lo, hi) int32 [T]."""
    lo, hi = np.zeros(max(T, 1), np.int32), np.zeros(max(T, 1), np.int32)
    sf, ef = _i32(sf), _i32(ef)
    _banded().emul_align_band(int(n_phones), _p(sf), _p(ef), int(T), _p(lo), _p(hi))
    return lo[:T].copy(), hi[:T].copy()


def align_run_banded(tp, sseq, ssid, tmatid, senscr, sf=None, ef=None, lo=None, hi=None):
    """state_align_search with the tokens kept in the band (by default the band rule's, else lo / hi).  Returns
    (status, start, dur, score per emitting state, tokens a phone outside the band would have written)."""
    tp = np.ascontiguousarray(tp, np.uint8)
    sseq = np.ascontiguousarray(sseq, np.uint16)
    ssid, tmatid, sf, ef = _i32(ssid), _i32(tmatid), _i32(sf), _i32(ef)
    senscr = np.ascontiguousarray(senscr, np.int16)
    T, n_sen = senscr.shape
    n_emit = tp.shape[1]
    if lo is None:
        lo, hi = band(len(ssid), T, sf, ef)
    lo, hi = np.append(_i32(lo), 0).astype(np.int32), np.append(_i32(hi), 0).astype(np.int32)
    out = np.zeros((3, max(1, len(ssid) * n_emit)), np.int32)
    n_out = np.zeros(1, np.int64)
    rc = _banded().emul_align_run_banded(n_emit, _p(tp), _p(sseq), len(ssid), _p(ssid), _p(tmatid), _p(sf), _p(ef),
                                         _p(senscr), n_sen, T, _p(out[0]), _p(out[1]), _p(out[2]), _p(lo), _p(hi),
                                         _p(n_out))
    k = len(ssid) * n_emit
    return int(rc), out[0, :k].copy(), out[1, :k].copy(), out[2, :k].copy(), int(n_out[0])
