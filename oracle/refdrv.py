"""ctypes binding for oracle/_ref/libpsref.so -- TEST INFRASTRUCTURE ONLY.

libpsref.so is the unmodified reference (cmusphinx/pocketsphinx 5.1.1) compiled by
oracle/Makefile plus oracle/ref_driver.c.  Only tests/, __graft_entry__.smoke() and
bench.py's CPU-baseline / --impl reference legs may import this module.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PSREF_LIB") or os.path.join(HERE, "_ref", "libpsref.so")   # PSREF_LIB: e.g. _ref/libpsref_fx.so

KIND_NAMES = {0: "ptm", 1: "s2_semi", 2: "ms"}

# Byte-for-byte mirror of hmm_t (src/hmm.h:169-182): 88 bytes on LP64.
HMM_DTYPE = np.dtype({
    "names": ["ctx", "score", "history", "out_score", "out_history", "ssid", "senid",
              "bestscore", "tmatid", "frame", "mpx", "n_emit_state"],
    "formats": ["<u8", ("<i4", 5), ("<i4", 5), "<i4", "<i4", "<u2", ("<u2", 5),
                "<i4", "<i2", "<i4", "u1", "u1"],
    "offsets": [0, 8, 28, 48, 52, 56, 58, 68, 72, 76, 80, 81],
    "itemsize": 88,
})


def available():
    return os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB_PATH)
        L.refdrv_open.restype = C.c_void_p
        L.refdrv_open.argtypes = [C.c_char_p, C.c_char_p]
        L.refdrv_close.argtypes = [C.c_void_p]
        L.refdrv_dims.argtypes = [C.c_void_p, C.c_void_p]
        L.refdrv_export.restype = C.c_long
        L.refdrv_export.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_long]
        L.refdrv_featurize.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_int]
        L.refdrv_reset.argtypes = [C.c_void_p]
        L.refdrv_fe_info.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.refdrv_fe_export.restype = C.c_long
        L.refdrv_fe_export.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_long]
        L.refdrv_mfcc.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_int]
        L.refdrv_fe_reset.argtypes = [C.c_void_p]
        L.refdrv_kws.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_long] + \
            [C.c_void_p] * 6 + [C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.refdrv_allphone.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.refdrv_allphone_lm.argtypes = L.refdrv_allphone.argtypes + [C.c_void_p]
        L.refdrv_align.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_long,
                                   C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                   C.c_void_p]
        L.refdrv_score.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.refdrv_score_active.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                          C.c_int, C.c_void_p, C.c_void_p]
        L.refdrv_time_score.restype = C.c_double
        L.refdrv_time_score.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.refdrv_hmmctx_new.restype = C.c_void_p
        L.refdrv_hmmctx_new.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.refdrv_hmmctx_free.argtypes = [C.c_void_p]
        L.refdrv_hmm_vit_eval.restype = C.c_int32
        L.refdrv_hmm_vit_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.refdrv_hmm_sweep.restype = None
        L.refdrv_hmm_sweep.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.refdrv_hmm_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.refdrv_hmm_enter.argtypes = [C.c_void_p, C.c_int, C.c_int32, C.c_int32, C.c_int]
        L.refdrv_hmm_clear.argtypes = [C.c_void_p, C.c_int]
        L.refdrv_hmm_clear_scores.argtypes = [C.c_void_p, C.c_int]
        L.refdrv_hmm_normalize.argtypes = [C.c_void_p, C.c_int, C.c_int32]
        L.refdrv_time_hmm_vit_eval.restype = C.c_double
        L.refdrv_time_hmm_vit_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.refdrv_phoneloop_run.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_char_p, C.c_int,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.refdrv_phoneloop_params.argtypes = [C.c_void_p, C.c_void_p]
        L.refdrv_decode.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_long, C.c_int,
                                    C.c_char_p, C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_void_p]
        L.refdrv_decode_senscr.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p,
                                           C.c_long, C.c_char_p, C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_void_p]
        assert L.refdrv_sizeof_hmm() == HMM_DTYPE.itemsize
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class RefModel:
    """One reference acmod_t (fe + feat + mdef + tmat + mgau back-end), all senones computed."""

    def __init__(self, hmmdir, **kv):
        s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode() or None
        self.h = lib().refdrv_open(hmmdir.encode(), s)
        if not self.h:
            raise RuntimeError("reference acmod_init failed for " + hmmdir)
        d = np.zeros(32, np.int32)
        lib().refdrv_dims(self.h, _p(d))
        self.kind = KIND_NAMES[int(d[0])]
        (self.n_sen, self.n_mgau, self.n_feat, self.n_density, self.topn, self.sumlen,
         self.n_emit_state, self.n_tmat, self.n_sseq, self.n_ciphone, self.n_ci_sen) = map(int, d[1:12])
        self.mixw_4bit = bool(d[12])
        self.logadd8_size = int(d[13])
        self.ds_ratio = int(d[14])
        self.aw = int(d[15])
        self.ms_logadd_size, self.ms_logadd_width, self.ms_logadd_zero = int(d[16]), int(d[17]), int(d[18])
        self.featlen = [int(x) for x in d[20:20 + self.n_feat]]

    def close(self):
        if self.h:
            lib().refdrv_close(self.h)
            self.h = None

    def export(self, what, dtype):
        n = lib().refdrv_export(self.h, what.encode(), None, 0)
        if n < 0:
            raise KeyError(what)
        buf = np.zeros(n // np.dtype(dtype).itemsize, dtype)
        if n:
            lib().refdrv_export(self.h, what.encode(), _p(buf), n)
        return buf

    def packed(self):
        """Model arrays in the layout pocketsphinx_b200.model.PackedModel expects."""
        m = dict(kind=self.kind, n_sen=self.n_sen, n_mgau=self.n_mgau, n_feat=self.n_feat,
                 n_density=self.n_density, topn=self.topn, featlen=np.array(self.featlen, np.int32),
                 n_emit_state=self.n_emit_state, aw=self.aw, ds_ratio=self.ds_ratio,
                 n_ciphone=self.n_ciphone, n_ci_sen=self.n_ci_sen,
                 mean=self.export("mean", np.float32), var=self.export("var", np.float32),
                 det=self.export("det", np.float32), mixw=self.export("mixw", np.uint8),
                 mixw_cb=self.export("mixw_cb", np.uint8), sen2cb=self.export("sen2cb", np.int32),
                 logadd8=self.export("logadd8", np.uint8),
                 tp=self.export("tp", np.uint8).reshape(self.n_tmat, self.n_emit_state, self.n_emit_state + 1),
                 sseq=self.export("sseq", np.uint16).reshape(self.n_sseq, self.n_emit_state),
                 phone_ssid=self.export("phone_ssid", np.int32),
                 phone_tmat=self.export("phone_tmat", np.int32))
        if self.kind == "ms":
            wdt = {1: np.uint8, 2: np.uint16, 4: np.uint32}[self.ms_logadd_width]
            m["logadd_ms"] = self.export("logadd_ms", wdt).astype(np.uint32)
            m["logadd_ms_zero"] = self.ms_logadd_zero
        if self.kind == "s2_semi":
            m["topn_beam"] = self.export("topn_beam", np.uint8)
        return m

    def fe_export(self, what, dtype):
        n = lib().refdrv_fe_export(self.h, what.encode(), None, 0)
        if n < 0:
            raise KeyError(what)
        buf = np.zeros(n // np.dtype(dtype).itemsize, dtype)
        if n:
            lib().refdrv_fe_export(self.h, what.encode(), _p(buf), n)
        return buf

    def fe_desc(self):
        """Front-end parameters and tables as the reference's fe_init left them (dict)."""
        i = np.zeros(16, np.int32)
        f = np.zeros(4, np.float32)
        lib().refdrv_fe_info(self.h, _p(i), _p(f))
        d = dict(frame_size=int(i[0]), frame_shift=int(i[1]), fft_size=int(i[2]), fft_order=int(i[3]),
                 n_filt=int(i[4]), n_cep=int(i[5]), remove_dc=int(i[6]), remove_noise=int(i[7]),
                 transform=int(i[8]), lifter_val=int(i[9]), log_spec=int(i[10]), dither=int(i[11]),
                 window=int(i[13]), cmn=int(i[14]), cepsize=int(i[15]),
                 alpha=np.float32(f[0]), sqrt_inv_n=np.float32(f[1]), sqrt_inv_2n=np.float32(f[2]),
                 sampling_rate=float(f[3]))
        d["hamming"] = self.fe_export("hamming", np.float64)
        d["ccc"] = self.fe_export("ccc", np.float64)
        d["sss"] = self.fe_export("sss", np.float64)
        for k in ("spec_start", "filt_start", "filt_width"):
            d[k] = self.fe_export(k, np.int16)
        d["filt_coeffs"] = self.fe_export("filt_coeffs", np.float32)
        d["mel_cosine"] = self.fe_export("mel_cosine", np.float32).reshape(d["n_cep"], d["n_filt"])
        d["lifter"] = self.fe_export("lifter", np.float32)
        return d

    def mfcc(self, pcm):
        """Cepstra before CMN from a fresh stream (noise tracker reset)."""
        pcm = np.ascontiguousarray(pcm, np.int16)
        i = np.zeros(16, np.int32); f = np.zeros(4, np.float32)
        lib().refdrv_fe_info(self.h, _p(i), _p(f))
        cap = len(pcm) // int(i[1]) + 16                    # more frames than the frame shift allows
        out = np.zeros((cap, int(i[5])), np.float32)
        T = lib().refdrv_mfcc(self.h, _p(pcm), len(pcm), _p(out), cap)
        if T > cap:
            raise RuntimeError("refdrv_mfcc made %d frames, more than the %d sized for" % (T, cap))
        return out[:T].copy()

    def _frame_cap(self, n_samples):
        """More frames than n_samples can make at this front end's own frame shift."""
        i = np.zeros(16, np.int32); f = np.zeros(4, np.float32)
        lib().refdrv_fe_info(self.h, _p(i), _p(f))
        return n_samples // int(i[1]) + 16

    def featurize_fresh(self, pcm):
        """featurize() as the first utterance of a fresh stream (noise tracker reset first)."""
        lib().refdrv_fe_reset(self.h)
        return self.featurize(pcm)

    def featurize(self, pcm, max_frames=None):
        pcm = np.ascontiguousarray(pcm, np.int16)
        cap = max_frames or self._frame_cap(len(pcm))
        out = np.zeros((cap, self.sumlen), np.float32)
        T = lib().refdrv_featurize(self.h, _p(pcm), len(pcm), _p(out), cap)
        if T > cap and not max_frames:
            raise RuntimeError("refdrv_featurize made %d frames, more than the %d sized for" % (T, cap))
        return out[:min(T, cap)].copy()

    def score(self, feats, reset=True, want_topn=False):
        feats = np.ascontiguousarray(feats, np.float32)
        T = feats.shape[0]
        scr = np.zeros((T, self.n_sen), np.int16)
        topn = None
        if want_topn and self.kind == "ptm":
            topn = np.zeros((T, self.n_mgau, self.n_feat, self.topn, 2), np.int32)
        elif want_topn and self.kind == "s2_semi":
            topn = np.zeros((T, self.n_feat, self.topn, 2), np.int32)
        lib().refdrv_score(self.h, _p(feats), T, _p(scr), int(reset), _p(topn))
        return (scr, topn) if want_topn else scr

    def score_active(self, feats, flags, reset=True):
        feats = np.ascontiguousarray(feats, np.float32)
        flags = np.ascontiguousarray(flags, np.uint8)
        T = feats.shape[0]
        scr = np.zeros((T, self.n_sen), np.int16)
        nact = np.zeros(T, np.int32)
        lists = np.zeros((T, self.n_sen), np.uint8)
        lib().refdrv_score_active(self.h, _p(feats), T, _p(flags), _p(scr), int(reset), _p(nact), _p(lists))
        return scr, nact, lists

    def time_score(self, feats, reps=1):
        feats = np.ascontiguousarray(feats, np.float32)
        return lib().refdrv_time_score(self.h, _p(feats), feats.shape[0], reps)

    def phoneloop(self, pcm, **kv):
        """The reference's phone_loop_search over one utterance.  Call it on a FRESH RefModel: the object's
        live-CMN state (after other utterances) and earlier pl_* settings are not undone, and both change
        the scores the phone loop sees."""
        pcm = np.ascontiguousarray(pcm, np.int16)
        kv.setdefault("pl_window", 5)
        s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode()
        cap = len(pcm) // 160 + 16
        np_ = self.n_ciphone
        hm = np.zeros((cap, np_), HMM_DTYPE)
        best = np.zeros(cap, np.int32)
        pen = np.zeros((cap, np_), np.int32)
        scr = np.zeros((cap, self.n_sen), np.int16)
        feat = np.zeros((cap, self.sumlen), np.float32)
        T = lib().refdrv_phoneloop_run(self.h, _p(pcm), len(pcm), s, cap, _p(hm), _p(best), _p(pen), _p(scr), _p(feat))
        par = np.zeros(8, np.int32)
        lib().refdrv_phoneloop_params(self.h, _p(par))
        params = dict(n_phones=int(par[0]), beam=int(par[1]), pbeam=int(par[2]), pip=int(par[3]),
                      window=int(par[4]), penalty_weight=float(par[6:8].view(np.float64)[0]))
        return dict(T=T, hmm=hm[:T], best=best[:T], pen=pen[:T], senscr=scr[:T], feat=feat[:T], params=params)


class RefHmmCtx:
    """hmm_context_t over caller-supplied tp / sseq tables; evaluates real 88-byte hmm_t arrays."""

    def __init__(self, tp, sseq):
        tp = np.ascontiguousarray(tp, np.uint8)
        sseq = np.ascontiguousarray(sseq, np.uint16)
        self.n_emit = tp.shape[1]
        assert tp.shape[2] == self.n_emit + 1 and sseq.shape[1] == self.n_emit
        self.h = lib().refdrv_hmmctx_new(self.n_emit, _p(tp), tp.shape[0], _p(sseq), sseq.shape[0])

    def close(self):
        if self.h:
            lib().refdrv_hmmctx_free(self.h)
            self.h = None

    def init(self, n, mpx, ssid, tmatid):
        hm = np.zeros(n, HMM_DTYPE)
        lib().refdrv_hmm_init(self.h, _p(hm), n, _p(np.ascontiguousarray(mpx, np.int32)),
                              _p(np.ascontiguousarray(ssid, np.int32)), _p(np.ascontiguousarray(tmatid, np.int32)))
        return hm

    def vit_eval(self, hmms, senscr):
        senscr = np.ascontiguousarray(senscr, np.int16)
        assert hmms.dtype == HMM_DTYPE and hmms.flags.c_contiguous
        return int(lib().refdrv_hmm_vit_eval(self.h, _p(hmms), len(hmms), _p(senscr)))

    def sweep(self, hmms, senscr):
        """T frames of hmm_vit_eval over the same records (updated in place); senscr int16 [T][n_sen];
        returns best int32 [T]."""
        senscr = np.ascontiguousarray(senscr, np.int16)
        assert hmms.dtype == HMM_DTYPE and hmms.flags.c_contiguous and senscr.ndim == 2
        best = np.zeros(len(senscr), np.int32)
        lib().refdrv_hmm_sweep(self.h, _p(hmms), len(hmms), _p(senscr), senscr.shape[1], len(senscr), _p(best))
        return best

    def time_vit_eval(self, hmms, senscr, reps=1):
        senscr = np.ascontiguousarray(senscr, np.int16)
        return lib().refdrv_time_hmm_vit_eval(self.h, _p(hmms), len(hmms), _p(senscr), reps)


def decode(hmmdir, lm, dic, pcm, use_cuda=False, libpath=None, twice=False, **kv):
    """Full reference decode (fwdtree + fwdflat + bestpath by default) of one utterance; with
    use_cuda the GMM back-end is the CUDA one bound through integration/ps_mgau_cuda.c."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode() or None
    hyp = C.create_string_buffer(4096)
    seg = C.create_string_buffer(65536)
    stats = np.zeros(4, np.int32)
    stats[3] = 1 if twice else 0          # twice: utt_us times the second of two passes over the utterance
    n = lib().refdrv_decode(hmmdir.encode(), lm.encode(), dic.encode(), s, _p(pcm), len(pcm), int(use_cuda),
                            libpath.encode() if libpath else None, hyp, 4096, seg, 65536, _p(stats))
    if n < 0:
        raise RuntimeError("refdrv_decode failed (%d)" % n)
    return dict(n_frames=n, hyp=hyp.value.decode(), seg=seg.value.decode(), score=int(stats[0]),
                cuda_calls=int(stats[1]), n_sen=int(stats[2]), utt_us=int(stats[3]))


def decode_senscr(hmmdir, lm, dic, senfile=None, pcm=None, senout=None, **kv):
    """-compallsen yes decode: from a senone dump (ps_decode_senscr) when senfile is given, else
    from PCM (optionally writing the reference's own dump to senout)."""
    s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode() or None
    hyp = C.create_string_buffer(4096)
    seg = C.create_string_buffer(65536)
    stats = np.zeros(4, np.int32)
    if pcm is not None:
        pcm = np.ascontiguousarray(pcm, np.int16)
    n = lib().refdrv_decode_senscr(hmmdir.encode(), lm.encode(), dic.encode(), s,
                                   senfile.encode() if senfile else None, _p(pcm), 0 if pcm is None else len(pcm),
                                   senout.encode() if senout else None, hyp, 4096, seg, 65536, _p(stats))
    if n < 0:
        raise RuntimeError("refdrv_decode_senscr failed (%d)" % n)
    return dict(n_frames=n, hyp=hyp.value.decode(), seg=seg.value.decode(), score=int(stats[0]))


def align(hmmdir, dictfile, words, pcm, **kv):
    """The reference's state_align_search on one utterance (compallsen, no look-ahead).
    Returns dict(n_frames, ssid, tmatid, start, dur, score, n_emit)."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode() or None
    cap = 4096
    ssid = np.zeros(cap, np.int32); tmat = np.zeros(cap, np.int32)
    st = np.zeros((3, cap * 5), np.int32)
    info = np.zeros(8, np.int32)
    rc = lib().refdrv_align(hmmdir.encode(), dictfile.encode(), s, words.encode(), _p(pcm), len(pcm),
                            _p(ssid), _p(tmat), cap, _p(st[0]), _p(st[1]), _p(st[2]), cap * 5, _p(info))
    if rc < 0:
        raise RuntimeError("refdrv_align failed: %d" % rc)
    nph, nst = int(info[1]), int(info[2])
    return dict(n_frames=int(info[0]), n_emit=int(info[3]), ssid=ssid[:nph].copy(), tmatid=tmat[:nph].copy(),
                start=st[0, :nst].copy(), dur=st[1, :nst].copy(), score=st[2, :nst].copy())


def kws(hmmdir, dictfile, pcm, keyphrase=None, keyfile=None, **kv):
    """The reference's kws_search on one utterance (compallsen, no look-ahead).  Returns the search
    configuration (phone loop, keyphrase HMM chains, thresholds, beam, plp) and its detections
    [n][5] = (keyphrase index, sf, ef, prob, ascr) in list order."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode() or None
    cap = 4096
    pl_ssid = np.zeros(cap, np.int32); pl_tmat = np.zeros(cap, np.int32)
    kp_off = np.zeros(cap, np.int32); kp_thr = np.zeros(cap, np.int32)
    kp_ssid = np.zeros(cap, np.int32); kp_tmat = np.zeros(cap, np.int32)
    det = np.zeros((cap, 5), np.int32)
    info = np.zeros(8, np.int32)
    rc = lib().refdrv_kws(hmmdir.encode(), dictfile.encode(), s, keyphrase.encode() if keyphrase else None,
                          keyfile.encode() if keyfile else None, _p(pcm), len(pcm), _p(pl_ssid), _p(pl_tmat), _p(kp_off),
                          _p(kp_thr), _p(kp_ssid), _p(kp_tmat), cap, _p(det), cap, _p(info))
    if rc < 0:
        raise RuntimeError("refdrv_kws failed: %d" % rc)
    n_pl, n_kp, n_k, n_det = int(info[1]), int(info[2]), int(info[3]), int(info[6])
    return dict(n_frames=int(info[0]), beam=int(info[4]), plp=int(info[5]), pl_ssid=pl_ssid[:n_pl].copy(),
                pl_tmat=pl_tmat[:n_pl].copy(), kp_off=kp_off[:n_kp + 1].copy(), kp_thresh=kp_thr[:n_kp].copy(),
                kp_ssid=kp_ssid[:n_k].copy(), kp_tmat=kp_tmat[:n_k].copy(), det=det[:n_det].copy())


def allphone(hmmdir, pcm, **kv):
    """The reference's allphone_search without a phone LM on one utterance: graph, parameters and
    the phone segmentation [n][5] = (ci, sf, ef, score, tscore)."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode() or None
    cap_n, cap_l, cap_s = 1 << 16, 1 << 22, 4096
    ci = np.zeros(cap_n, np.int32); ssid = np.zeros(cap_n, np.int32); tmat = np.zeros(cap_n, np.int32)
    soff = np.zeros(cap_n + 1, np.int32); succ = np.zeros(cap_l, np.int32)
    segs = np.zeros((cap_s, 5), np.int32)
    info = np.zeros(16, np.int32)
    lmt = np.zeros(64 * 64 + 64 * 64 * 64, np.int32)
    rc = lib().refdrv_allphone_lm(hmmdir.encode(), s, _p(pcm), len(pcm), _p(ci), _p(ssid), _p(tmat), _p(soff), cap_n,
                                  _p(succ), cap_l, _p(segs), cap_s, _p(info), _p(lmt))
    if rc < 0:
        raise RuntimeError("refdrv_allphone failed: %d" % rc)
    n, nl = int(info[1]), int(info[2])
    assert n <= cap_n and nl <= cap_l
    nc = int(info[10])
    extra = {}
    if info[9]:
        assert nc <= 64
        extra = dict(bg=lmt[:nc * nc].reshape(nc, nc).copy(), tg=lmt[nc * nc:nc * nc + nc ** 3].reshape(nc, nc, nc).copy())
    return dict(**extra, n_frames=int(info[0]), ci=ci[:n].copy(), ssid=ssid[:n].copy(), tmatid=tmat[:n].copy(),
                succ_off=soff[:n + 1].copy(), succ=succ[:nl].copy(), start=int(info[3]), beam=int(info[4]),
                pbeam=int(info[5]), inspen=int(info[6]), segs=segs[:int(info[7])].copy(), n_history=int(info[8]))


def fsg(hmmdir, dictfile, fsgfile, pcm, **kv):
    """The reference's fsg_search on one utterance (compallsen, no look-ahead, no bestpath): the
    flattened lextree, links, null arcs, beams, and the history table + hypothesis it produced."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode() or None
    L = lib()
    L.refdrv_fsg.restype = C.c_long
    L.refdrv_fsg.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_long, C.c_void_p,
                             C.c_long, C.c_void_p, C.c_char_p, C.c_int, C.c_char_p, C.c_int]
    cap = 1 << 22
    blob = np.zeros(cap, np.int32)
    info = np.zeros(16, np.int32)
    hyp = C.create_string_buffer(1 << 16)
    vocab = C.create_string_buffer(1 << 16)
    need = L.refdrv_fsg(hmmdir.encode(), dictfile.encode(), fsgfile.encode(), s, _p(pcm), len(pcm), _p(blob), cap,
                        _p(info), hyp, 1 << 16, vocab, 1 << 16)
    if need < 0 or need > cap:
        raise RuntimeError("refdrv_fsg failed: %d" % need)
    n_pn, n_state, n_link, n_null, n_hist = (int(x) for x in info[1:6])
    o = 0
    pnodes = blob[o:o + n_pn * 16].reshape(n_pn, 16).copy(); o += n_pn * 16
    roots = blob[o:o + n_state].copy(); o += n_state
    links = blob[o:o + n_link * 5].reshape(n_link, 5).copy(); o += n_link * 5
    nulloff = blob[o:o + n_state + 1].copy(); o += n_state + 1
    nullarc = blob[o:o + n_null].copy(); o += n_null
    hist = blob[o:o + n_hist * 13].reshape(n_hist, 13).copy()
    return dict(n_frames=int(info[0]), pnodes=pnodes, roots=roots, links=links, nulloff=nulloff, nullarc=nullarc,
                hist=hist, beam=int(info[6]), pbeam=int(info[7]), wbeam=int(info[8]), maxhmmpf=int(info[9]),
                silcipid=int(info[10]), n_ciphone=int(info[11]), start_state=int(info[12]),
                final_state=int(info[13]), score=int(info[14]), hyp=hyp.value.decode().split("\n")[0],
                seg=[l.split() for l in hyp.value.decode().split("\n")[1:] if l],   # word sf ef ascr lscr
                vocab=vocab.value.decode().split("\n")[:-1])


def fwdtree(hmmdir, lm, dictfile, pcm, dense_lm=True, **kv):
    """The reference's first pass (ngram_search_fwdtree; no fwdflat / bestpath / look-ahead) on one
    utterance: the flattened lextree, dictionary and dict2pid tables, the LM as a dense trigram score
    table, the search parameters, and the complete backpointer table + right-context score stack."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode() or None
    L = lib()
    L.refdrv_fwdtree.restype = C.c_long
    L.refdrv_fwdtree.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_long, C.c_void_p,
                                 C.c_long, C.c_void_p, C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_int]
    info = np.zeros(40, np.int32)
    hyp = C.create_string_buffer(4096)
    vocab = C.create_string_buffer(1 << 22)
    args = (hmmdir.encode(), lm.encode(), dictfile.encode(), s, _p(pcm), len(pcm))
    need = L.refdrv_fwdtree(*args, None, 0, _p(info), hyp, 4096, None, 0, int(dense_lm))
    if need < 0:
        raise RuntimeError("refdrv_fwdtree failed: %d" % need)
    blob = np.zeros(need, np.int32)
    if L.refdrv_fwdtree(*args, _p(blob), need, _p(info), hyp, 4096, vocab, 1 << 22, int(dense_lm)) != need:
        raise RuntimeError("refdrv_fwdtree: inconsistent size")
    keys = ("n_frame n_words n_root n_nonroot n_1ph_words n_1ph_LMwords n_ci sil beam pbeam wbeam lpbeam lponlybeam "
            "maxhmmpf maxwpf nwpen pip silpen fillpen start_wid finish_wid silence_wid filler_start filler_end bpidx "
            "bss_head n_lm score fwdflatbeam fwdflatwbeam min_ef_width max_sf_win lwf_bits n_pron").split()
    r = {k: int(info[i]) for i, k in enumerate(keys)}
    o = [0]

    def take(*shape):
        n = int(np.prod(shape))
        a = blob[o[0]:o[0] + n].reshape(shape).copy()
        o[0] += n
        return a
    nc, nl = r["n_ci"], r["n_lm"]
    r["roots"] = take(r["n_root"], 5); r["nonroot"] = take(r["n_nonroot"], 6); r["words"] = take(r["n_words"], 8)
    r["w1ph"] = take(r["n_1ph_words"]); r["r1ph"] = take(r["n_1ph_words"], 4)
    r["rs_n"] = take(nc, nc); r["rs_ssid"] = take(nc, nc, nc); r["rs_cimap"] = take(nc, nc, nc); r["ldiph"] = take(nc, nc, nc)
    r["lm"] = take(nl, nl + 1, nl + 1)
    r["inlm"] = take(r["n_words"]); r["pron_off"] = take(r["n_words"] + 1)
    r["pron_ci"] = take(r["n_pron"]); r["pron_ssid"] = take(r["n_pron"])
    r["bp"] = take(r["bpidx"], 10); r["bss"] = take(r["bss_head"]); r["bp_idx"] = take(r["n_frame"] + 1)
    assert o[0] == need
    r["hyp"] = hyp.value.decode()
    r["vocab"] = vocab.value.decode().split("\n")[:-1]
    r["info"] = info.copy()
    r["model"] = blob[:need - (r["bpidx"] * 10 + r["bss_head"] + r["n_frame"] + 1)].copy()
    return r


def fsg_roundtrip(hmmdir, dictfile, fsgfile, pcm, rows, n_frames, **kv):
    """Decode with the reference, replace its history table by `rows` through the maintainer-side binding
    (integration/ps_search_cuda.c: cuda_fsg_import) and let its own fsg_search_hyp answer."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    rows = np.ascontiguousarray(rows, np.int32)
    s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode() or None
    L = lib()
    L.refdrv_fsg_roundtrip.restype = C.c_long
    L.refdrv_fsg_roundtrip.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_long, C.c_void_p,
                                       C.c_int32, C.c_int32, C.c_char_p, C.c_int, C.c_void_p]
    hyp = C.create_string_buffer(4096)
    score = np.zeros(1, np.int32)
    n = L.refdrv_fsg_roundtrip(hmmdir.encode(), dictfile.encode(), fsgfile.encode(), s, _p(pcm), len(pcm), _p(rows), len(rows),
                               int(n_frames), hyp, 4096, _p(score))
    if n < 0:
        raise RuntimeError("refdrv_fsg_roundtrip failed: %d" % n)
    return dict(hyp=hyp.value.decode(), score=int(score[0]), n_entries=int(n))


def ngram_roundtrip(hmmdir, lm, dictfile, pcm, bp, bss, bp_idx, **kv):
    """Decode with the reference, wipe its backpointer table / score stack, import (bp, bss, bp_idx)
    through cuda_ngram_import and let its own ngram_search_hyp (lattice + bestpath when configured) and
    segment iterator answer."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    bp = np.ascontiguousarray(bp, np.int32); bss = np.ascontiguousarray(bss, np.int32)
    bp_idx = np.ascontiguousarray(bp_idx, np.int32)
    s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode() or None
    L = lib()
    L.refdrv_ngram_roundtrip.restype = C.c_long
    L.refdrv_ngram_roundtrip.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_long, C.c_void_p,
                                         C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_char_p, C.c_int,
                                         C.c_void_p, C.c_char_p, C.c_int]
    hyp = C.create_string_buffer(4096)
    seg = C.create_string_buffer(65536)
    score = np.zeros(1, np.int32)
    n = L.refdrv_ngram_roundtrip(hmmdir.encode(), lm.encode(), dictfile.encode(), s, _p(pcm), len(pcm), _p(bp), len(bp), _p(bss),
                                 len(bss), _p(bp_idx), len(bp_idx) - 1, hyp, 4096, _p(score), seg, 65536)
    if n < 0:
        raise RuntimeError("refdrv_ngram_roundtrip failed: %d" % n)
    return dict(hyp=hyp.value.decode(), score=int(score[0]), seg=seg.value.decode(), n_entries=int(n))


def lm_arrays(hmmdir, lm, dictfile, queries=None, **kv):
    """The LM behind an n-gram search as sorted arrays (integration/ps_search_cuda.c:cuda_ngram_export_lm) and
    the reference's own ngram_tg_score(...) >> SENSCR_SHIFT for `queries` [n][3] = (w, h1, h2) dictionary ids."""
    s = "\n".join("%s=%s" % (k, v) for k, v in kv.items()).encode() or None
    L = lib()
    L.refdrv_lm_arrays.restype = C.c_long
    L.refdrv_lm_arrays.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_long, C.c_void_p, C.c_long,
                                   C.c_void_p]
    need = L.refdrv_lm_arrays(hmmdir.encode(), lm.encode(), dictfile.encode(), s, None, 0, None, 0, None)
    if need < 0:
        raise RuntimeError("refdrv_lm_arrays failed: %d" % need)
    arr = np.zeros(need, np.int32)
    q = np.zeros((0, 3), np.int32) if queries is None else np.ascontiguousarray(queries, np.int32)
    scores = np.zeros(len(q), np.int32)
    if L.refdrv_lm_arrays(hmmdir.encode(), lm.encode(), dictfile.encode(), s, _p(arr), need, _p(q), len(q), _p(scores)) != need:
        raise RuntimeError("refdrv_lm_arrays: inconsistent size")
    return arr, scores
