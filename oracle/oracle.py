"""ctypes binding for oracle/_build/libpsoracle.so (our plain-C restatement, ps_oracle.c).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and bench.py's
CPU-baseline legs; never from pocketsphinx_b200/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "_build", "libpsoracle.so")

KIND_ID = {"ptm": 0, "s2_semi": 1, "ms": 2}
MAX_FEAT = 8

# same layout as the reference's 88-byte hmm_t (src/hmm.h:169-182)
HMM_DTYPE = np.dtype({
    "names": ["ctx", "score", "history", "out_score", "out_history", "ssid", "senid",
              "bestscore", "tmatid", "frame", "mpx", "n_emit_state"],
    "formats": ["<u8", ("<i4", 5), ("<i4", 5), "<i4", "<i4", "<u2", ("<u2", 5),
                "<i4", "<i2", "<i4", "u1", "u1"],
    "offsets": [0, 8, 28, 48, 52, 56, 58, 68, 72, 76, 80, 81],
    "itemsize": 88,
})


class _Model(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n_sen", C.c_int32), ("n_mgau", C.c_int32),
                ("n_feat", C.c_int32), ("n_density", C.c_int32), ("topn", C.c_int32),
                ("featlen", C.c_int32 * MAX_FEAT), ("ds_ratio", C.c_int32), ("aw", C.c_int32),
                ("mixw_4bit", C.c_int32), ("pdf_transposed", C.c_int32),
                ("logadd_ms_size", C.c_int32), ("logadd_ms_zero", C.c_int32),
                ("mean", C.c_void_p), ("var", C.c_void_p), ("det", C.c_void_p),
                ("mixw", C.c_void_p), ("mixw_cb", C.c_void_p), ("sen2cb", C.c_void_p),
                ("logadd8", C.c_void_p), ("logadd_ms", C.c_void_p), ("topn_beam", C.c_void_p),
                ("fixed_point", C.c_int32)]


class _HmmCtx(C.Structure):
    _fields_ = [("n_emit_state", C.c_int32), ("tp", C.c_void_p), ("sseq", C.c_void_p),
                ("senscore", C.c_void_p)]


def build(force=False):
    if force or not os.path.exists(LIB_PATH) or \
            os.path.getmtime(LIB_PATH) < os.path.getmtime(os.path.join(HERE, "ps_oracle.c")):
        subprocess.check_call(["make", "-s", "-C", HERE, "oracle"])


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH)
        L.pso_gmm_new.restype = C.c_void_p
        L.pso_gmm_new.argtypes = [C.c_void_p, C.c_int32]
        L.pso_gmm_free.argtypes = [C.c_void_p]
        L.pso_gmm_reset.argtypes = [C.c_void_p]
        L.pso_frame_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                     C.c_int32, C.c_int32]
        L.pso_score_utt.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.pso_flags2list.restype = C.c_int32
        L.pso_flags2list.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.pso_time_score_utt.restype = C.c_double
        L.pso_time_score_utt.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
        L.pso_hmm_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.pso_hmm_vit_eval_batch.restype = C.c_int32
        L.pso_hmm_vit_eval_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        L.pso_phoneloop_new.restype = C.c_void_p
        L.pso_phoneloop_new.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                        C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_double]
        L.pso_phoneloop_free.argtypes = [C.c_void_p]
        L.pso_phoneloop_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                        C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return None if a is None or (hasattr(a, "size") and a.size == 0) else a.ctypes.data


class OracleModel:
    """Wraps a pocketsphinx_b200.model.PackedModel (or equivalent dict) for the C oracle."""

    def __init__(self, pm):
        self.pm = pm
        m = _Model()
        m.kind = KIND_ID[pm.kind]
        m.n_sen, m.n_mgau, m.n_feat, m.n_density, m.topn = pm.n_sen, pm.n_mgau, pm.n_feat, pm.n_density, pm.topn
        for i, v in enumerate(pm.featlen):
            m.featlen[i] = int(v)
        m.ds_ratio = max(1, int(pm.ds_ratio))
        m.aw = int(pm.aw) if pm.aw else 1
        m.mixw_4bit = int(pm.mixw_4bit)
        m.pdf_transposed = int(pm.n_mgau == 1)
        m.logadd_ms_size = int(pm.logadd_ms.size)
        m.logadd_ms_zero = int(pm.logadd_ms_zero)
        m.mean, m.var, m.det = _p(pm.mean), _p(pm.var), _p(pm.det)
        m.mixw, m.mixw_cb, m.sen2cb = _p(pm.mixw), _p(pm.mixw_cb), _p(pm.sen2cb)
        m.logadd8, m.logadd_ms = _p(pm.logadd8), _p(pm.logadd_ms)
        m.topn_beam = _p(pm.topn_beam) if pm.topn_beam.size and pm.topn_beam.any() else None
        m.fixed_point = int(getattr(pm, "fixed_point", 0))
        self.c = m

    def score_utt(self, feats, want_topn=False, want_raw=False):
        """Scores [T][n_sen]; with want_topn the normalised top-N lists, with want_raw (ptm) the lists before
        normalisation, [T][n_mgau][n_feat][topn]{codeword, integer distance} (see ptm_records)."""
        pm = self.pm
        feats = np.ascontiguousarray(feats, np.float32)
        T = feats.shape[0]
        scr = np.zeros((T, pm.n_sen), np.int16)
        topn = raw = None
        if want_topn and pm.kind == "ptm":
            topn = np.zeros((T, pm.n_mgau, pm.n_feat, pm.topn, 2), np.int32)
        elif want_topn and pm.kind == "s2_semi":
            topn = np.zeros((T, pm.n_feat, pm.topn, 2), np.int32)
        if want_raw:
            assert pm.kind == "ptm", "raw top-N lists exist for ptm models"
            raw = np.zeros((T, pm.n_mgau, pm.n_feat, pm.topn, 2), np.int32)
        lib().pso_score_utt(C.byref(self.c), _p(feats), T, _p(scr), _p(topn), _p(raw))
        out = (scr,) + ((topn,) if want_topn else ()) + ((raw,) if want_raw else ())
        return out if len(out) > 1 else scr

    def time_score_utt(self, feats, reps=1):
        feats = np.ascontiguousarray(feats, np.float32)
        return lib().pso_time_score_utt(C.byref(self.c), _p(feats), feats.shape[0], reps)

    def decoder(self, n_hist=2):
        return OracleGmm(self, n_hist)


class OracleGmm:
    """One ps_mgau_t-like scorer with its top-N history ring and frame_idx."""

    def __init__(self, om, n_hist):
        self.om = om
        self.h = lib().pso_gmm_new(C.byref(om.c), n_hist)
        self.frame_idx_off = None

    def close(self):
        if self.h:
            lib().pso_gmm_free(self.h)
            self.h = None

    def reset(self):
        lib().pso_gmm_reset(self.h)

    def set_frame_idx(self, v):
        # pso_gmm_t: {m*, n_hist, frame_idx, ...}: frame_idx sits after an 8-byte ptr + int32
        C.c_int32.from_address(self.h + 12).value = int(v)

    def frame_eval(self, feat, frame, active_list=None, compallsen=True):
        pm = self.om.pm
        feat = np.ascontiguousarray(feat, np.float32)
        scr = np.zeros(pm.n_sen, np.int16)
        if active_list is not None:
            active_list = np.ascontiguousarray(active_list, np.uint8)
        n = 0 if active_list is None else len(active_list)
        lib().pso_frame_eval(self.h, _p(scr), _p(active_list), n, _p(feat), frame, int(compallsen))
        return scr

    def frame_eval_into(self, scr, feat, frame, active_list=None, compallsen=True):
        """Like frame_eval but writes into a caller buffer (stale entries kept, as the ms
        back-end leaves inactive senones untouched)."""
        feat = np.ascontiguousarray(feat, np.float32)
        if active_list is not None:
            active_list = np.ascontiguousarray(active_list, np.uint8)
        n = 0 if active_list is None else len(active_list)
        lib().pso_frame_eval(self.h, _p(scr), _p(active_list), n, _p(feat), frame, int(compallsen))
        return scr


def flags2list(flags):
    flags = np.ascontiguousarray(flags, np.uint8)
    out = np.zeros(len(flags), np.uint8)
    n = lib().pso_flags2list(_p(flags), len(flags), _p(out))
    return out[:n].copy()


SENSCR_SHIFT, MAX_NEG_ASCR = 10, 96


def ptm_records(raw):
    """Raw PTM lists [T][n_mgau][n_feat][4]{codeword, score} (score_utt(want_raw=True)) -> the device's top-N
    records int32 [T][n_mgau * n_feat][4] (psb_batch_get_topn): {s0 >> 10, the four codewords as bytes,
    min(255, (s0 >> 10) - (sj >> 10)) as bytes, 0}."""
    raw = np.asarray(raw)
    assert raw.shape[-2:] == (4, 2), "records hold four list entries"
    T = raw.shape[0]
    cw = raw[..., 0].reshape(T, -1, 4).astype(np.uint32)
    q = raw[..., 1].reshape(T, -1, 4) >> SENSCR_SHIFT
    e = np.minimum(255, q[..., :1] - q).astype(np.uint32)
    rec = np.zeros(cw.shape[:2] + (4,), np.int32)
    rec[..., 0] = q[..., 0]
    rec[..., 1] = (cw[..., 0] | cw[..., 1] << 8 | cw[..., 2] << 16 | cw[..., 3] << 24).view(np.int32)
    rec[..., 2] = (e[..., 0] | e[..., 1] << 8 | e[..., 2] << 16 | e[..., 3] << 24).view(np.int32)
    return rec


def ptm_norm_raw(raw):
    """ptm_mgau_codebook_norm (every codebook active) applied to raw lists: what score_utt(want_topn=True) returns."""
    out = np.array(raw, np.int32, copy=True)
    q = out[..., 1] >> SENSCR_SHIFT                               # [T][cb][f][topn]
    norm = q[:, :, :, 0].max(axis=1)                              # per frame and stream
    out[..., 1] = np.minimum(MAX_NEG_ASCR, norm[:, None, :, None] - q)
    return out


def assert_records_equal(got, want, what=""):
    """Top-N records [T][K][4]: equal, or an error naming the first differing (frame, pair) and field."""
    got, want = np.asarray(got, np.int32), np.asarray(want, np.int32)
    assert got.shape == want.shape, "%s: record shapes %s vs %s" % (what, got.shape, want.shape)
    g, w = got.view(np.uint32), want.view(np.uint32)          # codeword bytes compare as uint32
    bad = np.argwhere((g != w).any(-1))
    if bad.size:
        t, k = bad[0]
        names = ("top score >> 10", "codewords", "score offsets", "padding")
        fld = int(np.argmax(g[t, k] != w[t, k]))
        raise AssertionError("%s: %d records differ; first at frame %d, pair %d: field %s got 0x%08x want 0x%08x "
                             "(got %s, want %s)" % (what, len(bad), t, k, names[fld], g[t, k, fld], w[t, k, fld],
                                                    g[t, k].tolist(), w[t, k].tolist()))


class OracleHmmCtx:
    def __init__(self, tp, sseq):
        self.tp = np.ascontiguousarray(tp, np.uint8)
        self.sseq = np.ascontiguousarray(sseq, np.uint16)
        self.n_emit = self.tp.shape[1]
        c = _HmmCtx()
        c.n_emit_state = self.n_emit
        c.tp = _p(self.tp)
        c.sseq = _p(self.sseq)
        self.c = c

    def init(self, n, mpx, ssid, tmatid):
        hm = np.zeros(n, HMM_DTYPE)
        for i in range(n):
            lib().pso_hmm_init(C.byref(self.c), hm[i:i + 1].ctypes.data, int(mpx[i]), int(ssid[i]), int(tmatid[i]))
        return hm

    def vit_eval(self, hmms, senscr):
        senscr = np.ascontiguousarray(senscr, np.int16)
        assert hmms.dtype == HMM_DTYPE and hmms.flags.c_contiguous
        self.c.senscore = _p(senscr)
        return int(lib().pso_hmm_vit_eval_batch(C.byref(self.c), _p(hmms), len(hmms)))

    def sweep(self, hmms, senscr):
        """T frames of hmm_vit_eval over the same records (updated in place); senscr int16 [T][n_sen];
        returns best int32 [T] (the evaluate_channels loop over a fixed active set)."""
        senscr = np.ascontiguousarray(senscr, np.int16)
        return np.array([self.vit_eval(hmms, senscr[t]) for t in range(len(senscr))], np.int32)


WORST_SCORE = -0x20000000


def hmm_clear(hmms, i):
    """hmm_clear (hmm.c:181-196) on record i of an HMM_DTYPE array."""
    n = int(hmms["n_emit_state"][i])
    hmms["score"][i, :n] = WORST_SCORE
    hmms["history"][i, :n] = -1
    hmms["out_score"][i] = WORST_SCORE
    hmms["out_history"][i] = -1
    hmms["bestscore"][i] = WORST_SCORE
    hmms["frame"][i] = -1


def sweep_beam(ctx, hmms, senscr, frame0, beam, maxhmmpf=-1, clear=hmm_clear):
    """T frames of "evaluate the active instances, then prune to the beam" over a flat set of hmm_t
    (updated in place): evaluate_channels (ngram_search_fwdtree.c:702-715) and, of prune_channels
    (:1130-1181), the best score, the -maxhmmpf histogram (256 bins of width -beam / 256, walked until
    the running count exceeds maxhmmpf) and prune_nonroot_chan's decision (:811, :823-827, :872-874):
    bestscore BETTER_THAN best + dynamic beam -> frame = f + 1, else hmm_clear.  No transitions: an
    instance that leaves never returns.  ctx.vit_eval(records, row) is hmm_vit_eval over an array
    (OracleHmmCtx or the compiled reference's RefHmmCtx); clear(hmms, i) is hmm_clear.
    Returns (best int32 [T], n_evaluated int32 [T])."""
    senscr = np.ascontiguousarray(senscr, np.int16)
    T = len(senscr)
    best_out = np.full(T, WORST_SCORE, np.int32)
    n_out = np.zeros(T, np.int32)
    for t in range(T):
        f = frame0 + t
        idx = np.flatnonzero(hmms["frame"] == f)
        n_out[t] = len(idx)
        if len(idx) == 0:
            continue
        sub = np.ascontiguousarray(hmms[idx])
        best = ctx.vit_eval(sub, senscr[t])
        hmms[idx] = sub
        best_out[t] = best
        dyn = beam
        if maxhmmpf != -1 and len(idx) > maxhmmpf:
            bw = -beam // 256
            bins = np.zeros(256, np.int64)
            for i in idx:
                b = (best - int(hmms["bestscore"][i])) // bw        # both operands >= 0: C's truncation = floor
                bins[min(b, 255)] += 1
            nh, i = 0, 0
            while i < 256:
                nh += bins[i]
                if nh > maxhmmpf:
                    break
                i += 1
            dyn = -(i * bw)
        thresh = best + dyn
        for i in idx:
            if int(hmms["bestscore"][i]) > thresh:
                hmms["frame"][i] = f + 1
            else:
                clear(hmms, i)
    return best_out, n_out


def phoneloop_run(tp, sseq, ssid, tmatid, senscr, window, beam, pbeam, pip, penalty_weight):
    """phone_loop_search.c semantics over a [T][n_sen] senone score matrix."""
    tp = np.ascontiguousarray(tp, np.uint8)
    sseq = np.ascontiguousarray(sseq, np.uint16)
    ssid = np.ascontiguousarray(ssid, np.int32)
    tmatid = np.ascontiguousarray(tmatid, np.int32)
    senscr = np.ascontiguousarray(senscr, np.int16)
    T, n_sen = senscr.shape
    n = len(ssid)
    p = lib().pso_phoneloop_new(tp.shape[1], _p(tp), _p(sseq), n, _p(ssid), _p(tmatid),
                                window, beam, pbeam, pip, float(penalty_weight))
    hm = np.zeros((T, n), HMM_DTYPE)
    best = np.zeros(T, np.int32)
    pen = np.zeros((T, n), np.int32)
    lib().pso_phoneloop_run(p, _p(senscr), n_sen, T, _p(hm), _p(best), _p(pen))
    lib().pso_phoneloop_free(p)
    return dict(hmm=hm, best=best, pen=pen)


def align_run(tp, sseq, ssid, tmatid, senscr, sf=None, ef=None):
    """state_align_search.c semantics for one utterance over a [T][n_sen] score matrix.
    Returns (status, start, dur, score) per emitting state."""
    tp = np.ascontiguousarray(tp, np.uint8)
    sseq = np.ascontiguousarray(sseq, np.uint16)
    ssid = np.ascontiguousarray(ssid, np.int32)
    tmatid = np.ascontiguousarray(tmatid, np.int32)
    senscr = np.ascontiguousarray(senscr, np.int16)
    T, n_sen = senscr.shape
    n_emit = tp.shape[1]
    n_st = len(ssid) * n_emit
    out = np.zeros((3, n_st), np.int32)
    sf = None if sf is None else np.ascontiguousarray(sf, np.int32)
    ef = None if ef is None else np.ascontiguousarray(ef, np.int32)
    f = lib().pso_align_run
    f.restype = C.c_int32
    f.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    rc = f(n_emit, _p(tp), _p(sseq), len(ssid), _p(ssid), _p(tmatid), _p(sf), _p(ef), _p(senscr), n_sen, T,
           _p(out[0]), _p(out[1]), _p(out[2]))
    return int(rc), out[0].copy(), out[1].copy(), out[2].copy()


def kws_run(tp, sseq, pl_ssid, pl_tmat, kp_off, kp_thresh, kp_ssid, kp_tmat, beam, plp, senscr):
    """kws_search.c semantics for one utterance; returns the raw hits [n][5] =
    (frame, keyphrase, sf, prob, ascr) in the order the reference hands them to kws_detections_add."""
    tp = np.ascontiguousarray(tp, np.uint8); sseq = np.ascontiguousarray(sseq, np.uint16)
    a = [np.ascontiguousarray(x, np.int32) for x in (pl_ssid, pl_tmat, kp_off, kp_thresh, kp_ssid, kp_tmat)]
    senscr = np.ascontiguousarray(senscr, np.int16)
    T, n_sen = senscr.shape
    cap = max(1, T * (len(a[2]) - 1))
    hits = np.zeros((cap, 5), np.int32)
    f = lib().pso_kws_run
    f.restype = C.c_int32
    f.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                  C.c_void_p, C.c_int32]
    n = f(tp.shape[1], _p(tp), _p(sseq), len(a[0]), _p(a[0]), _p(a[1]), len(a[2]) - 1, _p(a[2]), _p(a[3]), _p(a[4]),
          _p(a[5]), int(beam), int(plp), _p(senscr), n_sen, T, _p(hits), cap)
    return hits[:n].copy()


def kws_detections(hits):
    """kws_detections_add (kws_detections.c:55-80) applied to raw hits in order: overlapping
    detections of one keyphrase keep the better one.  Returns rows (keyphrase, sf, ef, prob, ascr) in
    the reference's list order (newest first: glist_add_ptr prepends)."""
    lst = []
    for frame, k, sf, prob, ascr in hits.tolist():
        ef = frame
        for d in lst:
            if d[0] == k and d[1] < ef and d[2] > sf:
                if d[3] < prob:
                    d[1], d[2], d[3], d[4] = sf, ef, prob, ascr
                break
        else:
            lst.insert(0, [k, sf, ef, prob, ascr])
    return np.array(lst, np.int32).reshape(-1, 5)


def allphone_run(tp, sseq, ssid, tmatid, succ_off, succ, start, beam, pbeam, inspen, senscr, cap=None):
    """allphone_search.c (no phone LM) for one utterance; returns the history table
    [n][4] = (ef, node, hist, score)."""
    tp = np.ascontiguousarray(tp, np.uint8); sseq = np.ascontiguousarray(sseq, np.uint16)
    a = [np.ascontiguousarray(x, np.int32) for x in (ssid, tmatid, succ_off, succ)]
    senscr = np.ascontiguousarray(senscr, np.int16)
    T, n_sen = senscr.shape
    cap = cap or max(1, T * len(a[0]))
    hist = np.zeros((cap, 4), np.int32)
    f = lib().pso_allphone_run
    f.restype = C.c_int32
    f.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32]
    n = f(tp.shape[1], _p(tp), _p(sseq), len(a[0]), _p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), int(start), int(beam),
          int(pbeam), int(inspen), _p(senscr), n_sen, T, _p(hist), cap)
    return hist[:min(n, cap)].copy(), n


def allphone_backtrace(hist, node_ci, last_frame, inspen):
    """allphone_backtrace (allphone_search.c:765-840) over a history table: best entry ending in the
    last frame that has one, then the chain of predecessors.  Returns rows (ci, sf, ef, score, tscore)
    in the reference's segment-list order (time ascending)."""
    n = len(hist)
    hi = n - 1
    frm = last = last_frame
    while hi > 0:
        if hist[hi][0] <= last_frame:
            frm = last = int(hist[hi][0])
            break
        hi -= 1
    if hi < 0:
        return np.zeros((0, 5), np.int32)
    best, best_idx = -2**31, -1
    while frm == last and hi > 0:
        frm = int(hist[hi][0])
        if hist[hi][3] > best and frm == last:
            best, best_idx = int(hist[hi][3]), hi
        hi -= 1
    segs = []
    while best_idx > 0:
        ef, node, hh, score = [int(x) for x in hist[best_idx]]
        sf = int(hist[hh][0]) + 1 if hh > 0 else 0
        asc = score - (int(hist[hh][3]) if hh > 0 else 0) - inspen
        segs.insert(0, [int(node_ci[node]), sf, ef, asc, inspen])
        best_idx = hh
    return np.array(segs, np.int32).reshape(-1, 5)


def allphone_lm_run(tp, sseq, ssid, tmatid, succ_off, succ, start, beam, pbeam, node_ci, bg, tg, senscr, cap=None):
    """allphone_search.c with a phone LM (dense bigram / trigram tables); history rows
    [n][5] = (ef, node, hist, score, tscore)."""
    tp = np.ascontiguousarray(tp, np.uint8); sseq = np.ascontiguousarray(sseq, np.uint16)
    a = [np.ascontiguousarray(x, np.int32) for x in (ssid, tmatid, succ_off, succ, node_ci, bg, tg)]
    senscr = np.ascontiguousarray(senscr, np.int16)
    T, n_sen = senscr.shape
    n_ci = int(round(len(a[5].ravel()) ** 0.5))
    cap = cap or max(1, T * len(a[0]))
    hist = np.zeros((cap, 5), np.int32)
    f = lib().pso_allphone_lm_run
    f.restype = C.c_int32
    f.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                  C.c_int32, C.c_void_p, C.c_int32]
    n = f(tp.shape[1], _p(tp), _p(sseq), len(a[0]), _p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), int(start), int(beam),
          int(pbeam), n_ci, _p(a[4]), _p(a[5]), _p(a[6]), _p(senscr), n_sen, T, _p(hist), cap)
    return hist[:min(n, cap)].copy(), n


def allphone_backtrace_lm(hist, node_ci, last_frame):
    """allphone_backtrace for history rows that carry their own tscore (5 columns)."""
    n = len(hist)
    hi = n - 1
    frm = last = last_frame
    while hi > 0:
        if hist[hi][0] <= last_frame:
            frm = last = int(hist[hi][0])
            break
        hi -= 1
    best, best_idx = -2**31, -1
    while frm == last and hi > 0:
        frm = int(hist[hi][0])
        if hist[hi][3] > best and frm == last:
            best, best_idx = int(hist[hi][3]), hi
        hi -= 1
    segs = []
    while best_idx > 0:
        ef, node, hh, score, tscore = [int(x) for x in hist[best_idx]]
        sf = int(hist[hh][0]) + 1 if hh > 0 else 0
        asc = score - (int(hist[hh][3]) if hh > 0 else 0) - tscore
        segs.insert(0, [int(node_ci[node]), sf, ef, asc, tscore])
        best_idx = hh
    return np.array(segs, np.int32).reshape(-1, 5)


def fsg_run(tp, sseq, g, senscr, cap=None):
    """fsg_search.c for one utterance on a flattened lextree `g` (what refdrv.fsg / the golden file
    hold: pnodes, roots, links, nulloff, nullarc, beams, ...); returns the history table
    [n][13] = (link, frame, score, pred, lc, rc.bv[8])."""
    tp = np.ascontiguousarray(tp, np.uint8); sseq = np.ascontiguousarray(sseq, np.uint16)
    pn, roots, links, nulloff, nullarc = (np.ascontiguousarray(g[k], np.int32)
                                          for k in ("pnodes", "roots", "links", "nulloff", "nullarc"))
    senscr = np.ascontiguousarray(senscr, np.int16)
    T, n_sen = senscr.shape
    cap = cap or max(1024, 8 * T * max(1, len(links)))
    hist = np.zeros((cap, 13), np.int32)
    f = lib().pso_fsg_run
    f.restype = C.c_int32
    f.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                  C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int32] * 7 + [C.c_void_p, C.c_int32, C.c_int32,
                                                                            C.c_void_p, C.c_int32]
    n = f(tp.shape[1], _p(tp), _p(sseq), len(pn), _p(pn), len(roots), _p(roots), len(links), _p(links), _p(nulloff),
          _p(nullarc), int(g["n_ciphone"]), int(g["silcipid"]), int(g["start_state"]), int(g["beam"]), int(g["pbeam"]),
          int(g["wbeam"]), int(g["maxhmmpf"]), _p(senscr), n_sen, T, _p(hist), cap)
    assert n <= cap
    return hist[:n].copy()


def fsg_find_exit(hist, links, frame_idx, final_state, final=True):
    """fsg_search_find_exit (fsg_search.c:886-958): best word exit in the last frame <= frame_idx that
    has one (preferring, and when final requiring, the grammar's final state).  Returns (index, score)."""
    bp = len(hist) - 1
    frm = last = frame_idx
    while bp > 0:
        if hist[bp][1] <= frame_idx:
            frm = last = int(hist[bp][1])
            break
        bp -= 1
    if bp <= 0:
        return bp, None
    best, besthist = -(1 << 31), -1
    while frm == last:
        l, score = int(hist[bp][0]), int(hist[bp][2])
        if l < 0:
            break
        to = int(links[l][1])
        if score == best and to == final_state:
            besthist = bp
        elif score > best and (not final or to == final_state):
            best, besthist = score, bp
        bp -= 1
        if bp < 0:
            break
        frm = int(hist[bp][1])
    return besthist, (best if besthist >= 0 else None)


def fsg_hyp_wids(hist, links, bp):
    """The word ids along the predecessor chain of entry bp (fsg_search_hyp, fsg_search.c:1012-1060),
    in time order; null transitions (wid < 0) are kept out like in the reference."""
    out = []
    while bp > 0:
        l = int(hist[bp][0])
        if l >= 0 and links[l][2] >= 0:
            out.append(int(links[l][2]))
        bp = int(hist[bp][3])
    return out[::-1]


def fwdtree_run(tp, sseq, ci_tmat, info, model, senscr, pl_pen=None, pl_window=0, pen_in_force=None, lm_arrays=None):
    """ngram_search_fwdtree.c for one utterance on the flattened search `info` / `model`
    (refdrv.fwdtree / the golden file); returns (bp table [n][10], bscore_stack, bp_table_idx).
    pl_pen [T][n_ci] + pl_window: the phone loop's penalties after each of ITS steps and its window;
    frame t of the search runs after the phone loop has seen frame min(t + window, T - 1)
    (ps_search_forward / ps_end_utt, pocketsphinx.c:1172-1195, 1329-1333).  pen_in_force [T][n_ci]
    gives the penalties per SEARCH frame directly instead."""
    tp = np.ascontiguousarray(tp, np.uint8); sseq = np.ascontiguousarray(sseq, np.uint16)
    ci_tmat = np.ascontiguousarray(ci_tmat, np.int32)
    info = np.ascontiguousarray(info, np.int32); model = np.ascontiguousarray(model, np.int32)
    senscr = np.ascontiguousarray(senscr, np.int16)
    T, n_sen = senscr.shape
    bp_cap, bss_cap = 64 * (T + 16), 64 * (T + 16) * 64
    bp = np.zeros((bp_cap, 10), np.int32); bss = np.zeros(bss_cap, np.int32); bp_idx = np.zeros(T + 2, np.int32)
    bss_n = C.c_int32()
    pen = None
    if pen_in_force is not None and T > 0:
        pen = np.ascontiguousarray(pen_in_force, np.int32)
        assert pen.shape[0] == T
    elif pl_pen is not None and pl_window > 0 and T > 0:
        pen = np.ascontiguousarray(np.asarray(pl_pen, np.int32)[np.minimum(np.arange(T) + pl_window, T - 1)])
    f = lib().pso_fwdtree_run
    f.restype = C.c_int32
    f.argtypes = [C.c_int32] + [C.c_void_p] * 6 + [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                                    C.c_int32, C.c_void_p, C.c_void_p]
    lma = None if lm_arrays is None else np.ascontiguousarray(lm_arrays, np.int32)
    n = f(tp.shape[1], _p(tp), _p(sseq), _p(ci_tmat), _p(info), _p(model), _p(senscr), n_sen, T,
          _p(pen) if pen is not None else None, _p(lma) if lma is not None else None, _p(bp), bp_cap, _p(bss),
          bss_cap, C.byref(bss_n), _p(bp_idx))
    assert n <= bp_cap and bss_n.value <= bss_cap
    return bp[:n].copy(), bss[:bss_n.value].copy(), bp_idx[:T + 1].copy()


def fwdtree_find_exit(bp, bp_idx, n_frame, finish_wid):
    """ngram_search_find_exit (ngram_search.c:501-541) with frame_idx = -1: </s> in the last frame
    that has exits, else its best-scoring entry.  Returns (index or -1, score)."""
    if n_frame == 0:
        return -1, None
    f = n_frame - 1
    end = int(bp_idx[f])
    while f >= 0 and bp_idx[f] == end:
        f -= 1
    if f < 0:
        return -1, None
    best, best_exit = -0x20000000, -1
    for b in range(int(bp_idx[f]), end):
        if bp[b][2] == finish_wid or bp[b][4] > best:
            best, best_exit = int(bp[b][4]), b
        if bp[b][2] == finish_wid:
            break
    return best_exit, best


def fwdtree_hyp(bp, b, words, vocab, start_wid, finish_wid):
    """ngram_search_bp_hyp (:545-590): base strings of the real words (dict_real_word: neither
    filler nor <s> / </s>) along the backpointer chain."""
    out = []
    while b != -1:
        w = int(bp[b][2])
        b = int(bp[b][3])
        if not words[w][4] and int(words[w][5]) not in (start_wid, finish_wid):
            out.append(vocab[int(words[w][5])])
    return " ".join(reversed(out))


def fwdflat_run(tp, sseq, ci_tmat, ci_ssid, info, model, bp_first, senscr, lm_arrays=None):
    """ngram_search_fwdflat.c for one utterance: bp_first = the first pass's backpointer table,
    info / model from an export made with fwdflat=yes.  Returns (bp table, bscore_stack, bp_table_idx)."""
    tp = np.ascontiguousarray(tp, np.uint8); sseq = np.ascontiguousarray(sseq, np.uint16)
    ci_tmat = np.ascontiguousarray(ci_tmat, np.int32); ci_ssid = np.ascontiguousarray(ci_ssid, np.int32)
    info = np.ascontiguousarray(info, np.int32); model = np.ascontiguousarray(model, np.int32)
    n_first = -1 if bp_first is None else len(bp_first)                     # None: -fwdtree no
    bp_first = np.zeros((1, 10), np.int32) if bp_first is None else np.ascontiguousarray(bp_first, np.int32)
    senscr = np.ascontiguousarray(senscr, np.int16)
    T, n_sen = senscr.shape
    bp_cap, bss_cap = 64 * (T + 16), 64 * (T + 16) * 64
    bp = np.zeros((bp_cap, 10), np.int32); bss = np.zeros(bss_cap, np.int32); bp_idx = np.zeros(T + 2, np.int32)
    bss_n = C.c_int32()
    f = lib().pso_fwdflat_run
    f.restype = C.c_int32
    f.argtypes = [C.c_int32] + [C.c_void_p] * 7 + [C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                                    C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lma = None if lm_arrays is None else np.ascontiguousarray(lm_arrays, np.int32)
    n = f(tp.shape[1], _p(tp), _p(sseq), _p(ci_tmat), _p(ci_ssid), _p(info), _p(model), _p(bp_first), n_first,
          _p(senscr), n_sen, T, _p(lma) if lma is not None else None, _p(bp), bp_cap, _p(bss), bss_cap, C.byref(bss_n), _p(bp_idx))
    assert n <= bp_cap and bss_n.value <= bss_cap
    return bp[:n].copy(), bss[:bss_n.value].copy(), bp_idx[:T + 1].copy()


def lm_scores(lmarr, queries):
    """tg(w | h1, h2) >> SENSCR_SHIFT from the LM as sorted arrays, for queries [n][3] of dictionary ids."""
    lmarr = np.ascontiguousarray(lmarr, np.int32)
    q = np.ascontiguousarray(queries, np.int32)
    out = np.zeros(len(q), np.int32)
    f = lib().pso_lm_scores
    f.restype = None
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    f(_p(lmarr), _p(q), len(q), _p(out))
    return out
