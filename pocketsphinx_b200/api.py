"""Host-side mirror of the reference's operator interface for the hot path, over the C-ABI.

Names follow the reference: a `Mgau` is a ps_mgau_t-like scorer (frame_eval / transform /
free, acmod.h:98-125), `HmmContext.vit_eval` is the batched hmm_vit_eval (hmm.h:282),
`PhoneLoop` runs phone_loop_search.c's frame loop on the device.  Everything goes through
libpsb200.so; nothing here computes scores on the CPU.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import ModelDesc, PsbError, check, lib
from .model import PackedModel

KIND_ID = {"ptm": 0, "s2_semi": 1, "ms": 2}

# the reference's hmm_t, byte for byte (hmm.h:169-182)
HMM_DTYPE = np.dtype({
    "names": ["ctx", "score", "history", "out_score", "out_history", "ssid", "senid",
              "bestscore", "tmatid", "frame", "mpx", "n_emit_state"],
    "formats": ["<u8", ("<i4", 5), ("<i4", 5), "<i4", "<i4", "<u2", ("<u2", 5),
                "<i4", "<i2", "<i4", "u1", "u1"],
    "offsets": [0, 8, 28, 48, 52, 56, 58, 68, 72, 76, 80, 81],
    "itemsize": 88,
})


def _p(a):
    if a is None:
        return None
    if hasattr(a, "data_ptr"):          # torch tensor (host-pinned or device)
        return a.data_ptr()
    return a.ctypes.data if a.size else None


def device_count():
    return lib().psb_device_count()


class Model:
    """Device-resident acoustic model (psb_model_t)."""

    def __init__(self, pm: PackedModel, device=0, device_ptrs=None):
        self.pm = pm
        d = ModelDesc()
        d.kind = KIND_ID[pm.kind]
        d.n_sen, d.n_mgau, d.n_feat, d.n_density, d.topn = pm.n_sen, pm.n_mgau, pm.n_feat, pm.n_density, pm.topn
        for i, v in enumerate(pm.featlen):
            d.featlen[i] = int(v)
        d.ds_ratio = int(pm.ds_ratio)
        d.aw = int(pm.aw)
        d.logadd_ms_size = int(pm.logadd_ms.size)
        d.logadd_ms_zero = int(pm.logadd_ms_zero)
        d.fixed_point = int(getattr(pm, "fixed_point", 0))   # arrays then carry the FIXED_POINT build's int32 bit patterns
        if device_ptrs is None:
            d.on_device = 0
            d.mean, d.var, d.det, d.mixw = _p(pm.mean), _p(pm.var), _p(pm.det), _p(pm.mixw)
            d.mixw_cb = _p(pm.mixw_cb) if pm.mixw_4bit else None
            d.sen2cb, d.logadd8 = _p(pm.sen2cb), _p(pm.logadd8)
            d.logadd_ms = _p(pm.logadd_ms)
            d.topn_beam = _p(pm.topn_beam) if pm.topn_beam.size else None
        else:                           # e.g. torch tensors filled by an NCCL broadcast
            d.on_device = 1
            for k in ("mean", "var", "det", "mixw", "mixw_cb", "sen2cb", "logadd8", "logadd_ms", "topn_beam"):
                setattr(d, k, _p(device_ptrs.get(k)))
        self._keep = device_ptrs
        h = C.c_void_p()
        check(lib().psb_model_create(C.byref(d), device, C.byref(h)), "psb_model_create")
        self.h = h
        self.device = device

    def update_gaussians(self, mean, var, det):
        """ps_mgaufuncs_t.transform: re-upload MLLR-adapted Gaussians."""
        mean = np.ascontiguousarray(mean, np.float32)
        var = np.ascontiguousarray(var, np.float32)
        det = np.ascontiguousarray(det, np.float32)
        check(lib().psb_model_update_gaussians(self.h, _p(mean), _p(var), _p(det)), "psb_model_update_gaussians")

    def close(self):
        if self.h:
            lib().psb_model_free(self.h)
            self.h = None


class Mgau:
    """ps_mgau_t twin: one decoder's scorer with its history ring and frame_idx."""

    def __init__(self, model: Model, pl_window=0):
        self.model = model
        h = C.c_void_p()
        check(lib().psb_scorer_create(model.h, pl_window + 2, C.byref(h)), "psb_scorer_create")
        self.h = h

    @property
    def frame_idx(self):
        return lib().psb_scorer_get_frame_idx(self.h)

    @frame_idx.setter
    def frame_idx(self, v):
        check(lib().psb_scorer_set_frame_idx(self.h, int(v)), "psb_scorer_set_frame_idx")

    def reset(self):
        check(lib().psb_scorer_reset(self.h), "psb_scorer_reset")

    def frame_eval(self, feat_row, frame, senone_active=None, compallsen=True, out=None):
        """out: the caller-owned int16[n_sen] buffer (acmod->senone_scores); the ms back-end leaves
        the entries of unlisted senones untouched, so pass the same buffer across calls."""
        pm = self.model.pm
        feat_row = np.ascontiguousarray(feat_row, np.float32)
        ptrs = (C.c_void_p * pm.n_feat)()
        off = 0
        for f in range(pm.n_feat):
            ptrs[f] = feat_row.ctypes.data + 4 * off
            off += int(pm.featlen[f])
        scr = np.zeros(pm.n_sen, np.int16) if out is None else out
        n = 0
        if senone_active is not None:
            senone_active = np.ascontiguousarray(senone_active, np.uint8)
            n = len(senone_active)
        check(lib().psb_scorer_frame_eval(self.h, _p(scr), _p(senone_active), n, ptrs, int(frame), int(compallsen)),
              "psb_scorer_frame_eval")
        return scr

    def close(self):
        if self.h:
            lib().psb_scorer_free(self.h)
            self.h = None


class Batch:
    """Batched utterance scoring workspace (psb_batch_t)."""

    def __init__(self, model: Model, max_utts, max_frames):
        self.model = model
        h = C.c_void_p()
        check(lib().psb_batch_create(model.h, int(max_utts), int(max_frames), C.byref(h)), "psb_batch_create")
        self.h = h

    @staticmethod
    def offsets(lengths):
        off = np.zeros(len(lengths) + 1, np.int32)
        np.cumsum(lengths, out=off[1:])
        return off

    def score_host(self, feats, utt_off, out=None):
        """feats: [total][sumlen] float32 host array (numpy or pinned torch); returns int16 [total][n_sen]."""
        pm = self.model.pm
        total = int(utt_off[-1])
        if out is None:
            out = np.zeros((total, pm.n_sen), np.int16)
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        check(lib().psb_batch_score_host(self.h, _p(feats), _p(utt_off), len(utt_off) - 1, _p(out)),
              "psb_batch_score_host")
        return out

    def score_device(self, d_feats_ptr, utt_off, d_senscr_ptr=None):
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        check(lib().psb_batch_score_device(self.h, d_feats_ptr, _p(utt_off), len(utt_off) - 1, d_senscr_ptr),
              "psb_batch_score_device")

    def sync(self):
        check(lib().psb_batch_sync(self.h), "psb_batch_sync")

    def senscr_device_ptr(self):
        return lib().psb_batch_senscr_device(self.h)

    def last_kernel_ms(self):
        out = np.zeros(3, np.float32)
        check(lib().psb_batch_last_kernel_ms(self.h, _p(out)), "psb_batch_last_kernel_ms")
        return dict(transpose=float(out[0]), topn=float(out[1]), senone=float(out[2]))

    def set_pipeline(self, n):
        check(lib().psb_batch_set_pipeline(self.h, int(n)), "psb_batch_set_pipeline")

    def event_record(self, slot):
        check(lib().psb_batch_event_record(self.h, slot), "psb_batch_event_record")

    def event_elapsed_ms(self):
        ms = C.c_float()
        check(lib().psb_batch_event_elapsed_ms(self.h, C.byref(ms)), "psb_batch_event_elapsed_ms")
        return ms.value

    def run_phoneloop_device(self, phoneloop, utt_off, d_best_ptr=None, d_pen_ptr=None):
        """Phone loop over this batch's device-resident scores, on this batch's stream."""
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        check(lib().psb_phoneloop_run_device(phoneloop.h, self.senscr_device_ptr(), _p(utt_off), len(utt_off) - 1,
                                             d_best_ptr, d_pen_ptr, None, self.h), "psb_phoneloop_run_device")

    def decode_device(self, phoneloop, d_feats_ptr, utt_off):
        """Asynchronous device-resident decode; returns device addresses of best / penalties."""
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        pb, pp = C.c_void_p(), C.c_void_p()
        check(lib().psb_decode_batch_device(self.h, phoneloop.h, d_feats_ptr, _p(utt_off), len(utt_off) - 1,
                                            C.byref(pb), C.byref(pp)), "psb_decode_batch_device")
        return pb.value, pp.value

    def get_topn(self, n_frames):
        rec = np.zeros((n_frames, self.model.pm.n_mgau * self.model.pm.n_feat, 4), np.int32)
        check(lib().psb_batch_get_topn(self.h, _p(rec), n_frames), "psb_batch_get_topn")
        return rec

    TC_COUNTERS = ("rows", "from_filter_alone", "exact_distances", "tie_fixups", "over_cap", "lane_over",
                   "fallback_listed", "fallback_all", "split_lists", "fail_gap", "fail_straddle", "fail_sign",
                   "fail_saturation", "tiles_per_cta", "ctas_per_pair")

    def tc_check(self):
        """(max |filter value - exact distance| / bound, max candidates) of the tensor-core filter (PSB_TC_CHECK=1);
        tc_stats gets its decision-path counters by name (psb_batch_tc_counters)."""
        r, n = C.c_float(), C.c_int32()
        check(lib().psb_batch_tc_check(self.h, C.byref(r), C.byref(n), None), "psb_batch_tc_check")
        st = np.zeros(len(self.TC_COUNTERS), np.int64)
        check(lib().psb_batch_tc_counters(self.h, _p(st), len(st)), "psb_batch_tc_counters")
        self.tc_stats = {k: int(v) for k, v in zip(self.TC_COUNTERS, st)}
        return r.value, n.value

    MS_PLAN = ("tile", "fuse", "prefetch", "nt", "n_used", "all", "frames_per_cta", "tiles_x", "chunk", "n_chunks",
               "dist_bytes", "n_sm", "transposed", "tile_smem")

    def ms_plan(self, total_frames):
        """How a batch of total_frames frames on an ms model is scored (psb_batch_ms_plan), by name."""
        v = np.zeros(len(self.MS_PLAN), np.int64)
        check(lib().psb_batch_ms_plan(self.h, int(total_frames), _p(v), len(v)), "psb_batch_ms_plan")
        return {k: int(x) for k, x in zip(self.MS_PLAN, v)}

    TM_TOPN = ("tc_filter", "ptm_scan", "ptm_scalar", "semi_split", "fixed")
    TM_SENONE = ("ptm_senone4", "ptm_senone_8b", "ptm_senone_4b", "semi_senone4", "semi_senone_8b", "semi_senone_4b")

    def tm_plan(self, total_frames):
        """How a batch of total_frames frames on a ptm or semi-continuous model is scored (psb_batch_tm_plan): "topn",
        the top-N paths of its streams joined by "+"; "senone", the senone kernel; "threads", "n_bsen" and "smem" of
        the senone launch."""
        v = np.zeros(5, np.int64)
        check(lib().psb_batch_tm_plan(self.h, int(total_frames), _p(v), len(v)), "psb_batch_tm_plan")
        return dict(topn="+".join(n for i, n in enumerate(self.TM_TOPN) if int(v[0]) >> i & 1),
                    senone=self.TM_SENONE[int(v[1])], threads=int(v[2]), n_bsen=int(v[3]), smem=int(v[4]))

    def decode_host(self, phoneloop, feats, utt_off, want_senscr=False, best=None, pen=None, senscr=None):
        """End to end: host features -> senone scores -> phone-loop Viterbi -> host results."""
        pm = self.model.pm
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        total = int(utt_off[-1])
        if best is None:
            best = np.zeros(total, np.int32)
        if pen is None:
            pen = np.zeros((total, phoneloop.n_phones), np.int32)
        if want_senscr and senscr is None:
            senscr = np.zeros((total, pm.n_sen), np.int16)
        check(lib().psb_decode_batch_host(self.h, phoneloop.h, _p(feats), _p(utt_off), len(utt_off) - 1,
                                          _p(best), _p(pen), _p(senscr) if want_senscr else None),
              "psb_decode_batch_host")
        return (best, pen, senscr) if want_senscr else (best, pen)

    def decode_pcm_host(self, fe, phoneloop, pcm, samp_off, want_senscr=False):
        """Audio in, phone-loop results out: (frame_off, best, pen[, senscr])."""
        pm = self.model.pm
        pcm = np.ascontiguousarray(pcm, np.int16)
        samp_off = np.ascontiguousarray(samp_off, np.int64)
        n_utt = len(samp_off) - 1
        total = sum(fe.n_frames(int(samp_off[u + 1] - samp_off[u])) for u in range(n_utt))
        frame_off = np.zeros(n_utt + 1, np.int32)
        best = np.zeros(total, np.int32)
        pen = np.zeros((total, phoneloop.n_phones), np.int32)
        senscr = np.zeros((total, pm.n_sen), np.int16) if want_senscr else None
        check(lib().psb_decode_batch_pcm_host(self.h, fe.h, phoneloop.h, _p(pcm) if pcm.size else None, _p(samp_off), n_utt,
                                              _p(frame_off), _p(best), _p(pen), _p(senscr) if want_senscr else None),
              "psb_decode_batch_pcm_host")
        return (frame_off, best, pen, senscr) if want_senscr else (frame_off, best, pen)

    def score_pcm(self, fe, pcm, samp_off):
        """Audio in, senone scores out, all on the device: the front end's features go straight to the scorer and the
        scores stay at senscr_device_ptr() (ready when this returns).  Returns frame_off int32 [n_utt+1]."""
        pcm = np.ascontiguousarray(pcm, np.int16)
        samp_off = np.ascontiguousarray(samp_off, np.int64)
        n_utt = len(samp_off) - 1
        frame_off = np.zeros(n_utt + 1, np.int32)
        check(lib().psb_fe_process_host(fe.h, _p(pcm) if pcm.size else None, _p(samp_off), n_utt, None, None,
                                        _p(frame_off)), "psb_fe_process_host")
        if frame_off[-1]:
            self.score_device(lib().psb_fe_device_feats(fe.h), frame_off)
            self.sync()
        return frame_off

    def close(self):
        if self.h:
            lib().psb_batch_free(self.h)
            self.h = None


class HmmContext:
    """hmm_context_t twin (hmm.h:145-154) on the device."""

    def __init__(self, tp, sseq, n_sen, device=0):
        self.tp = np.ascontiguousarray(tp, np.uint8)
        self.sseq = np.ascontiguousarray(sseq, np.uint16)
        self.n_emit = self.tp.shape[1]
        self.n_sen = n_sen
        h = C.c_void_p()
        check(lib().psb_hmmctx_create(self.n_emit, _p(self.tp), self.tp.shape[0], _p(self.sseq),
                                      self.sseq.shape[0], n_sen, device, C.byref(h)), "psb_hmmctx_create")
        self.h = h

    def vit_eval(self, hmms, senscr):
        """In-place batched hmm_vit_eval over an array of 88-byte hmm_t records; returns best score."""
        assert hmms.dtype == HMM_DTYPE and hmms.flags.c_contiguous
        senscr = np.ascontiguousarray(senscr, np.int16)
        best = C.c_int32()
        check(lib().psb_hmm_vit_eval_batch(self.h, _p(hmms) if len(hmms) else None, len(hmms), _p(senscr),
                                           C.byref(best)), "psb_hmm_vit_eval_batch")
        return best.value

    def vit_eval_ptrs(self, hmms, index, senscr):
        """Same through an active list of pointers into `hmms` (chan_t* style)."""
        senscr = np.ascontiguousarray(senscr, np.int16)
        ptrs = (C.c_void_p * len(index))(*[hmms.ctypes.data + 88 * int(i) for i in index])
        best = C.c_int32()
        check(lib().psb_hmm_vit_eval_ptrs(self.h, ptrs, len(index), _p(senscr), C.byref(best)),
              "psb_hmm_vit_eval_ptrs")
        return best.value

    def allphone(self, d_senscr_ptr, utt_off, ssid, tmatid, succ_off, succ, start, beam, pbeam, inspen, cap=None):
        """allphone_search (no phone LM) over a batch.  Returns (list of history tables [n][4] =
        (ef, node, predecessor entry, score), counts)."""
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        a = [np.ascontiguousarray(x, np.int32) for x in (ssid, tmatid, succ_off, succ)]
        n_utt = len(utt_off) - 1
        if cap is None:
            cap = max(1, int(np.diff(utt_off).max(initial=1)) * len(a[0]))
        hist = np.zeros((max(1, n_utt), cap, 4), np.int32)
        n_hist = np.zeros(max(1, n_utt), np.int32)
        check(lib().psb_allphone_batch_device(self.h, C.c_void_p(d_senscr_ptr), _p(utt_off), n_utt, len(a[0]), _p(a[0]),
                                              _p(a[1]), _p(a[2]), _p(a[3]), int(start), int(beam), int(pbeam), int(inspen),
                                              _p(hist), cap, _p(n_hist)), "psb_allphone_batch_device")
        return [hist[u, :min(int(n_hist[u]), cap)].copy() for u in range(n_utt)], n_hist[:n_utt].copy()

    def fsg(self, d_senscr_ptr, utt_off, g, cap):
        """fsg_search over a batch, every utterance against the flattened grammar lextree `g` (a mapping
        with pnodes, roots, links, nulloff, nullarc, n_ciphone, silcipid, start_state, beam, pbeam,
        wbeam, maxhmmpf).  Returns the list of history tables [n][13] = (link, frame, score, pred,
        lc, rc.bv[8]) and the entry counts."""
        from ._lib import FsgDesc
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        n_utt = len(utt_off) - 1
        a = {k: np.ascontiguousarray(g[k], np.int32) for k in ("pnodes", "roots", "links", "nulloff", "nullarc")}
        d = FsgDesc(len(a["pnodes"]), a["pnodes"].ctypes.data, len(a["roots"]), a["roots"].ctypes.data,
                    len(a["links"]), a["links"].ctypes.data, a["nulloff"].ctypes.data,
                    a["nullarc"].ctypes.data if len(a["nullarc"]) else None, int(g["n_ciphone"]), int(g["silcipid"]),
                    int(g["start_state"]), int(g["beam"]), int(g["pbeam"]), int(g["wbeam"]), int(g["maxhmmpf"]))
        hist = np.zeros((max(n_utt, 1), int(cap), 13), np.int32)
        n_hist = np.zeros(max(n_utt, 1), np.int32)
        check(lib().psb_fsg_batch_device(self.h, C.byref(d), C.c_void_p(d_senscr_ptr), _p(utt_off), n_utt, _p(hist),
                                         int(cap), _p(n_hist)), "psb_fsg_batch_device")
        return [hist[u, :min(int(n_hist[u]), int(cap))] for u in range(n_utt)], n_hist[:n_utt]

    def ngram_fwdtree(self, d_senscr_ptr, utt_off, info, model, ci_tmat, bp_cap, bss_cap, d_pen_ptr=None, pl_window=0, lm_arrays=None):
        """ngram_search_fwdtree over a batch (flattened search `info` / `model`, see include/psb200.h).
        d_pen_ptr / pl_window: the phone loop's device penalty table and its window (look-ahead).
        Returns per utterance (bp table [n][10], bscore_stack, bp_table_idx [T+1])."""
        from ._lib import NgramDesc
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        n_utt = len(utt_off) - 1
        info = np.ascontiguousarray(info, np.int32); model = np.ascontiguousarray(model, np.int32)
        ci_tmat = np.ascontiguousarray(ci_tmat, np.int32)
        lma = None if lm_arrays is None else np.ascontiguousarray(lm_arrays, np.int32)
        d = NgramDesc(info.ctypes.data, model.ctypes.data, len(model), ci_tmat.ctypes.data, None,
                      None if lma is None else lma.ctypes.data, 0 if lma is None else len(lma))
        bp = np.zeros((max(n_utt, 1), int(bp_cap), 10), np.int32)
        bss = np.zeros((max(n_utt, 1), int(bss_cap)), np.int32)
        bp_idx = np.zeros(int(utt_off[-1]) + max(n_utt, 1), np.int32)
        res = np.zeros((max(n_utt, 1), 3), np.int32)
        check(lib().psb_ngram_fwdtree_batch_device(self.h, C.byref(d), C.c_void_p(d_senscr_ptr),
                                                   C.c_void_p(d_pen_ptr) if d_pen_ptr else None, int(pl_window), _p(utt_off), n_utt, _p(bp),
                                                   int(bp_cap), _p(bss), int(bss_cap), _p(bp_idx), _p(res)),
              "psb_ngram_fwdtree_batch_device")
        out = []
        for u in range(n_utt):
            T = int(utt_off[u + 1] - utt_off[u])
            o = int(utt_off[u]) + u
            out.append((bp[u, :res[u, 0]].copy(), bss[u, :res[u, 1]].copy(), bp_idx[o:o + T + 1].copy()))
        return out

    def ngram_fwdflat(self, d_senscr_ptr, utt_off, info, model, ci_tmat, ci_ssid, first_tables, bp_cap, bss_cap, lm_arrays=None):
        """ngram_search_fwdflat over a batch; first_tables = the first pass's bp table of every utterance.
        Returns per utterance (bp table [n][10], bscore_stack, bp_table_idx [T+1])."""
        from ._lib import NgramDesc
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        n_utt = len(utt_off) - 1
        info = np.ascontiguousarray(info, np.int32); model = np.ascontiguousarray(model, np.int32)
        ci_tmat = np.ascontiguousarray(ci_tmat, np.int32); ci_ssid = np.ascontiguousarray(ci_ssid, np.int32)
        lma = None if lm_arrays is None else np.ascontiguousarray(lm_arrays, np.int32)
        d = NgramDesc(info.ctypes.data, model.ctypes.data, len(model), ci_tmat.ctypes.data, ci_ssid.ctypes.data,
                      None if lma is None else lma.ctypes.data, 0 if lma is None else len(lma))
        cap_in = max([len(t) for t in first_tables] + [1])
        first = np.zeros((max(n_utt, 1), cap_in, 10), np.int32)
        n_first = np.zeros(max(n_utt, 1), np.int32)
        for u, t in enumerate(first_tables):
            first[u, :len(t)] = t
            n_first[u] = len(t)
        bp = np.zeros((max(n_utt, 1), int(bp_cap), 10), np.int32)
        bss = np.zeros((max(n_utt, 1), int(bss_cap)), np.int32)
        bp_idx = np.zeros(int(utt_off[-1]) + max(n_utt, 1), np.int32)
        res = np.zeros((max(n_utt, 1), 3), np.int32)
        check(lib().psb_ngram_fwdflat_batch_device(self.h, C.byref(d), C.c_void_p(d_senscr_ptr), _p(utt_off), n_utt, _p(first),
                                                   cap_in, _p(n_first), _p(bp), int(bp_cap), _p(bss), int(bss_cap), _p(bp_idx),
                                                   _p(res)), "psb_ngram_fwdflat_batch_device")
        out = []
        for u in range(n_utt):
            T = int(utt_off[u + 1] - utt_off[u])
            o = int(utt_off[u]) + u
            out.append((bp[u, :res[u, 0]].copy(), bss[u, :res[u, 1]].copy(), bp_idx[o:o + T + 1].copy()))
        return out

    def ngram_two_pass(self, d_senscr_ptr, utt_off, info, model, ci_tmat, ci_ssid, bp_cap, bss_cap, d_pen_ptr=None, pl_window=0,
                       first_cap=None, first_bss_cap=None, lm_arrays=None):
        """Both n-gram passes back to back on the device (first-pass tables never leave it).  Returns per
        utterance (bp table, bscore_stack, bp_table_idx) of the second pass, and the first pass's entry counts."""
        from ._lib import NgramDesc
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        n_utt = len(utt_off) - 1
        info = np.ascontiguousarray(info, np.int32); model = np.ascontiguousarray(model, np.int32)
        ci_tmat = np.ascontiguousarray(ci_tmat, np.int32); ci_ssid = np.ascontiguousarray(ci_ssid, np.int32)
        lma = None if lm_arrays is None else np.ascontiguousarray(lm_arrays, np.int32)
        d = NgramDesc(info.ctypes.data, model.ctypes.data, len(model), ci_tmat.ctypes.data, ci_ssid.ctypes.data,
                      None if lma is None else lma.ctypes.data, 0 if lma is None else len(lma))
        bp = np.zeros((max(n_utt, 1), int(bp_cap), 10), np.int32)
        bss = np.zeros((max(n_utt, 1), int(bss_cap)), np.int32)
        bp_idx = np.zeros(int(utt_off[-1]) + max(n_utt, 1), np.int32)
        res = np.zeros((max(n_utt, 1), 3), np.int32)
        res1 = np.zeros((max(n_utt, 1), 3), np.int32)
        check(lib().psb_ngram_two_pass_batch_device(self.h, C.byref(d), C.c_void_p(d_senscr_ptr),
                                                    C.c_void_p(d_pen_ptr) if d_pen_ptr else None, int(pl_window), _p(utt_off), n_utt,
                                                    int(first_cap or bp_cap), int(first_bss_cap or bss_cap), _p(bp), int(bp_cap), _p(bss),
                                                    int(bss_cap), _p(bp_idx), _p(res), _p(res1)), "psb_ngram_two_pass_batch_device")
        out = []
        for u in range(n_utt):
            T = int(utt_off[u + 1] - utt_off[u])
            o = int(utt_off[u]) + u
            out.append((bp[u, :res[u, 0]].copy(), bss[u, :res[u, 1]].copy(), bp_idx[o:o + T + 1].copy()))
        return out, res1[:n_utt, 0].copy()

    def allphone_lm(self, d_senscr_ptr, utt_off, ssid, tmatid, succ_off, succ, start, beam, pbeam, node_ci, bg, tg):
        """allphone_search with a phone LM (dense bigram / trigram tables).  History rows
        [n][5] = (ef, node, predecessor entry, score, tscore)."""
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        a = [np.ascontiguousarray(x, np.int32) for x in (ssid, tmatid, succ_off, succ, node_ci, bg, tg)]
        n_utt = len(utt_off) - 1
        n_ci = a[5].shape[0]
        assert a[5].shape == (n_ci, n_ci) and a[6].shape == (n_ci, n_ci, n_ci)
        cap = max(1, int(np.diff(utt_off).max(initial=1)) * len(a[0]))
        hist = np.zeros((max(1, n_utt), cap, 5), np.int32)
        n_hist = np.zeros(max(1, n_utt), np.int32)
        check(lib().psb_allphone_lm_batch_device(self.h, C.c_void_p(d_senscr_ptr), _p(utt_off), n_utt, len(a[0]), _p(a[0]),
                                                 _p(a[1]), _p(a[2]), _p(a[3]), int(start), int(beam), int(pbeam), n_ci,
                                                 _p(a[4]), _p(a[5]), _p(a[6]), _p(hist), cap, _p(n_hist)),
              "psb_allphone_lm_batch_device")
        return [hist[u, :min(int(n_hist[u]), cap)].copy() for u in range(n_utt)], n_hist[:n_utt].copy()

    def allphone_net(self, d_senscr_ptr, utt_off, net, beam, pbeam, inspen=0, bg=None, tg=None, cap=None,
                     want_hist=False, hist_budget=4 << 30):
        """allphone_search over a batch on a factored PHMM net (allphone_net.build_net: ssid, tmatid, ci,
        lc, rc, n_ci, start), with a phone LM when bg / tg are given.  The history table stays on the
        device; its backtrace runs there.  cap: history rows per utterance (default: frames x nodes,
        which cannot overflow).  Utterances go to the device in sub-batches whose history tables fit
        hist_budget bytes.  Returns a dict: status [n_utt] (0 ok, 1 history overflow), n_hist [n_utt],
        segs (list of [n][5] = (ci, sf, ef, score, tscore)), hist (list of [n][4] rows, if want_hist)."""
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        n_utt = len(utt_off) - 1
        H = len(net["ci"])
        a = [np.ascontiguousarray(net[k], np.int32) for k in ("ssid", "tmatid", "ci")]
        lc, rc = (np.ascontiguousarray(net[k], np.uint64) for k in ("lc", "rc"))
        if (bg is None) != (tg is None):
            raise ValueError("give both phone-LM tables or neither")
        bg = None if bg is None else np.ascontiguousarray(bg, np.int32)
        tg = None if tg is None else np.ascontiguousarray(tg, np.int32)
        lens = np.diff(utt_off)
        cap = int(cap or max(1, int(lens.max(initial=1)) * H))
        per = max(1, int(hist_budget) // (cap * 16))
        out = dict(status=np.zeros(n_utt, np.int32), n_hist=np.zeros(n_utt, np.int32), segs=[], hist=[] if want_hist else None)
        for u0 in range(0, max(n_utt, 1), per):
            u1 = min(n_utt, u0 + per)
            m = u1 - u0
            sub = utt_off[u0:u1 + 1] - utt_off[u0]
            seg_cap = max(1, int(np.diff(sub).max(initial=1)))          # a segment spans at least one frame
            res = np.zeros((max(m, 1), 3), np.int32)
            segs = np.zeros((max(m, 1), seg_cap, 5), np.int32)
            hist = np.zeros((max(m, 1), cap, 4), np.int32) if want_hist else None
            ptr = d_senscr_ptr + int(utt_off[u0]) * self.n_sen * 2 if m else d_senscr_ptr
            check(lib().psb_allphone_net_batch_device(self.h, C.c_void_p(ptr), _p(sub), m, H, _p(a[0]), _p(a[1]), _p(a[2]),
                                                      _p(lc), _p(rc), int(net["n_ci"]), int(net["start"]), int(beam), int(pbeam),
                                                      int(inspen), _p(bg) if bg is not None else None,
                                                      _p(tg) if tg is not None else None, cap, _p(res), _p(segs), seg_cap,
                                                      _p(hist) if want_hist else None), "psb_allphone_net_batch_device")
            for j in range(m):
                out["status"][u0 + j], out["n_hist"][u0 + j] = res[j, 0], res[j, 1]
                out["segs"].append(segs[j, :res[j, 2]].copy())
                if want_hist:
                    out["hist"].append(hist[j, :min(int(res[j, 1]), cap)].copy())
        return out

    def kws(self, d_senscr_ptr, utt_off, pl_ssid, pl_tmat, kp_off, kp_thresh, kp_ssid, kp_tmat, beam, plp, cap=None):
        """kws_search over a batch (scores on the device).  Returns a list of raw hit arrays
        [n][5] = (frame, keyphrase, start frame, prob, ascr), one per utterance, and the hit counts.
        cap: hit rows per utterance, rows past it dropped (counted all the same).  By default the rows
        start at two per frame (a frame has at most one per keyphrase, which for long lists would reserve
        far more than is ever written) and a batch that overflows them is searched again with as many as
        its fullest utterance needs."""
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        a = [np.ascontiguousarray(x, np.int32) for x in (pl_ssid, pl_tmat, kp_off, kp_thresh, kp_ssid, kp_tmat)]
        n_utt, n_kp = len(utt_off) - 1, len(a[2]) - 1
        grow = cap is None
        if grow:
            cap = max(1, int(np.diff(utt_off).max(initial=1)) * min(2, max(1, n_kp)))
        while True:
            hits = np.zeros((max(1, n_utt), cap, 5), np.int32)
            n_hits = np.zeros(max(1, n_utt), np.int32)
            check(lib().psb_kws_batch_device(self.h, C.c_void_p(d_senscr_ptr), _p(utt_off), n_utt, len(a[0]), _p(a[0]),
                                             _p(a[1]), n_kp, _p(a[2]), _p(a[3]), _p(a[4]), _p(a[5]), int(beam), int(plp),
                                             _p(hits), cap, _p(n_hits)), "psb_kws_batch_device")
            need = int(n_hits[:n_utt].max(initial=0))
            if not grow or need <= cap:
                break
            cap = need
        return [hits[u, :min(int(n_hits[u]), cap)].copy() for u in range(n_utt)], n_hits[:n_utt].copy()

    def align(self, senscr, utt_off, ph_off, ssid, tmatid, sf=None, ef=None, device_ptr=None):
        """state_align_search over a batch.  senscr: host int16 [frames][n_sen] (or device_ptr);
        returns (status [n_utt], start, dur, score per emitting state)."""
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        ph_off = np.ascontiguousarray(ph_off, np.int32)
        ssid = np.ascontiguousarray(ssid, np.int32)
        tmatid = np.ascontiguousarray(tmatid, np.int32)
        sf = None if sf is None else np.ascontiguousarray(sf, np.int32)
        ef = None if ef is None else np.ascontiguousarray(ef, np.int32)
        n_utt = len(utt_off) - 1
        n_st = max(1, int(ph_off[-1]) * self.n_emit)
        out = np.zeros((3, n_st), np.int32)
        status = np.zeros(max(1, n_utt), np.int32)
        if device_ptr is not None:
            check(lib().psb_align_batch_device(self.h, C.c_void_p(device_ptr), _p(utt_off), n_utt, _p(ph_off), _p(ssid),
                                               _p(tmatid), _p(sf), _p(ef), _p(out[0]), _p(out[1]), _p(out[2]), _p(status)),
                  "psb_align_batch_device")
        else:
            senscr = np.ascontiguousarray(senscr, np.int16)
            check(lib().psb_align_batch_host(self.h, _p(senscr), _p(utt_off), n_utt, _p(ph_off), _p(ssid), _p(tmatid),
                                             _p(sf), _p(ef), _p(out[0]), _p(out[1]), _p(out[2]), _p(status)),
                  "psb_align_batch_host")
        k = int(ph_off[-1]) * self.n_emit
        return status[:n_utt], out[0, :k], out[1, :k], out[2, :k]

    def close(self):
        if self.h:
            lib().psb_hmmctx_free(self.h)
            self.h = None


class HmmSet:
    """Device-resident HMM instances in segments (one per utterance): the batched
    evaluate_channels / fsg_search_hmm_eval / phmm_eval_all loop with state kept in HBM."""

    def __init__(self, ctx: HmmContext, n_max, n_seg_max):
        self.ctx = ctx
        h = C.c_void_p()
        check(lib().psb_hmmset_create(ctx.h, int(n_max), int(n_seg_max), C.byref(h)), "psb_hmmset_create")
        self.h = h
        self.n = 0
        self.n_seg = 0

    def upload(self, hmms, seg_off):
        assert hmms.dtype == HMM_DTYPE and hmms.flags.c_contiguous
        seg_off = np.ascontiguousarray(seg_off, np.int64)
        check(lib().psb_hmmset_upload(self.h, _p(hmms) if len(hmms) else None, len(hmms), _p(seg_off),
                                      len(seg_off) - 1), "psb_hmmset_upload")
        self.n, self.n_seg = len(hmms), len(seg_off) - 1

    def download(self, hmms=None):
        if hmms is None:
            hmms = np.zeros(self.n, HMM_DTYPE)
        assert hmms.dtype == HMM_DTYPE and hmms.flags.c_contiguous and len(hmms) == self.n
        check(lib().psb_hmmset_download(self.h, _p(hmms) if self.n else None), "psb_hmmset_download")
        return hmms

    def eval_host(self, senscr):
        """One frame; senscr int16 [n_seg][n_sen]; returns best int32 [n_seg]."""
        senscr = np.ascontiguousarray(senscr, np.int16)
        assert senscr.shape == (self.n_seg, self.ctx.n_sen)
        best = np.zeros(self.n_seg, np.int32)
        check(lib().psb_hmmset_eval_host(self.h, _p(senscr), _p(best)), "psb_hmmset_eval_host")
        return best

    def eval_frames_device(self, d_senscr, n_frames, d_best, d_row0=None, d_n_rows=None):
        """Device pointers (ints); returns the device time of the n_frames launches in ms."""
        ms = C.c_float()
        check(lib().psb_hmmset_eval_frames_device(self.h, C.c_void_p(d_senscr), C.c_void_p(d_row0) if d_row0 else None,
                                                  C.c_void_p(d_n_rows) if d_n_rows else None, int(n_frames),
                                                  C.c_void_p(d_best), C.byref(ms)), "psb_hmmset_eval_frames_device")
        return ms.value

    def sweep_device(self, d_senscr, rows_total, n_frames, d_best, d_row0=None, d_n_rows=None, timed=True):
        """The same steps fused in one launch (state in registers, score rows by TMA): device pointers
        (ints), rows_total = rows of the score matrix; returns the device time in ms (timed=False:
        asynchronous on the set's stream, returns None)."""
        ms = C.c_float()
        check(lib().psb_hmmset_sweep_device(self.h, C.c_void_p(d_senscr), int(rows_total), C.c_void_p(d_row0) if d_row0 else None,
                                            C.c_void_p(d_n_rows) if d_n_rows else None, int(n_frames),
                                            C.c_void_p(d_best), C.byref(ms) if timed else None), "psb_hmmset_sweep_device")
        return ms.value if timed else None

    def sweep_beam_device(self, d_senscr, rows_total, n_frames, frame0, beam, d_best, maxhmmpf=-1, d_n_active=None,
                          d_row0=None, d_n_rows=None, timed=True):
        """The fused sweep with beam pruning between frames (evaluate_channels + the beam part of prune_channels,
        ngram_search_fwdtree.c:702-715, :1130-1181, without transitions): instances whose frame field equals
        frame0 + t are evaluated in frame t, survivors of best + dynamic beam move on, the others are hmm_clear'ed.
        Device pointers (ints); d_n_active [n_frames][n_seg] int32 receives the evaluated counts."""
        ms = C.c_float()
        check(lib().psb_hmmset_sweep_beam_device(self.h, C.c_void_p(d_senscr), int(rows_total), C.c_void_p(d_row0) if d_row0 else None,
                                                 C.c_void_p(d_n_rows) if d_n_rows else None, int(n_frames), int(frame0), int(beam),
                                                 int(maxhmmpf), C.c_void_p(d_best), C.c_void_p(d_n_active) if d_n_active else None,
                                                 C.byref(ms) if timed else None), "psb_hmmset_sweep_beam_device")
        return ms.value if timed else None

    def use_batch_stream(self, batch):
        check(lib().psb_hmmset_use_batch_stream(self.h, batch.h if batch is not None else None), "psb_hmmset_use_batch_stream")

    def snapshot(self):
        check(lib().psb_hmmset_snapshot(self.h), "psb_hmmset_snapshot")

    def restore(self):
        check(lib().psb_hmmset_restore(self.h), "psb_hmmset_restore")

    def close(self):
        if self.h:
            lib().psb_hmmset_free(self.h)
            self.h = None


class PhoneLoop:
    """phone_loop_search.c on the device over batches of utterances."""

    def __init__(self, ctx: HmmContext, ssid, tmatid, window, beam, pbeam, pip, penalty_weight):
        self.ctx = ctx
        ssid = np.ascontiguousarray(ssid, np.int32)
        tmatid = np.ascontiguousarray(tmatid, np.int32)
        self.n_phones = len(ssid)
        h = C.c_void_p()
        check(lib().psb_phoneloop_create(ctx.h, self.n_phones, _p(ssid), _p(tmatid), window, beam, pbeam, pip,
                                         float(penalty_weight), C.byref(h)), "psb_phoneloop_create")
        self.h = h

    def run_host(self, senscr, utt_off, trace=False):
        senscr = np.ascontiguousarray(senscr, np.int16)
        utt_off = np.ascontiguousarray(utt_off, np.int32)
        total = int(utt_off[-1])
        best = np.zeros(total, np.int32)
        pen = np.zeros((total, self.n_phones), np.int32)
        tr = np.zeros((total, self.n_phones), HMM_DTYPE) if trace else None
        check(lib().psb_phoneloop_run_host(self.h, _p(senscr), _p(utt_off), len(utt_off) - 1, _p(best), _p(pen),
                                           _p(tr)), "psb_phoneloop_run_host")
        return dict(best=best, pen=pen, hmm=tr)

    def close(self):
        if self.h:
            lib().psb_phoneloop_free(self.h)
            self.h = None


def sendump_write(path, senscr, mdef_file="(none)", logbase=1.0001):
    """Write [T][n_sen] int16 scores as a reference senone dump (.sen)."""
    senscr = np.ascontiguousarray(senscr, np.int16)
    check(lib().psb_sendump_write(path.encode(), mdef_file.encode(), senscr.shape[1], float(logbase), _p(senscr),
                                  senscr.shape[0]), "psb_sendump_write")


def sendump_read(path, max_frames=1 << 20):
    n_sen = C.c_int32()
    n = lib().psb_sendump_read(path.encode(), C.byref(n_sen), None, 0)
    if n < 0:
        raise PsbError("psb_sendump_read failed: " + lib().psb_last_error().decode())
    size = (__import__("os").path.getsize(path) // (2 * n_sen.value)) + 1
    out = np.zeros((min(size, max_frames), n_sen.value), np.int16)
    n = lib().psb_sendump_read(path.encode(), C.byref(n_sen), _p(out), out.shape[0])
    if n < 0:
        raise PsbError("psb_sendump_read failed: " + lib().psb_last_error().decode())
    return out[:n]



def fsg_hyp(hist, links, n_frame, final_state, final=True, cap=4096):
    """ps_get_hyp / ps_seg_iter of a grammar search without -bestpath, on the table `HmmContext.fsg`
    returned (fsg_search_find_exit + fsg_search_seg_iter, fsg_search.c:883-954, 1122-1180).  Returns
    (entry, score, seg [n][7] = entry, link, wid, sf, ef, ascr, lscr); entry <= 0: no hypothesis."""
    hist = np.ascontiguousarray(hist, np.int32).reshape(-1, 13)
    links = np.ascontiguousarray(links, np.int32).reshape(-1, 5)
    entry, score = C.c_int32(-1), C.c_int32(0)
    check(lib().psb_fsg_find_exit(_p(hist), len(hist), _p(links), len(links), int(n_frame), int(final_state), int(bool(final)),
                                  C.byref(entry), C.byref(score)), "psb_fsg_find_exit")
    if entry.value <= 0:
        return entry.value, None, np.zeros((0, 7), np.int32)
    seg = np.zeros((cap, 7), np.int32)
    n = lib().psb_fsg_backtrace(_p(hist), len(hist), _p(links), len(links), entry.value, _p(seg), cap)
    check(min(n, 0), "psb_fsg_backtrace")
    return entry.value, score.value, seg[:min(n, cap)].copy()


def ngram_hyp(bp, bp_idx, n_frame, finish_wid, cap=4096):
    """ngram_search_find_exit + ngram_search_bp_iter (ngram_search.c:498-541, 958-997) on a backpointer
    table the n-gram entry points returned.  Returns (entry, score, seg [n][5] = entry, wid, sf, ef,
    path score); entry -1: no frame had a word exit."""
    bp = np.ascontiguousarray(bp, np.int32).reshape(-1, 10)
    bp_idx = np.ascontiguousarray(bp_idx, np.int32)
    entry, score = C.c_int32(-1), C.c_int32(0)
    check(lib().psb_ngram_find_exit(_p(bp), len(bp), _p(bp_idx), int(n_frame), int(finish_wid), C.byref(entry), C.byref(score)),
          "psb_ngram_find_exit")
    if entry.value < 0:
        return -1, None, np.zeros((0, 5), np.int32)
    seg = np.zeros((cap, 5), np.int32)
    n = lib().psb_ngram_backtrace(_p(bp), len(bp), entry.value, _p(seg), cap)
    check(min(n, 0), "psb_ngram_backtrace")
    return entry.value, score.value, seg[:min(n, cap)].copy()



def ngram_segments(info, model, bp, bss, entry, lm_arrays=None, second_pass=False, cap=4096):
    """ps_seg_iter of an n-gram search without -bestpath (ngram_search_bp2itor, ngram_search.c:886-928):
    seg [n][7] = entry, wid, sf, ef, path score, ascr, lscr.  second_pass: the tables come from fwdflat,
    LM scores are scaled by the float32 fwdflat_fwdtree_lw_ratio (its bits are info[32])."""
    from ._lib import NgramDesc
    info = np.ascontiguousarray(info, np.int32); model = np.ascontiguousarray(model, np.int32)
    bp = np.ascontiguousarray(bp, np.int32).reshape(-1, 10); bss = np.ascontiguousarray(bss, np.int32)
    lma = None if lm_arrays is None else np.ascontiguousarray(lm_arrays, np.int32)
    d = NgramDesc(info.ctypes.data, model.ctypes.data, len(model), None, None,
                  None if lma is None else lma.ctypes.data, 0 if lma is None else len(lma))
    lwf = np.float32(1.0)
    if second_pass:
        lwf = info[32:33].view(np.float32)[0]
    seg = np.zeros((cap, 7), np.int32)
    n = lib().psb_ngram_segments(C.byref(d), _p(bp), len(bp), _p(bss), len(bss), int(entry), C.c_float(float(lwf)), _p(seg), cap)
    check(min(n, 0), "psb_ngram_segments")
    return seg[:min(n, cap)].copy()


class FrontEnd:
    """fe/ + feat/ for whole batches on the device.  `desc` is the dict of fe_tables.make_fe_desc() -- or the
    same arrays taken out of the reference's fe_t.  `opts` (fe_tables.make_fe_opts(), optional) selects the
    feature type, CMN (including live, and -varnorm), -cmninit, AGC, an LDA transform and dither; without it every
    utterance is a fresh stream with desc's 1s_c_d_dd features and CMN.  feat_dim is the LDA output dimension when
    there is a transform.  The cepstra process_host returns (want_mfcc) are the ones after CMN and AGC."""

    def __init__(self, desc, device=0, opts=None):
        from ._lib import FeDesc, FeOpts
        self.desc = desc
        self._keep = {}
        d = FeDesc()
        for k in ("frame_size", "frame_shift", "fft_size", "fft_order", "n_filt", "n_cep", "remove_dc", "remove_noise",
                  "transform", "lifter_val", "window", "cmn"):
            setattr(d, k, int(desc[k]))
        d.pre_emphasis_alpha = float(desc["alpha"])
        d.sqrt_inv_n = float(desc["sqrt_inv_n"])
        d.sqrt_inv_2n = float(desc["sqrt_inv_2n"])
        for k, dt in (("hamming", np.float64), ("ccc", np.float64), ("sss", np.float64), ("spec_start", np.int16),
                      ("filt_start", np.int16), ("filt_width", np.int16), ("filt_coeffs", np.float32),
                      ("mel_cosine", np.float32), ("lifter", np.float32)):
            a = np.ascontiguousarray(desc[k], dt)
            self._keep[k] = a
            setattr(d, k, a.ctypes.data if a.size else None)
        d.n_coeffs = int(self._keep["filt_coeffs"].size)
        self.n_cep = int(desc["n_cep"])
        h = C.c_void_p()
        if opts is None:
            check(lib().psb_fe_create(C.byref(d), device, C.byref(h)), "psb_fe_create")
        else:
            o = FeOpts()
            for k in ("feat", "cmn", "varnorm", "dither", "seed"):
                setattr(o, k, int(opts[k]))
            ci = np.zeros(32, np.float32)
            v = np.asarray(opts["cmn_init"], np.float32).ravel()[:32]
            ci[:v.size] = v
            o.cmn_init[:] = ci.tolist()
            o.agc, o.agc_thresh = int(opts.get("agc", 0)), float(opts.get("agc_thresh", 2.0))
            if opts.get("lda") is not None:
                a = np.ascontiguousarray(opts["lda"], np.float32)
                assert a.ndim == 2
                self._keep["lda"] = a
                o.lda, (o.lda_rows, o.lda_cols), o.ldadim = a.ctypes.data, a.shape, int(opts.get("ldadim", 0))
            check(lib().psb_fe_create_ex(C.byref(d), C.byref(o), device, C.byref(h)), "psb_fe_create_ex")
        self.h = h
        self.feat_dim = lib().psb_fe_feat_dim(h)

    def initial_state(self):
        """The session state of a fresh decoder: -cmninit's mean and the dither generator seeded with -seed."""
        from ._lib import FeState
        s = FeState()
        check(lib().psb_fe_state_init(self.h, C.byref(s)), "psb_fe_state_init")
        return s

    def set_sessions(self, sess_off, states=None):
        """Names the sessions of the next process_* / Batch.decode_pcm_host call: session s is utterances
        sess_off[s] .. sess_off[s + 1] - 1, starting from states[s] (FeState objects; None: fresh)."""
        from ._lib import FeState
        sess_off = np.ascontiguousarray(sess_off, np.int32)
        n = len(sess_off) - 1
        arr = None
        if states is not None:
            assert len(states) == n
            arr = (FeState * max(n, 1))(*states)
        check(lib().psb_fe_set_sessions(self.h, _p(sess_off), n, arr), "psb_fe_set_sessions")

    def get_states(self, n_sess):
        """The sessions' states after the last call, as a list of FeState."""
        from ._lib import FeState
        arr = (FeState * max(n_sess, 1))()
        check(lib().psb_fe_get_states(self.h, arr, n_sess), "psb_fe_get_states")
        return [arr[i] for i in range(n_sess)]

    def set_stream_starts(self, starts, noise=None):
        """Names the stream starts of the next process_* / Batch.decode_pcm_host call: starts[u] true runs
        ps_start_stream before utterance u, false carries the noise tracker on from the utterance before it in its
        session, or for a session's first utterance from noise[s] (FeNoise objects, one per session of that call;
        None: a fresh tracker for every session).  Without this call every utterance starts a stream."""
        from ._lib import FeNoise
        starts = np.ascontiguousarray(np.asarray(starts, bool), np.uint8)
        arr, n = None, 0
        if noise is not None:
            n = len(noise)
            arr = (FeNoise * max(n, 1))(*noise)
        check(lib().psb_fe_set_stream_starts(self.h, _p(starts) if starts.size else None, len(starts), arr, n),
              "psb_fe_set_stream_starts")

    def get_noise_states(self, n_sess):
        """The sessions' noise trackers after the last call, which must have set stream starts, as a list of FeNoise."""
        from ._lib import FeNoise
        arr = (FeNoise * max(n_sess, 1))()
        check(lib().psb_fe_get_noise_states(self.h, arr, n_sess), "psb_fe_get_noise_states")
        return [arr[i] for i in range(n_sess)]

    def filterbanks(self, banks, bank_of_utt):
        """The arrays psb_fe_set_filterbanks takes, built and checked on the host (ValueError) without naming
        anything for the next call: utterance u reads banks[bank_of_utt[u]].  Each bank is a dict with make_fe_desc's
        spec_start / filt_start / filt_width / filt_coeffs, or a (warp_type, warp_params) pair built with this front
        end's own settings (fe_tables.make_filterbank over desc["bank_args"])."""
        from .fe_tables import make_filterbank
        nf = int(self.desc["n_filt"])
        ss, fs, fw, co, coeff_off = [], [], [], [], [0]
        for b in banks:
            if not isinstance(b, dict):
                if "bank_args" not in self.desc:
                    raise ValueError("(warp_type, warp_params) banks need a desc from make_fe_desc (its bank_args)")
                b = make_filterbank(warp_type=b[0], warp_params=b[1], **self.desc["bank_args"])
            for lst, k, dt in ((ss, "spec_start", np.int16), (fs, "filt_start", np.int16), (fw, "filt_width", np.int16)):
                a = np.ascontiguousarray(b[k], dt).ravel()
                if a.size != nf:
                    raise ValueError("a filter bank has %d filters, this front end %d" % (a.size, nf))
                lst.append(a)
            co.append(np.ascontiguousarray(b["filt_coeffs"], np.float32).ravel())
            coeff_off.append(coeff_off[-1] + co[-1].size)
        cat = lambda parts, dt: np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros(0, dt), dt)
        return (len(banks), cat(ss, np.int16), cat(fs, np.int16), cat(fw, np.int16), np.asarray(coeff_off, np.int32),
                cat(co, np.float32), np.ascontiguousarray(bank_of_utt, np.int32))

    def warp_filterbanks(self, warps, sess_off=None):
        """filterbanks() for one warp per utterance, or with sess_off one per session: a -warp_params string (under
        desc's warp_type), a (warp_type, warp_params) pair, a filter-bank dict, or None for desc's own bank."""
        if sess_off is not None:
            if len(warps) != len(sess_off) - 1:
                raise ValueError("%d warps for %d sessions" % (len(warps), len(sess_off) - 1))
            warps = [w for s, w in enumerate(warps) for _ in range(int(sess_off[s + 1]) - int(sess_off[s]))]
        banks, index, bank_of_utt = [], {}, []
        for w in warps:
            if isinstance(w, str):
                w = (self.desc.get("warp_type", "inverse_linear"), w)
            k = id(w) if isinstance(w, dict) else w
            if k not in index:
                index[k] = len(banks)
                banks.append(self.desc if w is None else w)
            bank_of_utt.append(index[k])
        return self.filterbanks(banks or [self.desc], bank_of_utt)

    def name_filterbanks(self, arrays):
        """Names the banks filterbanks() / warp_filterbanks() built for the next process_* / Batch.decode_pcm_host
        call (psb_fe_set_filterbanks).  Without it every utterance reads desc's bank."""
        n, ss, fs, fw, coeff_off, co, bank_of_utt = arrays
        check(lib().psb_fe_set_filterbanks(self.h, n, _p(ss) if ss.size else None, _p(fs) if fs.size else None,
                                           _p(fw) if fw.size else None, _p(coeff_off), _p(co) if co.size else None,
                                           _p(bank_of_utt) if bank_of_utt.size else None, len(bank_of_utt)),
              "psb_fe_set_filterbanks")

    def set_filterbanks(self, banks, bank_of_utt):
        """Per-utterance mel filter banks (VTLN) for the next call: name_filterbanks(filterbanks(...))."""
        self.name_filterbanks(self.filterbanks(banks, bank_of_utt))

    def set_warps(self, warps, sess_off=None):
        """Per-utterance (or with sess_off per-session) warps for the next call: name_filterbanks(warp_filterbanks(...))."""
        self.name_filterbanks(self.warp_filterbanks(warps, sess_off))

    def cancel_settings(self):
        """Drops what set_sessions, set_stream_starts and set_filterbanks named for the next call
        (psb_fe_cancel_settings): the next call runs with none of them."""
        check(lib().psb_fe_cancel_settings(self.h), "psb_fe_cancel_settings")

    def process_sessions(self, pcm, samp_off, sess_off, states=None, want_mfcc=False, starts=None, noise=None, warp=None):
        """process_host over named sessions; returns (feats, frame_off, outgoing states[, mfcc]).  With starts (one
        flag per utterance, set_stream_starts) the outgoing noise trackers follow as one more item at the end.  warp:
        one -warp_params string, (warp_type, warp_params) pair or filter-bank dict per session (None: desc's bank).
        A refused setting leaves nothing named for the next call."""
        banks = None if warp is None else self.warp_filterbanks(warp, sess_off=sess_off)
        try:
            self.set_sessions(sess_off, states)
            if starts is not None:
                self.set_stream_starts(starts, noise)
            if banks is not None:
                self.name_filterbanks(banks)
        except BaseException:
            self.cancel_settings()
            raise
        r = self.process_host(pcm, samp_off, want_mfcc)
        r = r[:2] + (self.get_states(len(sess_off) - 1),) + r[2:]
        return r + (self.get_noise_states(len(sess_off) - 1),) if starts is not None else r

    def n_frames(self, n_samples):
        return lib().psb_fe_n_frames(self.h, int(n_samples))

    @staticmethod
    def sample_offsets(lens):
        off = np.zeros(len(lens) + 1, np.int64)
        np.cumsum(lens, out=off[1:])
        return off

    def process_host(self, pcm, samp_off, want_mfcc=False):
        """pcm int16 (utterances back to back), samp_off int64 [n_utt+1] -> (feats [T][feat_dim],
        frame_off int32 [n_utt+1][, mfcc after CMN and AGC [T][n_cep]])."""
        pcm = np.ascontiguousarray(pcm, np.int16)
        samp_off = np.ascontiguousarray(samp_off, np.int64)
        n_utt = len(samp_off) - 1
        total = sum(self.n_frames(int(samp_off[u + 1] - samp_off[u])) for u in range(n_utt))
        feats = np.zeros((total, self.feat_dim), np.float32)
        mfcc = np.zeros((total, self.n_cep), np.float32) if want_mfcc else None
        frame_off = np.zeros(n_utt + 1, np.int32)
        check(lib().psb_fe_process_host(self.h, _p(pcm) if pcm.size else None, _p(samp_off), n_utt, _p(feats) if total else None,
                                        _p(mfcc) if (want_mfcc and total) else None, _p(frame_off)), "psb_fe_process_host")
        return (feats, frame_off, mfcc) if want_mfcc else (feats, frame_off)

    def process_device(self, d_pcm_ptr, samp_off, d_feats_ptr):
        """Device buffers; returns (frame_off int32 [n_utt+1], device ms of the two kernels)."""
        samp_off = np.ascontiguousarray(samp_off, np.int64)
        n_utt = len(samp_off) - 1
        frame_off = np.zeros(n_utt + 1, np.int32)
        ms = C.c_float()
        check(lib().psb_fe_process_device(self.h, C.c_void_p(d_pcm_ptr), _p(samp_off), n_utt, C.c_void_p(d_feats_ptr),
                                          None, _p(frame_off), C.byref(ms)), "psb_fe_process_device")
        return frame_off, ms.value

    def close(self):
        if self.h:
            lib().psb_fe_free(self.h)
            self.h = None


class Endpointer:
    """ps_endpointer_t for whole batches of int16 streams on the device (arguments as the reference's Python
    Endpointer: window, ratio, vad_mode, sample_rate, frame_length; 0 / None = the reference's default).  Every
    stream is one whole recording: ps_endpointer_process on each full frame, then ps_endpointer_end_stream with the
    rest -- also when the rest is empty, which the reference's Python Segmenter skips.  warmup: None (default), 0 (no
    warm-up: every chunk boundary of the parallel filter bank is repaired) or a frame count; results never depend on
    it.  Rates that map to 48 kHz (44.1 / 48 kHz input) are refused."""

    def __init__(self, window=0.3, ratio=0.9, vad_mode=0, sample_rate=16000, frame_length=0.03, device=0, warmup=None):
        from ._lib import VadOpts
        o = VadOpts()
        o.mode, o.sample_rate, o.frame_length = int(vad_mode), int(sample_rate or 0), float(frame_length or 0.0)
        o.window, o.ratio = float(window or 0.0), float(ratio or 0.0)
        o.warmup = 0 if warmup is None else (-1 if int(warmup) == 0 else int(warmup))
        h = C.c_void_p()
        check(lib().psb_vad_create(C.byref(o), device, C.byref(h)), "psb_vad_create")
        self.h = h
        L = lib()
        self.frame_size, self.frame_length, self.sample_rate = L.psb_vad_frame_size(h), L.psb_vad_frame_length(h), L.psb_vad_sample_rate(h)
        self.start_frames, self.end_frames, self.maxlen = L.psb_vad_start_frames(h), L.psb_vad_end_frames(h), L.psb_vad_maxlen(h)
        self.warmup = L.psb_vad_warmup(h)

    def process(self, streams):
        """(flags int8 [frames], frame_off int32 [n + 1], seg_n int32 [n], segs int64 [frames][2], times float64 [frames][2])."""
        streams = [np.ascontiguousarray(s, np.int16) for s in streams]
        n = len(streams)
        samp_off = np.zeros(n + 1, np.int64)
        samp_off[1:] = np.cumsum([len(s) for s in streams])
        pcm = np.concatenate(streams) if n else np.zeros(0, np.int16)
        total = int(sum(len(s) // self.frame_size for s in streams))
        flags = np.zeros(max(total, 1), np.int8)
        frame_off = np.zeros(n + 1, np.int32)
        seg_n = np.zeros(max(n, 1), np.int32)
        segs = np.zeros((max(total, 1), 2), np.int64)
        times = np.zeros((max(total, 1), 2), np.float64)
        check(lib().psb_vad_process_host(self.h, _p(pcm) if pcm.size else None, _p(samp_off), n, _p(flags), _p(frame_off),
                                         _p(seg_n), _p(segs), _p(times)), "psb_vad_process_host")
        return flags[:total], frame_off, seg_n[:n], segs, times

    def classify_batch(self, streams):
        """Per stream, int8 [full frames]: ps_vad_classify of each frame on a fresh VAD."""
        flags, frame_off = self.process(streams)[:2]
        return [flags[frame_off[i]:frame_off[i + 1]] for i in range(len(frame_off) - 1)]

    def segment_batch(self, streams):
        """Per stream, [(start_time, end_time, start_sample, end_sample)] with the reference's float64 times."""
        _, frame_off, seg_n, segs, times = self.process(streams)
        out = []
        for i in range(len(frame_off) - 1):
            r = range(int(frame_off[i]), int(frame_off[i]) + int(seg_n[i]))
            out.append([(float(times[j, 0]), float(times[j, 1]), int(segs[j, 0]), int(segs[j, 1])) for j in r])
        return out

    @property
    def last_repairs(self):
        """Chunk recomputations of the last call: chunks whose start state differed from their predecessor's end."""
        return int(lib().psb_vad_last_repairs(self.h))

    @property
    def last_passes(self):
        """Repair passes of the last call; the last pass recomputes nothing."""
        return int(lib().psb_vad_last_passes(self.h))

    def close(self):
        if self.h:
            lib().psb_vad_free(self.h)
            self.h = None


LIVE_STATUS = np.dtype([("in_speech", np.int32), ("reserved", np.int32), ("start_sample", np.int64), ("frames", np.int64),
                        ("speech_start", np.float64), ("speech_end", np.float64)])     # psb_vad_live_status_t


class LiveEndpointer(Endpointer):
    """ps_endpointer_t for n_slots live streams on the device: feed() hands each listed slot its next samples, in any
    lengths; the results are bit for bit the reference's when the same samples reach ps_endpointer_process one frame
    at a time across the same calls.  Options as Endpointer's; the whole-stream calls of Endpointer on this handle
    leave the slots alone."""

    def __init__(self, n_slots, window=0.3, ratio=0.9, vad_mode=0, sample_rate=16000, frame_length=0.03, device=0,
                 warmup=None):
        super().__init__(window, ratio, vad_mode, sample_rate, frame_length, device, warmup)
        try:
            check(lib().psb_vad_live_open(self.h, int(n_slots)), "psb_vad_live_open")
        except PsbError:
            self.close()
            raise
        self.n_slots = int(n_slots)

    def feed(self, chunks, slots=None, final=None):
        """chunks: int16 arrays, one per slot in `slots` (default: slots 0 .. len(chunks) - 1).  final: per slot, true
        to end the stream after these samples (ps_endpointer_end_stream; the samples after the last full frame are
        dropped, and a slot fed afterwards goes on like the reference's endpointer does).  Returns one dict per fed slot:
        flags (int8 per new frame), segments ended in this call [(start_time, end_time, start_sample, end_sample)],
        in_speech, speech_start, speech_end, start_sample (of the open segment, -1 when not in speech), frames (fed
        since the slot was made fresh)."""
        chunks = [np.ascontiguousarray(c, np.int16) for c in chunks]
        n = len(chunks)
        slots = np.arange(n, dtype=np.int32) if slots is None else np.ascontiguousarray(slots, np.int32)
        if len(slots) != n:
            raise ValueError("feed: %d chunks for %d slots" % (n, len(slots)))
        fin = None if final is None else np.ascontiguousarray([bool(f) for f in final], np.int8)
        if fin is not None and len(fin) != n:
            raise ValueError("feed: %d final flags for %d slots" % (len(fin), n))
        samp_off = np.zeros(n + 1, np.int64)
        samp_off[1:] = np.cumsum([len(c) for c in chunks])
        pcm = np.concatenate(chunks) if n else np.zeros(0, np.int16)
        cap = int(sum((len(c) + self.frame_size - 1) // self.frame_size for c in chunks))
        flags = np.zeros(max(cap, 1), np.int8)
        frame_off = np.zeros(n + 1, np.int32)
        seg_n = np.zeros(max(n, 1), np.int32)
        segs = np.zeros((cap + n + 1, 2), np.int64)
        times = np.zeros((cap + n + 1, 2), np.float64)
        status = np.zeros(max(n, 1), LIVE_STATUS)
        check(lib().psb_vad_feed_host(self.h, _p(slots) if n else None, n, _p(pcm) if pcm.size else None, _p(samp_off),
                                      _p(fin) if fin is not None else None, _p(flags), _p(frame_off), _p(seg_n), _p(segs),
                                      _p(times), _p(status)), "psb_vad_feed_host")
        out = []
        for i in range(n):
            r0 = int(frame_off[i]) + i
            st = status[i]
            out.append(dict(flags=flags[frame_off[i]:frame_off[i + 1]].copy(),
                            segments=[(float(times[j, 0]), float(times[j, 1]), int(segs[j, 0]), int(segs[j, 1]))
                                      for j in range(r0, r0 + int(seg_n[i]))],
                            in_speech=bool(st["in_speech"]), speech_start=float(st["speech_start"]),
                            speech_end=float(st["speech_end"]), start_sample=int(st["start_sample"]),
                            frames=int(st["frames"])))
        return out

    def reset(self, slots):
        """The listed slots start fresh streams (a new ps_endpointer_init)."""
        slots = np.ascontiguousarray(slots, np.int32)
        check(lib().psb_vad_live_reset(self.h, _p(slots) if len(slots) else None, len(slots)), "psb_vad_live_reset")


class Vad(Endpointer):
    """ps_vad_t for whole batches (arguments as the reference's Python Vad: mode, sample_rate, frame_length):
    classify_batch(streams) gives ps_vad_classify's decision for every full frame of each stream."""

    def __init__(self, mode=0, sample_rate=16000, frame_length=0.03, device=0, warmup=None):
        super().__init__(0.3, 0.9, mode, sample_rate, frame_length, device, warmup)


def pitch_main_reads(n_frames, smooth_window):
    """The reads pocketsphinx_pitch makes inside its frame loop that succeed (psb_pitch_main_reads): yin_t's uint16
    frame counter makes smooth_window + 1 of them fail after every 65 536 frames."""
    if smooth_window == 0:
        return n_frames
    r = n_frames % 65536
    return n_frames // 65536 * (65535 - smooth_window) + max(r - smooth_window, 0)


def pitch_result(period, bestdiff, main_reads, frame_shift, sample_rate):
    """One stream's reads as pocketsphinx_pitch prints them: period and bestdiff (uint16, as yin_read returns them),
    time (the samples of the main loop's reads before this one over the rate: every read after the loop shares the
    last time), voicing (1 - bestdiff / 32768, 0 above 32768) and pitch (sample_rate / period, sample_rate for 0)."""
    period = np.asarray(period, np.uint16)
    bestdiff = np.asarray(bestdiff, np.uint16)
    k = np.minimum(np.arange(len(period), dtype=np.int64), main_reads)
    bd = bestdiff.astype(np.float64)
    p = period.astype(np.float64)
    return dict(period=period, bestdiff=bestdiff,
                time=(k * frame_shift).astype(np.float64) / sample_rate,
                voicing=np.where(bestdiff > 32768, 0.0, 1.0 - bd / 32768),
                pitch=np.where(period == 0, float(sample_rate), float(sample_rate) / np.where(period == 0, 1.0, p)))


def pitch_lines(result, sample_rate):
    """pocketsphinx_pitch's output lines for one stream's result ("%.3f %.2f %.2f\\n" each: time, voicing, pitch, with
    voicing and pitch computed from bestdiff and period as the program computes them); joined, they are the program's
    output file byte for byte."""
    sps = float(sample_rate)
    return ["%.3f %.2f %.2f\n" % (t, 0.0 if bd > 32768 else 1.0 - bd / 32768.0, sps if p == 0 else sps / p)
            for t, p, bd in zip(result["time"].tolist(), result["period"].tolist(), result["bestdiff"].tolist())]


class PitchTracker:
    """YIN pitch tracking (the reference's pocketsphinx_pitch, fe/yin.c) for whole batches of int16 streams on the
    device.  Keywords are the program's options; each stream is tracked by a fresh yin_t, bit for bit."""

    def __init__(self, sample_rate=16000, flen=0.025, fshift=0.01, smooth_window=2, voice_thresh=0.1, search_range=0.2,
                 device=0):
        from ._lib import PitchOpts
        o = PitchOpts()
        o.sample_rate, o.smooth_window = int(sample_rate), int(smooth_window)
        o.flen, o.fshift = float(flen), float(fshift)
        o.voice_thresh, o.search_range = float(voice_thresh), float(search_range)
        h = C.c_void_p()
        check(lib().psb_pitch_create(C.byref(o), device, C.byref(h)), "psb_pitch_create")
        self.h = h
        L = lib()
        self.sample_rate, self.smooth_window = int(sample_rate), int(smooth_window)
        self.frame_size, self.frame_shift, self.ndiff = L.psb_pitch_frame_size(h), L.psb_pitch_frame_shift(h), L.psb_pitch_ndiff(h)

    def n_frames(self, n_samples):
        return 1 + (n_samples - self.frame_size) // self.frame_shift if n_samples >= self.frame_size else 0

    def track_batch(self, streams):
        """Per stream, a dict of period, bestdiff (uint16), time, voicing and pitch (float64): one entry per yin_read
        that succeeds, as pitch_result describes them."""
        streams = [np.ascontiguousarray(s, np.int16) for s in streams]
        n = len(streams)
        samp_off = np.zeros(n + 1, np.int64)
        samp_off[1:] = np.cumsum([len(s) for s in streams])
        pcm = np.concatenate(streams) if n else np.zeros(0, np.int16)
        frames = [self.n_frames(len(s)) for s in streams]
        cap = max(sum(frames), 1)                                      # at most one read per frame
        period = np.zeros(cap, np.uint16)
        bestdiff = np.zeros(cap, np.uint16)
        out_off = np.zeros(n + 1, np.int32)
        check(lib().psb_pitch_process_host(self.h, _p(pcm) if pcm.size else None, _p(samp_off), n, _p(out_off),
                                           _p(period), _p(bestdiff), None), "psb_pitch_process_host")
        return [pitch_result(period[out_off[i]:out_off[i + 1]].copy(), bestdiff[out_off[i]:out_off[i + 1]].copy(),
                             pitch_main_reads(frames[i], self.smooth_window), self.frame_shift, self.sample_rate)
                for i in range(n)]

    def close(self):
        if self.h:
            lib().psb_pitch_free(self.h)
            self.h = None


PITCH_LIVE_STATUS = np.dtype([("frames", np.int32), ("main_reads", np.int32), ("reads", np.int32),
                              ("ended", np.int32)])                               # psb_pitch_live_status_t


def pitch_live_result(period, bestdiff, status, frame_shift, sample_rate):
    """One slot's reads of one live call as pitch_result gives them for the whole stream: the call's reads are the
    stream's reads status["reads"] - len(period) .. status["reads"] - 1, so their times continue across calls.  Adds
    the slot's frames, main_reads (so far) and ended."""
    period = np.asarray(period, np.uint16)
    reads, main = int(status["reads"]), int(status["main_reads"])
    res = pitch_result(period, bestdiff, 0, frame_shift, sample_rate)
    k = np.minimum(np.arange(reads - len(period), reads, dtype=np.int64), main)
    res["time"] = (k * frame_shift).astype(np.float64) / sample_rate
    res.update(frames=int(status["frames"]), main_reads=main, ended=bool(status["ended"]))
    return res


class LivePitchTracker(PitchTracker):
    """YIN pitch tracking for n_slots live streams on the device: feed() hands each listed slot its next samples, in
    any lengths, and returns the reads those samples complete.  A slot's results joined over its calls are
    track_batch's for the whole stream, bit for bit, whatever the chunking.  Options as PitchTracker's; track_batch on
    this handle leaves the slots alone."""

    def __init__(self, n_slots, sample_rate=16000, flen=0.025, fshift=0.01, smooth_window=2, voice_thresh=0.1,
                 search_range=0.2, device=0):
        super().__init__(sample_rate, flen, fshift, smooth_window, voice_thresh, search_range, device)
        try:
            check(lib().psb_pitch_live_open(self.h, int(n_slots)), "psb_pitch_live_open")
        except PsbError:
            self.close()
            raise
        self.n_slots = int(n_slots)

    def feed(self, chunks, slots=None, final=None):
        """chunks: int16 arrays, one per slot in `slots` (default: slots 0 .. len(chunks) - 1).  final: per slot, true
        to end the stream after these samples (yin_end; the slot is then refused until reset).  Returns one dict per
        fed slot: period, bestdiff, time, voicing and pitch of this call's reads (as pitch_live_result), frames (fed
        since the slot was made fresh), main_reads and ended."""
        chunks = [np.ascontiguousarray(c, np.int16) for c in chunks]
        n = len(chunks)
        slots = np.arange(n, dtype=np.int32) if slots is None else np.ascontiguousarray(slots, np.int32)
        if len(slots) != n:
            raise ValueError("feed: %d chunks for %d slots" % (n, len(slots)))
        fin = None if final is None else np.ascontiguousarray([bool(f) for f in final], np.int8)
        if fin is not None and len(fin) != n:
            raise ValueError("feed: %d final flags for %d slots" % (len(fin), n))
        samp_off = np.zeros(n + 1, np.int64)
        samp_off[1:] = np.cumsum([len(c) for c in chunks])
        pcm = np.concatenate(chunks) if n else np.zeros(0, np.int16)
        # new frames + the drain of a final call, per slot
        cap = int(sum(-(-len(c) // self.frame_shift) + 2 * self.smooth_window for c in chunks))
        period = np.zeros(max(cap, 1), np.uint16)
        bestdiff = np.zeros(max(cap, 1), np.uint16)
        out_off = np.zeros(n + 1, np.int32)
        status = np.zeros(max(n, 1), PITCH_LIVE_STATUS)
        check(lib().psb_pitch_feed_host(self.h, _p(slots) if n else None, n, _p(pcm) if pcm.size else None, _p(samp_off),
                                        _p(fin) if fin is not None else None, _p(out_off), _p(period), _p(bestdiff),
                                        _p(status), None), "psb_pitch_feed_host")
        return [pitch_live_result(period[out_off[i]:out_off[i + 1]].copy(), bestdiff[out_off[i]:out_off[i + 1]].copy(),
                                  status[i], self.frame_shift, self.sample_rate) for i in range(n)]

    def reset(self, slots):
        """The listed slots start fresh streams (a new yin_init)."""
        slots = np.ascontiguousarray(slots, np.int32)
        check(lib().psb_pitch_live_reset(self.h, _p(slots) if len(slots) else None, len(slots)), "psb_pitch_live_reset")
