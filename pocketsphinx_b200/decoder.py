"""Batch n-gram decoding from audio to words on the device, configured like the reference's ps_decoder_t
(-hmm, -dict, -lm and the search settings by their reference names): front end -> senone scores -> phone
loop -> first pass -> second pass on the GPU, hypothesis and segments read from the returned tables
(ps_decode_raw + ps_get_hyp / ps_seg_iter with -bestpath no, pocketsphinx.c:1073-1345).  Everything the
reference loads from files is read here by the package itself (s3io, lmio, dict2pid, lextree).

STATUS: GPU-verified end to end (tests/test_gpu_zz_decoder.py).  Out of the
hot-path scope (SURVEY 8): kept small, not extended.
"""
import math
import os

import numpy as np

from . import api, lextree, s3io
from .fe_tables import AGC_TYPES, CMN_TYPES, FEAT_TYPES, make_fe_desc, make_fe_opts
from .model import PackedModel

# config_macro.h (the reference's defaults for every front-end / feature key this class looks at)
FE_REFERENCE_DEFAULTS = dict(feat="1s_c_d_dd", cmn="live", agc="none", agcthresh="2.0", varnorm="no", lda="", ldadim="0",
                             svspec="", dither="no",
                             round_filters="yes", ncep="13", frate="100", nfft="0", cmninit="40,3,-1", seed="-1", samprate="16000",
                             wlen="0.025625", nfilt="40", lowerf="133.33334", upperf="6855.4976", alpha="0.97",
                             transform="legacy", lifter="0", remove_noise="no", remove_dc="no", unit_area="yes", doublebw="no",
                             warp_type="inverse_linear", warp_params="")
PL_DEFAULTS = dict(pl_window="5", pl_beam="1e-10", pl_pbeam="1e-10", pl_pip="1.0", pl_weight="3.0")


def _logs(p, logbase=1.0001):
    return (-(1 << 31) >> 2 if p <= 0 else int(math.log(p) * (1.0 / math.log(logbase)))) >> 10


def acoustic_setup(hmm, cfg, device=0):
    """The acoustic model and the device front end for -hmm `hmm` and the reference-named settings cfg (strings), as
    ps_init configures them: the model's own settings (varfloor, tmatfloor, mixwfloor, topn, ds, aw); the front end
    from the reference's defaults (config_macro.h), overlaid by the model's feat.params, then by cfg.  Returns
    (PackedModel, api.FrontEnd, the front-end settings in force)."""
    pm = PackedModel.from_dir(hmm, **{k: v for k, v in cfg.items() if k in ("varfloor", "tmatfloor", "mixwfloor", "topn", "ds", "aw")})
    # front end: the reference's own defaults (config_macro.h), overlaid by the model's feat.params, then by the
    # caller -- like ps_init; whatever the device front end does not implement is refused, not ignored
    from .s3io import read_feat_params
    fp = dict(FE_REFERENCE_DEFAULTS)
    fp.update(read_feat_params(os.path.join(hmm, "feat.params")))
    fp.update({k: v for k, v in cfg.items() if k in FE_REFERENCE_DEFAULTS})
    yes = ("yes", "1", "true", "True")
    unsupported = []
    if fp["feat"] not in FEAT_TYPES: unsupported.append("-feat " + fp["feat"])
    if fp["cmn"] not in CMN_TYPES: unsupported.append("-cmn " + fp["cmn"])
    if fp["agc"] not in AGC_TYPES: unsupported.append("-agc " + fp["agc"])
    if fp["varnorm"] in yes and CMN_TYPES.get(fp["cmn"]) != 1: unsupported.append("-varnorm yes with -cmn " + fp["cmn"])
    if fp["svspec"] not in ("", "0-12/13-25/26-38"): unsupported.append("-svspec " + fp["svspec"])
    if int(fp["ncep"]) != 13: unsupported.append("-ncep " + fp["ncep"])
    if int(fp["frate"]) != 100: unsupported.append("-frate " + fp["frate"])
    if int(fp["nfft"]) != 0: unsupported.append("-nfft " + fp["nfft"])
    if unsupported:
        raise NotImplementedError("front end settings the device front end does not implement: " + ", ".join(unsupported))
    # -lda defaults to the model's feature_transform when there is one (ps_expand_model_config, pocketsphinx.c:119)
    if not fp["lda"] and os.path.exists(os.path.join(hmm, "feature_transform")):
        fp["lda"] = os.path.join(hmm, "feature_transform")
    if fp["lda"] and fp["svspec"]:
        # feat_dimension2 is the LDA output for every subvector, which no model's streams match (acmod_init fails)
        raise ValueError("-lda %s with -svspec %s: the reference cannot load this model either" % (fp["lda"], fp["svspec"]))
    lda = s3io.read_lda(fp["lda"])[0] if fp["lda"] else None
    opts = make_fe_opts(feat=fp["feat"], cmn=fp["cmn"], cmninit=fp["cmninit"], dither=fp["dither"] in yes,
                        seed=int(fp["seed"]), ncep=int(fp["ncep"]), varnorm=fp["varnorm"] in yes, agc=fp["agc"],
                        agcthresh=float(fp["agcthresh"]), lda=lda, ldadim=int(fp["ldadim"]))
    desc = make_fe_desc(samprate=float(fp["samprate"]), wlen=float(fp["wlen"]), nfilt=int(fp["nfilt"]),
                        lowerf=float(fp["lowerf"]), upperf=float(fp["upperf"]), alpha=float(fp["alpha"]),
                        transform=fp["transform"], lifter=int(fp["lifter"]), remove_noise=fp["remove_noise"] in yes,
                        remove_dc=fp["remove_dc"] in yes, unit_area=fp["unit_area"] in yes,
                        round_filters=fp["round_filters"] in yes, doublebw=fp["doublebw"] in yes,
                        warp_type=fp["warp_type"], warp_params=fp["warp_params"] or None)
    # 1s_c_d_dd with batch CMN and nothing else is the front end desc alone describes
    plain = (opts["feat"], opts["cmn"], opts["dither"], opts["varnorm"], opts["agc"], lda is None) == (0, 1, 0, 0, 0, True)
    # the dimension psb_fe_feat_dim will report: feat_read_lda's out_dim, else the feature type's
    dim = 51 if opts["feat"] == 1 else 3 * int(fp["ncep"])
    if lda is not None:
        dim = opts["ldadim"] if 0 < opts["ldadim"] <= lda.shape[0] else lda.shape[0]
    if dim != pm.sumlen:
        raise ValueError("the front end makes %d-dimensional features (-feat %s%s), the model in %s wants %d"
                         % (dim, fp["feat"], ", -lda %s" % fp["lda"] if fp["lda"] else "", hmm, pm.sumlen))
    fe = api.FrontEnd(desc, device) if plain else api.FrontEnd(desc, device, opts)
    return pm, fe, fp


class Decoder:
    def __init__(self, hmm, dict_file, lm_file, max_utts=64, max_frames=1 << 16, device=0, **config):
        cfg = {k: str(v) for k, v in config.items()}
        self.pm, self.fe, fp = acoustic_setup(hmm, cfg, device)
        search_cfg = {k: v for k, v in cfg.items() if k in lextree.DEFAULTS}
        self.search = lextree.ngram_search_from_files(hmm, dict_file, lm_file, **search_cfg)
        # -phone_align / -state_align (pocketsphinx_main.c; -state_align implies -phone_align): a second pass aligns
        # each utterance to its own word segments.  The alignment always has all three levels.
        yes = ("yes", "1", "true", "True")
        self.phone_align = cfg.get("phone_align", "no") in yes or cfg.get("state_align", "no") in yes
        self.align_tables = None
        if self.phone_align:
            from .align import AlignTables
            self.align_tables = AlignTables(hmm, dict_file)
        self.model = api.Model(self.pm, device)
        # the second pass scores every utterance after a copy of itself (_align_pass): twice the frames
        k = 2 if self.phone_align else 1
        self.batch = api.Batch(self.model, max_utts * k, max_frames * k)
        self.ctx = api.HmmContext(self.pm.tp, self.pm.sseq, self.pm.n_sen, device=device)
        self.device = device
        pl = dict(PL_DEFAULTS)
        pl.update({k: v for k, v in cfg.items() if k in PL_DEFAULTS})
        self.pl_window = int(pl["pl_window"])
        n_ci = self.pm.n_ciphone
        self.phoneloop = api.PhoneLoop(self.ctx, self.pm.phone_ssid[:n_ci], self.pm.phone_tmat[:n_ci], self.pl_window,
                                       _logs(float(pl["pl_beam"])), _logs(float(pl["pl_pbeam"])), _logs(float(pl["pl_pip"])),
                                       float(pl["pl_weight"]))
        self.second_pass = search_cfg.get("fwdflat", "yes") in ("yes", "1", "true", "True")
        self.bp_cap = int(cfg.get("latsize", 5000))
        self.sample_rate = int(float(fp["samprate"]))
        self.warp_params = fp["warp_params"] or None
        self.max_utts = max_utts

    def decode_raw_batch(self, utterances, sessions=None, start_stream="utterance", warp=None):
        """utterances: int16 arrays, each a whole utterance.  sessions: None (every utterance a fresh decoder) or one
        session id per utterance; the utterances of one id are one decoder's, in list order, from a fresh decoder
        (the front end's live CMN and dither state carry over).  start_stream says where that decoder calls
        ps_start_stream, which resets the -remove_noise tracker: "utterance" reproduces a reference program that calls
        ps_start_stream, ps_start_utt, ps_process_raw(full_utt), ps_end_utt for every utterance; "session" one that
        calls ps_start_stream once before a session's first utterance and then only ps_start_utt, ps_process_raw,
        ps_end_utt, so the tracker carries from one utterance to the next.  Returns one dict per utterance: hyp (the
        words, fillers and <s> / </s> left out), score, seg [n][7] = entry, wid, sf, ef, path score, ascr, lscr, and
        words().  With phone_align / state_align each dict also has alignment (align.Alignment: the words, phones and
        states of the second pass over seg; None where the reference's ps_set_alignment or search fails) and
        alignment_error (that failure's reason, else None).  warp: None, or one -warp_params string per utterance (under this decoder's -warp_type; None: the
        decoder's own -warp_params), so each utterance is decoded with its own VTLN warp; the utterances of one session
        are one decoder's and must name the same warp."""
        if start_stream not in ("utterance", "session"):
            raise ValueError("start_stream must be 'utterance' or 'session', not %r" % (start_stream,))
        if warp is not None:
            warp = list(warp)
            if len(warp) != len(utterances):
                raise ValueError("%d warps for %d utterances" % (len(warp), len(utterances)))
            # None is the decoder's own -warp_params, and "" is unset: both name the bank of the decoder's front end
            # when they mean its warp (None below)
            warp = [None if (self.warp_params if w is None else w or None) == self.warp_params else w for w in warp]
            if all(w is None for w in warp):
                warp = None
        if sessions is None:
            return self._decode(utterances, None, warp=warp)
        assert len(sessions) == len(utterances)
        if warp is not None:
            named = {}
            for sid, w in zip(sessions, warp):
                if named.setdefault(sid, w) != w:
                    raise ValueError("session %r names two warps, %r and %r: a session is one decoder, with one warp"
                                     % (sid, named[sid], w))
        first = {}
        for i, sid in enumerate(sessions):
            first.setdefault(sid, i)
        # the front end wants each session's utterances consecutive, in decode order
        order = sorted(range(len(utterances)), key=lambda i: (first[sessions[i]], i))
        sizes = [sessions.count(sid) for sid in sorted(first, key=first.get)]
        res = self._decode([utterances[i] for i in order], np.cumsum([0] + sizes), start_stream == "session",
                           None if warp is None else [warp[i] for i in order])
        out = [None] * len(utterances)
        for j, i in enumerate(order):
            out[i] = res[j]
        return out

    def decode_stream_batch(self, streams, vad_mode=0, vad_window=0.3, vad_ratio=0.9, vad_frame_length=0.03,
                            start_stream="utterance", warp=None):
        """Whole recordings in, words out: every stream is cut into speech segments by the device endpointer (at the
        model's sample rate; api.Endpointer), and all segments of all streams are decoded in one decode_raw_batch call
        with one session per stream, so a stream's segments are one decoder's utterances in order (live CMN and dither
        carry over, as for a reference decoder fed the segments one after another).  start_stream is decode_raw_batch's:
        "utterance" for a reference program that calls ps_start_stream before every segment, "session" for one that
        calls it once per recording, so the -remove_noise tracker carries across its segments.  Returns, per stream, a list of
        dicts: start_time, end_time (the endpointer's float64 seconds), start_sample, end_sample, and decode_raw_batch's
        hyp, score, seg, words, n_frames.  The segments count against max_utts / max_frames of this Decoder.  warp:
        None, or one -warp_params string per stream (decode_raw_batch's warp; None: the decoder's own)."""
        if warp is not None and len(warp) != len(streams):
            raise ValueError("%d warps for %d streams" % (len(warp), len(streams)))
        ep = api.Endpointer(vad_window, vad_ratio, vad_mode, self.sample_rate, vad_frame_length, self.device)
        try:
            segs = ep.segment_batch(streams)
        finally:
            ep.close()
        utts, sessions = [], []
        for i, (pcm, ss) in enumerate(zip(streams, segs)):
            for _, _, a, b in ss:
                utts.append(np.asarray(pcm)[a:b])
                sessions.append(i)
        if len(utts) > self.max_utts:
            raise ValueError("%d speech segments, more than this Decoder's max_utts (%d): create it with a larger max_utts"
                             % (len(utts), self.max_utts))
        res = self.decode_raw_batch(utts, sessions, start_stream, None if warp is None else [warp[i] for i in sessions]) \
            if utts else []
        out, k = [], 0
        for ss in segs:
            row = []
            for t0, t1, a, b in ss:
                d = dict(res[k])
                d.update(start_time=t0, end_time=t1, start_sample=a, end_sample=b)
                row.append(d)
                k += 1
            out.append(row)
        return out

    def _decode(self, utterances, sess_off, carry_noise=False, warp=None):
        import torch
        g = self.search
        info = g["info"]
        off = api.FrontEnd.sample_offsets([len(u) for u in utterances])
        pcm = np.concatenate([np.ascontiguousarray(u, np.int16) for u in utterances]) if utterances else np.zeros(0, np.int16)
        # the banks are built (and a refused warp raises) before anything is named for the front end's next call;
        # whatever is refused after that drops every setting, so none is left for a later call
        banks = None if warp is None else self.fe.warp_filterbanks(warp)
        try:
            if sess_off is not None:
                self.fe.set_sessions(sess_off)
                if carry_noise:
                    starts = np.zeros(len(utterances), bool)
                    starts[np.asarray(sess_off[:-1])[np.diff(sess_off) > 0]] = True
                    self.fe.set_stream_starts(starts)
            if banks is not None:
                self.fe.name_filterbanks(banks)
            frame_off, best, pen = self.batch.decode_pcm_host(self.fe, self.phoneloop, pcm, off)
        except BaseException:
            self.fe.cancel_settings()
            raise
        d_scr = self.batch.senscr_device_ptr()
        d_pen = (torch.from_numpy(np.ascontiguousarray(pen, np.int32)).to(torch.device("cuda", self.device))
                 if self.pl_window > 0 and len(pen) else None)
        pen_ptr, win = (d_pen.data_ptr(), self.pl_window) if d_pen is not None else (None, 0)
        # -latsize is an initial size in the reference (bp_table / bscore_stack double on demand,
        # ngram_search.c:326-339): a table that fills up is retried with doubled capacities
        # ... and streams start from a size that fits them (the 72 k-word en-us LM writes about eleven entries per frame
        # and twenty scores per entry on the reference's test data): a retry repeats the whole search, the reference's
        # realloc does not
        longest = int(np.diff(frame_off).max()) if len(frame_off) > 1 else 0
        cap = max(self.bp_cap, 12 * longest + 1000)
        for _ in range(6):
            try:
                if self.second_pass:
                    tabs, _ = self.ctx.ngram_two_pass(d_scr, frame_off, info, g["model"], g["ci_tmat"], g["ci_ssid"], cap, 24 * cap,
                                                      pen_ptr, win, first_cap=cap, first_bss_cap=24 * cap, lm_arrays=g["lm_arrays"])
                else:
                    tabs = self.ctx.ngram_fwdtree(d_scr, frame_off, info, g["model"], g["ci_tmat"], cap, 24 * cap, pen_ptr, win,
                                                  lm_arrays=g["lm_arrays"])
                break
            except api.PsbError as e:
                if "overflow" not in str(e):
                    raise
                cap *= 2
        else:
            raise RuntimeError("backpointer table still overflows at %d entries per utterance" % cap)
        out = []
        words, base, fs, fe_ = g["words"], g["base"], int(info[22]), int(info[23])
        for u, (bp, bss, idx) in enumerate(tabs):
            T = int(frame_off[u + 1] - frame_off[u])
            entry, score, _ = api.ngram_hyp(bp, idx, T, int(info[20]))
            seg = api.ngram_segments(info, g["model"], bp, bss, entry, lm_arrays=g["lm_arrays"], second_pass=self.second_pass)
            real = [words[base[w]] for w in seg[:, 1] if not (fs <= int(base[w]) <= fe_)]        # dict_real_word + dict_basestr
            out.append(dict(hyp=" ".join(real), score=score, seg=seg, words=[words[w] for w in seg[:, 1]], n_frames=T))
        if self.phone_align:
            self._align_pass(utterances, sess_off, carry_noise, warp, out)
        return out

    def _align_pass(self, utterances, sess_off, carry_noise, warp, out):
        """The second pass of `pocketsphinx single -phone_align yes` (decode_single, pocketsphinx_main.c:462-476):
        ps_set_alignment(ps, NULL) turns the segments into timed words (ps_alignment_add_word(wid, sf, ef - sf + 1)),
        and the same decoder decodes the same audio again, without ps_start_stream.  Its front end carries its state
        (live CMN, the -remove_noise tracker, dither) from the first decode into the second, so the second pass is
        scored as the utterance's own repeat in its session: every utterance is followed by a copy of itself, the
        copies are aligned, the originals get no phones."""
        from .align import align_batch
        n = len(utterances)
        lens = np.repeat([len(u) for u in utterances], 2)
        pcm2 = (np.concatenate([np.ascontiguousarray(u, np.int16) for u in utterances for _ in (0, 1)]) if n
                else np.zeros(0, np.int16))
        sess2 = np.arange(0, 2 * n + 1, 2, dtype=np.int32) if sess_off is None else 2 * np.asarray(sess_off, np.int32)
        starts = np.zeros(2 * n, bool)
        if carry_noise:
            starts[sess2[:-1][np.diff(sess2) > 0]] = True
        else:
            starts[0::2] = True
        banks = None if warp is None else self.fe.warp_filterbanks([w for w in warp for _ in (0, 1)])
        try:
            self.fe.set_sessions(sess2)
            self.fe.set_stream_starts(starts)
            if banks is not None:
                self.fe.name_filterbanks(banks)
            frame_off = self.batch.score_pcm(self.fe, pcm2, api.FrontEnd.sample_offsets(lens))
        except BaseException:
            self.fe.cancel_settings()
            raise
        chains = []
        for d in out:
            seg = d["seg"]
            # ps_seg_iter returns NULL for no segments, and ps_set_alignment fails
            chains += [None, (seg[:, 1].tolist(), seg[:, 2].astype(np.int64), (seg[:, 3] - seg[:, 2] + 1).astype(np.int64))
                       if len(seg) else None]
        res, self.last_align_token_bytes = align_batch(self.ctx, self.align_tables, self.batch.senscr_device_ptr(),
                                                       frame_off, chains, windows=True)
        for u, d in enumerate(out):
            a, why = res[2 * u + 1]
            d["alignment"] = a
            d["alignment_error"] = why if chains[2 * u + 1] is not None else "no word segments to align"

    def close(self):
        for o in (self.phoneloop, self.batch, self.ctx, self.model, self.fe):
            o.close()
