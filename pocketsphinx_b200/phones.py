"""Phone decoding from audio for whole batches, configured like the reference's allphone search (-hmm, -allphone
with a phone LM or none, -allphone_ci, and beam / pbeam / pip / lw / wip by their reference names): front end ->
senone scores -> allphone_net_kernel on the GPU (DESIGN 4.9), the phone segments read out as ps_get_hyp and
ps_seg_iter report them at the end of an utterance (allphone_search_hyp / allphone_search_fill_iter,
allphone_search.c:77-130, 877-915).  The PHMM net is built from the model definition alone (allphone_net); the
phone LM is read by the package (lmio) and tabulated once by psb_allphone_lm_tables; the model and front end are set
up as for the Decoder (decoder.acoustic_setup).
"""
import ctypes as C
import os

import numpy as np

from . import allphone_net, api, lmio, s3io
from ._lib import check, lib
from .decoder import acoustic_setup

# config_macro.h: the settings the allphone search reads, at the reference's defaults
ALLPHONE_DEFAULTS = dict(allphone_ci="yes", beam="1e-48", pbeam="1e-48", pip="1.0", lw="6.5", wip="0.65", logbase="1.0001")

_BOOL = {"yes": True, "true": True, "1": True, "no": False, "false": False, "0": False}


def phone_lm_tables(lm, ciname, sil, lw=6.5, wip=0.65, logbase=1.0001):
    """The phone LM's dense tables (bg [n_ci][n_ci], tg [n_ci][n_ci][n_ci], scores >> SENSCR_SHIFT) for a model whose
    CI phone names in CI order are `ciname` and whose silence phone is CI phone `sil`.  lm: lmio.read_lm_bin's result;
    lw / wip as ngram_model_read applies them.  ci2lmwid is allphone_search_init's (:552-577): a phone the LM does not
    know maps to SIL's LM word, and an LM without SIL is refused as the reference refuses it."""
    n_ci = len(ciname)
    if n_ci > 64:
        raise ValueError("%d CI phones: the phone net's context sets are 64-bit masks (at most 64)" % n_ci)
    wid = {}
    for i, w in enumerate(lm["words"]):
        wid.setdefault(w, i)                                 # duplicates: the first one wins (hash_table_enter)
    unk = wid.get("<UNK>", -1)                               # ngram_unknown_wid
    silwid = wid.get(ciname[sil], unk) if 0 <= sil < n_ci else unk
    if silwid == unk:
        raise ValueError("Phonetic LM does not have SIL phone in vocabulary")
    ci2lmwid = [wid.get(n, unk) for n in ciname]
    ci2lmwid = np.array([silwid if w == unk else w for w in ci2lmwid], np.int32)
    block = lmio.lm_arrays(lm, list(ciname), lw=lw, wip=wip, logbase=logbase)
    block[10:10 + n_ci] = ci2lmwid                           # the widmap: ci2lmwid, not the n-gram search's <UNK> rule
    bg = np.zeros((n_ci, n_ci), np.int32)
    tg = np.zeros((n_ci, n_ci, n_ci), np.int32)
    check(lib().psb_allphone_lm_tables(block.ctypes.data_as(C.c_void_p), n_ci, bg.ctypes.data_as(C.c_void_p),
                                       tg.ctypes.data_as(C.c_void_p)), "psb_allphone_lm_tables")
    return bg, tg


def phone_result(segs, status, n_frames, ciname):
    """One utterance's result from its allphone_net rows: segs [n][5] = (ci, sf, ef, score, tscore) in time order (the
    reference's phseg_t list after allphone_backtrace) and the search's status.  hyp: the phones' CI names joined by
    single spaces, SIL and fillers included (allphone_search_hyp), None when there is no segment; score:
    ps_get_hyp's out_score, the best history entry's path score, which the segments' score + tscore add up to
    (allphone never renormalises, and the backtrace starts each chain from 0); seg: ps_seg_iter's rows (name, sf, ef,
    ascr = score, lscr = tscore).  A status other than 0 (1: the utterance's history outgrew its table) leaves no
    hypothesis; `reason` then says why."""
    status = int(status)
    out = dict(hyp=None, score=None, seg=[], n_frames=int(n_frames), status=status, reason=None)
    if status != 0:
        out["reason"] = ("history table overflow: the search of this utterance stopped" if status == 1
                         else "search status %d" % status)
        return out
    rows = np.asarray(segs).reshape(-1, 5).tolist()
    if not rows:
        return out
    out["seg"] = [(ciname[c], sf, ef, sc, ts) for c, sf, ef, sc, ts in rows]
    out["hyp"] = " ".join(s[0] for s in out["seg"])
    out["score"] = int(sum(sc + ts for _, _, _, sc, ts in rows))
    return out


def search_setup(hmm, allphone=None, **config):
    """What allphone_search_init builds from -hmm, -allphone and the settings in config (strings, reference names;
    others are ignored): ciname (the CI phone names), net (allphone_net.build_net over the mdef), beam, pbeam,
    inspen (allphone_search_init :580-601; 0 with a phone LM, whose insertion penalty is its -wip), and bg / tg
    (phone_lm_tables; None without a phone LM).  Host work only: the model's other files are not read."""
    s = dict(ALLPHONE_DEFAULTS)
    s.update({k: str(v) for k, v in config.items() if k in ALLPHONE_DEFAULTS})
    ci_only = _BOOL.get(s["allphone_ci"].lower())
    if ci_only is None:
        raise ValueError("-allphone_ci %s: not a boolean" % s["allphone_ci"])
    md = s3io.read_mdef(os.path.join(hmm, "mdef"))
    ciname = list(md["ciname"])
    lw, logbase = float(s["lw"]), float(s["logbase"])
    beam, pbeam, inspen = allphone_net.search_params(float(s["beam"]), float(s["pbeam"]), float(s["pip"]), lw, logbase)
    bg = tg = None
    if allphone is not None:
        bg, tg = phone_lm_tables(lmio.read_lm_bin(allphone), ciname, int(md["sil"]), lw, float(s["wip"]), logbase)
        inspen = 0
    return dict(ciname=ciname, net=allphone_net.build_net(allphone_net.mdef_phones(md), ci_only), beam=beam,
                pbeam=pbeam, inspen=inspen, bg=bg, tg=tg)


class PhoneDecoder:
    """Phone decoding for batches of utterances, configured like the reference's ps_decoder_t with -allphone:
    allphone is the phone LM's path (a binary trie LM, e.g. en-us-phone.lm.bin) or None for the unconstrained phone
    loop.  config: allphone_ci (default yes: one node per CI phone; no: the context-dependent net of every phone of
    the mdef), beam, pbeam, pip, lw, wip, logbase, and every model and front-end setting the Decoder takes, by the
    reference's names.  Every senone is scored (the reference's -compallsen yes).  Each utterance is decoded by a
    fresh decoder.  max_utts / max_frames bound one batch (frames summed over its utterances)."""

    def __init__(self, hmm, allphone=None, max_utts=64, max_frames=1 << 16, device=0, **config):
        cfg = {k: str(v) for k, v in config.items()}
        self.search = search_setup(hmm, allphone, **cfg)
        self.ciname = self.search["ciname"]
        self.pm, self.fe, _ = acoustic_setup(hmm, cfg, device)
        self.model = api.Model(self.pm, device)
        self.batch = api.Batch(self.model, max_utts, max_frames)
        self.ctx = api.HmmContext(self.pm.tp, self.pm.sseq, self.pm.n_sen, device=device)
        self.max_utts, self.max_frames = max_utts, max_frames

    def decode_raw_batch(self, utterances):
        """utterances: int16 arrays, each a whole utterance.  Returns one dict per utterance (see decode_senscr)."""
        lens = [len(u) for u in utterances]
        frames = [self.fe.n_frames(n) for n in lens]
        if len(utterances) > self.max_utts:
            raise ValueError("%d utterances, more than this PhoneDecoder's max_utts (%d)" % (len(utterances), self.max_utts))
        if sum(frames) > self.max_frames:
            raise ValueError("%d frames in this batch (longest utterance %d), more than this PhoneDecoder's max_frames "
                             "(%d): create it with a larger max_frames" % (sum(frames), max(frames), self.max_frames))
        pcm = np.concatenate([np.ascontiguousarray(u, np.int16) for u in utterances]) if utterances else np.zeros(0, np.int16)
        frame_off = self.batch.score_pcm(self.fe, pcm, api.FrontEnd.sample_offsets(lens))
        return self.decode_senscr(self.batch.senscr_device_ptr(), frame_off)

    def decode_senscr(self, d_senscr_ptr, frame_off):
        """The search from senone scores already on the device (int16 [frames][n_sen], every senone), utterance u at
        frames frame_off[u] .. frame_off[u+1].  Returns one dict per utterance: hyp, score (ps_get_hyp), seg
        (ps_seg_iter: (phone, sf, ef, ascr, lscr)), n_frames, status (0, or 1: the history outgrew its table) and
        reason (None, or why there is no hypothesis)."""
        frame_off = np.ascontiguousarray(frame_off, np.int32)
        p = self.search
        r = self.ctx.allphone_net(d_senscr_ptr, frame_off, p["net"], p["beam"], p["pbeam"], p["inspen"], bg=p["bg"],
                                  tg=p["tg"])
        return [phone_result(r["segs"][u], r["status"][u], frame_off[u + 1] - frame_off[u], self.ciname)
                for u in range(len(frame_off) - 1)]

    def close(self):
        for o in (self.batch, self.ctx, self.model, self.fe):
            o.close()
