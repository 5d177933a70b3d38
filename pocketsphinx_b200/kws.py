"""Keyword spotting in batches of audio on the device, configured like the reference's kws search (-hmm, -dict,
-keyphrase or -kws, kws_threshold / kws_plp / kws_delay / beam by their reference names): front end -> senone
scores -> kws_kernel on the GPU, the raw hits reduced on the host by the reference's detection-list rules
(kws_detections_add, kws_detections.c:55-80) and reported as ps_get_hyp / ps_seg_iter report them at the end of an
utterance (kws_search.c:117-151, 672-684, kws_detections.c:83-121).  The keyphrase chains are built from the files
alone (dict2pid.keyphrase_phones); the model and front end are set up as for the Decoder (decoder.acoustic_setup).
"""
import os
import re

import numpy as np

from . import api, dict2pid, lmio, s3io
from .decoder import acoustic_setup
from .lextree import _logs

# cmdln_macro.h: the kws search's settings and their reference defaults
KWS_DEFAULTS = dict(kws_threshold="1e-30", kws_plp="1e-1", kws_delay="10", beam="1e-48", logbase="1.0001")

_FLOAT_PREFIX = re.compile(r"\s*[+-]?(?:inf(?:inity)?|nan|(?:\d+\.?\d*|\.\d+)(?:[eE][+-]?\d+)?)", re.IGNORECASE)


def _atof(s):
    """atof_c: the longest leading decimal number of s, 0 where there is none."""
    m = _FLOAT_PREFIX.match(s)
    return float(m.group(0)) if m else 0.0


def read_kws_list(path, def_threshold, logbase=1.0001):
    """kws_search_read_list (kws_search.c:337-382): one keyphrase per line, whitespace trimmed from both ends, blank
    lines and comment lines ('#' first) skipped; a line ending in '/' carries its own threshold between the last two
    slashes (logmath_log >> SENSCR_SHIFT), and its phrase is the text before that slash as it stands (a space before
    the slash stays part of it).  Returns [(phrase, threshold)] in the reference's list order: glist_add_ptr prepends
    and the list is never reversed, so the last line of the file comes first."""
    out = []
    with open(path, "rb") as f:
        lines = f.read().decode("utf-8", "surrogateescape").split("\n")          # fgets: lines end at '\n' only
    for n, raw in enumerate(lines):
        # lineiter_start_clean tests the first line for '#' before trimming it, lineiter_next every later one after
        if n == 0 and raw.startswith("#"):
            continue
        line = raw.strip(" \t\n\r\f")                                     # string_trim
        if not line or (n > 0 and line.startswith("#")):
            continue
        if line.endswith("/") and len(line) > 1:
            begin = len(line) - 2
            while line[begin] != "/" and begin > 0:
                begin -= 1
            thr = _logs(_atof(line[begin + 1:len(line) - 1]), logbase)
            line = line[:begin]
        else:
            thr = def_threshold
        out.append((line, thr))
    out.reverse()
    return out


def detections(hits, phrases):
    """kws_detections_add on the raw hits of one utterance, in the order the search produced them: a hit overlapping
    an earlier detection of the same keyphrase text replaces it when its prob is higher and is dropped otherwise.
    hits: [n][5] = (frame, keyphrase index, sf, prob, ascr); phrases: the keyphrase texts by index.  Returns the
    detection list in the reference's order (newest first), entries (keyphrase, sf, ef, prob, ascr)."""
    made, by_text = [], {}
    for ef, k, sf, prob, ascr in np.asarray(hits).tolist():
        text = phrases[k]
        # this text's detections oldest first, and the running maximum of their end frames: hits come in frame
        # order, so the scan (newest first) stops where no older detection ends after sf -- none of those overlaps
        same, top = by_text.setdefault(text, ([], []))
        i = len(same) - 1
        while i >= 0 and top[i] > sf:
            d = same[i]
            if d[1] < ef and d[2] > sf:
                if d[3] < prob:
                    d[1:] = [sf, ef, prob, ascr]
                    top[i:] = [ef] * (len(top) - i)    # ef is the latest frame yet
                break
            i -= 1
        else:
            d = [text, sf, ef, prob, ascr]
            same.append(d)
            top.append(ef)
            made.append(d)
    return [tuple(d) for d in reversed(made)]


def hyp_and_segments(dets, n_frames, delay):
    """What ps_get_hyp and ps_seg_iter report after an utterance of n_frames frames (kwss->frame) with -kws_delay
    `delay`: the hypothesis joins, oldest first, the keyphrases of the detections that end before n_frames - delay
    (None when there is none: ps_get_hyp's NULL); the segments skip the newest detections while they end after
    n_frames - delay and list all the rest, oldest first, as (keyphrase, sf, ef, prob, ascr)."""
    last = n_frames - delay
    words = [d[0] for d in reversed(dets) if d[2] < last]
    i = 0
    while i < len(dets) and dets[i][2] > last:
        i += 1
    return (" ".join(words) if words else None), list(reversed(dets[i:]))


class KeywordSpotter:
    """Keyword spotting for batches of utterances, configured like the reference's ps_decoder_t with -keyphrase or
    -kws: exactly one of keyphrase (one phrase) or kws (a keyphrase list file) is given.  config: kws_threshold,
    kws_plp, kws_delay, beam, and every model and front-end setting the Decoder takes, by the reference's names.
    Phrases with a word the dictionary lacks are left out, as the reference leaves them out (kws_search.c:533-548);
    they are in `dropped`.  `keyphrases` / `thresholds` are the spotted phrases in the reference's list order.
    max_utts / max_frames bound one batch (frames summed over its utterances); a stream is one utterance."""

    def __init__(self, hmm, dict_file, keyphrase=None, kws=None, max_utts=64, max_frames=1 << 16, device=0, **config):
        if (keyphrase is None) == (kws is None):
            raise ValueError("give exactly one of keyphrase and kws (the reference refuses both and neither)")
        cfg = {k: str(v) for k, v in config.items()}
        self.pm, self.fe, _ = acoustic_setup(hmm, cfg, device)
        k = dict(KWS_DEFAULTS)
        k.update({n: v for n, v in cfg.items() if n in KWS_DEFAULTS})
        logbase = float(k["logbase"])
        # kws_search_init (kws_search.c:397-411)
        self.beam, self.plp = _logs(float(k["beam"]), logbase), _logs(float(k["kws_plp"]), logbase)
        self.def_threshold, self.delay = _logs(float(k["kws_threshold"]), logbase), int(k["kws_delay"])
        listed = read_kws_list(kws, self.def_threshold, logbase) if kws is not None else [(keyphrase, self.def_threshold)]
        # kws_search_reinit (kws_search.c:479-594): the phone loop is every CI phone; each phrase one chain
        md = s3io.read_mdef(os.path.join(hmm, "mdef"))
        nd = os.path.join(hmm, "noisedict")
        words, prons, _, _ = lmio.read_dict(dict_file, nd if os.path.exists(nd) else None, md["ciname"])
        ci = {n: i for i, n in enumerate(md["ciname"])}
        idx = {}
        for i, w in enumerate(words):
            idx.setdefault(w, i)
        pr = [[ci[x] for x in p] for p in prons]
        tabs = dict2pid.build(md, pr)
        self.keyphrases, self.thresholds, self.dropped = [], [], []
        ssid, tmat, off = [], [], [0]
        for text, thr in listed:
            ws = [w for w in re.split(r"[ \t\n\v\f\r]+", text) if w]         # str2words: isspace_c separates
            if any(w not in idx for w in ws):
                self.dropped.append(text)
                continue
            s, t = dict2pid.keyphrase_phones(md, pr, tabs, [idx[w] for w in ws])
            self.keyphrases.append(text)
            self.thresholds.append(thr)
            ssid.append(s); tmat.append(t); off.append(off[-1] + len(s))
        n_ci = md["n_ciphone"]
        self.pl_ssid = md["phone_ssid"][:n_ci].astype(np.int32)
        self.pl_tmat = md["phone_tmat"][:n_ci].astype(np.int32)
        self.kp_off = np.array(off, np.int32)
        self.kp_thresh = np.array(self.thresholds, np.int32)
        self.kp_ssid = np.concatenate(ssid).astype(np.int32) if ssid else np.zeros(0, np.int32)
        self.kp_tmat = np.concatenate(tmat).astype(np.int32) if tmat else np.zeros(0, np.int32)
        self.model = api.Model(self.pm, device)
        self.batch = api.Batch(self.model, max_utts, max_frames)
        self.ctx = api.HmmContext(self.pm.tp, self.pm.sseq, self.pm.n_sen, device=device)
        self.max_utts, self.max_frames = max_utts, max_frames

    def spot_raw_batch(self, utterances):
        """utterances: int16 arrays, each one utterance (a whole recording is one stream, one utterance, as the
        reference searches it).  Returns one dict per utterance: detections, hyp, seg (see spot_senscr), n_frames."""
        lens = [len(u) for u in utterances]
        frames = [self.fe.n_frames(n) for n in lens]
        if len(utterances) > self.max_utts:
            raise ValueError("%d utterances, more than this KeywordSpotter's max_utts (%d)" % (len(utterances), self.max_utts))
        if sum(frames) > self.max_frames:
            raise ValueError("%d frames in this batch (longest utterance %d), more than this KeywordSpotter's max_frames "
                             "(%d): create it with a larger max_frames" % (sum(frames), max(frames), self.max_frames))
        pcm = np.concatenate([np.ascontiguousarray(u, np.int16) for u in utterances]) if utterances else np.zeros(0, np.int16)
        frame_off = self.batch.score_pcm(self.fe, pcm, api.FrontEnd.sample_offsets(lens))
        return self.spot_senscr(self.batch.senscr_device_ptr(), frame_off)

    def spot_senscr(self, d_senscr_ptr, frame_off):
        """The search from senone scores already on the device (int16 [frames][n_sen], every senone), utterance u
        at frames frame_off[u] .. frame_off[u+1].  Returns one dict per utterance: detections (the detection list,
        newest first, entries (keyphrase, sf, ef, prob, ascr)), hyp and seg (ps_get_hyp / ps_seg_iter at the end of
        the utterance, -kws_delay applied), n_frames."""
        frame_off = np.ascontiguousarray(frame_off, np.int32)
        hits, _ = self.ctx.kws(d_senscr_ptr, frame_off, self.pl_ssid, self.pl_tmat, self.kp_off, self.kp_thresh,
                               self.kp_ssid, self.kp_tmat, self.beam, self.plp)
        out = []
        for u, h in enumerate(hits):
            T = int(frame_off[u + 1] - frame_off[u])
            dets = detections(h, self.keyphrases)
            hyp, seg = hyp_and_segments(dets, T, self.delay)
            out.append(dict(detections=dets, hyp=hyp, seg=seg, n_frames=T))
        return out

    def close(self):
        for o in (self.batch, self.ctx, self.model, self.fe):
            o.close()
