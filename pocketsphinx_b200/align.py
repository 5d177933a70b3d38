"""Forced alignment from audio for whole batches, as the reference's state_align_search reports it through
ps_alignment_t: words, phones and HMM states, each with start, duration, score and parent.

`Aligner` aligns audio to transcripts (ps_alignment_add_word without timing, ps_alignment_populate,
ps_set_alignment, one decode).  `Decoder(..., phone_align="yes" / state_align="yes")` runs the second pass of
`pocketsphinx single -phone_align yes` over its own word segments (ps_set_alignment(ps, NULL)) through
`align_batch` below.  Both build the phone chains on the host (dict2pid.alignment_phones) and run one
psb_align_batch_device call per batch (align_kernel, DESIGN 4.7); the word and phone levels are
ps_alignment_propagate restated on the host.
"""
import os
import re
from collections import namedtuple

import numpy as np

from . import api, dict2pid, lmio, s3io
from .decoder import acoustic_setup

INT_MAX = 2**31 - 1

# ps_alignment_iter_name / ps_alignment_iter_seg: name, start, duration, score; parent: the index of the entry one
# level up (ps_alignment_entry_t.parent; -1 for words)
Entry = namedtuple("Entry", "name start duration score parent")


def failure_reason(status):
    """The reference's error for an align_kernel status: None for 0 (state_align_search_finish, :225-235)."""
    if status == 0:
        return None
    if status == -1:
        return "Failed to reach final state in alignment"
    return "Alignment failed in frame %d" % (-2 - status)


def phone_windows(starts, durations, n_emit):
    """state_align_search_init (:455-478): each phone's (sf, ef) from the start and duration it took from its word in
    ps_alignment_populate.  A window shorter than the phone's emitting states (min_nframes) means always active, as
    does a start of 0 for sf."""
    st = np.asarray(starts, np.int64)
    du = np.asarray(durations, np.int64)
    ok = du >= n_emit
    sf = np.where((st > 0) & ok, st, 0).astype(np.int32)
    ef = np.where(ok, st + du, INT_MAX).astype(np.int32)
    return sf, ef


def token_band(sf, ef, n_frames, n_phones):
    """The phones that can hold a token in each frame (psb_hmm.cu: align_band): lo[f], the first phone with ef >= f
    (phone 0 in frame 0), and hi[f], the last phone i with sf[j] <= f + 1 for every 1 <= j <= i; hi < lo is an empty
    band.  Returns (lo, hi) int64 [n_frames]; align_kernel keeps (hi - lo + 1) x n_emit tokens in frame f."""
    f = np.arange(n_frames, dtype=np.int64)
    if n_phones == 0:
        return np.zeros(n_frames, np.int64), np.full(n_frames, -1, np.int64)
    if ef is None:
        lo = np.zeros(n_frames, np.int64)
    else:
        lo = np.searchsorted(np.maximum.accumulate(np.asarray(ef, np.int64)), f, side="left").astype(np.int64)
        lo[:1] = 0
    if sf is None:
        hi = np.full(n_frames, n_phones - 1, np.int64)
    else:
        s = np.asarray(sf, np.int64).copy()
        s[0] = np.iinfo(np.int64).min
        hi = np.searchsorted(np.maximum.accumulate(s), f + 1, side="right").astype(np.int64) - 1
    return lo, np.maximum(hi, lo - 1)


def band_tokens(sf, ef, n_frames, n_phones, n_emit):
    """Tokens align_kernel keeps for one utterance (each 8 bytes: id and score)."""
    lo, hi = token_band(sf, ef, n_frames, n_phones)
    return int(((hi - lo + 1) * n_emit).sum())


class Alignment:
    """One utterance's alignment: `words`, `phones`, `states`, lists of Entry.  Word names are the dictionary's
    (dict_wordstr, alternates as "word(2)"), phone names the CI phones', state names the senone ids in decimal, as
    ps_alignment_iter_name gives them; start / duration in frames and score as ps_alignment_iter_seg gives them."""

    def __init__(self, words, phones, states):
        self.words, self.phones, self.states = words, phones, states

    def children(self, level, i):
        """ps_alignment_iter_children: the phones of word i (level "word") or the states of phone i ("phone")."""
        sub = {"word": self.phones, "phone": self.states}[level]
        return [e for e in sub if e.parent == i]

    def __repr__(self):
        return "Alignment(%s)" % " ".join("%s:%d+%d" % (w.name, w.start, w.duration) for w in self.words)


def propagate(word_names, word_start, word_dur, phone_names, phone_word, state_names, n_emit, st_start, st_dur,
              st_score):
    """The alignment after state_align_search_finish: states the backtrace visited (st_start >= 0) take its start,
    duration and score; the others keep what ps_alignment_populate gave them (their word's start and duration, score
    0).  State 0's score is never set by the backtrace (0).  Then ps_alignment_propagate (ps_alignment.c:315-350):
    each phone starts at its first state and sums its states' durations and scores, each word likewise over its
    phones."""
    n_ph = len(phone_names)
    ps_ = np.asarray(word_start, np.int64)[phone_word]
    pd_ = np.asarray(word_dur, np.int64)[phone_word]
    st_start, st_dur, st_score = (np.asarray(a, np.int64) for a in (st_start, st_dur, st_score))
    seen = st_start >= 0
    s_start = np.where(seen, st_start, np.repeat(ps_, n_emit))
    s_dur = np.where(seen, st_dur, np.repeat(pd_, n_emit))
    s_score = np.where(seen, st_score, 0)
    states = [Entry(state_names[k], int(s_start[k]), int(s_dur[k]), int(s_score[k]), k // n_emit)
              for k in range(n_ph * n_emit)]
    p_dur = s_dur.reshape(n_ph, n_emit).sum(1)
    p_score = s_score.reshape(n_ph, n_emit).sum(1)
    phones = [Entry(phone_names[i], int(s_start[i * n_emit]), int(p_dur[i]), int(p_score[i]), int(phone_word[i]))
              for i in range(n_ph)]
    words = []
    for w in range(len(word_names)):
        mine = [p for p in phones if p.parent == w]
        words.append(Entry(word_names[w], mine[0].start, sum(p.duration for p in mine), sum(p.score for p in mine), -1))
    return Alignment(words, phones, states)


class AlignTables:
    """The dictionary and context tables ps_alignment_populate reads: the model's mdef, the dictionary and filler
    dictionary in the reference's word-id order (lmio.read_dict, as the Decoder reads them), dict2pid's tables."""

    def __init__(self, hmm, dict_file, filler_dict=None):
        self.md = s3io.read_mdef(os.path.join(hmm, "mdef"))
        if filler_dict is None:
            nd = os.path.join(hmm, "noisedict")
            filler_dict = nd if os.path.exists(nd) else None
        self.words, prons, _, _ = lmio.read_dict(dict_file, filler_dict, self.md["ciname"])
        ci = {n: i for i, n in enumerate(self.md["ciname"])}
        self.prons = [[ci[x] for x in p] for p in prons]
        self.wid = {w: i for i, w in enumerate(self.words)}
        self.tabs = dict2pid.build(self.md, self.prons)
        self.n_emit = self.md["n_emit_state"]

    def lookup(self, text):
        """str2words + dict_wordid: whitespace-separated words, each the dictionary's exactly (fillers included).
        An unknown word raises ValueError naming it."""
        out = []
        for w in re.split(r"[ \t\n\v\f\r]+", text):
            if not w:
                continue
            if w not in self.wid:
                raise ValueError("word %r is not in the dictionary" % w)
            out.append(self.wid[w])
        return out

    def chain(self, wids):
        """ps_alignment_populate: (ssid, tmatid, cipid, word index) per phone."""
        ssid, tmat, cipid = dict2pid.alignment_phones(self.md, self.prons, self.tabs, wids)
        word = np.repeat(np.arange(len(wids)), [len(self.prons[w]) for w in wids])
        return ssid, tmat, cipid, word


def align_batch(ctx, tables, d_senscr, frame_off, chains, windows=None):
    """One psb_align_batch_device call for a batch.  chains: per utterance (wids, word_start, word_dur) or None (no
    alignment: no phones); windows: apply state_align_search_init's per-phone windows from the words' timing (the
    second pass) or not (transcripts: every phone always active).  Returns per utterance (Alignment or None, reason)
    and the token arena's bytes."""
    n = len(chains)
    md, sseq = tables.md, tables.md["sseq"]
    ph_off, ssid, tmat, sfs, efs, built = [0], [], [], [], [], []
    for c in chains:
        if c is None:
            built.append(None)
            ph_off.append(ph_off[-1])
            continue
        wids, w_st, w_du = c
        s, t, ci, word = tables.chain(wids)
        built.append((wids, w_st, w_du, ci, word, s))
        ssid.append(s); tmat.append(t)
        if windows:
            sf, ef = phone_windows(np.asarray(w_st)[word], np.asarray(w_du)[word], tables.n_emit)
        else:
            sf, ef = np.zeros(len(s), np.int32), np.full(len(s), INT_MAX, np.int32)
        sfs.append(sf); efs.append(ef)
        ph_off.append(ph_off[-1] + len(s))
    cat = lambda a: np.concatenate(a).astype(np.int32) if a else np.zeros(0, np.int32)
    status, st, du, sc = ctx.align(None, np.ascontiguousarray(frame_off, np.int32), np.array(ph_off, np.int32), cat(ssid),
                                   cat(tmat), cat(sfs), cat(efs), device_ptr=d_senscr)
    N = tables.n_emit
    out = []
    for u in range(n):
        b = built[u]
        if b is None:
            out.append((None, "no words to align"))
            continue
        reason = failure_reason(int(status[u]))
        if reason is not None:
            out.append((None, reason))
            continue
        wids, w_st, w_du, ci, word, s = b
        a, z = ph_off[u] * N, ph_off[u + 1] * N
        out.append((propagate([tables.words[w] for w in wids], w_st, w_du, [md["ciname"][c] for c in ci], word,
                              [str(int(x)) for x in sseq[s].reshape(-1)], N, st[a:z], du[a:z], sc[a:z]), None))
    return out, int(api.lib().psb_align_last_token_bytes(ctx.h))


class Aligner:
    """Forced alignment of audio to transcripts for batches of utterances, configured like the reference's
    ps_decoder_t (-hmm, -dict, -fdict as filler_dict, and every model and front-end setting the Decoder takes, by the
    reference's names).  Each utterance is aligned by a fresh decoder, as a program calling ps_set_alignment with an
    untimed word list and decoding once.  max_utts / max_frames bound one batch (frames summed over its
    utterances)."""

    def __init__(self, hmm, dict_file, max_utts=64, max_frames=1 << 16, device=0, filler_dict=None, **config):
        cfg = {k: str(v) for k, v in config.items()}
        self.pm, self.fe, _ = acoustic_setup(hmm, cfg, device)
        self.tables = AlignTables(hmm, dict_file, filler_dict)
        self.model = api.Model(self.pm, device)
        self.batch = api.Batch(self.model, max_utts, max_frames)
        self.ctx = api.HmmContext(self.pm.tp, self.pm.sseq, self.pm.n_sen, device=device)
        self.max_utts, self.max_frames = max_utts, max_frames
        self.reasons = []
        self.last_token_bytes = 0

    def align_raw_batch(self, utterances, texts):
        """utterances: int16 arrays, each a whole utterance; texts: one transcript per utterance (dictionary words
        separated by whitespace, fillers such as <sil>, <s>, </s> included).  Returns one Alignment per utterance, or
        None where the reference's search fails; `reasons` then holds its error for each utterance (None where it
        aligned).  An unknown word raises ValueError before anything runs on the device."""
        if len(texts) != len(utterances):
            raise ValueError("%d transcripts for %d utterances" % (len(texts), len(utterances)))
        wids = [self.tables.lookup(t) for t in texts]
        lens = [len(u) for u in utterances]
        frames = [self.fe.n_frames(n) for n in lens]
        if len(utterances) > self.max_utts:
            raise ValueError("%d utterances, more than this Aligner's max_utts (%d)" % (len(utterances), self.max_utts))
        if sum(frames) > self.max_frames:
            raise ValueError("%d frames in this batch, more than this Aligner's max_frames (%d): create it with a larger "
                             "max_frames" % (sum(frames), self.max_frames))
        pcm = np.concatenate([np.ascontiguousarray(u, np.int16) for u in utterances]) if utterances else np.zeros(0, np.int16)
        frame_off = self.batch.score_pcm(self.fe, pcm, api.FrontEnd.sample_offsets(lens))
        return self._align(self.batch.senscr_device_ptr(), frame_off, wids)

    def align_senscr(self, d_senscr_ptr, frame_off, texts):
        """align_raw_batch from senone scores already on the device (int16 [frames][n_sen], every senone), utterance
        u at frames frame_off[u] .. frame_off[u+1]."""
        if len(texts) != len(frame_off) - 1:
            raise ValueError("%d transcripts for %d utterances" % (len(texts), len(frame_off) - 1))
        return self._align(d_senscr_ptr, frame_off, [self.tables.lookup(t) for t in texts])

    def _align(self, d_senscr_ptr, frame_off, wids):
        # ps_alignment_add_word(al, wid, 0, 0): every phone always active
        chains = [(w, np.zeros(len(w), np.int64), np.zeros(len(w), np.int64)) if w else None for w in wids]
        res, self.last_token_bytes = align_batch(self.ctx, self.tables, d_senscr_ptr, frame_off, chains)
        self.reasons = [r for _, r in res]
        return [a for a, _ in res]

    def close(self):
        for o in (self.batch, self.ctx, self.model, self.fe):
            o.close()
