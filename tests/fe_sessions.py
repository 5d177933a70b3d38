"""TEST INFRASTRUCTURE: numpy restatement of the front-end options psb_fe_create_ex adds, on top of
oracle/fe_port.py (which covers one fresh, undithered utterance):
  - MT19937 (util/genrand.c) and the dither draw order of fe_process_frames + fe_end_utt
    (fe_interface.c:352-545, fe_sigproc.c:855-904);
  - cmn_live / cmn_live_shiftwin / cmn_live_update over a session (cmn_live.c, feat.c:917-938);
  - feat_s2_4x_cep2feat and feat_s3_1x39_cep2feat with replicated edges (feat.c:425-538).
Same float32 operations as the C code.  Pinned against the compiled reference by
tests/test_fe_sessions.py, and the device's output against it by tests/test_gpu_fe_sessions.py."""
import ctypes as C
import os

import numpy as np

from oracle import fe_port

F32 = np.float32
CMN_WIN, CMN_WIN_HWM = 500, 800
FEAT_DIM = {0: 39, 1: 51, 2: 39}


class MT19937:
    def __init__(self, seed=-1):
        mt = [0] * 624
        mt[0] = seed & 0xffffffff
        for i in range(1, 624):
            mt[i] = (1812433253 * (mt[i - 1] ^ (mt[i - 1] >> 30)) + i) & 0xffffffff
        self.mt, self.mti = mt, 624

    def _twist(self):
        mt = self.mt
        for kk in range(624):
            y = (mt[kk] & 0x80000000) | (mt[(kk + 1) % 624] & 0x7fffffff)
            mt[kk] = mt[(kk + 397) % 624] ^ (y >> 1) ^ (0x9908b0df if y & 1 else 0)
        self.mti = 0

    def int32(self):
        if self.mti >= 624:
            self._twist()
        y = self.mt[self.mti]
        self.mti += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9d2c5680
        y ^= (y << 15) & 0xefc60000
        y ^= y >> 18
        return y

    def int31(self):
        return self.int32() >> 1

    def dither_bits(self, n):
        return np.array([0 if self.int31() % 4 else 1 for _ in range(n)], np.int32)


def draw_plan(d, n):
    """(first sample of the last frame, full-frame draws, last-frame draws) of one n-sample utterance."""
    fs, sh = d["frame_size"], d["frame_shift"]
    if n <= 0:
        return 0, 0, 0
    full = 1 + (n - fs) // sh if n >= fs else 0
    main = fs + (full - 1) * sh if full else 0
    return full * sh, main, n - full * sh


def _wrap16(a):
    return ((a.astype(np.int32) + 32768) % 65536 - 32768).astype(np.int16)


def mfspec_dithered(d, pcm, rng):
    """fe_port.mfspec with dither: the full frames read sample i + draw i, the last frame its own fresh draws."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    n = len(pcm)
    t0, main, tail = draw_plan(d, n)
    dp = pcm.copy()
    dp[:main] = _wrap16(pcm[:main].astype(np.int32) + rng.dither_bits(main))
    tl = _wrap16(pcm[t0:t0 + tail].astype(np.int32) + rng.dither_bits(tail))
    T = fe_port.n_frames(d, n)
    if T == 0:
        return np.zeros((0, d["n_filt"]), np.float64)
    out = fe_port.mfspec(d, dp)
    # the last frame: its samples are the fresh copy, its pre-emphasis prior the full frames' sample before it
    last = np.concatenate([dp[:t0], tl])
    out[T - 1] = _last_frame(d, last, T - 1)
    return out


def _last_frame(d, pcm, k):
    x = fe_port._fft_real(d, fe_port._frame(d, pcm, k))
    N = d["fft_size"]
    spec = np.empty(N // 2 + 1, np.float64)
    spec[0] = x[0] * x[0]
    j = np.arange(1, N // 2 + 1)
    spec[1:] = x[j] * x[j] + x[N - j] * x[N - j]
    row = np.zeros(d["n_filt"], np.float64)
    for w in range(d["n_filt"]):
        acc = 0.0
        s0, f0 = int(d["spec_start"][w]), int(d["filt_start"][w])
        for i in range(int(d["filt_width"][w])):
            acc += spec[s0 + i] * float(d["filt_coeffs"][f0 + i])
        row[w] = acc
    return row


class CmnState:
    def __init__(self, cmn_init, nc=13):
        self.mean = np.asarray(cmn_init, np.float32)[:nc].copy()
        self.sum = (self.mean * F32(CMN_WIN)).astype(np.float32)
        self.nframe = CMN_WIN

    def utterance(self, cep):
        """cmn_live over one utterance's cepstra (returned normalised), then shiftwin / update."""
        cep = np.array(cep, np.float32, copy=True)
        for t in range(len(cep)):
            if cep[t, 0] < 0:
                continue
            self.sum = (self.sum + cep[t]).astype(np.float32)
            cep[t] = (cep[t] - self.mean).astype(np.float32)
            self.nframe += 1
        if self.nframe > CMN_WIN_HWM:
            sf = F32(1.0 / self.nframe)
            self.mean = (self.sum / F32(self.nframe)).astype(np.float32)
            self.sum = (self.sum * F32(F32(CMN_WIN) * sf)).astype(np.float32)
            self.nframe = CMN_WIN
        if self.nframe > 0:
            self.mean = (self.sum / F32(self.nframe)).astype(np.float32)
        return cep


def batch_cmn(cep):
    return fe_port.features(dict(cmn=1, window=3), cep)[1] if len(cep) else cep


def dyn_features(cep, feat):
    """cepstra after CMN [T][13] -> features [T][FEAT_DIM[feat]] (0 1s_c_d_dd, 1 s2_4x, 2 s3_1x39)."""
    T, nc = cep.shape
    if feat == 0:
        return fe_port.features(dict(cmn=0, window=3), cep)[0]
    idx = lambda t: min(max(t, 0), T - 1)
    out = np.zeros((T, FEAT_DIM[feat]), np.float32)
    for t in range(T):
        c = lambda k: cep[idx(t + k)]
        d2 = c(2) - c(-2)
        dd = (c(3) - c(-1)) - (c(1) - c(-3))
        if feat == 1:
            out[t, 0:12] = c(0)[1:]
            out[t, 12:24] = d2[1:]
            out[t, 24:36] = (c(4) - c(-4))[1:]
            out[t, 36:39] = (c(0)[0], d2[0], dd[0])
            out[t, 39:51] = dd[1:]
        else:
            out[t, 0:12] = c(0)[1:]
            out[t, 12:24] = d2[1:]
            out[t, 24:27] = (c(0)[0], d2[0], dd[0])
            out[t, 27:39] = dd[1:]
    return out


def session(d, opts, utterances, cmn_state=None, rng=None):
    """One session: utterances in decode order -> (list of features, list of cepstra after CMN, cmn, rng)."""
    if cmn_state is None:
        cmn_state = CmnState(opts["cmn_init"], d["n_cep"])
    if rng is None and opts["dither"]:
        rng = MT19937(opts["seed"])
    feats, ceps = [], []
    for pcm in utterances:
        mf = mfspec_dithered(d, pcm, rng) if opts["dither"] else fe_port.mfspec(d, np.ascontiguousarray(pcm, np.int16))
        cep = fe_port.cepstra(d, mf)
        cep = post_cepstra(opts, cep, cmn_state)
        feats.append(dyn_features(cep, opts["feat"]))
        ceps.append(cep)
    return feats, ceps, cmn_state, rng


def post_cepstra(opts, cep, cmn_state):
    if opts["cmn"] == 2:
        return cmn_state.utterance(cep)
    if opts["cmn"] == 1:
        return batch_cmn(cep)
    return cep


# ---- the compiled reference's own pieces, through ctypes (CPU pinning only) ----

class _Cmn(C.Structure):
    _fields_ = [("cmn_mean", C.POINTER(C.c_float)), ("cmn_var", C.POINTER(C.c_float)), ("sum", C.POINTER(C.c_float)),
                ("nframe", C.c_int32), ("veclen", C.c_int32), ("repr", C.c_char_p), ("refcount", C.c_int)]


def ref_lib():
    from oracle import refdrv
    L = refdrv.lib()
    L.genrand_seed.argtypes = [C.c_ulong]
    L.genrand_int31.restype = C.c_long
    L.cmn_init.restype = C.POINTER(_Cmn)
    L.cmn_init.argtypes = [C.c_int32]
    L.cmn_set_repr.argtypes = [C.POINTER(_Cmn), C.c_char_p]
    L.cmn_live.argtypes = [C.POINTER(_Cmn), C.c_void_p, C.c_int32, C.c_int32]
    L.cmn_live_update.argtypes = [C.POINTER(_Cmn)]
    L.cmn_free.argtypes = [C.POINTER(_Cmn)]
    return L


class RefCmn:
    """The reference's cmn_t, driven as feat_cmn (live, full utterance) and feat_update_stats drive it."""

    def __init__(self, cmninit, nc=13):
        self.L = ref_lib()
        self.c = self.L.cmn_init(nc)
        self.nc = nc
        self.L.cmn_set_repr(self.c, cmninit.encode())

    def utterance(self, cep):
        cep = np.array(cep, np.float32, copy=True)
        rows = (C.c_void_p * max(len(cep), 1))(*[cep[t].ctypes.data for t in range(len(cep))])
        self.L.cmn_live(self.c, rows, 0, len(cep))
        self.L.cmn_live_update(self.c)          # feat_cmn, endutt
        self.L.cmn_live_update(self.c)          # ps_end_utt -> feat_update_stats
        return cep

    def state(self):
        c = self.c.contents
        return (np.ctypeslib.as_array(c.cmn_mean, (self.nc,)).copy(), np.ctypeslib.as_array(c.sum, (self.nc,)).copy(),
                int(c.nframe))

    def close(self):
        self.L.cmn_free(self.c)


def ref_model_dir(name):
    from oracle import refdrv
    base = os.path.join(os.path.dirname(refdrv.LIB_PATH))
    return os.path.join(base, "model", {"tidigits": "tidigits_hmm", "en-us": "en-us", "an4": "an4_ci_cont"}[name])


def ref_session_decode(hmm, lm, dic, utterances, **feat_params):
    """One reference ps_decoder_t over several utterances (ps_start_stream, ps_start_utt, ps_process_raw(full_utt),
    ps_end_utt each); returns the hypotheses.  feat_params replace keys of the model's feat.params: ps_init parses
    that file after the caller's settings, so the overrides go into a copy of it."""
    import tempfile
    L = ref_lib()
    L.ps_config_init.restype = C.c_void_p
    L.ps_config_init.argtypes = [C.c_void_p]
    L.ps_config_set_str.restype = C.c_void_p
    L.ps_config_set_str.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    L.ps_init.restype = C.c_void_p
    L.ps_init.argtypes = [C.c_void_p]
    for f in ("ps_start_stream", "ps_start_utt", "ps_end_utt", "ps_free"):
        getattr(L, f).argtypes = [C.c_void_p]
    L.ps_config_free.argtypes = [C.c_void_p]
    L.ps_process_raw.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int]
    L.ps_get_hyp.restype = C.c_char_p
    L.ps_get_hyp.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
    params = {}
    for line in open(os.path.join(hmm, "feat.params")):
        parts = line.split()
        if len(parts) == 2:
            params[parts[0].lstrip("-")] = parts[1]
    params.update({k: str(v) for k, v in feat_params.items()})
    with tempfile.TemporaryDirectory() as tmp:
        fp = os.path.join(tmp, "feat.params")
        with open(fp, "w") as f:
            f.write("".join("-%s %s\n" % kv for kv in params.items()))
        cfg = L.ps_config_init(None)
        for k, v in (("hmm", hmm), ("lm", lm), ("dict", dic), ("featparams", fp)):
            L.ps_config_set_str(cfg, k.encode(), v.encode())
        ps = L.ps_init(cfg)
        assert ps, "ps_init failed"
        hyps = []
        for pcm in utterances:
            pcm = np.ascontiguousarray(pcm, np.int16)
            L.ps_start_stream(ps)
            L.ps_start_utt(ps)
            L.ps_process_raw(ps, pcm.ctypes.data, len(pcm), 0, 1)
            L.ps_end_utt(ps)
            score = C.c_int32()
            h = L.ps_get_hyp(ps, C.byref(score))
            hyps.append(h.decode() if h else "")
        L.ps_free(ps)
        L.ps_config_free(cfg)
    return hyps
