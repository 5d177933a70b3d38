"""Host-side mirror of the reference front end's INITIALISATION (fe_init, fe_create_hamming,
fe_create_twiddle, fe_build_melfilters, fe_compute_melcosine: src/fe/fe_interface.c:60-300,
src/fe/fe_sigproc.c:552-724, 774-934): the tables psb_fe_create takes are the arrays the
reference's own fe_t holds (a C host passes those), and this module rebuilds them for Python
hosts with the same float32 / float64 / libm steps.  tests/test_fe_tables.py pins every array
bit for bit against the compiled reference.  No per-frame arithmetic lives here."""
import math
import re
import warnings

import numpy as np

F32 = np.float32
TRANSFORMS = {"legacy": 0, "dct": 1, "htk": 2}       # fe_internal.h: LEGACY_DCT, DCT_II, DCT_HTK
CMN_TYPES = {"none": 0, "batch": 1, "current": 1, "live": 2}   # feat/cmn.h: CMN_NONE, CMN_BATCH, CMN_LIVE (cmn_type_str)
FEAT_TYPES = {"1s_c_d_dd": 0, "s2_4x": 1, "s3_1x39": 2, "1s_12c_12d_3p_12dd": 2}   # psb200.h: PSB_FEAT_*
AGC_TYPES = {"none": 0, "max": 1, "emax": 2, "noise": 3}          # feat/agc.h: agc_type_str, psb200.h: PSB_AGC_*


WARP_TYPES = ("inverse_linear", "affine", "piecewise_linear")   # fe_warp.c name2id
_WARP_ALIASES = ("inverse", "linear", "piecewise")              # fe_warp.c __name2id: the same ids, in order
_STRTOD = re.compile(r"[+-]?(\d+\.?\d*|\.\d+)([eE][+-]?\d+)?")


def _atof_c(tok):
    # atof_c: the longest decimal prefix, 0 without one
    m = _STRTOD.match(tok)
    return float(m.group(0)) if m else 0.0


class Warp:
    """One frequency warp as fe_warp_set + fe_warp_set_parameters leave it (fe_warp*.c, float32 throughout) when
    the parameter string is newly set: the reference keeps the parameters in process-global statics and skips a
    string equal to the last one set, which this class does not reproduce (DESIGN 4.6).  params None or "" is
    unset: neutral, as is a slope of 0 (which the clamp to [0.1, 10] never leaves)."""

    def __init__(self, warp_type="inverse_linear", params=None, samprate=16000.0):
        if warp_type in WARP_TYPES:
            self.kind = WARP_TYPES.index(warp_type)
        elif warp_type in _WARP_ALIASES:
            self.kind = _WARP_ALIASES.index(warp_type)
        else:
            raise ValueError("unimplemented warping function %r (implemented: %s)" % (warp_type, ", ".join(WARP_TYPES)))
        sr = F32(samprate)
        self.nyquist = nyq = F32(sr / F32(2))
        self.neutral = params is None or params == ""
        if self.neutral:
            return
        n_param = 1 if self.kind == 0 else 2
        p = [F32(0)] * 2
        toks = [t for t in re.split("[ \t]", params[:255]) if t]          # strtok(" \t") on a 256-byte copy
        for i, t in enumerate(toks[:n_param]):
            p[i] = F32(_atof_c(t))
        if p[0] < F32(0.1):
            p[0] = F32(0.1)
        elif p[0] > F32(10.0):
            p[0] = F32(10.0)
        self.final = [F32(0), F32(0)]
        if self.kind == 1:                                          # affine: b in [-nyquist, nyquist]
            if p[1] < -nyq:
                p[1] = -nyq
            elif p[1] > nyq:
                p[1] = nyq
        elif self.kind == 2:                                        # piecewise: F in [0, nyquist]
            if p[1] < 0:
                p[1] = F32(0)
            elif p[1] > nyq:
                p[1] = nyq
            if p[1] < sr:
                if p[1] == 0:
                    p[1] = F32(sr * F32(0.85))
                a, f = p
                with np.errstate(all="ignore"):                     # F at Nyquist: inf / NaN, as in C
                    self.final = [F32(F32(nyq - F32(a * f)) / F32(nyq - f)),
                                  F32(F32(F32(nyq * f) * F32(a - F32(1))) / F32(nyq - f))]
        self.a, self.b = p
        if self.a == 0:
            self.neutral = True

    def to_warped(self, x):
        # *_unwarped_to_warped
        x = F32(x)
        if self.neutral:
            return x
        if self.kind == 0:
            return F32(x / self.a)
        if self.kind == 1:
            return F32(F32(x * self.a) + self.b)
        with np.errstate(all="ignore"):
            return F32(x * self.a) if x < self.b else F32(F32(self.final[0] * x) + self.final[1])

    def to_unwarped(self, x):
        # *_warped_to_unwarped
        x = F32(x)
        if self.neutral:
            return x
        if self.kind == 0:
            return F32(x * self.a)
        if self.kind == 1:
            return F32(F32(x - self.b) / self.a)
        if x < F32(self.a * self.b):
            return F32(x / self.a)
        with np.errstate(all="ignore"):
            return F32(F32(x - self.final[1]) / self.final[0])


def _c_int(x):
    # (int) of a double on x86-64 (cvttsd2si): NaN and values out of int32 range give INT_MIN
    return int(x) if -2147483649.0 < x < 2147483648.0 else -(1 << 31)


def _mel(x, warp=None):
    # fe_mel (fe_sigproc.c:536-542); a warp can take log10 below 0, where C's log10 gives -inf / NaN
    w = F32(x) if warp is None else warp.to_warped(x)
    v = 1.0 + float(w) / 700.0
    # glibc: log10(NaN) is that NaN, log10(0) -inf, log10(x < 0) the default NaN of x86 (sign bit set)
    return F32(2595.0 * (math.log10(v) if v > 0 or v != v else -math.inf if v == 0 else -math.nan))


def _melinv(x, warp=None):
    # fe_melinv (fe_sigproc.c:544-549); pow overflows to inf as in C
    try:
        p = math.pow(10.0, float(F32(x)) / 2595.0)
    except OverflowError:
        p = math.inf
    w = F32(700.0 * (p - 1.0))
    return w if warp is None else warp.to_unwarped(w)


def make_filterbank(samprate=16000.0, fft_size=512, nfilt=25, lowerf=130.0, upperf=6800.0, unit_area=True,
                    round_filters=True, doublebw=False, warp_type="inverse_linear", warp_params=None):
    """fe_build_melfilters (fe_sigproc.c:552-683) under a warp, float32 throughout: dict of spec_start, filt_start,
    filt_width (int16 [nfilt]) and filt_coeffs (float32).  A filter no DFT point falls in keeps what calloc left:
    spec_start -1, filt_start 0, filt_width 0.  With doublebw and an outer edge outside [0, Nyquist] every filter is
    empty at spec_start 0 (fe_init ignores the builder's error), with a warning.  NaN edges (a piecewise F clamped to
    Nyquist divides by zero) pass the reference's range tests and give its NaN-filled bank.  Where the reference's
    process ends (E_FATAL: a filter its own coefficient pass rejects) this raises ValueError."""
    sr = F32(samprate)
    warp = Warp(warp_type, warp_params, samprate)
    melmin, melmax = _mel(lowerf, warp), _mel(upperf, warp)
    melbw = F32(melmax - melmin) / F32(nfilt + 1)
    if doublebw:
        melmin = F32(melmin - melbw)
        melmax = F32(melmax + melbw)
        lo, hi = _melinv(melmin, warp), _melinv(melmax, warp)
        if lo < 0 or hi > F32(sr / F32(2)):
            # fe_build_melfilters returns FE_INVALID_PARAM_ERROR here, which fe_init ignores: the bank is what
            # calloc left, every filter empty at spec_start 0, and every mel energy is 0
            warnings.warn("doublebw filter edges %g .. %g Hz outside 0 .. %g Hz: every mel filter is empty, as in the "
                          "reference" % (lo, hi, sr / 2))
            z = np.zeros(nfilt, np.int16)
            return dict(spec_start=z, filt_start=z.copy(), filt_width=z.copy(), filt_coeffs=np.zeros(0, np.float32))
    fftfreq = sr / F32(fft_size)

    def edges(i):
        fr = []
        for j in range(3):
            k = (i + j * 2) if doublebw else (i + j)
            f = _melinv(F32(F32(k) * melbw) + melmin, warp)
            if round_filters:
                f = F32(_c_int(float(F32(f / fftfreq)) + 0.5)) * fftfreq
            fr.append(F32(f))
        return fr

    spec_start, filt_start, filt_width, coeffs = [], [], [], []
    for i in range(nfilt):
        fr = edges(i)
        start, width, fstart = -1, 0, 0
        for j in range(fft_size // 2 + 1):
            hz = F32(j) * fftfreq
            if hz < fr[0]:
                continue
            elif hz > fr[2] or j == fft_size // 2:
                width = j - start
                fstart = len(coeffs)
                break
            if start == -1:
                start = j
        spec_start.append(start); filt_start.append(fstart); filt_width.append(width)
        for j in range(width):
            hz = F32(start + j) * fftfreq
            if hz < fr[0] or hz > fr[2]:                             # a NaN edge passes, as in C
                raise ValueError("filter %d: frequency %g Hz outside %g .. %g Hz (fe_build_melfilters: range does not "
                                 "match)" % (i, hz, fr[0], fr[2]))
            lo = F32(hz - fr[0]) / F32(fr[1] - fr[0])
            hi = F32(fr[2] - hz) / F32(fr[2] - fr[1])
            if unit_area:
                s = F32(2) / F32(fr[2] - fr[0])
                lo = F32(lo * s)
                hi = F32(hi * s)
            coeffs.append(lo if lo < hi else hi)
    return dict(spec_start=np.array(spec_start, np.int16), filt_start=np.array(filt_start, np.int16),
                filt_width=np.array(filt_width, np.int16), filt_coeffs=np.array(coeffs, np.float32))


def make_fe_desc(samprate=16000.0, frate=100, wlen=0.025625, nfft=0, nfilt=25, lowerf=130.0, upperf=6800.0,
                 ncep=13, alpha=0.97, transform="dct", lifter=22, remove_noise=True, remove_dc=False,
                 unit_area=True, round_filters=True, doublebw=False, cmn="batch", window=3,
                 warp_type="inverse_linear", warp_params=None):
    """Defaults = model/en-us/en-us/feat.params on top of config_macro.h.  warp_type / warp_params: -warp_type and
    -warp_params (Warp); the filter bank is the warped one.  desc["bank_args"] holds make_filterbank's arguments, so
    the same front end can build banks under other warps (api.FrontEnd.set_filterbanks)."""
    sr = F32(samprate)
    frame_shift = int(float(sr / F32(frate)) + 0.5)                   # fe_interface.c:234
    frame_size = int(float(F32(wlen) * sr) + 0.5)                     # :235
    if nfft == 0:                                                     # :101-108
        order, size = 0, 1
        while size < frame_size:
            order += 1
            size <<= 1
    else:
        size, order = nfft, int(math.log2(nfft))
        assert 1 << order == size and size >= frame_size
    d = dict(frame_size=frame_size, frame_shift=frame_shift, fft_size=size, fft_order=order, n_filt=nfilt,
             n_cep=ncep, remove_dc=int(remove_dc), remove_noise=int(remove_noise),
             transform=TRANSFORMS[transform], lifter_val=int(lifter), window=window, cmn=CMN_TYPES[cmn],
             alpha=F32(alpha), sampling_rate=float(sr))
    # fe_create_hamming (:774-789): first half, float64
    d["hamming"] = np.array([0.54 - 0.46 * math.cos(2 * math.pi * i / (float(frame_size) - 1.0))
                             for i in range(frame_size // 2)], np.float64)
    # fe_create_twiddle (:916-934)
    d["ccc"] = np.array([math.cos(2 * math.pi * i / size) for i in range(size // 4)], np.float64)
    d["sss"] = np.array([math.sin(2 * math.pi * i / size) for i in range(size // 4)], np.float64)
    # fe_warp_set + fe_warp_set_parameters (fe_interface.c:166-177), then fe_build_melfilters (:552-683)
    d["warp_type"], d["warp_params"] = warp_type, warp_params
    d["bank_args"] = dict(samprate=float(sr), fft_size=size, nfilt=nfilt, lowerf=lowerf, upperf=upperf,
                          unit_area=unit_area, round_filters=round_filters, doublebw=doublebw)
    d.update(make_filterbank(warp_type=warp_type, warp_params=warp_params, **d["bank_args"]))
    # fe_compute_melcosine (:686-724)
    freqstep = math.pi / nfilt
    d["mel_cosine"] = np.array([[math.cos(freqstep * i * (j + 0.5)) for j in range(nfilt)] for i in range(ncep)],
                               np.float64).astype(np.float32)
    d["sqrt_inv_n"] = F32(math.sqrt(1.0 / nfilt))
    d["sqrt_inv_2n"] = F32(math.sqrt(2.0 / nfilt))
    if lifter:
        d["lifter"] = np.array([1 + (lifter // 2) * math.sin(i * math.pi / lifter) for i in range(ncep)],
                               np.float64).astype(np.float32)
    else:
        d["lifter"] = np.zeros(0, np.float32)
    return d


def make_fe_opts(feat="1s_c_d_dd", cmn="live", cmninit="40,3,-1", varnorm=False, dither=False, seed=-1, ncep=13,
                 agc="none", agcthresh=2.0, lda=None, ldadim=0):
    """psb_fe_opts_t from the feat.params / command-line keys -feat, -cmn, -cmninit, -varnorm, -dither, -seed,
    -agc, -agcthresh and -ldadim; the defaults are config_macro.h's.  cmn_init is what cmn_set_repr
    (cmn.c:119-146) parses out of -cmninit: up to ncep comma-separated values, the rest 0.  lda: None or the
    transform matrix [m][n] (s3io.read_lda(path)[0])."""
    init = np.zeros(32, np.float32)
    vals = cmninit.split(",") if cmninit else []
    for i, v in enumerate(vals[:ncep]):
        if v != "":
            init[i] = F32(float(v))
    return dict(feat=FEAT_TYPES[feat], cmn=CMN_TYPES[cmn], varnorm=int(bool(varnorm)), dither=int(bool(dither)),
                seed=int(seed), cmn_init=init, agc=AGC_TYPES[agc], agc_thresh=F32(agcthresh),
                lda=None if lda is None else np.ascontiguousarray(lda, np.float32), ldadim=int(ldadim))


def n_frames(desc, n_samples):
    """Frames of one utterance: fe_process_frames + fe_end_utt (fe_interface.c:352-520)."""
    if n_samples <= 0:
        return 0
    full = 1 + (n_samples - desc["frame_size"]) // desc["frame_shift"] if n_samples >= desc["frame_size"] else 0
    return full + 1
