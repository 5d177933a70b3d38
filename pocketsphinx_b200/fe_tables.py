"""Host-side mirror of the reference front end's INITIALISATION (fe_init, fe_create_hamming,
fe_create_twiddle, fe_build_melfilters, fe_compute_melcosine: src/fe/fe_interface.c:60-300,
src/fe/fe_sigproc.c:552-724, 774-934): the tables psb_fe_create takes are the arrays the
reference's own fe_t holds (a C host passes those), and this module rebuilds them for Python
hosts with the same float32 / float64 / libm steps.  tests/test_fe_tables.py pins every array
bit for bit against the compiled reference.  No per-frame arithmetic lives here."""
import math

import numpy as np

F32 = np.float32
TRANSFORMS = {"legacy": 0, "dct": 1, "htk": 2}       # fe_internal.h: LEGACY_DCT, DCT_II, DCT_HTK
CMN_TYPES = {"none": 0, "batch": 1, "current": 1, "live": 2}   # feat/cmn.h: CMN_NONE, CMN_BATCH, CMN_LIVE (cmn_type_str)
FEAT_TYPES = {"1s_c_d_dd": 0, "s2_4x": 1, "s3_1x39": 2, "1s_12c_12d_3p_12dd": 2}   # psb200.h: PSB_FEAT_*
AGC_TYPES = {"none": 0, "max": 1, "emax": 2, "noise": 3}          # feat/agc.h: agc_type_str, psb200.h: PSB_AGC_*


def _mel(x):
    # fe_mel (fe_sigproc.c:536-542), neutral warping
    return F32(2595.0 * math.log10(1.0 + float(F32(x)) / 700.0))


def _melinv(x):
    # fe_melinv (fe_sigproc.c:544-549)
    return F32(700.0 * (math.pow(10.0, float(F32(x)) / 2595.0) - 1.0))


def make_fe_desc(samprate=16000.0, frate=100, wlen=0.025625, nfft=0, nfilt=25, lowerf=130.0, upperf=6800.0,
                 ncep=13, alpha=0.97, transform="dct", lifter=22, remove_noise=True, remove_dc=False,
                 unit_area=True, round_filters=True, doublebw=False, cmn="batch", window=3):
    """Defaults = model/en-us/en-us/feat.params on top of config_macro.h."""
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
    # fe_build_melfilters (:552-683), float32 throughout
    melmin, melmax = _mel(lowerf), _mel(upperf)
    melbw = F32(melmax - melmin) / F32(nfilt + 1)
    if doublebw:
        melmin = F32(melmin - melbw)
        melmax = F32(melmax + melbw)
    fftfreq = sr / F32(size)

    def edges(i):
        fr = []
        for j in range(3):
            k = (i + j * 2) if doublebw else (i + j)
            f = _melinv(F32(F32(k) * melbw) + melmin)
            if round_filters:
                f = F32(int(float(F32(f / fftfreq)) + 0.5)) * fftfreq
            fr.append(F32(f))
        return fr

    spec_start, filt_start, filt_width, coeffs = [], [], [], []
    for i in range(nfilt):
        fr = edges(i)
        start = -1
        width = None
        for j in range(size // 2 + 1):
            hz = F32(j) * fftfreq
            if hz < fr[0]:
                continue
            elif hz > fr[2] or j == size // 2:
                width = j - start
                break
            if start == -1:
                start = j
        assert width is not None and start >= 0
        spec_start.append(start); filt_start.append(len(coeffs)); filt_width.append(width)
        for j in range(width):
            hz = F32(start + j) * fftfreq
            assert fr[0] <= hz <= fr[2]
            lo = F32(hz - fr[0]) / F32(fr[1] - fr[0])
            hi = F32(fr[2] - hz) / F32(fr[2] - fr[1])
            if unit_area:
                s = F32(2) / F32(fr[2] - fr[0])
                lo = F32(lo * s)
                hi = F32(hi * s)
            coeffs.append(lo if lo < hi else hi)
    d["spec_start"] = np.array(spec_start, np.int16)
    d["filt_start"] = np.array(filt_start, np.int16)
    d["filt_width"] = np.array(filt_width, np.int16)
    d["filt_coeffs"] = np.array(coeffs, np.float32)
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
