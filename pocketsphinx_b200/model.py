"""Packed acoustic model: the flat arrays the C-ABI (include/psb200.h) takes.

This is host-side data plumbing only (no arithmetic from the hot path lives here).  Arrays are
in the reference's in-memory order after its loaders ran (ms_gauden.c:264-308 precompute,
ptm_mgau.c:457-661 sendump, tmat.c:215-236, bin_mdef.h:121-147):

  mean, var   float32 [n_mgau][n_feat][n_density][featlen[f]]  (var = precomputed 1/(2s^2) in log units)
  det         float32 [n_mgau][n_feat][n_density]
  mixw        uint8   ptm/semi: [n_feat][n_density][row], row = n_sen (8 bit) or (n_sen+1)//2 (4 bit)
                      ms: pdf[sen][feat][cw] (n_mgau>1) or pdf[feat][cw][sen] (n_mgau==1)
  mixw_cb     uint8   [16] when the sendump is 4-bit clustered, else empty
  sen2cb      int32   [n_sen]
  logadd8     uint8   [256] add table of logmath_init(base, 10, 1)
  tp          uint8   [n_tmat][n_emit][n_emit+1]; sseq uint16 [n_sseq][n_emit]
"""
from dataclasses import dataclass, field

import numpy as np

KINDS = ("ptm", "s2_semi", "ms")


@dataclass
class PackedModel:
    kind: str
    n_sen: int
    n_mgau: int
    n_feat: int
    n_density: int
    topn: int
    featlen: np.ndarray
    mean: np.ndarray
    var: np.ndarray
    det: np.ndarray
    mixw: np.ndarray
    sen2cb: np.ndarray
    logadd8: np.ndarray
    mixw_cb: np.ndarray = field(default_factory=lambda: np.zeros(0, np.uint8))
    n_emit_state: int = 3
    tp: np.ndarray = field(default_factory=lambda: np.zeros((0, 3, 4), np.uint8))
    sseq: np.ndarray = field(default_factory=lambda: np.zeros((0, 3), np.uint16))
    phone_ssid: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    phone_tmat: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    n_ciphone: int = 0
    n_ci_sen: int = 0
    ds_ratio: int = 1
    aw: int = 1
    logadd_ms: np.ndarray = field(default_factory=lambda: np.zeros(0, np.uint32))
    logadd_ms_zero: int = 0
    topn_beam: np.ndarray = field(default_factory=lambda: np.zeros(0, np.uint8))

    def __post_init__(self):
        assert self.kind in KINDS
        self.featlen = np.ascontiguousarray(self.featlen, np.int32)
        self.mean = np.ascontiguousarray(self.mean, np.float32).ravel()
        self.var = np.ascontiguousarray(self.var, np.float32).ravel()
        self.det = np.ascontiguousarray(self.det, np.float32).ravel()
        self.mixw = np.ascontiguousarray(self.mixw, np.uint8).ravel()
        self.mixw_cb = np.ascontiguousarray(self.mixw_cb, np.uint8).ravel()
        self.sen2cb = np.ascontiguousarray(self.sen2cb, np.int32).ravel()
        self.logadd8 = np.ascontiguousarray(self.logadd8, np.uint8).ravel()
        self.tp = np.ascontiguousarray(self.tp, np.uint8)
        self.sseq = np.ascontiguousarray(self.sseq, np.uint16)
        self.phone_ssid = np.ascontiguousarray(self.phone_ssid, np.int32)
        self.phone_tmat = np.ascontiguousarray(self.phone_tmat, np.int32)
        self.logadd_ms = np.ascontiguousarray(self.logadd_ms, np.uint32).ravel()
        self.topn_beam = np.ascontiguousarray(self.topn_beam, np.uint8).ravel()
        n = self.n_mgau * self.n_density * self.sumlen
        assert self.mean.size == n and self.var.size == n, (self.mean.size, n)
        assert self.det.size == self.n_mgau * self.n_feat * self.n_density
        assert self.sen2cb.size == self.n_sen
        assert len(self.featlen) == self.n_feat

    @property
    def sumlen(self):
        return int(np.sum(self.featlen))

    @property
    def mixw_4bit(self):
        return self.mixw_cb.size == 16

    @property
    def mixw_row(self):
        return (self.n_sen + 1) // 2 if self.mixw_4bit else self.n_sen

    def to_npz_dict(self):
        d = {}
        for k, v in self.__dict__.items():
            d[k] = np.array(v) if not isinstance(v, np.ndarray) else v
        return d

    def save(self, path):
        np.savez_compressed(path, **self.to_npz_dict())

    @classmethod
    def from_dict(cls, d):
        kw = {}
        for k in cls.__dataclass_fields__:
            if k not in d:
                continue
            v = d[k]
            if isinstance(v, np.ndarray) and v.ndim == 0:
                v = v.item()
            if k == "kind":
                v = str(v)
            kw[k] = v
        return cls(**kw)

    @classmethod
    def from_dir(cls, path, **config):
        """An acoustic-model directory as the reference ships them (s3io.read_model_dir: mdef, means,
        variances, transition_matrices, sendump / mixture_weights, feat.params), loaded without the reference."""
        from . import s3io
        return cls.from_dict(s3io.read_model_dir(path, **config))

    @classmethod
    def load(cls, path):
        return cls.from_dict(load_npz(path))


class NpzArrays(dict):
    """The arrays of an .npz file by name; `.files` lists the names like np.load's result."""

    @property
    def files(self):
        return list(self)


def load_npz(path):
    """All arrays of `path`.  A large file is stored in parts (name.npz, name.part1.npz, ...) so that each part stays
    under 1 MB: an array found in several parts is their concatenation along axis 0, in part order."""
    import glob
    import re
    stem = path[:-len(".npz")]
    parts = sorted(glob.glob(glob.escape(stem) + ".part*.npz"), key=lambda p: int(re.search(r"\.part(\d+)\.npz$", p).group(1)))
    out = NpzArrays()
    for p in [path] + parts:
        with np.load(p, allow_pickle=False) as z:
            for k in z.files:
                out[k] = np.concatenate([out[k], z[k]]) if k in out else z[k]
    return out


def make_logadd8(base=1.0001, shift=10):
    """The 8-bit add table of logmath_init(base, 10, TRUE) (util/logmath.c:63-162): entry i is
    round(log_base(1 + base^-(i<<shift))) >> shift, first writer wins, at least 256 entries.
    Uses float64 like the reference; validated against the reference table in tests."""
    import math
    inv = 1.0 / math.log(base)
    table = np.zeros(256, np.uint8)
    byx = 1.0
    i = 0
    while True:
        lobyx = math.log(1.0 + byx) * inv
        k = int(lobyx + 0.5 * (1 << shift)) >> shift
        idx = i >> shift
        if idx < 256 and table[idx] == 0:
            table[idx] = k & 0xff
        if k <= 0:
            break
        byx /= base
        i += 1
    return table


SEN2CB_LAYOUTS = ("cuts", "small", "single", "identity")


def _ptm_sen2cb(rng, layout, n_sen, n_mgau, n_ci, n_emit_state):
    """The senone -> codebook map of synth_ptm (see there)."""
    if layout == "cuts":
        sen2cb = np.empty(n_sen, np.int32)
        sen2cb[:n_ci] = np.repeat(np.arange(n_mgau), n_emit_state)
        cuts = np.sort(rng.choice(np.arange(1, n_sen - n_ci), n_mgau - 1, replace=False))
        sizes = np.diff(np.concatenate([[0], cuts, [n_sen - n_ci]]))
        sen2cb[n_ci:] = np.repeat(np.arange(n_mgau), sizes)
        return sen2cb
    if layout == "small":
        sizes = []
        while sum(sizes) < n_sen:
            sizes.append(int(rng.integers(1, 4)))
        sizes[-1] -= sum(sizes) - n_sen
        return np.repeat(np.arange(len(sizes)) % n_mgau, sizes).astype(np.int32)
    if layout == "single":
        return np.zeros(n_sen, np.int32)
    assert layout == "identity" and n_mgau == n_sen, "sen2cb='identity' needs n_mgau == n_sen"
    return np.arange(n_sen, dtype=np.int32)


def _pack_4bit(rng, q, n_sen):
    """Cluster 8-bit mixture weights [f][cw][sen] to 16 values and pack them as a clustered sendump stores them:
    row (n_sen + 1) // 2 bytes, senone 2i in the low nibble of byte i, 2i + 1 in the high one, an odd last senone
    alone in the low nibble of the last byte.  Returns (packed, mixw_cb)."""
    mixw_cb = np.sort(rng.choice(np.arange(0, 160), 16, replace=False)).astype(np.uint8)
    idx = np.abs(q[..., None].astype(np.int32) - mixw_cb.astype(np.int32)).argmin(-1).astype(np.uint8)
    row = (n_sen + 1) // 2
    packed = np.zeros(q.shape[:-1] + (row,), np.uint8)
    packed[..., :n_sen // 2] |= idx[..., 0:n_sen - (n_sen & 1):2]
    packed[..., :n_sen // 2] |= idx[..., 1:n_sen:2] << 4
    if n_sen & 1:
        packed[..., row - 1] |= idx[..., n_sen - 1]
    return packed, mixw_cb


def synth_ptm(seed=0, n_mgau=42, n_feat=3, n_density=256, featlen=13, n_sen=5138, topn=4,
              n_tmat=None, n_emit_state=3, skip_arcs=False, four_bit=False, sen2cb="cuts", featlens=None,
              return_raw=False):
    """Synthetic PTM model of the BASELINE.json shape (42 cb x 3 streams x 256 Gaussians x 13
    dims, 5138 senones).  Generated as RAW parameters (means, variances, transition
    probabilities, quantised mixture weights) and passed through mirrors of the reference's
    loaders (s3io.precompute_gaussians / quantize_tmat), so that the same model can also be
    written as Sphinx-3 files (s3io.write_model_dir) and loaded by the unmodified reference.
    featlens: stream lengths (n_feat streams of featlen dimensions by default).
    four_bit: clustered 4-bit mixture weights (mixw_cb), packed as _pack_4bit describes.
    sen2cb: "cuts" (CI senones first, n_emit_state per codebook, the rest in contiguous per-codebook runs cut at
    random), "small" (runs of 1-3 senones, codebooks in turn), "single" (every senone on codebook 0) or "identity"
    (n_mgau == n_sen, senone s on codebook s).  Only "cuts" is a map the reference derives from an mdef."""
    from . import s3io
    rng = np.random.default_rng(seed)
    fl = np.array(featlens if featlens is not None else [featlen] * n_feat, np.int32)
    n_feat = len(fl)
    scale = np.array([3.0, 1.0, 0.5] + [1.0] * max(0, n_feat - 3), np.float32)[:n_feat]
    if featlens is None:
        mean = (rng.normal(0.0, 1.0, (n_mgau, n_feat, n_density, featlen)) * scale[None, :, None, None]).astype(np.float32)
        var_raw = (rng.uniform(0.05, 2.0, (n_mgau, n_feat, n_density, featlen))
                   * (scale[None, :, None, None].astype(np.float64) ** 2)).astype(np.float32)
    else:
        mean, var_raw = _synth_gaussians(rng, n_mgau, fl, n_density, scale)
    var, det = s3io.precompute_gaussians(var_raw, n_mgau, n_feat, n_density, fl)
    n_ci = n_mgau * n_emit_state
    assert sen2cb != "cuts" or n_sen > n_ci
    s2c = _ptm_sen2cb(rng, sen2cb, n_sen, n_mgau, n_ci, n_emit_state)
    # mixture weights as the sendump stores them: 0..159, most mass on few codewords
    lb = np.log(1.0001)
    w = rng.gamma(0.3, 1.0, (n_sen, n_feat, n_density)) + 1e-7
    w /= w.sum(-1, keepdims=True)
    q = (np.trunc(-np.log(w) / lb).astype(np.int64)) >> 10
    mixw = np.minimum(q, 159).astype(np.uint8).transpose(1, 2, 0).copy()    # [f][cw][sen]
    mixw_cb = np.zeros(0, np.uint8)
    if four_bit:
        mixw, mixw_cb = _pack_4bit(rng, mixw, n_sen)
    n_tmat = n_tmat or n_mgau
    tp_float = synth_tmat_float(rng, n_tmat, n_emit_state, skip_arcs)
    tp = s3io.quantize_tmat(tp_float)
    n_sseq = 4096
    sseq = np.empty((n_sseq, n_emit_state), np.uint16)
    sseq[:n_mgau] = np.arange(n_ci).reshape(n_mgau, n_emit_state) % n_sen
    sseq[n_mgau:] = rng.integers(0, n_sen, (n_sseq - n_mgau, n_emit_state))
    pm = PackedModel(kind="ptm", n_sen=n_sen, n_mgau=n_mgau, n_feat=n_feat, n_density=n_density,
                     topn=topn, featlen=fl, mean=mean, var=var, det=det, mixw=mixw, mixw_cb=mixw_cb, sen2cb=s2c,
                     logadd8=make_logadd8(), n_emit_state=n_emit_state, tp=tp, sseq=sseq,
                     phone_ssid=np.arange(n_mgau, dtype=np.int32),
                     phone_tmat=np.arange(n_mgau, dtype=np.int32) % n_tmat,
                     n_ciphone=n_mgau, n_ci_sen=min(n_ci, n_sen))
    if return_raw:
        return pm, dict(mean=mean, var_raw=var_raw, tp_float=tp_float, mixw_q=mixw,
                        mixw_cb=mixw_cb if four_bit else None)
    return pm


def synth_tmat_float(rng, n_tmat, n_emit_state, skip_arcs=False):
    """float32 tp[n_tmat][n][n+1] for a Bakis topology (upper triangular, at most one skip)."""
    n = n_emit_state
    tp = np.zeros((n_tmat, n, n + 1), np.float32)
    for t in range(n_tmat):
        for i in range(n):
            nxt = [i, i + 1] + ([i + 2] if skip_arcs and i + 2 <= n else [])
            p = rng.dirichlet(np.ones(len(nxt)) * 2.0)
            for j, pj in zip(nxt, p):
                tp[t, i, j] = pj
    return tp


def synth_tmat(rng, n_tmat, n_emit_state, skip_arcs=False):
    """uint8 tp[n_tmat][n][n+1] = min(255, (-log_base p) >> 10) for a Bakis topology
    (tmat.c:215-236); impossible arcs are 255."""
    n = n_emit_state
    tp = np.full((n_tmat, n, n + 1), 255, np.uint8)
    lb = np.log(1.0001)
    for t in range(n_tmat):
        for i in range(n):
            nxt = [i, i + 1] + ([i + 2] if skip_arcs and i + 2 <= n else [])
            p = rng.dirichlet(np.ones(len(nxt)) * 2.0)
            for j, pj in zip(nxt, p):
                tp[t, i, j] = min(255, int(-np.log(pj) / lb) >> 10)
    return tp


def synth_feats(model, n_utt, n_frames, seed=0, rho=0.9, noise=0.15):
    """Synthetic dynamic-feature trajectories [n_utt][n_frames][sumlen] (float32): an AR(1)
    walk between Gaussian means of the model so that frame-to-frame top-N churn is
    speech-like (SURVEY 8d: 'feat ~ N(mu_cb, sigma_cb) mixtures drawn from the model')."""
    rng = np.random.default_rng(seed)
    D = model.sumlen
    fl = model.featlen
    offs = np.concatenate([[0], np.cumsum(fl)]).astype(np.int64)
    per_cb = model.n_density * D
    seg = 8
    n_seg = (n_frames + seg - 1) // seg + 1
    cbs = rng.integers(0, model.n_mgau, (n_utt, n_seg))
    tgt = np.empty((n_utt, n_seg, D), np.float32)
    for f in range(model.n_feat):
        cws = rng.integers(0, model.n_density, (n_utt, n_seg))
        base = cbs * per_cb + offs[f] * model.n_density + cws * int(fl[f])
        idx = base[..., None] + np.arange(int(fl[f]))
        tgt[:, :, offs[f]:offs[f + 1]] = model.mean[idx]
    out = np.empty((n_utt, n_frames, D), np.float32)
    x = tgt[:, 0].copy()
    for t in range(n_frames):
        x = np.float32(rho) * x + np.float32(1 - rho) * tgt[:, t // seg + 1]
        out[:, t] = x
    out += rng.normal(0, noise, out.shape).astype(np.float32)
    return out


def _synth_gaussians(rng, n_mgau, featlens, n_density, scale=None):
    """Random raw Gaussians, flattened [n_mgau][n_feat][n_density][len]: (mean, raw variance)."""
    means, varis = [[] for _ in range(n_mgau)], [[] for _ in range(n_mgau)]
    for f, fl in enumerate(featlens):
        sc = 1.0 if scale is None else scale[f]
        mu = (rng.normal(0, 1, (n_mgau, n_density, fl)) * sc).astype(np.float32)
        s2 = (rng.uniform(0.05, 2.0, (n_mgau, n_density, fl)) * sc * sc).astype(np.float32)
        for cb in range(n_mgau):
            means[cb].append(mu[cb].ravel())
            varis[cb].append(s2[cb].ravel())
    mean = np.concatenate([np.concatenate(m) for m in means])
    var_raw = np.concatenate([np.concatenate(v) for v in varis])
    return mean, var_raw


def synth_semi(seed=0, featlens=(12, 24, 3, 12), n_density=256, n_sen=670, topn=4, four_bit=False,
               topn_beam=None, return_raw=False):
    """Synthetic semi-continuous model (one shared codebook, s2_semi_mgau.c), 8-bit or 4-bit
    clustered mixture weights."""
    from . import s3io
    rng = np.random.default_rng(seed)
    n_feat = len(featlens)
    mean, var_raw = _synth_gaussians(rng, 1, featlens, n_density)
    var, det = s3io.precompute_gaussians(var_raw, 1, n_feat, n_density, featlens)
    lb = np.log(1.0001)
    w = rng.gamma(0.3, 1.0, (n_sen, n_feat, n_density)) + 1e-7
    w /= w.sum(-1, keepdims=True)
    q = np.minimum((np.trunc(-np.log(w) / lb).astype(np.int64)) >> 10, 159).astype(np.uint8)
    q = q.transpose(1, 2, 0).copy()                        # [f][cw][sen]
    mixw_cb = np.zeros(0, np.uint8)
    if four_bit:
        q, mixw_cb = _pack_4bit(rng, q, n_sen)
    tp_float = synth_tmat_float(rng, 10, 3)
    pm = PackedModel(kind="s2_semi", n_sen=n_sen, n_mgau=1, n_feat=n_feat, n_density=n_density, topn=topn,
                     featlen=np.array(featlens, np.int32), mean=mean, var=var, det=det, mixw=q, mixw_cb=mixw_cb,
                     sen2cb=np.zeros(n_sen, np.int32), logadd8=make_logadd8(), tp=s3io.quantize_tmat(tp_float),
                     topn_beam=np.array(topn_beam if topn_beam is not None else [0] * n_feat, np.uint8))
    if return_raw:
        return pm, dict(mean=mean, var_raw=var_raw, tp_float=tp_float, mixw_q=q, mixw_cb=mixw_cb if four_bit else None)
    return pm


def synth_ms(seed=0, n_sen=5138, n_density=8, featlens=(39,), topn=4, n_mgau=None, aw=1, return_raw=False):
    """Synthetic model for the generic ms back-end.  n_mgau=None: continuous (.cont.: one codebook
    per senone, pdf[sen][feat][cw]); n_mgau=1: pdf[feat][cw][sen]; other: PTM-like tying."""
    from . import s3io
    rng = np.random.default_rng(seed)
    n_feat = len(featlens)
    cont = n_mgau is None
    n_mgau = n_sen if cont else n_mgau
    mean, var_raw = _synth_gaussians(rng, n_mgau, featlens, n_density)
    var, det = s3io.precompute_gaussians(var_raw, n_mgau, n_feat, n_density, featlens)
    w = (rng.gamma(0.5, 1.0, (n_sen, n_feat, n_density)) + 1e-7).astype(np.float32)
    pdf = s3io.quantize_mixw_ms(w)                          # [sen][feat][cw]
    if n_mgau == 1:
        pdf = pdf.transpose(1, 2, 0).copy()
    sen2cb = np.arange(n_sen, dtype=np.int32) if cont else rng.integers(0, n_mgau, n_sen).astype(np.int32)
    tab = make_logadd8().astype(np.uint32)                  # same table, used on non-negated logs
    tp_float = synth_tmat_float(rng, 10, 3)
    pm = PackedModel(kind="ms", n_sen=n_sen, n_mgau=n_mgau, n_feat=n_feat, n_density=n_density, topn=topn,
                     featlen=np.array(featlens, np.int32), mean=mean, var=var, det=det, mixw=pdf,
                     sen2cb=sen2cb, logadd8=make_logadd8(), aw=aw, logadd_ms=tab, tp=s3io.quantize_tmat(tp_float),
                     logadd_ms_zero=-(1 << 31) >> 12)
    if return_raw:
        return pm, dict(mean=mean, var_raw=var_raw, tp_float=tp_float, mixw_float=w)
    return pm


def quantize_for_ties(pm, seed=0):
    """Return (model, feature generator) whose Gaussian exponents are small integers so that many
    codewords tie exactly at the float and int level: exercises the order-dependent tie rules of
    eval_topn / eval_cb (SURVEY A.1.2)."""
    import copy
    q = copy.deepcopy(pm)
    rng = np.random.default_rng(seed)
    q.mean = np.round(q.mean).astype(np.float32)
    q.var = (rng.integers(1, 4, q.var.shape) * 256).astype(np.float32)
    q.det = (rng.integers(-6, 1, q.det.shape) * 512).astype(np.float32)

    def feats(n_utt, n_frames, s=1):
        r = np.random.default_rng(s)
        return r.integers(-3, 4, (n_utt, n_frames, q.sumlen)).astype(np.float32)
    return q, feats
