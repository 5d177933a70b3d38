"""TEST INFRASTRUCTURE: numpy restatement of the feature transforms between CMN and the GMM that
psb_fe_create_ex adds on top of tests/fe_sessions.py, in the order feat_s2mfc2feat_block_utt
(feat.c:1277-1307) runs them, each in the reference's float32 / float64 operations:
  - batch CMN with -varnorm yes (cmn.c:165-232);
  - AGC on c0: agc_max, agc_emax + agc_emax_update, agc_noise (agc.c:110-216);
  - the LDA transform (feat_lda_transform, lda.c:139-159).
Pinned against the compiled reference by tests/test_fe_xform.py, and the device's output against it by
tests/test_gpu_fe_xform.py.  Also derives LDA models from a shipped continuous model."""
import os
import shutil

import numpy as np

import fe_sessions as fs

F32 = np.float32


def cmn_varnorm(cep):
    """cmn() with varnorm: the mean over frames with c0 >= 0, the variance over all frames."""
    cep = np.array(cep, F32, copy=True)
    T, nc = cep.shape
    if T == 0:
        return cep
    s, n = np.zeros(nc, F32), 0
    for t in range(T):
        if cep[t, 0] < 0:
            continue
        s = (s + cep[t]).astype(F32)
        n += 1
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = (s / F32(n)).astype(F32)
        var = np.zeros(nc, F32)
        for t in range(T):
            d = (cep[t] - mean).astype(F32)
            var = (var + (d * d).astype(F32)).astype(F32)
        istd = np.sqrt(np.float64(T) / var.astype(np.float64)).astype(F32)
        return ((cep - mean).astype(F32) * istd).astype(F32)


class Agc:
    """agc_t after agc_init + agc_emax_set, driven as feat_agc (beginutt, endutt) and feat_update_stats drive it."""

    def __init__(self, kind, cmn_none=False, thresh=2.0):
        self.kind = kind
        self.max, self.obs_max, self.obs_max_sum = F32(10.0 if cmn_none else 5.0), F32(0), F32(0)
        self.obs_frame, self.obs_utt = 0, 0
        self.thresh = F32(thresh)

    def utterance(self, cep):
        cep = np.array(cep, F32, copy=True)
        T = len(cep)
        c0 = cep[:, 0]
        if self.kind == "max" and T:
            m = c0[0]
            for x in c0[1:]:
                if x > m:
                    m = x
            cep[:, 0] = (c0 - m).astype(F32)
        elif self.kind == "noise" and T:
            lo = c0[0]
            for x in c0:
                if x < lo:
                    lo = x
            lim = F32(lo + self.thresh)
            s, n = F32(0), 0
            for x in c0:
                if x < lim:
                    s = F32(s + x)
                    n += 1
            if n:
                cep[:, 0] = (c0 - F32(s / F32(n))).astype(F32)
        elif self.kind == "emax":
            for x in c0:
                if x > self.obs_max:
                    self.obs_max, self.obs_frame = x, 1
            if T:
                cep[:, 0] = (c0 - self.max).astype(F32)
            self.update()          # feat_agc, endutt
            self.update()          # ps_end_utt -> feat_update_stats
        return cep

    def update(self):
        if self.obs_frame:
            self.obs_max_sum = F32(self.obs_max_sum + self.obs_max)
            self.obs_utt += 1
            self.max = F32(self.obs_max_sum / F32(self.obs_utt))
            if self.obs_utt == 16:
                self.obs_max_sum = F32(self.obs_max_sum / F32(2))
                self.obs_utt = 8
        self.obs_frame = 0
        self.obs_max = F32(-1000.0)

    def state(self):
        return self.max, self.obs_max, self.obs_max_sum, self.obs_frame, self.obs_utt


def lda(feats, a, ldadim=0):
    """feat_lda_transform with lda[0] = a [m][n] and feat_read_lda's output dimension."""
    m = ldadim if 0 < ldadim <= a.shape[0] else a.shape[0]
    x = np.asarray(feats, F32)
    acc = np.zeros((len(x), m), F32)
    for k in range(a.shape[1]):
        acc = (acc + (x[:, k:k + 1] * a[None, :m, k]).astype(F32)).astype(F32)
    return acc


def features(cep, cmn="batch", varnorm=False, agc=None, a=None, ldadim=0, feat=0):
    """Cepstra before CMN [T][n_cep] -> (features, cepstra after CMN and AGC), as feat_s2mfc2feat_block_utt;
    agc: an Agc (its state carries over between calls) or None."""
    if cmn == "batch":
        cep = cmn_varnorm(cep) if varnorm else fs.batch_cmn(np.asarray(cep, F32))
    cep = np.asarray(cep, F32)
    if agc is not None:
        cep = agc.utterance(cep)
    f = fs.dyn_features(cep, feat) if len(cep) else np.zeros((0, fs.FEAT_DIM[feat]), F32)
    if a is not None:
        f = lda(f, a, ldadim)
    return f, cep


def emax_session():
    """More than 16 utterances (the emax history decays at 16), an empty one first, an all-silent one (every c0 < 0
    without CMN: it counts only once obs_max has dropped to -1000) and a sub-frame one."""
    from oracle import fe_golden
    go = fe_golden.goforward()
    noise = lambda n, seed, amp: (np.random.default_rng(seed).standard_normal(n) * amp).astype(np.int16)
    u = [np.zeros(0, np.int16), np.zeros(4000, np.int16), go, noise(50, 3, 3000)]
    u += [go[i * 2000:i * 2000 + 9000 + 500 * i] for i in range(15)]
    u += [noise(6000, 9, 200), go]
    return u


def orthonormal(m, n, seed):
    """The first m rows of a random n x n orthogonal matrix (float32)."""
    q, _ = np.linalg.qr(np.random.default_rng(seed).standard_normal((n, n)))
    return q[:m].astype(F32)


def block_rotation(seed, n=39, block=13):
    """A full-rank block-diagonal rotation (one random rotation per 13-dimensional block)."""
    a = np.zeros((n, n), F32)
    for b in range(0, n, block):
        a[b:b + block, b:b + block] = orthonormal(block, block, seed + b)
    return a


def copy_model(src, dst):
    """A writable copy of a model directory (the source tree may be read-only, and copytree keeps its modes)."""
    os.makedirs(dst)
    for f in os.listdir(src):
        shutil.copyfile(os.path.join(src, f), os.path.join(dst, f))
    return dst


def derive_lda_model(src, dst, a, write_transform=True):
    """Copy the continuous model in src to dst with its Gaussians mapped through a [m][n]: means A mu,
    variances diag(A Sigma A^T); feature_transform = a (when write_transform).  feat.params is copied as it is."""
    from pocketsphinx_b200 import s3io
    copy_model(src, dst)
    m, n = a.shape
    a64 = a.astype(np.float64)
    for name, f in (("means", lambda x: x @ a64.T), ("variances", lambda x: x @ (a64 * a64).T)):
        n_mgau, n_feat, n_density, featlen, arr = s3io.read_gauden(os.path.join(src, name))
        assert n_feat == 1 and int(featlen[0]) == n
        out = f(arr.reshape(-1, n).astype(np.float64)).astype(F32)
        s3io.write_gauden(os.path.join(dst, name), out, n_mgau, 1, n_density, [m])
    if write_transform:
        s3io.write_lda(os.path.join(dst, "feature_transform"), a[None])
    return dst
