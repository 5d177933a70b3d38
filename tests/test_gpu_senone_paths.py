"""GPU (-m gpu): every path the tied-mixture senone stage takes, bit-exact against the C oracle.  psb_launch_ptm_batch
picks its senone kernel from the model: ptm_senone4_kernel (four senones per thread, 16x2 arithmetic biased by
SEN_BIAS) or ptm_senone_kernel<8-bit | 4-bit> for PTM, semi_senone4_kernel or semi_senone_kernel<8-bit | 4-bit> for
semi-continuous models.  Each batch case reads the plan the launcher runs (Batch.tm_plan), asserts the kernel it is
meant to reach, scores a ragged batch and compares every utterance's int16 scores with oracle.OracleModel.score_utt.
The per-frame scorer (scorer_senone_kernel, scorer_semi_senone_kernel) is compared call by call with the oracle's
ps_mgau twin.  Where a case exists to reach an edge, it asserts from the oracle's own top-N lists that the edge is
reached.  test_cases_cover_every_kernel fails if a threshold change silently moves a case to another kernel.

The oracle is pinned to the compiled reference at these shapes by tests/test_tm_ref_shapes.py: the 4-bit PTM
sendump, -logbase 1.0000325 / 1.000031, -topn 1 / 2 / 8 and PTM stream counts 1, 2, 4 and 8.  The sen2cb layouts
other than random cuts rest on the oracle alone."""
import copy

import numpy as np
import pytest

from pocketsphinx_b200.model import SEN2CB_LAYOUTS, make_logadd8, synth_feats, synth_ptm, synth_semi

pytestmark = pytest.mark.gpu

SEN_BIAS = 64                       # psb_ptm.cu: the 16x2 kernels' bias
BASE_MAX21, BASE_MAX22 = 1.0000325, 1.000031


@pytest.fixture(scope="module")
def api():
    from pocketsphinx_b200 import api
    assert api.device_count() > 0, "no CUDA device visible"
    return api


# ---------------------------------------------------------------------------------------
# helpers

def _ragged(total, rng, lo, hi):
    """Utterance lengths in [lo, hi] summing to total."""
    lens = []
    while sum(lens) < total:
        lens.append(int(rng.integers(lo, hi + 1)))
    lens[-1] -= sum(lens) - total
    if lens[-1] <= 0:
        lens[-2] += lens.pop()
    return lens


def _feats(pm, total, seed, far=0.0):
    """Features [total][sumlen]; a fraction `far` of the frames moved far from every Gaussian."""
    x = synth_feats(pm, 1, total, seed=seed)[0]
    if far:
        rng = np.random.default_rng(seed)
        x[rng.random(total) < far] += np.float32(40)
    return x


def _plan(api, pm, total=64):
    m = api.Model(pm)
    b = api.Batch(m, 1, 1)
    try:
        return b.tm_plan(total)
    finally:
        b.close()
        m.close()


def _expect(plan, want):
    got = {k: plan[k] for k in want}
    assert got == want, "plan %s, expected %s" % (plan, want)


def _score_vs_oracle(api, pm, feats, lens, want=None):
    """Score the ragged batch on the device, compare each utterance with the oracle; returns the plan."""
    from oracle import oracle
    m = api.Model(pm)
    off = api.Batch.offsets(lens)
    total = int(off[-1])
    b = api.Batch(m, len(lens), total + 2)
    plan = b.tm_plan(total)
    if want is not None:
        _expect(plan, want)
    scr = b.score_host(np.ascontiguousarray(feats, np.float32), off)
    b.close()
    m.close()
    om = oracle.OracleModel(pm)
    for u in range(len(lens)):
        want_s = om.score_utt(feats[off[u]:off[u + 1]])
        got = scr[off[u]:off[u + 1]]
        bad = np.argwhere(got != want_s)
        assert bad.size == 0, "utt %d of %d (frames %d..%d): %d mismatches, first (frame, senone) %s: got %s want %s" % (
            u, len(lens), off[u], off[u + 1], len(bad), bad[0].tolist(), got[tuple(bad[0])], want_s[tuple(bad[0])])
    return plan


def _n_bsen(sen2cb):
    """ptm_senone4_kernel's one-by-one senones: every member of a quad that is incomplete or spans two codebooks."""
    n = len(sen2cb)
    out = 0
    for s0 in range(0, n, 4):
        q = sen2cb[s0:s0 + 4]
        if len(q) < 4 or (q != q[0]).any():
            out += len(q)
    return out


def _ptm4_threads(K, n_sen):
    n_quads = (n_sen + 3) // 4
    iters = (n_quads + 511) // 512
    r32 = lambda x: (x + 31) // 32 * 32
    return min(512, max(256, r32(K), r32(-(-n_quads // iters))))


def _weights(pm, f, cw, s):
    """Mixture weights of senones s at codewords cw of stream f (broadcasting), as the reference reads them: 4-bit PTM
    picks the nibble by the low bit of the byte (ptm_mgau.c:376-377), 4-bit semi by the senone's parity."""
    rows = pm.mixw.reshape(pm.n_feat, pm.n_density, pm.mixw_row)
    if not pm.mixw_4bit:
        return rows[f, cw, s].astype(np.int64)
    b = rows[f, cw, s // 2].astype(np.int64)
    odd = (b & 1) if pm.kind == "ptm" else (s & 1)
    return pm.mixw_cb[np.where(odd == 1, b >> 4, b & 15)].astype(np.int64)


def _semi_counts(lists, beam):
    """Entries inside topn_beam per (frame, stream) from normalised lists [T][f][topn]{cw, score} (mgau_norm,
    s2_semi_mgau.c:186-203: the first entry over the beam ends the list)."""
    sc = lists[..., 1]
    over = (sc > np.asarray(beam)[None, :, None]) & (np.asarray(beam)[None, :, None] > 0)
    return np.where(over.any(-1), over.argmax(-1), sc.shape[-1])


def _trace(pm, feats):
    """Restate the log-add chains of every (frame, senone, stream) from the oracle's normalised top-N lists: returns
    (lowest intermediate, largest |x - y| a fast_logmath_add sees)."""
    from oracle import oracle
    _, lists = oracle.OracleModel(pm).score_utt(feats, want_topn=True)
    tab = np.zeros(512, np.int64)
    tab[:256] = pm.logadd8
    s = np.arange(pm.n_sen)
    lo, dmax = 0, 0
    for f in range(pm.n_feat):
        if pm.kind == "ptm":
            L = lists[:, pm.sen2cb, f]                                  # [T][n_sen][topn]{cw, score}
            n = np.full(L.shape[:2], pm.topn)
        else:
            L = np.broadcast_to(lists[:, None, f], (len(feats), pm.n_sen) + lists.shape[2:])
            beam = pm.topn_beam if pm.topn_beam.size else np.zeros(pm.n_feat, np.uint8)
            n = np.broadcast_to(np.maximum(1, _semi_counts(lists, beam)[:, None, f]), L.shape[:2])
        y = _weights(pm, f, L[..., 0], s[None, :, None]) + L[..., 1]
        x = y[..., 0]
        for j in range(1, pm.topn):
            d = np.abs(x - y[..., j])
            live = j < n
            dmax = max(dmax, int(d[live].max(initial=0)))
            x = np.where(live, np.minimum(x, y[..., j]) - tab[np.minimum(d, 511)], x)
            lo = min(lo, int(x.min()))
    return lo, dmax


def _low_point(tab):
    """The lowest value three fast_logmath_adds can reach from non-negative inputs: every input 0."""
    x = 0
    for _ in range(3):
        x -= int(tab[-x])
    return x


# ---------------------------------------------------------------------------------------
# A: 4-bit PTM weights (ptm_senone_kernel<true>), odd and even n_sen

@pytest.mark.parametrize("n_sen", [301, 300])
def test_ptm_four_bit_batch(api, n_sen):
    pm = synth_ptm(seed=20 + n_sen, n_mgau=8, n_density=32, n_sen=n_sen, four_bit=True)
    rows = pm.mixw.reshape(pm.n_feat, pm.n_density, -1)
    # the nibble quirk shows only where a byte's low bit differs from its senone's parity: both must occur
    assert ((rows & 1) == 0).any() and ((rows & 1) == 1).any()
    lens = _ragged(257, np.random.default_rng(n_sen), 5, 60)
    _score_vs_oracle(api, pm, _feats(pm, sum(lens), seed=2), lens, dict(senone="ptm_senone_4b", threads=512))


# ---------------------------------------------------------------------------------------
# B: the 16x2 kernels' bias bound.  make_logadd8(1.0000325) peaks at 21, the largest table they accept
# (3 * 21 < SEN_BIAS); 1.000031 peaks at 22 and takes the per-senone kernels.  From non-negative inputs three
# fast_logmath_adds reach at most -42 (21) / -44 (22): x - tab[-x] from 0, every input 0.  3 * max (-63 / -66) is the
# launcher's bound, not a reachable value.  Mixture weights 0 and normalised scores 0 on one codebook drive the
# chains to that low point.

def _low_model(kind, base, seed):
    if kind == "ptm":
        pm = copy.deepcopy(synth_ptm(seed=seed, n_mgau=6, n_density=32, n_sen=303))
        fl = int(pm.featlen[0])
        mean = pm.mean.reshape(pm.n_mgau, pm.n_feat, pm.n_density, fl)
        var = pm.var.reshape(pm.n_mgau, pm.n_feat, pm.n_density, fl)
        det = pm.det.reshape(pm.n_mgau, pm.n_feat, pm.n_density)
        # codebook 0: identical Gaussians (ties -> every normalised score 0), boosted to win every stream
        mean[0] = mean[0, :, :1]
        var[0] = var[0, :, :1]
        det[0] = det[0, :, :1] + np.float32(2e5)
        pm.mean, pm.var, pm.det = mean.ravel(), var.ravel(), det.ravel()
        zero = pm.sen2cb == 0
    else:
        pm = copy.deepcopy(synth_semi(seed=seed, n_sen=303))
        offs = np.concatenate([[0], np.cumsum(pm.featlen)]) * pm.n_density
        det = pm.det.reshape(pm.n_feat, pm.n_density)
        for f, fl in enumerate(pm.featlen):
            g = pm.mean[offs[f]:offs[f + 1]].reshape(pm.n_density, fl)
            v = pm.var[offs[f]:offs[f + 1]].reshape(pm.n_density, fl)
            g[:8] = g[:1]
            v[:8] = v[:1]
            det[f, :8] = det[f, 0] + np.float32(2e5)
        pm.det = det.ravel()
        zero = np.arange(pm.n_sen) % 3 == 0
    mw = pm.mixw.reshape(pm.n_feat, pm.n_density, pm.mixw_row).copy()
    mw[:, :, zero] = 0
    pm.mixw = mw.ravel()
    pm.logadd8 = make_logadd8(base=base)
    return pm


@pytest.mark.parametrize("kind,base,kernel", [
    ("ptm", BASE_MAX21, "ptm_senone4"), ("ptm", BASE_MAX22, "ptm_senone_8b"),
    ("s2_semi", BASE_MAX21, "semi_senone4"), ("s2_semi", BASE_MAX22, "semi_senone_8b")])
def test_add_table_bias_bound(api, kind, base, kernel):
    pm = _low_model(kind, base, seed=30)
    tab_max = int(pm.logadd8.max())
    assert tab_max == (21 if base == BASE_MAX21 else 22)
    assert (3 * tab_max < SEN_BIAS) == kernel.endswith("4")
    lens = _ragged(223, np.random.default_rng(3), 5, 50)
    feats = _feats(pm, sum(lens), seed=4)
    _score_vs_oracle(api, pm, feats, lens, dict(senone=kernel))
    lo, _ = _trace(pm, feats)
    assert lo == _low_point(pm.logadd8), "the chains reach %d, not their low point %d" % (lo, _low_point(pm.logadd8))
    assert -SEN_BIAS < lo == -2 * tab_max


# ---------------------------------------------------------------------------------------
# C: PTM stream counts, K above 256 (ptm_senone4's CTA sized from K) and the refusals

STREAMS = {
    # name: (synth_ptm arguments, K)
    "nfeat1": (dict(featlens=(13,), n_mgau=8), 8),
    "nfeat2": (dict(featlens=(13, 13), n_mgau=8), 16),
    "nfeat4": (dict(featlens=(4, 4, 4, 4), n_mgau=8), 32),
    "nfeat8": (dict(featlens=(4,) * 8, n_mgau=8), 64),
    "K300": (dict(featlens=(13, 13, 13), n_mgau=100), 300),
    "K512": (dict(featlens=(4,) * 8, n_mgau=64), 512),
}


def _stream_model(name):
    kw, _ = STREAMS[name]
    return synth_ptm(seed=40 + len(name), n_density=32, n_sen=701, **kw)


@pytest.mark.parametrize("name", list(STREAMS))
def test_stream_counts_and_wide_K(api, name):
    pm = _stream_model(name)
    K = STREAMS[name][1]
    assert pm.n_mgau * pm.n_feat == K
    lens = _ragged(181, np.random.default_rng(K), 5, 50)
    plan = _score_vs_oracle(api, pm, _feats(pm, sum(lens), seed=5), lens,
                            dict(senone="ptm_senone4", threads=_ptm4_threads(K, pm.n_sen), n_bsen=_n_bsen(pm.sen2cb)))
    if K > 256:
        assert plan["threads"] >= K > 256, plan


def test_refusals(api):
    from pocketsphinx_b200.api import PsbError
    cases = [
        (synth_ptm(seed=50, n_mgau=171, n_density=32, n_sen=1200), "at most 512"),             # K = 513
        (synth_ptm(seed=51, n_mgau=8, n_density=32, n_sen=300, topn=2), "-topn 4"),
        (synth_semi(seed=52, n_density=64, n_sen=300, topn=8), "-topn 4"),
        # 120 000 int16 scores exceed one CTA's shared memory
        (synth_ptm(seed=53, n_mgau=1, n_feat=1, n_density=32, n_sen=120000), "shared memory"),
    ]
    for pm, msg in cases:
        m = api.Model(pm)
        b = api.Batch(m, 1, 8)
        with pytest.raises(PsbError, match=msg):
            b.tm_plan(8)
        with pytest.raises(PsbError, match=msg):
            b.score_host(_feats(pm, 8, seed=1), np.array([0, 8], np.int32))
        b.close()
        m.close()


# ---------------------------------------------------------------------------------------
# D: quads and the boundary list -- n_sen % 4 in {0, 1, 2, 3} x every sen2cb layout

def _quad_model(layout, r):
    if layout == "identity":                        # n_mgau == n_sen: every quad goes through bsen
        n_sen = 200 + r
        return synth_ptm(seed=60 + r, n_mgau=n_sen, n_feat=1, n_density=32, n_sen=n_sen, sen2cb=layout)
    return synth_ptm(seed=60 + r, n_mgau=8, n_density=32, n_sen=300 + r, sen2cb=layout)


@pytest.mark.parametrize("r", [0, 1, 2, 3])
@pytest.mark.parametrize("layout", SEN2CB_LAYOUTS)
def test_quad_layouts(api, layout, r):
    pm = _quad_model(layout, r)
    assert pm.n_sen % 4 == r
    nb = _n_bsen(pm.sen2cb)
    if layout == "identity":
        assert nb == pm.n_sen
    elif layout == "single":
        assert nb == r
    elif layout == "small":
        sizes = np.diff(np.flatnonzero(np.diff(np.concatenate([[-1], pm.sen2cb, [-1]]))))
        assert set(sizes.tolist()) >= {1, 2, 3}, "codebooks of 1, 2 and 3 senones"
    lens = _ragged(97, np.random.default_rng(r), 5, 40)
    _score_vs_oracle(api, pm, _feats(pm, sum(lens), seed=6), lens, dict(senone="ptm_senone4", n_bsen=nb))


# ---------------------------------------------------------------------------------------
# E: semi_senone4_kernel -- tail senones, the unaligned short4 fallback, streams with 1..4 entries in the beam

def _semi_beam_model(n_sen):
    """A semi-continuous model whose topn_beam gives, in some frame, streams with 1, 2, 3 and 4 entries in the beam.
    The normalised lists do not depend on the beam, so the beam is chosen from the lists of a beam-less model."""
    from oracle import oracle
    pm = copy.deepcopy(synth_semi(seed=70, n_sen=n_sen))
    feats = _feats(pm, 600, seed=7)
    _, lists = oracle.OracleModel(pm).score_utt(feats, want_topn=True)
    for b in range(1, 96):
        c = _semi_counts(lists, [b] * pm.n_feat)
        if (np.sort(c, -1) == [1, 2, 3, 4]).all(-1).any():
            pm.topn_beam = np.full(pm.n_feat, b, np.uint8)
            return pm, feats, c
    raise AssertionError("no beam gives streams with 1, 2, 3 and 4 entries in one frame")


@pytest.mark.parametrize("n_sen", [601, 602, 603])
def test_semi_senone4_tails_and_beam(api, n_sen):
    from oracle import oracle
    pm, feats, counts = _semi_beam_model(n_sen)
    _, lists = oracle.OracleModel(pm).score_utt(feats, want_topn=True)
    # mgau_norm stops normalising at the first entry over the beam: count from the normalised prefix
    c = np.array([[next((j for j in range(4) if lists[t, f, j, 1] > pm.topn_beam[f]), 4) for f in range(pm.n_feat)]
                  for t in range(len(feats))])
    assert np.array_equal(c, counts)
    assert (np.sort(c, -1) == [1, 2, 3, 4]).all(-1).any()
    lens = _ragged(len(feats), np.random.default_rng(n_sen), 40, 200)
    _score_vs_oracle(api, pm, feats, lens, dict(senone="semi_senone4", topn="semi_split"))


# ---------------------------------------------------------------------------------------
# F: mixture weights 255 next to 0 with normalised scores at the 96 clamp: |x - y| up to 351, past the 256-entry table

@pytest.mark.parametrize("kind,base,kernel", [
    ("ptm", 1.0001, "ptm_senone4"), ("ptm", BASE_MAX22, "ptm_senone_8b"),
    ("s2_semi", 1.0001, "semi_senone4"), ("s2_semi", BASE_MAX22, "semi_senone_8b")])
def test_weights_past_the_table(api, kind, base, kernel):
    if kind == "ptm":
        pm = copy.deepcopy(synth_ptm(seed=80, n_mgau=6, n_density=32, n_sen=402))
    else:
        pm = copy.deepcopy(synth_semi(seed=80, n_sen=402))
    rng = np.random.default_rng(81)
    pm.mixw = np.where(rng.random(pm.mixw.size) < 0.5, 0, 255).astype(np.uint8)
    pm.logadd8 = make_logadd8(base=base)
    lens = _ragged(211, np.random.default_rng(8), 5, 50)
    feats = _feats(pm, sum(lens), seed=9, far=0.3)
    _score_vs_oracle(api, pm, feats, lens, dict(senone=kernel))
    _, dmax = _trace(pm, feats)
    assert dmax >= 255 + 96, "largest |x - y| is %d" % dmax


# ---------------------------------------------------------------------------------------
# G: the per-frame scorer at -topn 1..8 (PTM and semi, 8- and 4-bit): compall, active lists with bridged gaps, and
# frames re-scored from the history ring

def _scorer_vs_oracle(api, pm, feats, rng, p_active=0.3, lookback=2):
    """Mgau.frame_eval and the oracle's frame_eval with identical call sequences: all senones, sparse lists, a gap
    of more than 255 senones (bridged in the delta list), and frames re-scored later from the ring.  Returns the
    frames scored with an active list."""
    from oracle import oracle
    m = api.Model(pm)
    s = api.Mgau(m, pl_window=0)
    dec = oracle.OracleModel(pm).decoder(n_hist=2)
    host = np.zeros(pm.n_sen, np.int16)
    want = np.zeros(pm.n_sen, np.int16)
    listed = []
    for t in range(len(feats)):
        mode = t % 3
        if mode == 0:
            lst, compall = None, True
        else:
            fl = (rng.random(pm.n_sen) < p_active).astype(np.uint8)
            if mode == 2:
                fl[pm.n_sen // 3: pm.n_sen // 3 + 300] = 0
            lst, compall = oracle.flags2list(fl), False
            listed.append(t)
        got = s.frame_eval(feats[t], t, lst, compallsen=compall, out=host)
        dec.frame_eval_into(want, feats[t], t, lst, compallsen=compall)
        assert np.array_equal(got, want), "frame %d (mode %d): %d senones differ" % (t, mode, (got != want).sum())
        if t >= lookback:
            lst = oracle.flags2list((rng.random(pm.n_sen) < p_active).astype(np.uint8))
            got = s.frame_eval(feats[t - lookback], t - lookback, lst, compallsen=False, out=host)
            dec.frame_eval_into(want, feats[t - lookback], t - lookback, lst, compallsen=False)
            assert np.array_equal(got, want), "re-scored frame %d" % (t - lookback)
        s.frame_idx = t + 1
        dec.set_frame_idx(t + 1)
    s.close(); dec.close(); m.close()
    return listed


def _scorer_model(kind, four_bit, topn, seed=90):
    if kind == "ptm":
        return synth_ptm(seed=seed, n_mgau=6, n_density=32, n_sen=651, topn=topn, four_bit=four_bit)
    return synth_semi(seed=seed, n_density=64, n_sen=651, topn=topn, four_bit=four_bit)


SCORER_TOPN = [1, 2, 3, 5, 8]


@pytest.mark.parametrize("topn", SCORER_TOPN)
@pytest.mark.parametrize("four_bit", [False, True], ids=["8bit", "4bit"])
@pytest.mark.parametrize("kind", ["ptm", "s2_semi"])
def test_per_frame_scorer_topn(api, kind, four_bit, topn):
    pm = _scorer_model(kind, four_bit, topn)
    _scorer_vs_oracle(api, pm, _feats(pm, 21, seed=91, far=0.2), np.random.default_rng(92))


@pytest.mark.parametrize("n_in_beam", [6, 7])
def test_semi_four_bit_wrap_boundary(api, n_in_beam):
    """get_scores_4b_feat_{1..6} add mixw_cb + score in uint8 (s2_semi_mgau.c:453-463); from 7 entries on the sum is
    an int.  Cluster values near 255 make the uint8 sum wrap; the beam leaves exactly 6 or exactly 7 entries in
    list-mode frames."""
    from oracle import oracle
    pm = copy.deepcopy(_scorer_model("s2_semi", True, 8, seed=93))
    pm.mixw_cb = np.array([0, 10, 30, 60, 90, 120, 150, 180, 200, 220, 235, 245, 250, 252, 254, 255], np.uint8)
    feats = _feats(pm, 45, seed=94)
    _, lists = oracle.OracleModel(pm).score_utt(feats, want_topn=True)
    listed = np.array([t for t in range(len(feats)) if t % 3])
    beam = None
    for b in range(1, 96):
        c = _semi_counts(lists, [b] * pm.n_feat)
        if (c[listed] == n_in_beam).sum() >= 5:
            beam = b
            break
    assert beam is not None, "no beam leaves %d entries in list-mode frames" % n_in_beam
    pm.topn_beam = np.full(pm.n_feat, beam, np.uint8)
    # a byte overflows where cluster value 255 meets a positive normalised score inside the beam
    inside = lists[listed, :, :n_in_beam, 1]
    assert ((c[listed] == n_in_beam)[..., None] & (inside > 0)).any()
    rows = pm.mixw.reshape(pm.n_feat, pm.n_density, pm.mixw_row)
    assert ((rows & 15) == 15).any() and ((rows >> 4) == 15).any()
    _scorer_vs_oracle(api, pm, feats, np.random.default_rng(95))


# ---------------------------------------------------------------------------------------
# every kernel, from the plans of the cases above

def test_cases_cover_every_kernel(api):
    plans = []
    for n_sen in (301, 300):
        plans.append(_plan(api, synth_ptm(seed=20 + n_sen, n_mgau=8, n_density=32, n_sen=n_sen, four_bit=True)))
    for kind, base in [("ptm", BASE_MAX21), ("ptm", BASE_MAX22), ("s2_semi", BASE_MAX21), ("s2_semi", BASE_MAX22)]:
        plans.append(_plan(api, _low_model(kind, base, seed=30)))
    for name in STREAMS:
        plans.append(_plan(api, _stream_model(name)))
    for layout in SEN2CB_LAYOUTS:
        for r in range(4):
            plans.append(_plan(api, _quad_model(layout, r)))
    plans.append(_plan(api, synth_semi(seed=70, n_sen=602)))
    kernels = {p["senone"] for p in plans}
    assert kernels >= {"ptm_senone4", "ptm_senone_8b", "ptm_senone_4b", "semi_senone4", "semi_senone_8b"}, kernels
    # semi_senone_4b and both widths of both per-frame kernels: the per-frame cases' models, and one 4-bit semi plan
    assert _plan(api, _scorer_model("s2_semi", True, 4))["senone"] == "semi_senone_4b"
    assert any(p["threads"] > 256 for p in plans if p["senone"] == "ptm_senone4")
    assert any(p["n_bsen"] == 0 for p in plans if p["senone"] == "ptm_senone4")
    per_frame = {(pm.kind, pm.mixw_4bit) for pm in (_scorer_model(k, fb, 1) for k in ("ptm", "s2_semi") for fb in (0, 1))}
    assert per_frame == {("ptm", False), ("ptm", True), ("s2_semi", False), ("s2_semi", True)}
