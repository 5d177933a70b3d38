"""GPU (-m gpu): every path the ms (continuous / generic multi-stream) batch stage takes, bit-exact against the C
oracle.  psb_launch_ms_batch picks its kernels from the model and the batch: tiled or streamed distances, senones
fused into the tile kernel or evaluated by ms_senone_kernel, the tile kernel's feature prefetch or in-place staging,
the list width NT and compute_dist_all, frames per CTA and chunks.  Each case reads the plan the launcher runs
(Batch.ms_plan), asserts the path it is meant to take, scores a ragged batch and compares every utterance's int16
scores with oracle.OracleModel.score_utt.  test_cases_cover_every_path fails if a threshold change silently moves a
case to another path.

The oracle is pinned to the compiled reference at these shapes by tests/test_ms_ref_shapes.py and
tests/test_s3io_vs_ref.py, for continuous models.  Tied codebooks with an arbitrary sen2cb (cases G, L2, M, N) and
the single shared codebook with transposed weights (H, J, P) rest on the oracle alone."""
import copy

import numpy as np
import pytest

from pocketsphinx_b200.model import synth_feats, synth_ms

pytestmark = pytest.mark.gpu

INT_MIN = -(1 << 31)


@pytest.fixture(scope="module")
def api():
    from pocketsphinx_b200 import api
    assert api.device_count() > 0, "no CUDA device visible"
    return api


# ---------------------------------------------------------------------------------------
# helpers

def _ragged(total, rng, lo, hi):
    """Utterance lengths in [lo, hi] summing to total, none a multiple of 4 (so none of 64)."""
    while True:
        lens = []
        while sum(lens) < total:
            n = int(rng.integers(lo, hi + 1))
            lens.append(n + 1 if n % 4 == 0 else n)
        lens[-1] -= sum(lens) - total
        if lens[-1] > 0 and lens[-1] % 4:
            return lens


def _feats(pm, total, seed):
    return synth_feats(pm, 1, total, seed=seed)[0]


def _plan(api, pm, total):
    m = api.Model(pm)
    b = api.Batch(m, 1, 1)
    try:
        return b.ms_plan(total)
    finally:
        b.close()
        m.close()


def _expect(plan, **want):
    got = {k: plan[k] for k in want}
    assert got == {k: int(v) for k, v in want.items()}, "plan %s, expected %s" % (plan, want)
    if plan["fuse"]:
        assert plan["dist_bytes"] == 0, plan


def _score_vs_oracle(api, pm, feats, lens, plan_want=None):
    """Score the ragged batch on the device, compare each utterance with the oracle; returns (plan, scores, off)."""
    from oracle import oracle
    m = api.Model(pm)
    off = api.Batch.offsets(lens)
    total = int(off[-1])
    b = api.Batch(m, len(lens), total + 2)
    plan = b.ms_plan(total)
    if plan_want is not None:
        _expect(plan, **plan_want)
    scr = b.score_host(np.ascontiguousarray(feats, np.float32), off)
    b.close()
    m.close()
    om = oracle.OracleModel(pm)
    for u in range(len(lens)):
        want = om.score_utt(feats[off[u]:off[u + 1]])
        got = scr[off[u]:off[u + 1]]
        bad = np.argwhere(got != want)
        assert bad.size == 0, "utt %d of %d (frames %d..%d): first mismatch (frame, senone) %s: got %s want %s" % (
            u, len(lens), off[u], off[u + 1], bad[0].tolist(), got[tuple(bad[0])], want[tuple(bad[0])])
    return plan, scr, off


def _smallest_total(api, pm, ok, hi=1 << 20):
    """The smallest frame count whose plan satisfies ok(plan), then the next one that is not a multiple of 64 (so
    the last CTA's range ends inside a block)."""
    m = api.Model(pm)
    b = api.Batch(m, 1, 1)
    lo = 1
    assert ok(b.ms_plan(hi)), b.ms_plan(hi)
    while lo < hi:
        mid = (lo + hi) // 2
        if ok(b.ms_plan(mid)):
            hi = mid
        else:
            lo = mid + 1
    while lo % 64 == 0 or not ok(b.ms_plan(lo)):
        lo += 1
    b.close()
    m.close()
    return lo


# ---------------------------------------------------------------------------------------
# the cases: model, and the plan it must get

CASES = {
    # name: (synth_ms arguments, plan fields)
    "A_tile_fused_nt1": (dict(seed=41, n_sen=301, n_density=8, topn=1),
                         dict(tile=1, fuse=1, prefetch=1, nt=1, all=0, n_used=1)),
    "B_tile_fused_nt2": (dict(seed=42, n_sen=301, n_density=8, topn=2),
                         dict(tile=1, fuse=1, prefetch=1, nt=2, all=0, n_used=2)),
    "C_tile_fused_nt8": (dict(seed=43, n_sen=201, n_density=16, featlens=(13,), topn=8),
                         dict(tile=1, fuse=1, prefetch=1, nt=8, all=0, n_used=8)),
    "D_all_nd3": (dict(seed=44, n_sen=250, n_density=3, topn=4),
                  dict(tile=1, fuse=1, prefetch=1, nt=4, all=1, n_used=3)),
    "D_all_nd4_nt8": (dict(seed=45, n_sen=250, n_density=4, topn=8),
                      dict(tile=1, fuse=1, prefetch=1, nt=8, all=1, n_used=4)),
    "E_three_streams": (dict(seed=46, n_sen=230, n_density=4, featlens=(13, 13, 13), topn=2),
                        dict(tile=1, fuse=1, prefetch=1, nt=2, all=0, n_used=2)),
    "F_staged_s2_4x": (dict(seed=47, n_sen=230, n_density=4, featlens=(12, 24, 3, 12), topn=4),
                       dict(tile=1, fuse=1, prefetch=0, nt=4, all=1, n_used=4)),
    "G_tile_tied": (dict(seed=48, n_sen=500, n_mgau=42, n_density=4, topn=2),
                    dict(tile=1, fuse=0, prefetch=1, nt=2, all=0, transposed=0)),
    "H_tile_transposed": (dict(seed=49, n_sen=300, n_mgau=1, n_density=8, topn=4),
                          dict(tile=1, fuse=0, prefetch=1, nt=4, all=0, transposed=1)),
    "I_partial_tile_20": (dict(seed=50, n_sen=20, n_density=8, topn=4),
                          dict(tile=1, fuse=1, tiles_x=1)),
    "I_partial_tile_33": (dict(seed=51, n_sen=33, n_density=8, topn=4),
                          dict(tile=1, fuse=1, tiles_x=2)),
    "J_streamed_cont": (dict(seed=52, n_sen=300, n_density=16, topn=4),
                        dict(tile=0, fuse=0, nt=4, all=0, transposed=0)),
    "J_streamed_transposed": (dict(seed=54, n_sen=300, n_mgau=1, n_density=16, topn=4),
                              dict(tile=0, fuse=0, nt=4, all=0, transposed=1)),
    "O_topn3_nd2": (dict(seed=53, n_sen=150, n_density=2, topn=3),
                    dict(tile=1, fuse=1, nt=4, all=1, n_used=2)),
}


def _model(name):
    return synth_ms(**CASES[name][0])


@pytest.mark.parametrize("name", [k for k in CASES if not k.startswith("O_")])
def test_path_matches_oracle(api, name):
    pm = _model(name)
    rng = np.random.default_rng(len(name))
    lens = _ragged(227, rng, 5, 70)
    _score_vs_oracle(api, pm, _feats(pm, sum(lens), seed=3), lens, CASES[name][1])


# ---------------------------------------------------------------------------------------
# K: several 64-frame blocks per CTA (the cross-block prefetch and the per-block sscr reset); L: several chunks

BIG = {
    # name: (synth_ms arguments, plan fields, condition on the plan that sizes the batch)
    "K_config4": (dict(seed=0, n_sen=5138, n_density=8, featlens=(39,), topn=4),
                  dict(tile=1, fuse=1, prefetch=1, nt=4, n_chunks=1),
                  lambda p: p["frames_per_cta"] >= 4 * 64),
    "K_staged": (dict(seed=61, n_sen=1000, n_density=4, featlens=(12, 24, 3, 12), topn=4),
                 dict(tile=1, fuse=1, prefetch=0, nt=4, n_chunks=1),
                 lambda p: p["frames_per_cta"] >= 4 * 64),
    # fused: only the 65535-frame grid limit splits the batch
    "L_fused_chunks": (dict(seed=62, n_sen=40, n_density=2, featlens=(13,), topn=2),
                       dict(tile=1, fuse=1, dist_bytes=0),
                       lambda p: p["n_chunks"] >= 2),
    # not fused: the 2 GiB list budget splits it (4096 codebooks x 4 streams x 8 entries x 8 bytes = 1 MiB per frame)
    "L_unfused_chunks": (dict(seed=63, n_sen=4500, n_mgau=4096, n_density=8, featlens=(3, 3, 3, 3), topn=8),
                         dict(tile=1, fuse=0, nt=8, all=1),
                         lambda p: p["n_chunks"] >= 2),
}


def _big_total(api, name, pm):
    kw, want, ok = BIG[name]
    total = _smallest_total(api, pm, ok)
    if name.startswith("L_"):
        total += 36                   # a partial last chunk after a boundary inside an utterance
    return total


@pytest.mark.parametrize("name", list(BIG))
def test_frame_blocks_and_chunks_match_oracle(api, name):
    kw, want, ok = BIG[name]
    pm = synth_ms(**kw)
    total = _big_total(api, name, pm)
    rng = np.random.default_rng(7)
    lens = _ragged(total, rng, 150, 400)
    off = api.Batch.offsets(lens)
    plan, _, _ = _score_vs_oracle(api, pm, _feats(pm, total, seed=9), lens, want)
    assert ok(plan), plan
    if name.startswith("K_"):
        ctas_y = -(-total // plan["frames_per_cta"])
        assert (total - (ctas_y - 1) * plan["frames_per_cta"]) % 64, "the last CTA's range must end inside a block"
    else:
        bounds = np.arange(1, plan["n_chunks"]) * plan["chunk"]
        assert all(b not in set(off.tolist()) for b in bounds), "a chunk boundary must fall inside an utterance"
        assert total % plan["chunk"], "the last chunk must be partial"


# ---------------------------------------------------------------------------------------
# M: extremes -- the fden floor, both int16 clamps, weights 0 / 255, aw with negative sums

EXTREME_SHAPES = {
    # sorted lists: a Gaussian below INT_MIN never enters them, so far frames keep the WORST_DIST entries (id 0)
    "fused_sorted": (dict(n_sen=200, n_density=8, topn=4), dict(tile=1, fuse=1, all=0)),
    # compute_dist_all lists every Gaussian: the only lists where a distance below INT_MIN meets the fden floor
    "fused_all": (dict(n_sen=200, n_density=4, topn=4), dict(tile=1, fuse=1, all=1)),
    "unfused_tied_all": (dict(n_sen=200, n_mgau=42, n_density=4, topn=4), dict(tile=1, fuse=0, transposed=0, all=1)),
    "streamed_tied_all": (dict(n_sen=200, n_mgau=42, n_density=8, featlens=(12, 24, 3, 12), topn=8),
                          dict(tile=0, transposed=0, all=1)),
}


def _restate(pm, feats):
    """float64 distances [T][n_mgau][n_feat][nd] of every Gaussian (ms_gauden.c compute_dist without the list)."""
    T, nd = len(feats), pm.n_density
    out = np.empty((T, pm.n_mgau, pm.n_feat, nd))
    mean = pm.mean.astype(np.float64)
    var = pm.var.astype(np.float64)
    det = pm.det.astype(np.float64).reshape(pm.n_mgau, pm.n_feat, nd)
    x = feats.astype(np.float64)
    o = 0
    for f, fl in enumerate(pm.featlen):
        fl = int(fl)
        idx = (np.arange(pm.n_mgau)[:, None, None] * nd * pm.sumlen + o * nd
               + np.arange(nd)[None, :, None] * fl + np.arange(fl)[None, None, :])
        mu, vv = mean[idx], var[idx]                                         # [cb][d][j]
        diff = x[:, None, None, o:o + fl] - mu[None]
        out[:, :, f] = det[None, :, f] - (diff * diff * vv[None]).sum(-1)
        o += fl
    return out


def _restate_raw(pm, dist):
    """Approximate raw senone scores (before the first clamp) [T][n_sen] and, per (frame, codebook, stream),
    whether every listed distance is below INT_MIN.  The log-add of the list is taken as its maximum, which is
    below the exact value by at most the table's largest entry."""
    n = min(pm.topn, pm.n_density)
    order = np.argsort(-dist, axis=-1, kind="stable")[..., :n]
    top = np.take_along_axis(dist, order, -1)                               # [T][cb][f][n]
    floored = (top < INT_MIN).all(-1)
    fden = np.where(top < INT_MIN, INT_MIN >> 10, np.floor((top + 1023) / 1024))
    sen = np.arange(pm.n_sen)
    cb = pm.sen2cb
    if pm.n_mgau == 1:
        w = pm.mixw.reshape(pm.n_feat, pm.n_density, pm.n_sen)              # [f][d][sen]
        ww = w[np.arange(pm.n_feat)[None, None, :, None], order[:, cb], sen[None, :, None, None]]
    else:
        w = pm.mixw.reshape(pm.n_sen, pm.n_feat, pm.n_density)
        ww = w[sen[None, :, None, None], np.arange(pm.n_feat)[None, None, :, None], order[:, cb]]
    fscr = (fden[:, cb] - ww).max(-1)                                       # [T][sen][f]
    return -fscr.sum(-1) / pm.aw, floored


def _extreme_model(shape, aw, seed):
    kw, want = EXTREME_SHAPES[shape]
    pm = synth_ms(seed=seed, aw=aw, **kw)
    rng = np.random.default_rng(seed)
    mw = pm.mixw.copy()
    mask = rng.random(mw.shape) < 0.5
    mw[mask] = np.where(rng.random(mask.sum()) < 0.5, 0, 255).astype(mw.dtype)
    pm.mixw = np.ascontiguousarray(mw)
    # sharp Gaussians: positive distances, so negative senone sums; the sharpest reach the negative first clamp
    det = pm.det.copy()
    r = rng.random(det.shape)
    det[r < 0.05] = np.float32(1.5e9)
    det[(r >= 0.05) & (r < 0.15)] += np.float32(2e7)
    pm.det = det
    return pm, want


def _extreme_feats(pm, total, seed):
    rng = np.random.default_rng(seed)
    x = _feats(pm, total, seed)
    kind = rng.integers(0, 4, total)
    x[kind == 1] += np.float32(40)                                          # far: the positive first clamp
    x[kind == 2] = (rng.choice([-1, 1], (int((kind == 2).sum()), pm.sumlen)) * 1e4).astype(np.float32)  # below INT_MIN
    return x


@pytest.mark.parametrize("shape", list(EXTREME_SHAPES))
@pytest.mark.parametrize("aw", [3, 512])
def test_extremes_match_oracle(api, shape, aw):
    """aw 3: both clamps and C truncation of negative sums.  aw 512: on the all-path the fden floor shows in
    unclamped scores (a floored stream contributes 2^21 + w, and even four such streams / 512 stay inside int16)."""
    pm, want = _extreme_model(shape, aw, seed=70 + aw)
    lens = _ragged(149, np.random.default_rng(aw), 5, 40)
    feats = _extreme_feats(pm, sum(lens), seed=aw)
    _, scr, _ = _score_vs_oracle(api, pm, feats, lens, want)
    raw, floored = _restate_raw(pm, _restate(pm, feats))
    assert (np.asarray(pm.mixw) == 0).any() and (np.asarray(pm.mixw) == 255).any()
    # frames where a codebook's whole list is far below INT_MIN
    dist_ok = floored.any(axis=(1, 2))
    assert dist_ok.sum() >= 10, "no frame reaches the fden floor"
    if aw == 3:
        assert (raw > 40000).any(), "the first clamp (32767) is never reached"
        assert (raw < -40000).any(), "the first clamp (-32768) is never reached"
        neg = (raw < -100) & (raw > -30000)
        assert neg.sum() > 50, "too few negative sums for C truncation to matter"
        best = np.maximum(np.minimum(raw, 32767), -32768).min(1, keepdims=True)
        second = np.maximum(np.minimum(raw, 32767), -32768) - best > 33000
        assert second.any(), "the second clamp is never reached"
        assert (scr[second] == 32767).all()
    elif want["all"]:
        unclamped = floored.all(axis=(2,))[:, pm.sen2cb] & (np.abs(raw) < 30000)
        assert unclamped.sum() > 100, "no unclamped score carries the fden floor"


# ---------------------------------------------------------------------------------------
# N: exact ties -- the tile kernel's swap chain and the streamed kernel's strict-'<' scan

TIE_SHAPES = {
    "fused_nt2": (dict(seed=80, n_sen=230, n_density=8, topn=2), dict(tile=1, fuse=1, nt=2, all=0)),
    "fused_nt4": (dict(seed=81, n_sen=230, n_density=8, topn=4), dict(tile=1, fuse=1, nt=4, all=0)),
    "streamed_tied_nt2": (dict(seed=82, n_sen=300, n_mgau=42, n_density=16, topn=2),
                          dict(tile=0, nt=2, all=0, transposed=0)),
    "streamed_tied_nt4": (dict(seed=83, n_sen=300, n_mgau=42, n_density=16, topn=4),
                          dict(tile=0, nt=4, all=0, transposed=0)),
}


def _tie_model(name, seed=6):
    """quantize_for_ties for ms models: small integer means, variance terms and dets, and integer features.  With
    39 dimensions summed, quantize_for_ties itself leaves ties rare among the top entries, so only about one
    dimension in ten keeps a variance term (0 elsewhere) and the means and features stay within +-2."""
    pm = copy.deepcopy(synth_ms(**TIE_SHAPES[name][0]))
    rng = np.random.default_rng(seed)
    pm.mean = np.clip(np.round(pm.mean), -2, 2).astype(np.float32)
    pm.var = ((rng.random(pm.var.shape) < 0.1) * rng.integers(1, 3, pm.var.shape) * 256).astype(np.float32)
    pm.det = (rng.integers(-2, 1, pm.det.shape) * 512).astype(np.float32)

    def feats(total, s):
        return np.random.default_rng(s).integers(-2, 3, (total, pm.sumlen)).astype(np.float32)
    return pm, feats


@pytest.mark.parametrize("name", list(TIE_SHAPES))
def test_ties_match_oracle(api, name):
    pm, gen = _tie_model(name)
    lens = _ragged(131, np.random.default_rng(5), 5, 40)
    feats = gen(sum(lens), s=9)
    _score_vs_oracle(api, pm, feats, lens, TIE_SHAPES[name][1])
    # integer inputs: every distance is an exact integer in float32, so int64 gives the exact lists
    d = _restate(pm, feats)
    assert np.array_equal(d, np.round(d)) and np.abs(d).max() < 2 ** 24
    n = pm.topn
    # the reference inserts before the first entry that is not better: among equal distances the later Gaussian
    # comes first
    di = d.astype(np.int64)
    key = di * (pm.n_density + 1) + np.arange(pm.n_density)
    top = np.sort(key, -1)[..., ::-1][..., :n] // (pm.n_density + 1)
    assert (top[..., :-1] == top[..., 1:]).mean() > 0.05, "too few ties among adjacent list entries"


# ---------------------------------------------------------------------------------------
# O: refusals

def test_refused_topn(api):
    """A -topn that is not a power of two below the Gaussian count is refused by the batch stage, before any
    launch; one above 8 is refused when the model is created."""
    from pocketsphinx_b200.api import PsbError
    pm = synth_ms(seed=90, n_sen=64, n_density=8, topn=3)
    m = api.Model(pm)
    b = api.Batch(m, 1, 8)
    with pytest.raises(PsbError, match="power-of-two -topn"):
        b.ms_plan(8)
    with pytest.raises(PsbError, match="power-of-two -topn"):
        b.score_host(_feats(pm, 8, seed=1), np.array([0, 8], np.int32))
    b.close()
    m.close()
    for nd in (8, 32):
        with pytest.raises(PsbError, match="topn 16 out of range"):
            api.Model(synth_ms(seed=90, n_sen=64, n_density=nd, topn=16))


def test_topn_above_two_gaussians_matches_oracle(api):
    pm = _model("O_topn3_nd2")
    lens = _ragged(101, np.random.default_rng(2), 5, 40)
    _score_vs_oracle(api, pm, _feats(pm, sum(lens), seed=4), lens, CASES["O_topn3_nd2"][1])


# ---------------------------------------------------------------------------------------
# P: the per-frame scorer (the ps_mgau_t drop-in)

def _scorer_vs_oracle(api, pm, feats, rng, p_active=0.3, lookback=2):
    """Mgau.frame_eval and the oracle's frame_eval with identical call sequences: all senones, sparse lists, a gap
    of more than 255 senones, and frames re-scored later."""
    from oracle import oracle
    m = api.Model(pm)
    s = api.Mgau(m, pl_window=0)
    dec = oracle.OracleModel(pm).decoder(n_hist=2)
    host = np.zeros(pm.n_sen, np.int16)
    want = np.zeros(pm.n_sen, np.int16)
    for t in range(len(feats)):
        mode = t % 3
        if mode == 0:
            lst, compall = None, True
        else:
            fl = (rng.random(pm.n_sen) < p_active).astype(np.uint8)
            if mode == 2:
                fl[pm.n_sen // 3: pm.n_sen // 3 + 300] = 0
            lst, compall = oracle.flags2list(fl), False
        got = s.frame_eval(feats[t], t, lst, compallsen=compall, out=host)
        dec.frame_eval_into(want, feats[t], t, lst, compallsen=compall)
        assert np.array_equal(got, want), "frame %d (mode %d)" % (t, mode)
        if t >= lookback:
            lst = oracle.flags2list((rng.random(pm.n_sen) < p_active).astype(np.uint8))
            got = s.frame_eval(feats[t - lookback], t - lookback, lst, compallsen=False, out=host)
            dec.frame_eval_into(want, feats[t - lookback], t - lookback, lst, compallsen=False)
            assert np.array_equal(got, want), "re-scored frame %d" % (t - lookback)
        s.frame_idx = t + 1
        dec.set_frame_idx(t + 1)
    s.close(); dec.close(); m.close()


@pytest.mark.parametrize("kw", [dict(n_sen=700, n_mgau=1, n_density=8, topn=4),
                                dict(n_sen=600, n_density=8, topn=1),
                                dict(n_sen=650, n_density=4, featlens=(12, 24, 3, 12), topn=4)],
                         ids=["shared_codebook", "topn1", "s2_4x"])
def test_per_frame_scorer_matches_oracle(api, kw):
    pm = synth_ms(seed=95, **kw)
    _scorer_vs_oracle(api, pm, _feats(pm, 24, seed=96), np.random.default_rng(97))


# ---------------------------------------------------------------------------------------
# every path, from the plans of the cases above

def test_cases_cover_every_path(api):
    plans = {}
    for name in CASES:
        plans[name] = _plan(api, _model(name), 227)
    for name, (kw, want, ok) in BIG.items():
        pm = synth_ms(**kw)
        plans[name] = _plan(api, pm, _big_total(api, name, pm))
    for shape in EXTREME_SHAPES:
        plans["M_" + shape] = _plan(api, _extreme_model(shape, 3, seed=73)[0], 149)
    for name in TIE_SHAPES:
        plans["N_" + name] = _plan(api, _tie_model(name)[0], 131)
    wants = dict({k: v[1] for k, v in CASES.items()}, **{k: v[1] for k, v in BIG.items()},
                 **{"M_" + k: v[1] for k, v in EXTREME_SHAPES.items()}, **{"N_" + k: v[1] for k, v in TIE_SHAPES.items()})
    for name, p in plans.items():
        _expect(p, **wants[name])

    def path(p):
        if p["tile"] and p["fuse"]:
            return "tile fused " + ("prefetch" if p["prefetch"] else "staged")
        if p["tile"]:
            return "tile unfused " + ("transposed" if p["transposed"] else "sen2cb")
        return "streamed " + ("transposed" if p["transposed"] else "sen2cb")
    paths = {path(p) for p in plans.values()}
    assert paths >= {"tile fused prefetch", "tile fused staged", "tile unfused sen2cb", "tile unfused transposed",
                     "streamed sen2cb", "streamed transposed"}, paths
    # sen2cb on the streamed path: both an identity map (continuous) and tied codebooks
    assert plans["J_streamed_cont"]["tile"] == 0 and plans["N_streamed_tied_nt2"]["tile"] == 0
    tile = [p for p in plans.values() if p["tile"]]
    assert {p["nt"] for p in tile if not p["all"]} == {1, 2, 4, 8}
    assert {p["nt"] for p in tile if p["all"]} >= {4, 8}
    for pre in (0, 1):
        assert any(p["frames_per_cta"] > 64 for p in tile if p["fuse"] and p["prefetch"] == pre), pre
    for fuse in (0, 1):
        assert any(p["n_chunks"] > 1 for p in tile if p["fuse"] == fuse), fuse
    assert all(p["dist_bytes"] == 0 for p in plans.values() if p["fuse"])
