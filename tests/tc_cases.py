"""Inputs built to drive each decision of the PTM tensor-core filter (psb_ptm_tc.cu), and a float64 numpy mirror of
that decision which shows on the CPU where every row lands.

Crafted pairs: all codewords of a (codebook, stream) pair share one mean, and crafted frames sit exactly on it, so a
codeword's exponent is its determinant, bit for bit; the determinants then place candidates by n-tile, quad lane and
half.  Separations are either well below the bound eps (near-ties of 0.15 - 1) or far above it (1e5, 1024), so the
float64 stand-in for the GEMM value cannot move a row between regimes.
"""
import copy

import numpy as np

TC_CAP = 18
LOW = -1.0e5                       # every codeword that must never be a candidate sits this far below the cluster


# ---------------------------------------------------------------------------------------
# mirror of the filter's decision

def _f32(x):
    return np.float32(x)


def pair_bounds(pm):
    """psb_tc_prepare's centre and bound coefficients per pair: cen [K][FL], A/B [K][FL], C [K] (float32)."""
    FL, nd = int(pm.featlen[0]), pm.n_density
    mean = pm.mean.reshape(pm.n_mgau, pm.n_feat, nd, FL).astype(np.float64)
    var = pm.var.reshape(pm.n_mgau, pm.n_feat, nd, FL).astype(np.float64)
    det = pm.det.reshape(pm.n_mgau, pm.n_feat, nd).astype(np.float64)
    cen = (mean.sum(2) / nd).astype(np.float32)                                     # [cb][f][FL]
    mp = mean - cen[:, :, None, :].astype(np.float64)
    A = np.nextafter((np.abs(var).max(2).astype(np.float32) * _f32(1.0001)), np.float32(np.inf))
    B = np.nextafter((np.abs(2.0 * var * mp).max(2).astype(np.float32) * _f32(1.0001)), np.float32(np.inf))
    C = ((np.abs(det) + (np.abs(var) * mp * mp).sum(-1)).max(-1) * 1.0001).astype(np.float32)
    K = pm.n_mgau * pm.n_feat
    return cen.reshape(K, FL), A.reshape(K, FL), B.reshape(K, FL), C.reshape(K)


def decide(pm, feats):
    """The filter's decision per (frame, pair) for features [T][sumlen], exact float64 distances in place of the GEMM
    values: dict of [T][K] arrays (n, n_h0, n_h1, over, listed, certain, fail_* flags)."""
    FL, nd = int(pm.featlen[0]), pm.n_density
    T, K = feats.shape[0], pm.n_mgau * pm.n_feat
    cen, A, B, C = pair_bounds(pm)
    mean = pm.mean.reshape(K, nd, FL).astype(np.float64)
    var = pm.var.reshape(K, nd, FL).astype(np.float64)
    det = pm.det.reshape(K, nd).astype(np.float64)
    col = np.arange(nd)
    tile, q4 = col // 8, (col % 8) // 2
    grp = tile // (nd // 64)
    half = q4 // 2
    keys = ("n", "n_h0", "n_h1", "over", "listed", "certain", "fail_gap", "fail_straddle", "fail_sign", "fail_saturation")
    out = {k: np.zeros((T, K), np.int64 if k.startswith("n") else bool) for k in keys}
    for k in range(K):
        f = k % pm.n_feat
        x = feats[:, f * FL:(f + 1) * FL].astype(np.float32)
        y = (x - cen[k]).astype(np.float32)
        S = C[k] + (A[k] * (y.astype(np.float64) ** 2)).sum(1) + (B[k] * np.abs(y.astype(np.float64))).sum(1)
        eps = S * 2.0 ** -18 + 2.0
        d = det[k][None, :] - (var[k][None] * (x[:, None, :].astype(np.float64) - mean[k][None]) ** 2).sum(-1)
        gm = np.full((T, 8), -np.inf)
        for g in range(8):
            gm[:, g] = d[:, grp == g].max(1)
        L0 = -np.sort(-gm, 1)[:, 4]                                                  # fifth largest group maximum
        thr = np.floor(L0 - eps) - 1.0 - eps
        cand = d >= thr[:, None]
        # each quad lane stores the pairs (8 i + 2 q4, + 1) whose larger value passes; the walk reads TC_CAP per lane
        pair_pass = np.maximum(d[:, 0::2], d[:, 1::2]) >= thr[:, None]             # [T][nd / 2], pair p = col // 2
        pq4 = q4[0::2]
        over = np.zeros(T, bool)
        nh = np.zeros((T, 2), np.int64)
        for lane in range(4):
            idx = np.nonzero(pq4 == lane)[0]                                         # ascending n-tile order
            pp = pair_pass[:, idx]
            over |= pp.sum(1) > TC_CAP
            walked = pp & (np.cumsum(pp, 1) <= TC_CAP)
            vals = cand[:, 2 * idx] & walked
            vals2 = cand[:, 2 * idx + 1] & walked
            nh[:, lane // 2] += vals.sum(1) + vals2.sum(1)
        n = nh.sum(1)
        listed = (n >= 5) & (n <= TC_CAP) & ~over
        a = -np.sort(-np.where(cand, d, -np.inf), 1)[:, :5]
        gap = 2 * eps + 1
        fail_gap = ((a[:, :4] - a[:, 1:5]) <= gap[:, None]).any(1)
        lo = np.ceil(a[:, :4] - eps[:, None]).astype(np.int64) >> 10
        hi = np.ceil(a[:, :4] + eps[:, None]).astype(np.int64) >> 10
        fail_str = (lo != hi).any(1)
        fail_sign = ~(a[:, 0] + eps < -2.0)
        fail_sat = ~(a[:, 4] > -2.0e9)
        out["n"][:, k], out["n_h0"][:, k], out["n_h1"][:, k] = n, nh[:, 0], nh[:, 1]
        out["over"][:, k], out["listed"][:, k] = over, listed
        out["fail_gap"][:, k], out["fail_straddle"][:, k] = listed & fail_gap, listed & fail_str
        out["fail_sign"][:, k], out["fail_saturation"][:, k] = listed & fail_sign, listed & fail_sat
        out["certain"][:, k] = listed & ~(fail_gap | fail_str | fail_sign | fail_sat)
    return out


# ---------------------------------------------------------------------------------------
# crafted models and features

def _columns(nd, h, count):
    """`count` columns of half h (quad lanes 2 h, 2 h + 1), one per n-tile first and the 8 groups in turn, so that any
    five of them lie in five different groups; no lane gets more than TC_CAP pairs for count <= TC_CAP."""
    npg = nd // 64
    cols = [8 * (g * npg + r) + 4 * h + o for o in (0, 2, 1, 3) for r in range(npg) for g in range(8)]
    return cols[:count]


def layout_split(nd, n0, n1, base):
    """Near-tied candidates: n0 in half 0, n1 in half 1, the best ones in half 1."""
    det = np.full(nd, base + LOW)
    cols = _columns(nd, 1, n1) + _columns(nd, 0, n0)
    det[cols] = base - 0.15 * np.arange(len(cols))
    return det


def layout_lane_over(nd, base):
    """The 32 codewords at columns 8 i (quad lane 0) one apart (in doubt, but with distinct integer scores, so no tie
    fix-up repairs a wrong list), the best ones at i >= TC_CAP: lane 0 stores 23 pairs with one passing value each,
    its walk stops after 18 of them."""
    det = np.full(nd, base + LOW)
    i = np.arange(nd // 8)
    det[8 * i] = base - 1.0 * (i[::-1])
    return det


def layout_boundary(nd, delta):
    """Five well-separated candidates, each 1024 k + delta: the >> 10 of a +- eps differs at both ends."""
    det = np.full(nd, -9000.0 + LOW)
    det[_columns(nd, 0, 5)] = -1024.0 * np.arange(3, 8) + delta
    return det


SPLITS = [(18, 0), (0, 18), (9, 9), (17, 2), (10, 9), (5, 0), (0, 5)]


def crafted_model(nd, layouts, seed=3, n_mgau=8, duplicate_pairs=()):
    """synth_ptm with pairs k = 0 .. len(layouts) - 1 (row-major over codebook, stream) given the determinant layouts and
    one shared mean per stream; `duplicate_pairs` also share one variance vector (identical codewords).  Returns the
    model and the crafted frame (every stream on its shared mean)."""
    from pocketsphinx_b200.model import synth_ptm
    pm = synth_ptm(seed=seed, n_mgau=n_mgau, n_density=nd, n_sen=n_mgau * 3 + 40)
    FL, K = 13, n_mgau * 3
    assert len(layouts) <= K
    mean = pm.mean.reshape(n_mgau, 3, nd, FL).copy()
    var = pm.var.reshape(n_mgau, 3, nd, FL).copy()
    det = pm.det.reshape(n_mgau, 3, nd).copy()
    rng = np.random.default_rng(seed)
    frame = rng.normal(0, 1, (3, FL)).astype(np.float32)
    for k, lay in enumerate(layouts):
        cb, f = divmod(k, 3)
        mean[cb, f] = frame[f]
        det[cb, f] = np.asarray(lay, np.float32)
        if k in duplicate_pairs:
            var[cb, f] = var[cb, f, 0]
    q = copy.deepcopy(pm)
    q.mean, q.var, q.det = mean.ravel(), var.ravel(), det.ravel()
    return q, frame.ravel()


def utterances(pm, frame, lens, seed, p_crafted=0.7, scale=1.0):
    """Ragged utterances mixing the crafted frame (probability p_crafted) with synthetic trajectories."""
    from pocketsphinx_b200.model import synth_feats
    rng = np.random.default_rng(seed)
    T = max(lens) if lens else 1
    base = synth_feats(pm, len(lens), max(T, 1), seed=seed)
    out = []
    for u, n in enumerate(lens):
        f = base[u, :n].copy()
        f[rng.random(n) < p_crafted] = frame
        out.append(np.ascontiguousarray(f * np.float32(scale), np.float32))
    return out


def case(name):
    """(model, utterances, the counters it must drive above 0) of one crafted case; counters as in api.Batch.TC_COUNTERS."""
    if name.startswith("lane_over"):
        pm, fr = crafted_model(256, [layout_lane_over(256, -6000.3)] * 6)
        return pm, utterances(pm, fr, [1, 40, 77, 3, 130], 1), {"lane_over"}
    if name.startswith("split"):
        nd = int(name.split("_")[1])
        lays = [layout_split(nd, a, b, -6000.3) for a, b in SPLITS]
        pm, fr = crafted_model(nd, lays * 3)
        return pm, utterances(pm, fr, [5, 64, 1, 100, 33], 2), {"split_lists", "over_cap", "fail_gap"}
    if name.startswith("dup"):
        nd = int(name.split("_")[1])
        pm, fr = crafted_model(nd, [np.full(nd, -5000.5)] * 12, duplicate_pairs=range(12))
        return pm, utterances(pm, fr, [0, 1, 2, 129, 17, 64, 65, 200], 3, p_crafted=0.5), {"over_cap", "tie_fixups"}
    if name.startswith("boundary"):
        nd = int(name.split("_")[1])
        pm, fr = crafted_model(nd, [layout_boundary(nd, dl) for dl in (-0.75, -0.25, 0.0, 0.25)] * 3)
        return pm, utterances(pm, fr, [50, 77, 1], 4), {"fail_straddle"}
    if name.startswith("positive"):
        nd = int(name.split("_")[1])
        lays = [layout_split(nd, a, b, 60.3) for a, b in SPLITS]
        pm, fr = crafted_model(nd, (lays * 4)[:24])
        lens = [300, 211, 1, 250, 129, 64]                  # 955 frames x 24 pairs >= 16384 rows, nearly all in doubt
        return pm, utterances(pm, fr, lens, 5, p_crafted=0.95), {"fail_sign", "fallback_listed", "fallback_all",
                                                                   "split_lists"}
    if name.startswith("saturation"):
        pm, fr = crafted_model(256, [])
        return pm, utterances(pm, fr, [40, 27], 6, p_crafted=0.0, scale=1.0e4), {"fail_saturation"}
    raise KeyError(name)


CASES = ["lane_over_256", "split_64", "split_128", "split_256", "dup_64", "dup_128", "dup_256", "boundary_128",
         "boundary_256", "positive_64", "positive_256", "saturation_256"]


# ---------------------------------------------------------------------------------------
# device runs (GPU tests and their PSB_TC_CHECK child processes)

def score_vs_oracle(api, oracle, pm, chunks, batch=None):
    """Score the utterances in one batch; compare every utterance's scores and top-N records with the oracle's.
    Returns (records, batch) -- the batch stays open when it was passed in."""
    lens = [len(c) for c in chunks]
    off = api.Batch.offsets(lens)
    own = batch is None
    m = None
    if own:
        m = api.Model(pm)
        batch = api.Batch(m, len(chunks) + 1, int(off[-1]) + 1)
    scr = batch.score_host(np.concatenate(chunks) if chunks else np.zeros((0, pm.sumlen), np.float32), off)
    rec = batch.get_topn(int(off[-1]))
    om = oracle.OracleModel(pm)
    for u, c in enumerate(chunks):
        if not len(c):
            continue
        want, raw = om.score_utt(c, want_raw=True)
        a, b = off[u], off[u + 1]
        oracle.assert_records_equal(rec[a:b], oracle.ptm_records(raw), "utterance %d (frames %d..%d)" % (u, a, b))
        assert np.array_equal(scr[a:b], want), "utterance %d: scores" % u
    if own:
        batch.close()
        m.close()
    return rec, batch


def child(script, timeout=900):
    """Run `script` in a fresh interpreter with PSB_TC_CHECK=1 (read once per process); `script` prints one JSON line
    last, which is returned parsed."""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    prelude = "import sys\nsys.path.insert(0, %r)\nsys.path.insert(0, %r)\n" % (os.path.dirname(here), here)
    r = subprocess.run([sys.executable, "-c", prelude + script], capture_output=True, text=True, timeout=timeout,
                       env=dict(os.environ, PSB_TC_CHECK="1"))
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])
