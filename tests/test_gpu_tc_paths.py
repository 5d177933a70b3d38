"""GPU (-m gpu): every decision path of the PTM tensor-core filter, at the record level.  The crafted cases of
tests/tc_cases.py (their regimes are shown on the CPU by tests/test_tc_decisions.py) are compared record by record and
score by score with the oracle; a PSB_TC_CHECK child process shows through the filter's counters that each path ran."""
import numpy as np
import pytest

import tc_cases as tc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from pocketsphinx_b200 import api
    assert api.device_count() > 0, "no CUDA device visible"
    return api


@pytest.mark.parametrize("name", tc.CASES)
def test_crafted_case_records_match_oracle(api, name):
    from oracle import oracle
    pm, utts, _ = tc.case(name)
    tc.score_vs_oracle(api, oracle, pm, utts)


def test_work_list_overflow_is_deterministic(api):
    """Which rows fall back to the filter kernel depends on the order of atomics; the records must not."""
    from oracle import oracle
    pm, utts, _ = tc.case("positive_256")
    r1, _ = tc.score_vs_oracle(api, oracle, pm, utts)
    r2, _ = tc.score_vs_oracle(api, oracle, pm, utts)
    oracle.assert_records_equal(r2, r1, "second run")


CHECK_CASES = r"""
import json, numpy as np
import tc_cases as tc
from oracle import oracle
from pocketsphinx_b200 import api
out = {}
for name in tc.CASES:
    pm, utts, want = tc.case(name)
    m = api.Model(pm)
    b = api.Batch(m, len(utts) + 1, sum(len(u) for u in utts) + 1)
    tc.score_vs_oracle(api, oracle, pm, utts, batch=b)
    r, n = b.tc_check()
    out[name] = dict(b.tc_stats, ratio=float(r), max_candidates=int(n), total=sum(len(u) for u in utts),
                     K=pm.n_mgau * pm.n_feat, want=sorted(want))
    b.close(); m.close()
print(json.dumps(out))
"""


def test_crafted_cases_drive_every_counted_path():
    """Each case drives every counter it was built for."""
    out = tc.child(CHECK_CASES)
    print(out)
    for name, v in out.items():
        assert 0.0 <= v["ratio"] < 0.8, (name, v)
        assert v["rows"] == v["total"] * v["K"], (name, v)
        for c in v["want"]:
            assert v[c] > 0, (name, c, v)


def _tpc_rule(tiles, K, P):
    """launch_wgmma's tiles-per-CTA rule for P resident CTAs."""
    t = 1
    while t < 32 and (tiles // (t * 2)) * K >= P * 4:
        t *= 2
    return t


def test_geometry_ragged_totals_and_tiles_per_cta_vs_oracle(api):
    """Ragged batches of 1 .. 191 frames (partial tiles, an empty second warpgroup) and batches sized so that a CTA walks
    1, 2, 8 and 32 tiles with a partial last CTA: every record of every utterance equals the oracle's."""
    import torch
    from oracle import oracle
    lays = [tc.layout_split(64, a, b, -6000.3) for a, b in tc.SPLITS]
    pm, fr = tc.crafted_model(64, lays * 3)
    K = pm.n_mgau * pm.n_feat
    P = torch.cuda.get_device_properties(0).multi_processor_count      # one filter CTA per SM (asserted below)
    rng = np.random.default_rng(7)
    for total in (1, 63, 64, 65, 127, 128, 129, 191, 192):
        lens = [total] if total < 60 else [total - 60, 1, 59]
        tc.score_vs_oracle(api, oracle, pm, tc.utterances(pm, fr, lens, total, p_crafted=0.5))
    seen = set()
    for target in (1, 2, 8, 32):
        tiles = next(t for t in range(2, 4096) if _tpc_rule(t, K, P) == target and (target == 1 or t % target))
        total = tiles * 128 - 37
        lens, left = [], total
        while left:
            n = int(min(left, rng.integers(1, 700)))
            lens.append(n)
            left -= n
        utts = tc.utterances(pm, fr, lens, target, p_crafted=0.3)
        feats, off = np.concatenate(utts), api.Batch.offsets(lens)
        m = api.Model(pm)
        b = api.Batch(m, len(lens) + 1, total + 1)
        b.score_host(feats, off)
        rec = b.get_topn(total)
        b.tc_check()
        st = b.tc_stats
        b.close(); m.close()
        assert st["tiles_per_cta"] == target and st["ctas_per_pair"] == -(-tiles // target), (target, tiles, st)
        seen.add(st["tiles_per_cta"])
        om = oracle.OracleModel(pm)
        for u in range(len(lens)):
            _, raw = om.score_utt(utts[u], want_raw=True)
            oracle.assert_records_equal(rec[off[u]:off[u + 1]], oracle.ptm_records(raw),
                                        "%d tiles per CTA, utterance %d" % (target, u))
    assert seen == {1, 2, 8, 32}


# ---------------------------------------------------------------------------------------
# psb_model_update_gaussians (ps_mgaufuncs_t.transform: MLLR)

def _mllr(pm, raw, seed):
    """A near-identity affine map of the means per stream and scaled variances; dets recomputed like the reference."""
    import copy
    from pocketsphinx_b200 import s3io
    rng = np.random.default_rng(seed)
    q = copy.deepcopy(pm)
    mean = raw["mean"].reshape(-1).astype(np.float32).copy()
    var_raw = raw["var_raw"].reshape(-1).astype(np.float32) * np.float32(1.3)
    pos = 0
    for cb in range(pm.n_mgau):
        for f, fl in enumerate(pm.featlen):
            n = pm.n_density * int(fl)
            blk = mean[pos:pos + n].reshape(pm.n_density, int(fl))
            A = np.eye(int(fl)) + rng.normal(0, 0.02, (int(fl), int(fl)))
            mean[pos:pos + n] = (blk @ A.T + rng.normal(0, 0.1, int(fl))).astype(np.float32).ravel()
            pos += n
    q.var, q.det = s3io.precompute_gaussians(var_raw, pm.n_mgau, pm.n_feat, pm.n_density, pm.featlen)
    q.mean = mean
    q.var, q.det = q.var.ravel(), q.det.ravel()
    return q


@pytest.mark.parametrize("kind", ["ptm", "ptm_scan", "semi", "ms"])
def test_batch_after_gaussian_update_matches_oracle(api, kind):
    """ptm: 13-dimensional streams, the tensor-core filter; ptm_scan: 12-dimensional streams, the scan."""
    from oracle import oracle
    from pocketsphinx_b200.model import synth_feats, synth_ms, synth_ptm, synth_semi
    if kind.startswith("ptm"):
        pm, raw = synth_ptm(seed=17, n_mgau=6, n_density=128, n_sen=120, featlen=12 if kind == "ptm_scan" else 13,
                            return_raw=True)
    elif kind == "semi":
        pm, raw = synth_semi(seed=17, n_sen=300, return_raw=True)
    else:
        pm, raw = synth_ms(seed=17, n_sen=200, n_density=8, return_raw=True)
    pm2 = _mllr(pm, raw, 3)
    feats = synth_feats(pm, 6, 30, seed=4)
    utts = [feats[u] for u in range(6)]
    off = api.Batch.offsets([30] * 6)
    m = api.Model(pm)
    b = api.Batch(m, 8, 200)                                   # created before the update, reused after it
    b.score_host(feats.reshape(-1, pm.sumlen), off)
    m.update_gaussians(pm2.mean, pm2.var, pm2.det)
    scr = b.score_host(feats.reshape(-1, pm.sumlen), off)
    om = oracle.OracleModel(pm2)
    for u in range(6):
        if kind.startswith("ptm"):
            want, rawl = om.score_utt(utts[u], want_raw=True)
            oracle.assert_records_equal(b.get_topn(180)[off[u]:off[u + 1]], oracle.ptm_records(rawl), "utt %d" % u)
        else:
            want = om.score_utt(utts[u])
        assert np.array_equal(scr[off[u]:off[u + 1]], want), "utterance %d" % u
    assert not np.array_equal(want, oracle.OracleModel(pm).score_utt(utts[-1]))     # the update changed the scores
    b.close(); m.close()


def test_frame_scorer_after_gaussian_update_between_utterances(api):
    from oracle import oracle
    from pocketsphinx_b200.model import synth_feats, synth_ptm
    pm, raw = synth_ptm(seed=19, n_mgau=6, n_density=64, n_sen=120, return_raw=True)
    pm2 = _mllr(pm, raw, 5)
    f = synth_feats(pm, 2, 20, seed=8)
    m = api.Model(pm)
    s = api.Mgau(m, pl_window=0)
    for model, feats in ((pm, f[0]), (pm2, f[1])):
        if model is pm2:
            m.update_gaussians(pm2.mean, pm2.var, pm2.det)
        s.reset()
        s.frame_idx = 0
        dec = oracle.OracleModel(model).decoder(n_hist=2)
        for t in range(len(feats)):
            assert np.array_equal(s.frame_eval(feats[t], t), dec.frame_eval(feats[t], t)), "frame %d" % t
            s.frame_idx = t + 1
            dec.set_frame_idx(t + 1)
        dec.close()
    s.close(); m.close()


CHECK_UPDATE = r"""
import copy, json, numpy as np
import tc_cases as tc
from oracle import oracle
from pocketsphinx_b200 import api
from pocketsphinx_b200.model import synth_feats, synth_ptm
pm = synth_ptm(seed=23, n_mgau=6, n_density=64, n_sen=120)
bad = copy.deepcopy(pm)                                  # one codeword with a variance whose bound is not finite
v = bad.var.reshape(pm.n_mgau, pm.n_feat, pm.n_density, 13).copy(); v[2, 1, 7] = 3.0e38
mu = bad.mean.reshape(v.shape).copy(); mu[2, 1, 7] += 5.0
bad.var, bad.mean = v.ravel(), mu.ravel()
utts = [u for u in synth_feats(pm, 4, 25, seed=3)]
out = {}
def step(name, m, b, model):
    tc.score_vs_oracle(api, oracle, model, utts, batch=b)
    b.tc_check()
    out[name] = b.tc_stats["rows"]
m = api.Model(pm); b = api.Batch(m, 5, 101)
step("good", m, b, pm)
m.update_gaussians(bad.mean, bad.var, bad.det); step("to_degenerate", m, b, bad)
m.update_gaussians(pm.mean, pm.var, pm.det); step("back", m, b, pm)
b.close(); m.close()
m = api.Model(bad); b = api.Batch(m, 5, 101)
step("created_degenerate", m, b, bad)
m.update_gaussians(pm.mean, pm.var, pm.det); step("updated_good", m, b, pm)
b.close(); m.close()
out["per_run"] = 100 * pm.n_mgau * pm.n_feat
print(json.dumps(out))
"""


def test_gaussian_update_switches_the_filter_off_and_on():
    """tc_ok follows the Gaussians: bounds that are not finite leave the scan kernels in charge (no filter rows), the
    update back brings the filter back, and a model created degenerate gets its filter operands on its first good
    update."""
    out = tc.child(CHECK_UPDATE)
    print(out)
    n = out["per_run"]
    assert out["good"] == n and out["to_degenerate"] == n and out["back"] == 2 * n, out
    assert out["created_degenerate"] == 0 and out["updated_good"] == n, out
