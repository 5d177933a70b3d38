"""CPU, build container only (skipped without oracle/_ref): continuous models of the shapes the ms batch kernels
take their less common paths at, written as Sphinx-3 files and loaded by the UNMODIFIED reference, must score
exactly like the C oracle.  This pins the oracle -- which tests/test_gpu_ms_paths.py holds the device to -- against
the reference at three 13-dimensional streams, the four s2_4x streams (12/24/3/12), top-N 1, and top-N above the
number of Gaussians (ms_mgau_init clamps it, and compute_dist_all lists every Gaussian in order).

The reference's continuous (.cont.) loader ties senone s to codebook s.  Tied codebooks with an arbitrary sen2cb and
the single shared codebook with transposed weights are not covered here: the device tests of those shapes rest on
the oracle alone."""
import numpy as np
import pytest

from oracle import oracle, refdrv
from pocketsphinx_b200 import s3io
from pocketsphinx_b200.model import PackedModel, synth_feats, synth_ms

pytestmark = pytest.mark.skipif(not refdrv.available(), reason="oracle/_ref/libpsref.so not built")

FEAT_3x13 = "-feat 1s_c_d_dd\n-svspec 0-12/13-25/26-38\n-cmn batch\n-agc none\n"
FEAT_S2_4X = "-feat s2_4x\n-cmn batch\n-agc none\n"
FEAT_CONT = "-feat 1s_c_d_dd\n-cmn batch\n-agc none\n"


def _ref_model(tmp_path, pm, raw, feat_params, **kv):
    d = str(tmp_path / "model")
    sen2ci = np.concatenate([np.repeat(np.arange(10), 3), np.arange(pm.n_sen - 30) % 10]).astype(np.int32)
    s3io.write_model_dir(d, kind="ms", n_mgau=pm.n_mgau, n_feat=pm.n_feat, n_density=pm.n_density,
                         featlen=pm.featlen, mean=raw["mean"], var_raw=raw["var_raw"], tp_float=raw["tp_float"],
                         sen2ci=sen2ci, n_ci=10, n_emit=3, n_ci_sen=30, mixw_float=raw["mixw_float"],
                         feat_params=feat_params)
    return refdrv.RefModel(d, senmgau=".cont.", **kv)


@pytest.mark.parametrize("name,kw,feat_params,ref_kw", [
    ("three_streams", dict(featlens=(13, 13, 13), n_density=4, topn=2), FEAT_3x13, {}),
    ("s2_4x", dict(featlens=(12, 24, 3, 12), n_density=4, topn=4), FEAT_S2_4X, {}),
    ("s2_4x_aw3", dict(featlens=(12, 24, 3, 12), n_density=8, topn=2, aw=3), FEAT_S2_4X, dict(aw="3")),
    ("topn1", dict(n_density=8, topn=1), FEAT_CONT, {}),
    ("topn_above_nd", dict(n_density=3, topn=4), FEAT_CONT, {}),
])
def test_ms_shapes_through_reference(tmp_path, name, kw, feat_params, ref_kw):
    pm, raw = synth_ms(seed=31, n_sen=120, return_raw=True, **kw)
    ref = _ref_model(tmp_path, pm, raw, feat_params, topn=str(pm.topn), **ref_kw)
    assert (ref.kind, ref.n_sen, ref.n_mgau, ref.n_feat, ref.n_density) == ("ms", 120, 120, pm.n_feat, pm.n_density)
    assert ref.featlen == [int(x) for x in pm.featlen] and ref.aw == pm.aw
    got = PackedModel.from_dict(ref.packed())
    for k in ("mean", "var", "det", "mixw", "sen2cb", "logadd_ms"):
        assert np.array_equal(getattr(got, k), getattr(pm, k)), "model array %s differs after the reference loaded it" % k
    om = oracle.OracleModel(pm)
    feats = synth_feats(pm, 3, 23, seed=7)
    feats[2, 5:9] *= np.float32(40)                  # frames far from every Gaussian: large negative distances
    for u in range(3):
        want = ref.score(feats[u])
        got_scr = om.score_utt(feats[u])
        bad = np.argwhere(got_scr != want)
        assert bad.size == 0, "%s utt %d: first mismatch (frame, senone) %s: oracle %s reference %s" % (
            name, u, bad[0].tolist(), got_scr[tuple(bad[0])], want[tuple(bad[0])])
    ref.close()
