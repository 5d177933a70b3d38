"""CPU, build container only (skipped without oracle/_ref): tied-mixture models of the shapes the senone kernels take
their less common paths at, written as Sphinx-3 files and loaded by the UNMODIFIED reference, must score exactly like
the C oracle.  This pins the oracle -- which tests/test_gpu_senone_paths.py holds the device to -- against the
reference at:

- a clustered (4-bit) PTM sendump, odd and even senone counts (the nibble quirk of ptm_mgau.c:376-377);
- -logbase 1.0000325 and 1.000031, whose add tables peak at 21 and 22 (the 16x2 kernels' bias bound);
- PTM and semi-continuous -topn 1, 2 and 8;
- PTM with 1, 2, 4 and 8 streams, as -svspec selects them from 1s_c_d_dd.

The reference derives a PTM model's senone -> codebook map from its mdef (CI senones first, then runs per CI
phone), so the other sen2cb layouts of the device tests (codebooks of 1-3 senones, one codebook, n_mgau == n_sen)
cannot be written for it; those cases rest on the oracle alone."""
import numpy as np
import pytest

from oracle import oracle, refdrv
from pocketsphinx_b200 import s3io
from pocketsphinx_b200.model import PackedModel, make_logadd8, synth_feats, synth_ptm, synth_semi

pytestmark = pytest.mark.skipif(not refdrv.available(), reason="oracle/_ref/libpsref.so not built")

FEAT_PTM = "-feat 1s_c_d_dd\n-svspec 0-12/13-25/26-38\n-cmn batch\n-agc none\n"
FEAT_SC = "-feat s2_4x\n-cmn batch\n-agc none\n"


def _feat_svspec(spec):
    return "-feat 1s_c_d_dd\n" + ("-svspec %s\n" % spec if spec else "") + "-cmn batch\n-agc none\n"


def _ref_model(tmp_path, pm, raw, feat_params, **kv):
    d = str(tmp_path / "model")
    if pm.kind == "ptm":
        sen2ci, n_ci = pm.sen2cb, pm.n_mgau
    else:
        sen2ci = np.concatenate([np.repeat(np.arange(10), 3), np.arange(pm.n_sen - 30) % 10]).astype(np.int32)
        n_ci = 10
    s3io.write_model_dir(d, kind=pm.kind, n_mgau=pm.n_mgau, n_feat=pm.n_feat, n_density=pm.n_density,
                         featlen=pm.featlen, mean=raw["mean"], var_raw=raw["var_raw"], tp_float=raw["tp_float"],
                         sen2ci=sen2ci, n_ci=n_ci, n_emit=3, n_ci_sen=n_ci * 3, mixw_q=raw["mixw_q"],
                         mixw_cb=raw.get("mixw_cb"), feat_params=feat_params)
    return refdrv.RefModel(d, **{k: str(v) for k, v in kv.items()})


def _check_scores(ref, pm, name, n_utt=3, T=23):
    """The reference's arrays as it loaded them (its own log base) drive the oracle; both score the same features."""
    got = PackedModel.from_dict(ref.packed())
    for k in ("mixw", "mixw_cb", "sen2cb"):
        assert np.array_equal(getattr(got, k), getattr(pm, k)), "%s: %s differs after the reference loaded it" % (name, k)
    om = oracle.OracleModel(got)
    feats = synth_feats(pm, n_utt, T, seed=7)
    feats[n_utt - 1, 5:9] *= np.float32(40)          # frames far from every Gaussian
    for u in range(n_utt):
        want = ref.score(feats[u])
        have = om.score_utt(feats[u])
        bad = np.argwhere(have != want)
        assert bad.size == 0, "%s utt %d: first mismatch (frame, senone) %s: oracle %s reference %s" % (
            name, u, bad[0].tolist(), have[tuple(bad[0])], want[tuple(bad[0])])
    return got


@pytest.mark.parametrize("n_sen", [201, 200])
def test_ptm_four_bit_sendump(tmp_path, n_sen):
    pm, raw = synth_ptm(seed=11, n_mgau=6, n_density=64, n_sen=n_sen, four_bit=True, return_raw=True)
    ref = _ref_model(tmp_path, pm, raw, FEAT_PTM)
    assert ref.kind == "ptm" and ref.mixw_4bit and ref.n_sen == n_sen
    # the quirk is observable only if some byte's low bit disagrees with its senone's parity
    b = pm.mixw.reshape(pm.n_feat, pm.n_density, -1)
    assert ((b & 1) == 0).any() and ((b & 1) == 1).any()
    _check_scores(ref, pm, "ptm 4-bit n_sen %d" % n_sen)
    ref.close()


@pytest.mark.parametrize("base,tab_max", [(1.0000325, 21), (1.000031, 22)])
@pytest.mark.parametrize("kind", ["ptm", "s2_semi"])
def test_logbase_add_table(tmp_path, kind, base, tab_max):
    if kind == "ptm":
        pm, raw = synth_ptm(seed=12, n_mgau=6, n_density=64, n_sen=150, return_raw=True)
        feat = FEAT_PTM
    else:
        pm, raw = synth_semi(seed=12, n_sen=150, return_raw=True)
        feat = FEAT_SC
    ref = _ref_model(tmp_path, pm, raw, feat, logbase=base)
    got = _check_scores(ref, pm, "%s logbase %s" % (kind, base))
    assert np.array_equal(got.logadd8, make_logadd8(base=base)) and int(got.logadd8.max()) == tab_max
    ref.close()


@pytest.mark.parametrize("topn", [1, 2, 8])
@pytest.mark.parametrize("kind", ["ptm", "s2_semi"])
def test_topn_widths(tmp_path, kind, topn):
    if kind == "ptm":
        pm, raw = synth_ptm(seed=13, n_mgau=6, n_density=64, n_sen=150, topn=topn, return_raw=True)
        feat = FEAT_PTM
    else:
        pm, raw = synth_semi(seed=13, n_sen=150, topn=topn, return_raw=True)
        feat = FEAT_SC
    ref = _ref_model(tmp_path, pm, raw, feat, topn=topn)
    assert ref.topn == topn
    got = _check_scores(ref, pm, "%s topn %d" % (kind, topn))
    assert got.topn == topn
    ref.close()


@pytest.mark.parametrize("featlens,svspec", [
    ((39,), None),
    ((13, 13), "0-12/13-25"),
    ((4, 4, 4, 4), "0-3/4-7/8-11/12-15"),
    ((4,) * 8, "/".join("%d-%d" % (4 * i, 4 * i + 3) for i in range(8))),
], ids=["1", "2", "4", "8"])
def test_ptm_stream_counts(tmp_path, featlens, svspec):
    pm, raw = synth_ptm(seed=14, n_mgau=5, n_density=32, n_sen=120, featlens=featlens, return_raw=True)
    ref = _ref_model(tmp_path, pm, raw, _feat_svspec(svspec))
    assert ref.n_feat == len(featlens) and ref.featlen == list(featlens)
    _check_scores(ref, pm, "ptm %d streams" % len(featlens))
    ref.close()
