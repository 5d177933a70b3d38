"""CPU, build container (needs oracle/_ref/libpsref_fx.so = `make -C oracle fx`): the oracle's
restatement of the FIXED_POINT build's PTM arithmetic (SURVEY A.1.11: Q12 features and means,
FIXMUL truncated to 32 bits, GMMSUB as gcc compiles it, early exits that are not result-neutral)
against the reference compiled with -DFIXED_POINT, on its own features of goforward.raw.  This pins
the oracle for the fixed-point kernels (tests/test_gpu_fixed_point.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import refdrv

from conftest import fx_case, golden

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FX = os.path.join(os.path.dirname(refdrv.LIB_PATH), "libpsref_fx.so")
needs_fx = pytest.mark.skipif(not os.path.exists(FX), reason="oracle/_ref/libpsref_fx.so not built (make -C oracle fx)")


@pytest.mark.parametrize("name", ["en_us", "tidigits"])
def test_fixed_point_oracle_matches_committed_fixture(name):
    """Runs anywhere: the restatement against tests/golden/fx_*.npz (the FIXED_POINT reference's features,
    top-N lists and scores on goforward.raw)."""
    from oracle import oracle
    pm, feats, want, want_topn = fx_case(name)
    got, topn = oracle.OracleModel(pm).score_utt(feats, want_topn=True)
    assert np.array_equal(topn, want_topn) and np.array_equal(got, want)


DUMP = r"""
import sys, numpy as np
sys.path.insert(0, %r)
from oracle import refdrv
ref = refdrv.RefModel(%r)
pcm = np.fromfile(%r, np.int16)
feats = ref.featurize(pcm)                       # mfcc_t = int32 (Q12) in this build, carried as 4-byte words
scr, topn = ref.score(feats, want_topn=True)
pk = ref.packed()
np.savez(%r, feats=feats.view(np.int32), senscr=scr, topn=topn,
         mean=ref.export("mean", np.int32), var=ref.export("var", np.int32), det=ref.export("det", np.int32))
"""


@needs_fx
def test_fixed_point_semi_oracle_matches_fixed_point_reference(tmp_path):
    """The semi-continuous back-end (tidigits, 4-bit clustered weights) in the fixed-point build."""
    from oracle import oracle
    from pocketsphinx_b200.model import PackedModel
    ref_dir = os.path.dirname(refdrv.LIB_PATH)
    out = str(tmp_path / "fxs.npz")
    code = DUMP % (ROOT, os.path.join(ref_dir, "model", "tidigits_hmm"), os.path.join(ref_dir, "data", "goforward.raw"), out)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, PSREF_LIB=FX), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    fx = np.load(out)
    pm = PackedModel.load(os.path.join(HERE, "golden", "tidigits_sc_model.npz"))
    pm.mean, pm.var, pm.det = fx["mean"].view(np.float32), fx["var"].view(np.float32), fx["det"].view(np.float32)
    pm.fixed_point = 1
    got, topn = oracle.OracleModel(pm).score_utt(fx["feats"].view(np.float32), want_topn=True)
    assert np.array_equal(topn, fx["topn"]) and np.array_equal(got, fx["senscr"])


@needs_fx
def test_fixed_point_ptm_oracle_matches_fixed_point_reference(tmp_path):
    from oracle import oracle
    from pocketsphinx_b200.model import PackedModel
    ref_dir = os.path.dirname(refdrv.LIB_PATH)
    out = str(tmp_path / "fx.npz")
    code = DUMP % (ROOT, os.path.join(ref_dir, "model", "en-us"), os.path.join(ref_dir, "data", "goforward.raw"), out)
    env = dict(os.environ, PSREF_LIB=FX)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    fx = np.load(out)
    pm = PackedModel.load(os.path.join(HERE, "golden", "en_us_ptm_model.npz"))     # mixw, sen2cb, add table: same in both builds
    assert fx["mean"].size == pm.mean.size
    pm.mean, pm.var, pm.det = fx["mean"].view(np.float32), fx["var"].view(np.float32), fx["det"].view(np.float32)
    pm.fixed_point = 1
    om = oracle.OracleModel(pm)
    got, topn = om.score_utt(fx["feats"].view(np.float32), want_topn=True)
    assert np.array_equal(topn, fx["topn"]), "top-N lists differ first in frame %d" % int(
        np.argwhere((topn != fx["topn"]).reshape(len(topn), -1).any(1))[0, 0])
    assert np.array_equal(got, fx["senscr"])
    # and the two builds really differ (otherwise this test would prove nothing)
    flt = golden("en_us_goforward.npz")["senscr"]
    assert (got != flt).mean() > 0.2
