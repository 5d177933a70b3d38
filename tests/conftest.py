import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def golden(name):
    from pocketsphinx_b200.model import load_npz
    return load_npz(os.path.join(GOLDEN, name))


@pytest.fixture(scope="session")
def en_us():
    from pocketsphinx_b200.model import PackedModel
    return PackedModel.load(os.path.join(GOLDEN, "en_us_ptm_model.npz"))


@pytest.fixture(scope="session")
def tidigits():
    from pocketsphinx_b200.model import PackedModel
    return PackedModel.load(os.path.join(GOLDEN, "tidigits_sc_model.npz"))


@pytest.fixture(scope="session")
def an4():
    from pocketsphinx_b200.model import PackedModel
    return PackedModel.load(os.path.join(GOLDEN, "an4_cont_model.npz"))


def fx_case(name):
    """The FIXED_POINT build's golden case `name` ("en_us" PTM, "tidigits" semi-continuous, 4-bit weights):
    (PackedModel with fixed_point = 1 and int32 Gaussians carried in float32-typed arrays, Q12 features
    viewed as float32, expected int16 scores, expected top-N lists).  tests/golden/fx_<name>.npz holds
    differences from the float build's goldens (oracle/make_golden.py:make_fixed_point)."""
    from pocketsphinx_b200.model import PackedModel
    gm, gg = {"en_us": ("en_us_ptm_model.npz", "en_us_goforward.npz"),
              "tidigits": ("tidigits_sc_model.npz", "tidigits_goforward.npz")}[name]
    fx = golden("fx_%s.npz" % name)
    pm = PackedModel.load(os.path.join(GOLDEN, gm))
    mean = (pm.mean.astype(np.float32) * np.float32(4096)).astype(np.int32) + fx["dmean"]
    var = pm.var.astype(np.int32) + fx["dvar"]
    det = pm.det.astype(np.int32)
    pm.mean, pm.var, pm.det = mean.view(np.float32), var.view(np.float32), det.view(np.float32)
    pm.fixed_point = 1
    senscr = (golden(gg)["senscr"].astype(np.int32) + fx["dsenscr"]).astype(np.int16)
    return pm, np.ascontiguousarray(fx["feats"]).view(np.float32), senscr, fx["topn"]


def hmm_view(raw):
    """uint8 [..., 88] golden dump -> structured hmm_t array."""
    from oracle.oracle import HMM_DTYPE
    return np.ascontiguousarray(raw).view(HMM_DTYPE).reshape(raw.shape[:-1])


HMM_FIELDS = ["score", "history", "out_score", "out_history", "ssid", "senid", "bestscore", "tmatid",
              "frame", "mpx", "n_emit_state"]


def assert_hmm_equal(a, b, n_emit, what=""):
    for k in HMM_FIELDS:
        x, y = a[k], b[k]
        if k in ("score", "history", "senid"):
            x, y = x[..., :n_emit], y[..., :n_emit]
        assert np.array_equal(x, y), "%s: hmm field %s differs at %s" % (
            what, k, np.argwhere(x != y)[:5].tolist())


def beam_case(n_emit, n, seed, frame0=7):
    """n plain hmm_t drawn from the golden hmm_vit_eval records, all entered with spread-out scores; nine in ten active
    in frame0 (frame field), the others not (never touched by a beam sweep)."""
    g = golden("hmm_vit_eval.npz")
    tp, sseq = g["n%d_tp" % n_emit], g["n%d_sseq" % n_emit]
    hm = hmm_view(g["n%d_before" % n_emit]).copy()
    hm = hm[hm["mpx"] == 0]
    rng = np.random.default_rng(seed)
    hm = np.ascontiguousarray(hm[rng.integers(0, len(hm), n)])
    hm["score"][:, 0] = -rng.integers(0, 4000, n).astype(np.int32)          # every instance entered, scores spread out
    hm["frame"] = frame0
    hm["frame"][rng.random(n) < 0.1] = frame0 - 1                              # not active: never touched
    hm["frame"][rng.random(n) < 0.05] = -1
    n_sen = len(g["n%d_senscr" % n_emit])
    return tp, sseq, hm, n_sen
