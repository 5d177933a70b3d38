"""CPU: the crafted inputs of tests/tc_cases.py land where they are meant to in the tensor-core filter's decision
(the numpy mirror of psb_ptm_tc.cu's threshold, lane storage, byte list and certainty tests)."""
import numpy as np
import pytest

import tc_cases as tc


def _on_frame(name):
    """The decision on the crafted frame alone (every crafted pair sits on its mean)."""
    pm, utts, _ = tc.case(name)
    feats = np.concatenate(utts)
    # the crafted frame is the most common row
    rows, counts = np.unique(feats, axis=0, return_counts=True)
    return tc.decide(pm, rows[np.argmax(counts)][None, :])


def test_lane_overflow_is_flagged_and_the_walk_stops_at_the_cap():
    d = _on_frame("lane_over_256")
    assert d["over"][0, :6].all() and not d["listed"][0, :6].any()
    assert (d["n"][0, :6] == tc.TC_CAP).all() and (d["n_h1"][0, :6] == 0).all()      # would look "listed" without it


@pytest.mark.parametrize("nd", [64, 128, 256])
def test_split_lists_fill_each_half_as_laid_out(nd):
    d = _on_frame("split_%d" % nd)
    for k, (a, b) in enumerate(tc.SPLITS):
        assert (d["n_h0"][0, k], d["n_h1"][0, k]) == (a, b), (nd, k)
        assert d["listed"][0, k] == (a + b <= tc.TC_CAP) and not d["over"][0, k]
        if d["listed"][0, k]:
            assert d["fail_gap"][0, k] and not d["certain"][0, k]


@pytest.mark.parametrize("nd", [64, 128, 256])
def test_duplicates_take_every_codeword(nd):
    d = _on_frame("dup_%d" % nd)
    assert (d["n"][0, :12] > tc.TC_CAP).all() or d["over"][0, :12].all()
    assert not d["listed"][0, :12].any()


@pytest.mark.parametrize("nd", [128, 256])
def test_1024_boundary_fails_only_the_straddle_test(nd):
    d = _on_frame("boundary_%d" % nd)
    assert d["listed"][0, :12].all() and d["fail_straddle"][0, :12].all()
    assert not (d["fail_gap"] | d["fail_sign"] | d["fail_saturation"])[0, :12].any()


@pytest.mark.parametrize("nd", [64, 256])
def test_positive_exponents_fail_the_sign_guard_and_fill_the_work_list(nd):
    pm, utts, _ = tc.case("positive_%d" % nd)
    feats = np.concatenate(utts)
    total, K = len(feats), pm.n_mgau * pm.n_feat
    assert total * K >= 16384
    d = tc.decide(pm, feats)
    doubt = ~d["certain"]
    cap = max(4096, total * K // 4) * 9 // 8                # psb_launch_ptm_tc's work-list capacity
    assert doubt.sum() > cap * 1.5
    on = _on_frame("positive_%d" % nd)
    listed = on["listed"][0]
    assert listed.any() and on["fail_sign"][0][listed].all()
    assert (on["listed"][0] & (on["n_h0"][0] > 0) & (on["n_h1"][0] > 0)).any()      # split lists among them
    assert (~on["listed"][0]).any()                                                   # and all-codeword rows


def test_saturated_features_fail_the_saturation_guard():
    pm, utts, _ = tc.case("saturation_256")
    d = tc.decide(pm, np.concatenate(utts))
    assert d["fail_saturation"].sum() > 100
