"""CPU: the filter banks under -warp_type / -warp_params (fe_tables.make_filterbank / Warp, restating fe_warp*.c and
fe_build_melfilters) against the banks inside the compiled reference's fe_t, byte for byte, on three front-end
configurations and a grid of warps that covers the parameter parsing, the clamps and the piecewise special cases."""
import warnings

import numpy as np
import pytest

from oracle import refdrv

import fe_warp_cases as wc

pytestmark = pytest.mark.skipif(not refdrv.available(), reason="compiled reference not built")

# name -> (refdrv settings, make_fe_desc arguments)
CONFIGS = {
    "en-us": ({}, {}),
    "tidigits": (dict(samprate="8000"), dict(samprate=8000, wlen=0.025, nfilt=20, lowerf=1, upperf=4000,
                                              round_filters=False, remove_dc=True, remove_noise=False, lifter=0)),
    "an4": ({}, dict(nfilt=40, lowerf=133.3334, upperf=6855.4976, transform="legacy", lifter=0, remove_noise=False)),
}
GRID = [("inverse_linear", None), ("inverse_linear", "")]                            # unset
GRID += [("inverse_linear", p) for p in ("1.0", "0.8", "0.88", "1.12", "1.2",
                                         "0.05", "0", "-3", "12", "abc",              # clamp to 0.1 / 10
                                         "0.9 2 3", "1.1\t7", "  0.95  ", "1.05xyz")]  # extra tokens, separators
GRID += [("affine", p) for p in ("0.9", "1.1 -300", "0.95 150", "0.9 1e6", "1.2 50 9", "0.01 -20")]
GRID += [("piecewise_linear", p) for p in ("0.9 0", "1.1 0", "0.9 5000", "1.1 1e6", "0.9", "1.12", "0.9 3000 8",
                                           "0.9 -5", "20 2000")]
GRID += [("inverse", "0.9"), ("linear", "1.1 -100"), ("piecewise", "0.9 2000")]         # fe_warp.c's aliases
BANK = ("spec_start", "filt_start", "filt_width", "filt_coeffs")


def _ours(mk, warp_type, warp_params):
    from pocketsphinx_b200.fe_tables import make_fe_desc
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return make_fe_desc(warp_type=warp_type, warp_params=warp_params, **mk)


def _same(ours, ref, what):
    for k in BANK:
        assert ours[k].dtype == ref[k].dtype and ours[k].shape == ref[k].shape, (what, k)
        assert ours[k].tobytes() == ref[k].tobytes(), (what, k)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_warped_banks_match_reference(name):
    kv, mk = CONFIGS[name]
    fatal = []
    for warp_type, warp_params in GRID:
        try:
            ours = _ours(mk, warp_type, warp_params)
        except ValueError:
            fatal.append((warp_type, warp_params))       # the reference ends its process here: not run
            continue
        r = wc.ref_model(name, warp_type, warp_params or None, **kv)
        _same(ours, r.fe_desc(), (name, warp_type, warp_params))
        r.close()
    # on tidigits a piecewise a of 20 (clamped to 10) with F at 2000 Hz puts a * F far above Nyquist: the final piece
    # runs backwards and the coefficient pass rejects a filter.  (F clamped to Nyquist, "0.9 5000" and "1.1 1e6", makes
    # every edge NaN; those banks are compared above, NaN coefficients included.)
    assert fatal == ([("piecewise_linear", "20 2000")] if name == "tidigits" else [])
    # the grid's warps change the bank
    plain = _ours(mk, "inverse_linear", None)
    assert _ours(mk, "inverse_linear", "0.8")["filt_coeffs"].tobytes() != plain["filt_coeffs"].tobytes()
    assert _ours(mk, "piecewise_linear", "1.12")["spec_start"].tobytes() != plain["spec_start"].tobytes()


def test_warps_that_end_the_reference_are_refused():
    """Under these warps the reference's own filter pass rejects a filter and ends the process (E_FATAL in
    fe_build_melfilters): with -round_filters yes, a b of -Nyquist takes the low edges below -700 Hz, where the mel
    scale is NaN, and (int) of NaN puts the rounded edges at INT_MIN DFT points; on tidigits a piecewise a * F far
    above Nyquist leaves a filter whose first point lies past its right edge.  The restatement raises ValueError
    instead; the reference is not run on them."""
    for name, warp_type, warp_params in (("en-us", "affine", "1.0 -1e6"), ("an4", "affine", "1 -8000"),
                                         ("tidigits", "piecewise_linear", "20 2000")):
        with pytest.raises(ValueError, match="range does not match"):
            _ours(CONFIGS[name][1], warp_type, warp_params)


def test_parameter_parsing_and_clamps():
    from pocketsphinx_b200.fe_tables import Warp
    f = np.float32
    assert Warp("inverse_linear", None).neutral and Warp("inverse_linear", "").neutral
    assert Warp("inverse_linear", "0").a == f(0.1) and Warp("inverse_linear", "99").a == f(10)
    assert Warp("inverse_linear", "0.9 5").a == f(0.9)
    w = Warp("affine", "0.9", 16000)
    assert (w.a, w.b) == (f(0.9), f(0))                                  # missing tokens are 0
    assert Warp("affine", "1 -1e9", 16000).b == f(-8000) and Warp("affine", "1 1e9", 8000).b == f(4000)
    w = Warp("piecewise_linear", "0.9 0", 16000)
    assert w.b == f(16000) * f(0.85)                                     # F = 0: 0.85 x the sampling rate
    assert Warp("piecewise_linear", "0.9 1e9", 16000).b == f(8000)
    assert Warp("piecewise_linear", "0.9 -1", 16000).b == f(16000) * f(0.85)
    with pytest.raises(ValueError, match="unimplemented warping function"):
        Warp("bilinear", "0.9")


def test_doublebw_out_of_range_banks_match_reference():
    """fe_build_melfilters refuses doublebw edges outside [0, Nyquist], and fe_init ignores the refusal: the bank
    stays as calloc left it, every filter empty.  The restatement gives those arrays (and warns)."""
    from pocketsphinx_b200.fe_tables import make_fe_desc
    kv, mk = CONFIGS["tidigits"]                    # lowerf 1 Hz: the doubled band starts below 0 Hz, warped or not
    for wp in (None, "0.9", "1.2"):
        name = "tidigits"
        with pytest.warns(UserWarning, match="every mel filter is empty"):
            ours = make_fe_desc(doublebw=True, warp_params=wp, **mk)
        assert (ours["filt_width"] == 0).all() and ours["filt_coeffs"].size == 0
        r = wc.ref_model(name, "inverse_linear", wp, doublebw="yes", **kv)
        _same(ours, r.fe_desc(), (name, wp))
        r.close()
    # in range, doublebw banks are ordinary ones
    ours = make_fe_desc(doublebw=True, warp_params="1.1")
    assert (ours["filt_width"] > 0).all()
    r = wc.ref_model("en-us", "inverse_linear", "1.1", doublebw="yes")
    _same(ours, r.fe_desc(), "en-us doublebw 1.1")
    r.close()


def test_unknown_warp_type_is_refused():
    """fe_warp_set fails fe_init for a name outside fe_warp.c's tables (the reference is not run on it: its process
    does not survive the failed init)."""
    from pocketsphinx_b200.fe_tables import make_fe_desc
    with pytest.raises(ValueError, match="unimplemented warping function"):
        make_fe_desc(warp_type="log", warp_params="0.9")


def test_filters_without_dft_points_keep_the_calloc_form():
    """A filter no DFT point falls in (its left edge above the last point) keeps spec_start -1, filt_start 0 and
    width 0; fe_init's upper-frequency check keeps the reference's own banks clear of it, so this pins the builder."""
    from pocketsphinx_b200.fe_tables import make_filterbank
    b = make_filterbank(samprate=8000, fft_size=256, nfilt=20, lowerf=1, upperf=6000, round_filters=False)
    empty = b["filt_width"] == 0
    assert empty.any() and (b["spec_start"][empty] == -1).all() and (b["filt_start"][empty] == 0).all()
    assert b["filt_coeffs"].size == int(b["filt_width"].sum())
