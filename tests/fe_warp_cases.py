"""TEST INFRASTRUCTURE: the compiled reference under -warp_type / -warp_params, shared by
tests/test_fe_warp_tables.py (CPU: the filter banks) and tests/test_gpu_fe_warp.py (device features and decodes).

The reference keeps each warp type's parameters in process-global statics (fe_warp_*.c: params, is_neutral, p_str) and
*_set_parameters returns early when the string equals the last one set for that type.  So in one process "0.9",
then unset, then "0.9" builds a neutral bank the third time, and a string set again at another sampling rate keeps
the clamps and the piecewise line of the first rate.  fresh() keeps every reference run clear of that: before a
string this process already set last for the type, it sets another one, so each run builds what fe_init builds when
the string is newly set -- which is what fe_tables.make_filterbank restates."""
import os

from oracle import refdrv

REF = os.path.dirname(refdrv.LIB_PATH)
MODELS = {"en-us": "en-us", "tidigits": "tidigits_hmm", "an4": "an4_ci_cont"}
_ALIAS = {"inverse": "inverse_linear", "linear": "affine", "piecewise": "piecewise_linear"}
_last = {}           # warp type -> the string this process set last (p_str starts as "")


def model_dir(name):
    return os.path.join(REF, "model", MODELS[name])


def fresh(warp_type, warp_params):
    """Make the next reference fe_init parse warp_params for warp_type anew (see above)."""
    if warp_params is None or warp_params == "":
        return                                    # NULL (refdrv maps "" to NULL): neutral, p_str untouched
    kind = _ALIAS.get(warp_type, warp_type)
    if _last.get(kind, "") == warp_params:
        other = "0.5" if warp_params != "0.5" else "0.6"
        refdrv.RefModel(model_dir("an4"), warp_type=kind, warp_params=other).close()
    _last[kind] = warp_params


def ref_model(name, warp_type="inverse_linear", warp_params=None, **kv):
    """refdrv.RefModel of one of MODELS under a warp, parsed anew."""
    fresh(warp_type, warp_params)
    kv = dict(kv, warp_type=warp_type)
    if warp_params is not None:
        kv["warp_params"] = warp_params
    return refdrv.RefModel(model_dir(name), **kv)


def ref_decode(hmm, lm, dic, pcm, warp_type="inverse_linear", warp_params=None, **kv):
    """refdrv.decode under a warp, parsed anew."""
    fresh(warp_type, warp_params)
    kv = dict(kv, warp_type=warp_type)
    if warp_params is not None:
        kv["warp_params"] = warp_params
    return refdrv.decode(hmm, lm, dic, pcm, **kv)
