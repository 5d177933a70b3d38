"""CPU: the C-ABI library builds, loads, and exports every symbol include/psb200.h declares."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from pocketsphinx_b200 import _lib
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "psb200.h")).read()
    declared = set(re.findall(r"\b(psb_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"psb_status_e"}
    bound = {name for name, _, _ in _lib.SYMBOLS}
    assert declared == bound, (declared ^ bound)
    for name in declared:
        assert hasattr(L, name)
    assert L.psb_abi_version() == 2


def test_hmm_struct_is_88_bytes():
    from pocketsphinx_b200.api import HMM_DTYPE
    assert HMM_DTYPE.itemsize == 88
    assert HMM_DTYPE.fields["bestscore"][1] == 68 and HMM_DTYPE.fields["frame"][1] == 76


def test_no_cpu_fallback_without_gpu():
    """Without a device the product must fail loudly, not compute on the CPU."""
    import pytest
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.model import synth_ptm
    if api.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(api.PsbError):
        api.Model(synth_ptm(n_density=32, n_sen=200))


def test_no_fused_multiply_add_in_distance_kernels():
    """The Gaussian exponent must round the product and the subtraction separately
    (ptm_mgau.c:64-69).  ptxas contracts mul+add pairs -- including packed mul.rn.f32x2 /
    add.rn.f32x2 even with explicit .rn -- so the build is checked: no FFMA / FFMA2 / HFMA-free
    distance kernels only (a contracted FMA would silently break bit-exactness)."""
    import shutil
    import subprocess
    import pytest
    from pocketsphinx_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    fn, bad = None, []
    for line in sass.splitlines():
        if "Function :" in line:
            fn = line.split("Function :")[1].strip()
        elif fn and any(k in fn for k in ("topn", "ms_dist", "semi_dist", "ptm_tc", "ptm_wgmma", "ptm_fixup")) and "FFMA" in line:
            bad.append((fn[:60], line.strip()[:80]))
    assert not bad, bad[:5]
    assert "HGMMA" in sass, "warpgroup tensor-core filter missing from the build"


def test_header_is_plain_c_and_the_example_compiles(tmp_path):
    """include/psb200.h must stay a C header (the reference is C): the example host program is
    compiled as C11 with -Wall -Wextra -pedantic -Werror."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("gcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([gcc, "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(root, "include"),
                        "-c", os.path.join(root, "integration", "example_batch.c"), "-o", str(tmp_path / "example.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_fe_create_rejects_bad_descriptors_before_touching_the_device():
    """Argument errors are reported (return < 0 + psb_last_error) without a GPU."""
    import ctypes as C
    from pocketsphinx_b200 import _lib
    from pocketsphinx_b200.fe_tables import make_fe_desc
    L = _lib.lib()
    d = make_fe_desc()
    keep = {}

    def desc(**over):
        x = _lib.FeDesc()
        for k in ("frame_size", "frame_shift", "fft_size", "fft_order", "n_filt", "n_cep", "remove_dc", "remove_noise",
                  "transform", "lifter_val", "window", "cmn"):
            setattr(x, k, int(over.get(k, d[k])))
        x.pre_emphasis_alpha, x.sqrt_inv_n, x.sqrt_inv_2n = float(d["alpha"]), float(d["sqrt_inv_n"]), float(d["sqrt_inv_2n"])
        for k in ("hamming", "ccc", "sss", "spec_start", "filt_start", "filt_width", "filt_coeffs", "mel_cosine", "lifter"):
            keep[k] = d[k]
            setattr(x, k, None if over.get(k, 1) is None else d[k].ctypes.data)
        x.n_coeffs = int(over.get("n_coeffs", d["filt_coeffs"].size))
        return x

    h = C.c_void_p()
    for over, word in ((dict(fft_size=500), "power of two"), (dict(transform=7), "transform"), (dict(cmn=2), "cmn"),
                       (dict(window=2), "1s_c_d_dd"), (dict(hamming=None), "missing table"), (dict(n_coeffs=3), "n_coeffs"),
                       (dict(n_filt=200), "n_cep <= n_filt")):
        rc = L.psb_fe_create(C.byref(desc(**over)), 0, C.byref(h))
        assert rc < 0 and word in L.psb_last_error().decode(), (over, L.psb_last_error())


def test_model_create_refuses_a_semi_model_with_several_codebooks_before_touching_the_device():
    """A semi-continuous model has one codebook (the reference refuses others, s2_semi_mgau.c:1269): psb_model_create
    says so without a GPU."""
    import copy
    import pytest
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.model import synth_semi
    pm = copy.copy(synth_semi(n_density=64, n_sen=100))
    pm.n_mgau = 2
    with pytest.raises(api.PsbError, match="one codebook"):
        api.Model(pm)
