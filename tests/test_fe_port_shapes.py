"""CPU, skipped without the compiled reference: oracle/fe_port.py (the numpy restatement of the front end the
device front end is checked against) bit for bit against the reference run live, at every shape of
tests/fe_shape_cases.GRID -- sample rates of 8 to 32 kHz, odd frame sizes, 256- to 1024-point FFTs, frame shifts of
80 to 320 samples, pre-emphasis off, 64 filters, 1 to 32 cepstra -- on lengths around each shape's own frame
boundaries, speech and noise.  Also: the tables fe_tables.make_fe_desc builds are the reference's own there, and
the reference driver sizes its output by the shape's frame shift."""
import numpy as np
import pytest

import fe_shape_cases as sc
from oracle import fe_port, refdrv
from pocketsphinx_b200.fe_tables import make_fe_desc

pytestmark = pytest.mark.skipif(not refdrv.available(), reason="oracle/_ref/libpsref.so not built")

TABLES = ("hamming", "ccc", "sss", "spec_start", "filt_start", "filt_width", "filt_coeffs", "mel_cosine", "lifter")
SCALARS = ("frame_size", "frame_shift", "fft_size", "fft_order", "n_filt", "n_cep", "remove_dc", "remove_noise",
           "transform", "lifter_val", "window", "cmn", "alpha", "sqrt_inv_n", "sqrt_inv_2n")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("entry", sc.GRID, ids=[e["id"] for e in sc.GRID])
def test_fe_port_matches_reference(entry, tmp_path):
    ref = sc.ref_model(entry, tmp_path)
    d = ref.fe_desc()
    assert (d["frame_size"], d["frame_shift"], d["fft_size"]) == entry["shape"]
    mk = make_fe_desc(**entry["mk"])
    for k in SCALARS:
        assert mk[k] == d[k], k
    for k in TABLES:
        a, b = np.asarray(mk[k]), np.asarray(d[k])
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), k
    nc = d["n_cep"]
    for pcm in sc.utterances(entry):
        what = "%s, %d samples" % (entry["id"], len(pcm))
        want_c = ref.mfcc(pcm)
        got_c = fe_port.cepstra(d, fe_port.mfspec(d, pcm))
        assert got_c.shape == want_c.shape == (fe_port.n_frames(d, len(pcm)), nc), what
        assert np.array_equal(_bits(got_c), _bits(want_c)), "cepstra, " + what
        got = fe_port.featurize(d, pcm)
        assert got.shape == (len(got_c), 3 * nc), what
        if len(pcm):
            want = ref.featurize_fresh(pcm)
            assert np.array_equal(_bits(got), _bits(want)), "features, " + what
    ref.close()


def test_reference_driver_keeps_every_frame_at_short_shifts():
    """RefModel.mfcc / featurize size their output by the front end's own frame shift: at 8 kHz (80 samples)
    a cap sized for 160 would keep 72 of the 111 frames of 8960 samples."""
    e = sc.BY_ID["8k"]
    ref = sc.ref_model(e, None)
    pcm = sc.goforward()[:8960]
    n = fe_port.n_frames(ref.fe_desc(), len(pcm))
    assert n == 111 > len(pcm) // 160 + 16
    assert len(ref.mfcc(pcm)) == n and len(ref.featurize_fresh(pcm)) == n
    ref.close()
