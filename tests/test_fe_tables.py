"""CPU: the Python mirror of the reference front end's initialisation (fe_tables.make_fe_desc)
against the tables inside the compiled reference's fe_t, bit for bit; frame counting."""
import numpy as np

from oracle import fe_golden


def test_fe_tables_match_reference():
    from pocketsphinx_b200.fe_tables import make_fe_desc, n_frames
    m = fe_golden.Recorded()
    ref = m.fe_desc()
    ours = make_fe_desc()
    for k in ("frame_size", "frame_shift", "fft_size", "fft_order", "n_filt", "n_cep", "remove_dc", "remove_noise",
              "transform", "lifter_val", "window", "cmn"):
        assert ours[k] == ref[k], k
    for k in ("alpha", "sqrt_inv_n", "sqrt_inv_2n"):
        assert np.float32(ours[k]).tobytes() == np.float32(ref[k]).tobytes(), k
    for k in ("hamming", "ccc", "sss", "spec_start", "filt_start", "filt_width", "filt_coeffs", "mel_cosine", "lifter"):
        assert ours[k].dtype == ref[k].dtype and ours[k].shape == ref[k].shape, k
        assert ours[k].tobytes() == ref[k].tobytes(), k
    for pcm in fe_golden.frame_count_inputs():
        assert n_frames(ours, len(pcm)) == len(m.mfcc(pcm)), len(pcm)
    m.close()
