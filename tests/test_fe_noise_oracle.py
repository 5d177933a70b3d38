"""CPU: the reference driven with ps_start_stream at chosen utterances only (tests/fe_noise_cases.py).  The
refdrv_featurize driver, which the GPU tests compare the device with, gives the same cepstra bit for bit as a
plain ps_decoder_t fed ps_start_stream once and then ps_start_utt / ps_process_raw(full_utt) / ps_end_utt per
utterance, on the en-us model's own settings (-remove_noise yes); and with the tracker carried the cepstra of
the later utterances are not those of fresh streams."""
import os

import numpy as np
import pytest

import fe_noise_cases as N
import fe_sessions as fs
from oracle import fe_golden, refdrv

pytestmark = pytest.mark.skipif(not refdrv.available(), reason="compiled reference not built")


def _utterances():
    go = fe_golden.goforward()
    return [go[:20000], N.pcm(9000, 1, amp=300), go[15000:], N.pcm(250, 2, amp=4000), N.pcm(12000, 3, amp=6000)]


@pytest.mark.parametrize("starts", [[1, 0, 0, 0, 0], [1, 0, 1, 0, 0]])
def test_featurize_driver_is_a_decoder_with_stream_starts(starts):
    hmm = fs.ref_model_dir("en-us")
    data = os.path.join(os.path.dirname(refdrv.LIB_PATH), "data")
    lm, dic = os.path.join(data, "turtle.lm.bin"), os.path.join(data, "turtle.dic")
    if not os.path.exists(lm):
        pytest.skip("reference data files not present")
    utts = _utterances()
    dec = N.ref_decoder(hmm, lm, dic, utts, starts)
    # -cmn none: 1s_c_d_dd's first 13 columns are the cepstra themselves
    r = refdrv.RefModel(hmm, cmn="none")
    carried = N.ref_stream_features(r, utts, starts)
    fresh = N.ref_stream_features(r, utts, [1] * len(utts))
    r.close()
    r = refdrv.RefModel(hmm)                                 # the model's own batch CMN
    feats = N.ref_stream_features(r, utts, starts)
    r.close()
    for u, d in enumerate(dec):
        assert d["cep"].shape[0] == carried[u].shape[0] > 0
        assert d["cep"].tobytes() == np.ascontiguousarray(carried[u][:, :13]).tobytes(), u
        assert fs.dyn_features(fs.batch_cmn(d["cep"]), 0).tobytes() == feats[u].tobytes(), u
        if starts[u]:
            assert carried[u].tobytes() == fresh[u].tobytes(), u
        else:
            assert np.abs(carried[u] - fresh[u]).max() > 0.1, u
