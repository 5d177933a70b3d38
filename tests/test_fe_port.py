"""CPU: the numpy restatement of the front end (oracle/fe_port.py, structured like psb_fe.cu)
against the compiled reference on real and synthetic PCM -- bit-exact (same libm)."""
import numpy as np
import pytest

from oracle import fe_golden, fe_port


@pytest.mark.parametrize("kv", fe_golden.PORT_CONFIGS)
def test_fe_port_matches_reference(kv):
    ref = fe_golden.Recorded(**kv)
    d = ref.fe_desc()
    for pcm in fe_golden.port_inputs(fe_golden.goforward()):
        want_c = ref.mfcc(pcm)
        got_c = fe_port.cepstra(d, fe_port.mfspec(d, pcm))
        assert got_c.shape == want_c.shape
        assert np.array_equal(got_c.view(np.uint32), want_c.view(np.uint32)), "cepstra, %d samples" % len(pcm)
        want = ref.featurize_fresh(pcm)
        got = fe_port.featurize(d, pcm)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "features, %d samples" % len(pcm)
    ref.close()
