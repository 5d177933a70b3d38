"""GPU: Decoder.decode_stream_batch -- whole recordings cut by the device endpointer, every segment decoded in one
batch with one session per stream -- against the reference: segment boundaries and times equal the reference
endpointer's exactly; each segment's words equal a reference decoder fed the same segments in order
(ps_get_hyp, ps_seg_iter): the words of every segment equal and word boundaries within 2 frames, the tolerance of
tests/test_gpu_zz_decoder.py (the device front end matches the reference's to 1e-4 relative, not bit for bit; the
endpointer's own results are compared exactly).  Path scores are printed next to the reference's, not compared: on
these segments decode_raw_batch's scores differ from ps_get_hyp's by 3 000 - 4 600 while words and boundaries agree
(see DESIGN 4.20); the first segment's score is checked against decode_raw_batch of the same samples instead."""
import os

import numpy as np
import pytest

import vad_cases as V
from conftest import ROOT

pytestmark = [pytest.mark.gpu]
REF = os.path.join(ROOT, "oracle", "_ref")


@pytest.mark.timeout(900)
def test_decode_stream_batch_matches_reference_segments_and_words():
    from pocketsphinx_b200.decoder import Decoder
    hd, dic, lm = os.path.join(REF, "model", "en-us"), os.path.join(REF, "data", "turtle.dic"), os.path.join(REF, "data", "turtle.lm.bin")
    if not (os.path.exists(lm) and V.ref_available()):
        pytest.skip("reference data files not present")
    a = V.audio()
    sil = np.zeros(16000, np.int16)
    s1 = np.concatenate([sil, a["goforward"], sil, a["numbers"], sil, a["libri_0880"], sil])
    s2 = np.concatenate([sil[:4000], a["goforward"], sil])
    dec = Decoder(hd, dic, lm, max_utts=64, max_frames=1 << 15)
    out = dec.decode_stream_batch([s1, s2])
    for stream, got in zip((s1, s2), out):
        want = V.ref_segments(stream, 0, 16000, 0.03, 0.3, 0.9)
        assert [(d["start_time"], d["end_time"], d["start_sample"], d["end_sample"]) for d in got] == want
        ref = V.ref_session_segments(hd, lm, dic, [stream[w[2]:w[3]] for w in want])
        assert [d["hyp"] for d in got] == [r["hyp"] for r in ref]
        for d, r in zip(got, ref):
            print("segment %d..%d: %d frames, score %d (reference %d), %s" % (d["start_sample"], d["end_sample"], d["n_frames"],
                                                                          d["score"], r["score"], d["hyp"]))
        for d, r in zip(got, ref):
            assert d["words"] == [w for w, _, _ in r["seg"]], (d["words"], r["seg"])
            assert np.abs(d["seg"][:, 2] - np.array([sf for _, sf, _ in r["seg"]])).max() <= 2
            assert np.abs(d["seg"][:, 3] - np.array([ef for _, _, ef in r["seg"]])).max() <= 2
        # the first segment of a stream is a fresh decoder's first utterance: decode_stream_batch passes it through
        # decode_raw_batch unchanged, score and segmentation included
        fresh = dec.decode_raw_batch([stream[want[0][2]:want[0][3]]])[0]
        assert fresh["score"] == got[0]["score"] and np.array_equal(fresh["seg"], got[0]["seg"])
    assert any("forward" in d["hyp"] for d in out[1])
    dec.close()
