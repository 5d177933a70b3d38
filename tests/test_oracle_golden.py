"""CPU: the plain-C oracle (oracle/ps_oracle.c) against fixtures produced by the compiled reference."""
import numpy as np
import pytest

from conftest import assert_hmm_equal, golden, hmm_view
from oracle import oracle


def test_ptm_goforward_bit_exact(en_us):
    g = golden("en_us_goforward.npz")
    om = oracle.OracleModel(en_us)
    scr, topn = om.score_utt(g["feats"], want_topn=True)
    assert scr.shape == (278, 5126)
    assert np.array_equal(scr, g["senscr"])
    assert np.array_equal(topn[0], g["topn_first"]) and np.array_equal(topn[-1], g["topn_last"])


def test_ptm_raw_lists_normalise_to_the_reference_lists(en_us):
    """The lists before ptm_norm (what the device's records hold) give, normalised, exactly the lists the
    reference hands out -- the en-us golden's first and last frame included -- and the same scores."""
    from pocketsphinx_b200.model import synth_feats, synth_ptm
    g = golden("en_us_goforward.npz")
    om = oracle.OracleModel(en_us)
    scr, topn, raw = om.score_utt(g["feats"], want_topn=True, want_raw=True)
    assert np.array_equal(scr, g["senscr"])
    norm = oracle.ptm_norm_raw(raw)
    assert np.array_equal(norm, topn)
    assert np.array_equal(norm[0], g["topn_first"]) and np.array_equal(norm[-1], g["topn_last"])
    assert np.array_equal(raw[..., 0], topn[..., 0])
    s = raw[..., 1]
    assert (s[..., :-1] >= s[..., 1:]).all() and (s < 0).all()            # descending integer distances
    for ds in (1, 2):
        pm = synth_ptm(seed=4, n_density=64, n_sen=300)
        pm.ds_ratio = ds
        f = synth_feats(pm, 1, 30, seed=1)[0]
        om = oracle.OracleModel(pm)
        scr, topn, raw = om.score_utt(f, want_topn=True, want_raw=True)
        assert np.array_equal(oracle.ptm_norm_raw(raw), topn) and np.array_equal(scr, om.score_utt(f))


def test_ptm_records_layout():
    """ptm_records packs {s0 >> 10, codeword bytes, min(255, offsets) bytes, 0}; assert_records_equal names the
    first differing (frame, pair) and field."""
    raw = np.zeros((2, 1, 2, 4, 2), np.int32)
    raw[0, 0, 0] = [[7, -1025], [255, -2047], [0, -2048], [9, -400000]]
    raw[0, 0, 1] = [[1, -1], [2, -2], [3, -3], [4, -1025]]
    raw[1] = raw[0]
    rec = oracle.ptm_records(raw)
    assert rec.shape == (2, 2, 4)
    assert rec[0, 0].view(np.uint32).tolist() == [(-2) & 0xffffffff, 0x0900ff07, 0xff000000, 0]
    assert rec[0, 1].view(np.uint32).tolist() == [(-1) & 0xffffffff, 0x04030201, 0x01000000, 0]
    oracle.assert_records_equal(rec, rec.copy())
    bad = rec.copy()
    bad[1, 1, 1] ^= np.int32(-0x80000000)                       # top codeword byte: compared as uint32
    with pytest.raises(AssertionError, match="frame 1, pair 1: field codewords"):
        oracle.assert_records_equal(bad, rec)


def test_ptm_active_lists(en_us):
    g = golden("en_us_active.npz")
    gf = golden("en_us_goforward.npz")
    n_sen = int(g["n_sen"])
    flags = np.unpackbits(g["flags"], axis=1)[:, :n_sen]
    om = oracle.OracleModel(en_us)
    dec = om.decoder(n_hist=2)
    for t in range(flags.shape[0]):
        lst = oracle.flags2list(flags[t])
        assert len(lst) == g["nact"][t]
        scr = dec.frame_eval(gf["feats"][t], t, lst, compallsen=False)
        dec.set_frame_idx(t + 1)
        assert np.array_equal(scr, g["senscr"][t]), "frame %d" % t
    dec.close()


def test_flags2list_bridges_gaps():
    flags = np.zeros(2000, np.uint8)
    flags[[3, 4, 300, 1999]] = 1
    lst = oracle.flags2list(flags)
    # 3, +1, then 296 = 255 + 41, then 1699 = 6*255 + 169
    assert lst.tolist() == [3, 1, 255, 41] + [255] * 6 + [169]
    assert int(np.cumsum(lst.astype(np.int64))[-1]) == 1999


def test_semi_tidigits_bit_exact(tidigits):
    g = golden("tidigits_goforward.npz")
    assert tidigits.kind == "s2_semi" and tidigits.mixw_4bit
    om = oracle.OracleModel(tidigits)
    scr, topn = om.score_utt(g["feats"], want_topn=True)
    assert np.array_equal(topn, g["topn"])
    assert np.array_equal(scr, g["senscr"])


def test_ms_an4_bit_exact(an4):
    g = golden("an4_goforward.npz")
    assert an4.kind == "ms"
    om = oracle.OracleModel(an4)
    scr = om.score_utt(g["feats"])
    assert np.array_equal(scr, g["senscr"])


@pytest.mark.parametrize("n_emit", [3, 5, 4, 1])
def test_hmm_vit_eval(n_emit):
    g = golden("hmm_vit_eval.npz")
    ctx = oracle.OracleHmmCtx(g["n%d_tp" % n_emit], g["n%d_sseq" % n_emit])
    hm = hmm_view(g["n%d_before" % n_emit]).copy()
    want = hmm_view(g["n%d_after" % n_emit])
    best = ctx.vit_eval(hm, g["n%d_senscr" % n_emit])
    assert best == int(g["n%d_best" % n_emit])
    assert_hmm_equal(hm, want, n_emit, "n_emit=%d" % n_emit)


def test_phoneloop_goforward(en_us):
    g = golden("en_us_goforward.npz")
    n, beam, pbeam, pip, window = [int(x) for x in g["pl_params"]]
    o = oracle.phoneloop_run(en_us.tp, en_us.sseq, en_us.phone_ssid[:n], en_us.phone_tmat[:n], g["senscr"],
                             window, beam, pbeam, pip, float(g["pl_weight"]))
    assert np.array_equal(o["best"], g["pl_best"])
    assert np.array_equal(o["pen"], g["pl_pen"])
    assert_hmm_equal(o["hmm"], hmm_view(g["pl_hmm"]), 3, "phone loop")
