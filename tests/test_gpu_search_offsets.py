"""GPU (-m gpu): every whole-utterance entry point on an HMM context refuses utterance offsets that
decrease.  The offsets used, [0, 50, 20, 100] over 100 frames, stay inside the score buffer, so an entry
point that did not check them would run without touching memory out of range and simply not raise."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

UTT_OFF = np.array([0, 50, 20, 100], np.int32)
N_FRAMES = 100


@pytest.fixture(scope="module")
def setup():
    import torch
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.model import synth_ptm
    assert api.device_count() > 0, "no CUDA device visible"
    pm = synth_ptm(seed=61, n_density=32, n_sen=300, n_emit_state=3)
    rng = np.random.default_rng(5)
    scr = rng.integers(0, 300, (N_FRAMES, pm.n_sen)).astype(np.int16)
    d_scr = torch.from_numpy(scr).cuda()
    ctx = api.HmmContext(pm.tp, pm.sseq, pm.n_sen)
    n = 6
    ssid = rng.integers(0, len(pm.sseq), n).astype(np.int32)
    tmat = rng.integers(0, pm.tp.shape[0], n).astype(np.int32)
    yield api, ctx, scr, d_scr, ssid, tmat
    ctx.close()


def _phoneloop(api, ctx, ssid, tmat):
    return api.PhoneLoop(ctx, ssid, tmat, 0, -1000, -1000, -20, 0.0)


def _fsg_desc():
    return dict(pnodes=np.zeros((1, 16), np.int32), roots=np.zeros(1, np.int32), links=np.zeros((1, 4), np.int32),
                nulloff=np.zeros(2, np.int32), nullarc=np.zeros(0, np.int32), n_ciphone=1, silcipid=0, start_state=0,
                beam=-1000, pbeam=-1000, wbeam=-1000, maxhmmpf=-1)


NGRAM = dict(info=np.zeros(16, np.int32), model=np.zeros(16, np.int32), ci_tmat=np.zeros(1, np.int32),
             ci_ssid=np.zeros(1, np.int32))


def _call(name, api, ctx, scr, d_scr, ssid, tmat):
    d = d_scr.data_ptr()
    ph_off = np.array([0, 2, 4, 6], np.int32)
    succ_off = np.arange(len(ssid) + 1, dtype=np.int32)
    succ = np.roll(np.arange(len(ssid), dtype=np.int32), -1)
    if name == "phoneloop_run_host":
        pl = _phoneloop(api, ctx, ssid, tmat)
        try:
            pl.run_host(scr, UTT_OFF)
        finally:
            pl.close()
    elif name == "phoneloop_run_device":
        pl = _phoneloop(api, ctx, ssid, tmat)
        try:
            api.check(api.lib().psb_phoneloop_run_device(pl.h, C.c_void_p(d), UTT_OFF.ctypes.data, len(UTT_OFF) - 1,
                                                         None, None, None, None), "psb_phoneloop_run_device")
        finally:
            pl.close()
    elif name == "align_batch_device":
        ctx.align(None, UTT_OFF, ph_off, ssid, tmat, device_ptr=d)
    elif name == "align_batch_host":
        ctx.align(scr, UTT_OFF, ph_off, ssid, tmat)
    elif name == "kws_batch_device":
        ctx.kws(d, UTT_OFF, ssid[:3], tmat[:3], np.array([0, 3], np.int32), np.array([-100], np.int32), ssid[3:], tmat[3:],
                -1000, -20)
    elif name == "allphone_batch_device":
        ctx.allphone(d, UTT_OFF, ssid, tmat, succ_off, succ, 0, -1000, -1000, 0)
    elif name == "allphone_lm_batch_device":
        ctx.allphone_lm(d, UTT_OFF, ssid, tmat, succ_off, succ, 0, -1000, -1000, np.zeros(len(ssid), np.int32),
                        np.zeros((1, 1), np.int32), np.zeros((1, 1, 1), np.int32))
    elif name == "fsg_batch_device":
        ctx.fsg(d, UTT_OFF, _fsg_desc(), 16)
    elif name == "ngram_fwdtree_batch_device":
        ctx.ngram_fwdtree(d, UTT_OFF, NGRAM["info"], NGRAM["model"], NGRAM["ci_tmat"], 16, 16)
    elif name == "ngram_fwdflat_batch_device":
        ctx.ngram_fwdflat(d, UTT_OFF, NGRAM["info"], NGRAM["model"], NGRAM["ci_tmat"], NGRAM["ci_ssid"],
                          [np.zeros((0, 10), np.int32)] * (len(UTT_OFF) - 1), 16, 16)
    elif name == "ngram_two_pass_batch_device":
        ctx.ngram_two_pass(d, UTT_OFF, NGRAM["info"], NGRAM["model"], NGRAM["ci_tmat"], NGRAM["ci_ssid"], 16, 16)
    else:
        raise AssertionError(name)


@pytest.mark.parametrize("name", ["phoneloop_run_host", "phoneloop_run_device", "align_batch_device", "align_batch_host",
                                  "kws_batch_device", "allphone_batch_device", "allphone_lm_batch_device",
                                  "fsg_batch_device", "ngram_fwdtree_batch_device", "ngram_fwdflat_batch_device",
                                  "ngram_two_pass_batch_device"])
def test_decreasing_utt_off_is_refused(setup, name):
    api = setup[0]
    with pytest.raises(api.PsbError, match="not monotone"):
        _call(name, *setup)


def test_decreasing_kp_off_is_refused(setup):
    """The keyphrase offsets are checked before they size the HMM tables: kp_off = [0, -1] would make the table
    shorter than the phone loop that is written into it."""
    api, ctx, scr, d_scr, ssid, tmat = setup
    with pytest.raises(api.PsbError, match="kp_off not monotone"):
        ctx.kws(d_scr.data_ptr(), np.array([0, N_FRAMES], np.int32), ssid[:3], tmat[:3], np.array([0, -1], np.int32),
                np.array([-100], np.int32), ssid[3:], tmat[3:], -1000, -20)
