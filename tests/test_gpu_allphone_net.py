"""GPU (-m gpu): psb_allphone_net_batch_device -- phone decoding over the factored PHMM net, the
context-dependent one (-allphone_ci no) included -- against the reference's own results on
goforward.raw (tests/golden/en_us_allphone_cd.npz, en_us_allphone.npz) and against the C restatement
(pso_allphone_run / pso_allphone_lm_run) on the link-list expansion of the same nets."""
import ctypes as C

import numpy as np
import pytest

from conftest import golden
from test_allphone_net_emul import cd_phones, synth_case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from pocketsphinx_b200 import api
    assert api.device_count() > 0, "no CUDA device visible"
    return api


@pytest.fixture(scope="module")
def goforward(api, en_us):
    import torch
    scr = golden("en_us_goforward.npz")["senscr"]
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    yield ctx, scr, torch.from_numpy(np.concatenate([scr, scr[:100]])).cuda()
    ctx.close()


def _cd_net():
    from pocketsphinx_b200 import allphone_net as A
    g = golden("en_us_allphone_cd.npz")
    return g, A.build_net(cd_phones(g), ci_only=False)


def test_cd_goforward_matches_reference(goforward, en_us):
    from oracle import oracle
    from pocketsphinx_b200 import allphone_net as A
    ctx, scr, d = goforward
    g, net = _cd_net()
    r = ctx.allphone_net(d.data_ptr(), np.array([0, 278, 378], np.int32), net, int(g["beam"]), int(g["pbeam"]),
                         int(g["inspen"]), want_hist=True)
    assert list(r["status"]) == [0, 0]
    assert r["n_hist"][0] == int(g["n_history"]) and np.array_equal(r["segs"][0], g["segs"])
    so, s = A.expand_links(net)
    want, wn = oracle.allphone_run(en_us.tp, en_us.sseq, net["ssid"], net["tmatid"], so, s, net["start"], int(g["beam"]),
                                   int(g["pbeam"]), int(g["inspen"]), scr[:100])
    assert r["n_hist"][1] == wn and np.array_equal(r["hist"][1], want)
    assert np.array_equal(r["segs"][1], oracle.allphone_backtrace(want, net["ci"], 99, int(g["inspen"])))
    assert r["hist"][0][-1, 0] == 277 and len(r["hist"][0]) == int(g["n_history"])


def test_cd_goforward_phone_lm_matches_reference(goforward):
    ctx, scr, d = goforward
    g, net = _cd_net()
    r = ctx.allphone_net(d.data_ptr(), np.array([0, 278], np.int32), net, int(g["lm_beam"]), int(g["lm_pbeam"]),
                         bg=g["lm_bg"], tg=g["lm_tg"])
    assert r["status"][0] == 0 and r["n_hist"][0] == int(g["lm_n_history"])
    assert np.array_equal(r["segs"][0], g["lm_segs"])
    assert " ".join(g["ciname"][r["segs"][0][:, 0]]) == "SIL G OW F AO R W ER D T AE N M IY IH ZH ER Z S V SIL"


def test_ci_net_matches_reference(goforward):
    from pocketsphinx_b200 import allphone_net as A
    ctx, scr, d = goforward
    ga = golden("en_us_allphone.npz")
    net = A.build_net(cd_phones(golden("en_us_allphone_cd.npz")), ci_only=True)
    uo = np.array([0, 278], np.int32)
    r = ctx.allphone_net(d.data_ptr(), uo, net, int(ga["beam"]), int(ga["pbeam"]), int(ga["inspen"]))
    assert r["n_hist"][0] == int(ga["n_history"]) and np.array_equal(r["segs"][0], ga["segs"])
    r = ctx.allphone_net(d.data_ptr(), uo, net, int(ga["beam"]), int(ga["pbeam"]), bg=ga["lm_bg"], tg=ga["lm_tg"])
    assert r["n_hist"][0] == int(ga["lm_n_history"]) and np.array_equal(r["segs"][0], ga["lm_segs"])


@pytest.mark.parametrize("n_emit", [3, 5])
def test_ragged_synthetic_batch_matches_oracle(api, n_emit):
    import torch
    from oracle import oracle
    from pocketsphinx_b200 import allphone_net as A
    pm, net, bg, tg = synth_case(n_emit, 7 + n_emit)
    so, s = A.expand_links(net)
    rng = np.random.default_rng(n_emit)
    frames = [90, 1, 40, 200, 0, 7]
    scr = [(rng.integers(0, 24, (t, pm.n_sen)) * 16).astype(np.int16) for t in frames]
    uo = np.concatenate([[0], np.cumsum(frames)]).astype(np.int32)
    ctx = api.HmmContext(pm.tp, pm.sseq, pm.n_sen)
    d = torch.from_numpy(np.concatenate(scr)).cuda()
    total = 0
    for beam, pbeam, inspen in ((-1080, -1080, 0), (-200, -90, -35)):
        for lm in (False, True):
            kw = dict(bg=bg, tg=tg) if lm else {}
            r = ctx.allphone_net(d.data_ptr(), uo, net, beam, pbeam, inspen, want_hist=True, **kw)
            wants = []
            for u, T in enumerate(frames):
                if lm:
                    want, wn = oracle.allphone_lm_run(pm.tp, pm.sseq, net["ssid"], net["tmatid"], so, s, net["start"], beam,
                                                      pbeam, net["ci"], bg, tg, scr[u])
                    segs = oracle.allphone_backtrace_lm(want, net["ci"], T - 1) if T else np.zeros((0, 5), np.int32)
                    want = want[:, :4]
                else:
                    want, wn = oracle.allphone_run(pm.tp, pm.sseq, net["ssid"], net["tmatid"], so, s, net["start"], beam, pbeam,
                                                   inspen, scr[u])
                    segs = oracle.allphone_backtrace(want, net["ci"], T - 1, inspen) if T else np.zeros((0, 5), np.int32)
                assert r["status"][u] == 0 and r["n_hist"][u] == wn, (u, beam, lm)
                assert np.array_equal(r["hist"][u], want) and np.array_equal(r["segs"][u], segs), (u, beam, lm)
                wants.append(wn)
                total += wn
            # a small history capacity: exactly the utterances that outgrow it report it, the others are unchanged
            cap = sorted(wants)[len(wants) // 2]
            r2 = ctx.allphone_net(d.data_ptr(), uo, net, beam, pbeam, inspen, cap=cap, want_hist=True, **kw)
            for u in range(len(frames)):
                if wants[u] > cap:
                    assert r2["status"][u] == 1 and len(r2["segs"][u]) == 0, u
                    assert np.array_equal(r2["hist"][u], r["hist"][u][:cap]), u
                else:
                    assert r2["status"][u] == 0 and r2["n_hist"][u] == wants[u], u
                    assert np.array_equal(r2["segs"][u], r["segs"][u]) and np.array_equal(r2["hist"][u], r["hist"][u]), u
            # sub-batches (one utterance per launch) give the same
            r3 = ctx.allphone_net(d.data_ptr(), uo, net, beam, pbeam, inspen, hist_budget=1, **kw)
            assert np.array_equal(r3["n_hist"], r["n_hist"]) and all(np.array_equal(a, b) for a, b in zip(r3["segs"], r["segs"]))
    assert total > 5000
    ctx.close()


def test_malformed_input_is_refused_before_launch(api, goforward):
    from pocketsphinx_b200 import _lib
    ctx, scr, d = goforward
    L = _lib.lib()
    g, net = _cd_net()
    uo = np.array([0, 10], np.int32)
    before = L.psb_kernel_launch_count()

    def call(n_ci=42, start=None, ci=None, lc=None, rc=None, tg_only=False):
        a = {k: np.ascontiguousarray(net[k], np.int32) for k in ("ssid", "tmatid", "ci")}
        if ci is not None:
            a["ci"] = ci
        m = {k: np.ascontiguousarray(v, np.uint64) for k, v in (("lc", net["lc"] if lc is None else lc),
                                                                ("rc", net["rc"] if rc is None else rc))}
        res, segs = np.zeros((1, 3), np.int32), np.zeros((1, 10, 5), np.int32)
        tg = np.zeros(42 ** 3, np.int32)
        P = lambda x: x.ctypes.data_as(C.c_void_p)   # noqa: E731
        rc_ = L.psb_allphone_net_batch_device(ctx.h, C.c_void_p(d.data_ptr()), P(uo), 1, len(a["ci"]), P(a["ssid"]),
                                              P(a["tmatid"]), P(a["ci"]), P(m["lc"]), P(m["rc"]), n_ci,
                                              int(net["start"]) if start is None else start, -1080, -1080, 0, None,
                                              P(tg) if tg_only else None, 1000, P(res), P(segs), 10, None)
        return rc_, L.psb_last_error().decode()

    assert call(n_ci=65)[0] < 0 and "64" in call(n_ci=65)[1]
    big = net["lc"].copy()
    big[5] |= np.uint64(1) << np.uint64(42)
    rc_, msg = call(lc=big)
    assert rc_ < 0 and "context bit" in msg
    rc_, msg = call(rc=big)
    assert rc_ < 0 and "context bit" in msg
    bad = np.ascontiguousarray(net["ci"], np.int32).copy()
    bad[7] = 42
    assert call(ci=bad)[0] < 0 and "out of range" in call(ci=bad)[1]
    assert call(start=len(net["ci"]))[0] < 0 and "start" in call(start=len(net["ci"]))[1]
    assert call(start=-1)[0] < 0
    assert call(tg_only=True)[0] < 0
    assert L.psb_kernel_launch_count() == before
