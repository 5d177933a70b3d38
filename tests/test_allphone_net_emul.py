"""CPU: phone decoding over the factored PHMM net (-allphone_ci no / yes).

* The net builder (pocketsphinx_b200/allphone_net.py) on the mdef phone table of
  tests/golden/en_us_allphone_cd.npz reproduces the net the reference's phmm_build / phmm_link made:
  node order, ssid, tmatid, ci, start, and the successor lists expanded from the lc / rc masks; also
  the context-independent net of en_us_allphone.npz, and the search parameters.
* The phase code of the device search (pocketsphinx_b200/csrc/psb_apn_core.h, the source
  allphone_net_kernel is compiled from), built for the host by tests/emul/apn_emul.cpp and run one
  "thread" at a time in ascending and descending order, reproduces the reference's history count and
  segmentation on goforward.raw (CD net, without and with the phone LM), and the C restatement's
  history rows (pso_allphone_run / pso_allphone_lm_run) on the link-list expansion of synthetic nets,
  with a data-race count of 0 in the race-check build."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, golden

ARGT = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32] + [C.c_void_p] * 5 + [C.c_int32] * 5 + [C.c_void_p] * 3 + \
    [C.c_int32] * 2 + [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def cd_phones(g):
    return dict(n_ciphone=len(g["ciname"]), phone_ssid=g["ph_ssid"], phone_tmat=g["ph_tmat"], phone_ctx=g["ph_ctx"],
                phone_filler=g["ph_filler"], sil=int(g["sil"]))


def build_emul(tmp, order, race=False):
    from oracle import oracle
    oracle.build()
    out = str(tmp / ("libapnemul_%s%s.so" % (order, "_race" if race else "")))
    odir = os.path.dirname(oracle.LIB_PATH)
    cmd = ["g++", "-O1", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-ffp-contract=off",
           "-I" + os.path.join(ROOT, "tests", "emul")]
    if order == "descending":
        cmd.append("-DPSB_FSG_EMUL_REVERSE")
    if race:
        cmd.append("-DPSB_FSG_RACECHECK")
    cmd += ["-o", out, os.path.join(ROOT, "tests", "emul", "apn_emul.cpp"), "-L" + odir, "-lpsoracle", "-Wl,-rpath," + odir]
    subprocess.check_call(cmd)
    L = C.CDLL(out)
    L.apn_emul_run.restype = C.c_int32
    L.apn_emul_run.argtypes = ARGT
    L.emul_race_count.restype = C.c_long
    return L


def run_emul(L, tp, sseq, net, beam, pbeam, inspen, scr, bg=None, tg=None, cap=None):
    """Returns (status, n_hist, history rows [n][4], segments [n][5])."""
    tp = np.ascontiguousarray(tp, np.uint8)
    sseq = np.ascontiguousarray(sseq, np.uint16)
    a = [np.ascontiguousarray(net[k], np.int32) for k in ("ssid", "tmatid", "ci")]
    lc, rc = (np.ascontiguousarray(net[k], np.uint64) for k in ("lc", "rc"))
    bg = None if bg is None else np.ascontiguousarray(bg, np.int32)
    tg = None if tg is None else np.ascontiguousarray(tg, np.int32)
    scr = np.ascontiguousarray(scr, np.int16)
    T, n_sen = scr.shape
    H = len(a[0])
    cap = cap or max(1, T * H)
    hist = np.zeros((cap, 4), np.int32)
    segs = np.zeros((max(T, 1), 5), np.int32)
    res = np.zeros(3, np.int32)
    L.apn_emul_run(tp.shape[1], _p(tp), _p(sseq), H, _p(a[0]), _p(a[1]), _p(a[2]), _p(lc), _p(rc), int(net["n_ci"]),
                   int(net["start"]), int(beam), int(pbeam), int(inspen), _p(bg), _p(tg), _p(scr), n_sen, T, _p(hist), cap,
                   _p(segs), len(segs), _p(res))
    return int(res[0]), int(res[1]), hist[:min(int(res[1]), cap)], segs[:int(res[2])]


def synth_net(rng, n_ci, H, start_ci=0, p_ctx=0.15):
    """A random factored net: every CI phone has at least one node; sparse random context masks, CI
    phone 0 / 1 acting as fillers in some contexts."""
    ci = np.sort(np.concatenate([np.arange(n_ci), rng.integers(0, n_ci, H - n_ci)])).astype(np.int32)
    bits = np.uint64(1) << np.arange(n_ci, dtype=np.uint64)
    lc = np.array([np.bitwise_or.reduce(bits[rng.random(n_ci) < p_ctx], initial=np.uint64(0)) for _ in range(H)], np.uint64)
    rc = np.array([np.bitwise_or.reduce(bits[rng.random(n_ci) < p_ctx], initial=np.uint64(0)) for _ in range(H)], np.uint64)
    first = np.searchsorted(ci, np.arange(n_ci))
    full = np.uint64((1 << n_ci) - 1)
    lc[first] = full
    rc[first] = full
    return dict(ci=ci, lc=lc, rc=rc, n_ci=n_ci, start=int(first[start_ci]))


def synth_case(n_emit, seed):
    from pocketsphinx_b200.model import synth_ptm
    pm = synth_ptm(seed=51, n_density=32, n_sen=300, n_emit_state=n_emit, skip_arcs=(n_emit == 5))
    rng = np.random.default_rng(seed)
    net = synth_net(rng, 11, 240)
    H = len(net["ci"])
    net["ssid"] = rng.integers(0, len(pm.sseq), H).astype(np.int32)
    net["tmatid"] = rng.integers(0, pm.tp.shape[0], H).astype(np.int32)
    n = net["n_ci"]
    bg = -(rng.integers(0, 12, (n, n)) * 16).astype(np.int32)        # quantized: ties between paths
    tg = -(rng.integers(0, 12, (n, n, n)) * 16).astype(np.int32)
    return pm, net, bg, tg


@pytest.fixture(scope="module", params=["ascending", "descending"])
def emul(request, tmp_path_factory):
    return build_emul(tmp_path_factory.mktemp("apnemul"), request.param)


@pytest.fixture(scope="module")
def race(tmp_path_factory):
    return build_emul(tmp_path_factory.mktemp("apnrace"), "ascending", race=True)


def test_builder_reproduces_reference_cd_net():
    from pocketsphinx_b200 import allphone_net as A
    g = golden("en_us_allphone_cd.npz")
    net = A.build_net(cd_phones(g), ci_only=False)
    for k in ("ssid", "tmatid", "ci"):
        assert np.array_equal(net[k], g[k]), k
    assert net["start"] == int(g["start"]) and len(net["ci"]) == 29324
    so, s = A.expand_links(net)
    assert np.array_equal(so, g["succ_off"])
    for p in range(len(so) - 1):                                          # as sets per node (and in fact in order)
        assert set(s[so[p]:so[p + 1]].tolist()) == set(g["succ"][g["succ_off"][p]:g["succ_off"][p + 1]].tolist())
    assert np.array_equal(s, g["succ"])
    n_ci = int(net["n_ci"])
    assert not ((net["lc"] | net["rc"]) >> np.uint64(n_ci)).any()


def test_builder_reproduces_reference_ci_net():
    from pocketsphinx_b200 import allphone_net as A
    g, ga = golden("en_us_allphone_cd.npz"), golden("en_us_allphone.npz")
    net = A.build_net(cd_phones(g), ci_only=True)
    for k in ("ssid", "tmatid", "ci"):
        assert np.array_equal(net[k], ga[k]), k
    assert net["start"] == int(ga["start"])
    so, s = A.expand_links(net)
    assert np.array_equal(so, ga["succ_off"]) and np.array_equal(s, ga["succ"])


def test_search_params_match_reference():
    from pocketsphinx_b200 import allphone_net as A
    g = golden("en_us_allphone_cd.npz")
    assert A.search_params() == (int(g["beam"]), int(g["pbeam"]), int(g["inspen"]))
    assert A.search_params(beam=1e-20, pbeam=1e-10, lw=2.0)[:2] == (int(g["lm_beam"]), int(g["lm_pbeam"]))
    assert A.search_params(pip=0.5, lw=6.5)[2] == (int(np.log(0.5) / np.log(1.0001)) * 6) >> 10


def test_builder_on_real_mdef_matches_reference_driver():
    from oracle import refdrv
    if not refdrv.available() or not os.path.isdir("/root/reference/model/en-us/en-us"):
        pytest.skip("the compiled reference and its model are not present")
    from pocketsphinx_b200 import allphone_net as A, s3io
    hmm = "/root/reference/model/en-us/en-us"
    net = A.build_net(A.mdef_phones(s3io.read_mdef(os.path.join(hmm, "mdef"))), ci_only=True)
    a = refdrv.allphone(hmm, np.zeros(1600, np.int16))
    for k in ("ssid", "tmatid", "ci"):
        assert np.array_equal(net[k], a[k]), k
    so, s = A.expand_links(net)
    assert np.array_equal(so, a["succ_off"]) and np.array_equal(s, a["succ"]) and net["start"] == a["start"]


def test_phase_code_reproduces_reference_cd(emul):
    from pocketsphinx_b200 import allphone_net as A
    g, m = golden("en_us_allphone_cd.npz"), golden("en_us_ptm_model.npz")
    scr = golden("en_us_goforward.npz")["senscr"]
    net = A.build_net(cd_phones(g), ci_only=False)
    st, n, _, segs = run_emul(emul, m["tp"], m["sseq"], net, int(g["beam"]), int(g["pbeam"]), int(g["inspen"]), scr)
    assert st == 0 and n == int(g["n_history"]) and np.array_equal(segs, g["segs"])


def test_phase_code_reproduces_reference_cd_lm(emul):
    from pocketsphinx_b200 import allphone_net as A
    g, m = golden("en_us_allphone_cd.npz"), golden("en_us_ptm_model.npz")
    scr = golden("en_us_goforward.npz")["senscr"]
    net = A.build_net(cd_phones(g), ci_only=False)
    st, n, _, segs = run_emul(emul, m["tp"], m["sseq"], net, int(g["lm_beam"]), int(g["lm_pbeam"]), 0, scr,
                              bg=g["lm_bg"], tg=g["lm_tg"])
    assert st == 0 and n == int(g["lm_n_history"]) and np.array_equal(segs, g["lm_segs"])
    assert " ".join(g["ciname"][segs[:, 0]]) == "SIL G OW F AO R W ER D T AE N M IY IH ZH ER Z S V SIL"


@pytest.mark.parametrize("n_emit", [3, 5])
def test_phase_code_matches_oracle_on_synthetic_nets(emul, n_emit):
    from oracle import oracle
    from pocketsphinx_b200 import allphone_net as A
    pm, net, bg, tg = synth_case(n_emit, 7 + n_emit)
    so, s = A.expand_links(net)
    rng = np.random.default_rng(n_emit)
    total = 0
    for T in (1, 2, 60, 150):
        scr = (rng.integers(0, 24, (T, pm.n_sen)) * 16).astype(np.int16)    # quantized scores: ties
        for beam, pbeam, inspen in ((-1080, -1080, 0), (-200, -90, -35), (-60, -30, 0)):
            want, wn = oracle.allphone_run(pm.tp, pm.sseq, net["ssid"], net["tmatid"], so, s, net["start"], beam, pbeam, inspen, scr)
            st, n, hist, segs = run_emul(emul, pm.tp, pm.sseq, net, beam, pbeam, inspen, scr)
            assert st == 0 and n == wn and np.array_equal(hist, want), (T, beam)
            assert np.array_equal(segs, oracle.allphone_backtrace(want, net["ci"], T - 1, inspen)), (T, beam)
            lwant, lwn = oracle.allphone_lm_run(pm.tp, pm.sseq, net["ssid"], net["tmatid"], so, s, net["start"], beam, pbeam,
                                                net["ci"], bg, tg, scr)
            st, n, hist, segs = run_emul(emul, pm.tp, pm.sseq, net, beam, pbeam, 0, scr, bg=bg, tg=tg)
            assert st == 0 and n == lwn and np.array_equal(hist, lwant[:, :4]), (T, beam, "lm")
            assert np.array_equal(segs, oracle.allphone_backtrace_lm(lwant, net["ci"], T - 1)), (T, beam, "lm")
            total += wn + lwn
    assert total > 5000


def test_phase_code_reports_history_overflow(emul):
    from oracle import oracle
    from pocketsphinx_b200 import allphone_net as A
    pm, net, _, _ = synth_case(3, 3)
    so, s = A.expand_links(net)
    scr = np.random.default_rng(1).integers(0, 300, (40, pm.n_sen)).astype(np.int16)
    want, wn = oracle.allphone_run(pm.tp, pm.sseq, net["ssid"], net["tmatid"], so, s, net["start"], -1080, -1080, 0, scr)
    st, n, hist, segs = run_emul(emul, pm.tp, pm.sseq, net, -1080, -1080, 0, scr, cap=wn)
    assert st == 0 and n == wn and np.array_equal(hist, want)
    st, n, hist, segs = run_emul(emul, pm.tp, pm.sseq, net, -1080, -1080, 0, scr, cap=wn - 1)
    assert st == 1 and len(segs) == 0 and np.array_equal(hist, want[:wn - 1])


def test_phase_code_is_race_free(race):
    from oracle import oracle
    from pocketsphinx_b200 import allphone_net as A
    g, ga, m = golden("en_us_allphone_cd.npz"), golden("en_us_allphone.npz"), golden("en_us_ptm_model.npz")
    scr = golden("en_us_goforward.npz")["senscr"]
    net = A.build_net(cd_phones(g), ci_only=True)
    st, n, _, segs = run_emul(race, m["tp"], m["sseq"], net, int(ga["beam"]), int(ga["pbeam"]), int(ga["inspen"]), scr)
    assert st == 0 and n == int(ga["n_history"]) and np.array_equal(segs, ga["segs"])
    st, n, _, segs = run_emul(race, m["tp"], m["sseq"], net, int(ga["beam"]), int(ga["pbeam"]), 0, scr,
                              bg=ga["lm_bg"], tg=ga["lm_tg"])
    assert st == 0 and n == int(ga["lm_n_history"]) and np.array_equal(segs, ga["lm_segs"])
    for n_emit in (3, 5):
        pm, snet, bg, tg = synth_case(n_emit, 2)
        so, s = A.expand_links(snet)
        sc = (np.random.default_rng(4).integers(0, 24, (50, pm.n_sen)) * 16).astype(np.int16)
        want, wn = oracle.allphone_lm_run(pm.tp, pm.sseq, snet["ssid"], snet["tmatid"], so, s, snet["start"], -200, -90,
                                          snet["ci"], bg, tg, sc)
        st, n, hist, _ = run_emul(race, pm.tp, pm.sseq, snet, -200, -90, 0, sc, bg=bg, tg=tg)
        assert st == 0 and n == wn and np.array_equal(hist, want[:, :4])
    assert race.emul_race_count() == 0
