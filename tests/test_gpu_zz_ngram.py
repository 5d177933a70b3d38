"""GPU (-m gpu): psb_ngram_fwdtree_batch_device (the first pass of the n-gram search on the device)
against the reference's golden backpointer tables and against the oracle on ragged batches.

The phase code is also checked on the host against the reference (tests/test_ngs_emul.py,
tests/test_ngf_emul.py)."""

import os

import numpy as np
import pytest

from conftest import golden

pytestmark = [pytest.mark.gpu]

TAGS = ("default", "wide", "narrow", "maxwpf", "abs", "pen", "lookahead")


def _case(g, tag):
    return {k[len(tag) + 1:]: g[k] for k in g.files if k.startswith(tag + ".")}


@pytest.fixture(scope="module")
def api():
    from pocketsphinx_b200 import api
    assert api.device_count() > 0, "no CUDA device visible"
    return api


@pytest.mark.timeout(300)
@pytest.mark.parametrize("tag", TAGS)
def test_fwdtree_batch_matches_reference_and_oracle(api, en_us, tag):
    import torch
    from oracle import oracle
    gf = golden("en_us_goforward.npz")
    scr = gf["senscr"]
    c = _case(golden("en_us_fwdtree.npz"), tag)
    n_ci = int(c["info"][6])
    cit = en_us.phone_tmat[:n_ci]
    parts = [scr, scr[:0], scr[:1], scr[:100], scr]
    utt_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int32)
    d_scr = torch.from_numpy(np.ascontiguousarray(np.concatenate(parts))).cuda()
    d_pen, win, la = None, 0, [{} for _ in parts]
    if tag == "lookahead":
        win = int(gf["pl_params"][4])
        # the phone loop's own table per utterance (prefixes of the utterance see the same phone-loop history)
        d_pen = torch.from_numpy(np.ascontiguousarray(np.concatenate([gf["pl_pen"][:len(p)] for p in parts]), np.int32)).cuda()
        la = [dict(pl_pen=gf["pl_pen"][:len(p)], pl_window=win) for p in parts]
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    out = ctx.ngram_fwdtree(d_scr.data_ptr(), utt_off, c["info"], c["model"], cit, len(c["bp"]) + 64, len(c["bss"]) + 4096,
                            d_pen.data_ptr() if d_pen is not None else None, win)
    for u in (0, 4):                                            # the reference's own tables
        bp, bss, idx = out[u]
        assert np.array_equal(bp, c["bp"]) and np.array_equal(bss, c["bss"]) and np.array_equal(idx, c["bp_idx"]), u
    for u in (1, 2, 3):
        want = oracle.fwdtree_run(en_us.tp, en_us.sseq, cit, c["info"], c["model"], parts[u], **la[u])
        bp, bss, idx = out[u]
        assert np.array_equal(bp, want[0]) and np.array_equal(bss, want[1]) and np.array_equal(idx, want[2]), u
    ctx.close()


@pytest.mark.timeout(300)
def test_fwdtree_full_table_is_an_error(api, en_us):
    import torch
    from pocketsphinx_b200._lib import PsbError
    gf = golden("en_us_goforward.npz")
    c = _case(golden("en_us_fwdtree.npz"), "default")
    d_scr = torch.from_numpy(np.ascontiguousarray(gf["senscr"])).cuda()
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    with pytest.raises(PsbError):
        ctx.ngram_fwdtree(d_scr.data_ptr(), np.array([0, 278], np.int32), c["info"], c["model"],
                          en_us.phone_tmat[:int(c["info"][6])], 100, 100000)
    ctx.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("tag", ("flat_default", "flat_wide", "flat_narrow"))
def test_fwdflat_batch_matches_reference_and_oracle(api, en_us, tag):
    """Second pass on the device behind the first pass on the device (ngs_fwdflat_kernel)."""
    import torch
    from oracle import oracle
    gf = golden("en_us_goforward.npz")
    scr = gf["senscr"]
    c = _case(golden("en_us_fwdtree.npz"), tag)
    n_ci = int(c["info"][6])
    cit, cis = en_us.phone_tmat[:n_ci], en_us.phone_ssid[:n_ci]
    parts = [scr, scr[:0], scr[:1], scr[:120], scr]
    utt_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int32)
    d_scr = torch.from_numpy(np.ascontiguousarray(np.concatenate(parts))).cuda()
    d_pen, win, la = None, 0, [{} for _ in parts]
    if tag == "flat_default":
        win = int(gf["pl_params"][4])
        d_pen = torch.from_numpy(np.ascontiguousarray(np.concatenate([gf["pl_pen"][:len(p)] for p in parts]), np.int32)).cuda()
        la = [dict(pl_pen=gf["pl_pen"][:len(p)], pl_window=win) for p in parts]
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    first = ctx.ngram_fwdtree(d_scr.data_ptr(), utt_off, c["info"], c["model"], cit, 8192, 1 << 18,
                              d_pen.data_ptr() if d_pen is not None else None, win)
    out = ctx.ngram_fwdflat(d_scr.data_ptr(), utt_off, c["info"], c["model"], cit, cis, [t[0] for t in first],
                            len(c["bp"]) + 64, len(c["bss"]) + 4096)
    for u in (0, 4):
        bp, bss, idx = out[u]
        assert np.array_equal(bp, c["bp"]) and np.array_equal(bss, c["bss"]) and np.array_equal(idx, c["bp_idx"]), u
    for u in (1, 2, 3):
        bp1 = oracle.fwdtree_run(en_us.tp, en_us.sseq, cit, c["info"], c["model"], parts[u], **la[u])[0]
        assert np.array_equal(first[u][0], bp1), u
        want = oracle.fwdflat_run(en_us.tp, en_us.sseq, cit, cis, c["info"], c["model"], bp1, parts[u])
        bp, bss, idx = out[u]
        assert np.array_equal(bp, want[0]) and np.array_equal(bss, want[1]) and np.array_equal(idx, want[2]), u
    ctx.close()


@pytest.mark.timeout(600)
def test_all_searches_on_tidigits_against_the_live_reference(api, tidigits):
    """5-state HMMs, another phone set, dictionary, grammar and LM: the reference runs live on the GPU
    box (oracle/_ref travels with its copy of the tidigits model)."""
    import torch
    from oracle import refdrv
    if not refdrv.available():
        pytest.skip("oracle/_ref/libpsref.so not built")
    ref_dir = os.path.dirname(refdrv.LIB_PATH)
    hd = os.path.join(ref_dir, "model", "tidigits_hmm")
    dic = os.path.join(ref_dir, "model", "tidigits_lm", "tidigits.dic")
    pcm = np.fromfile(os.path.join(ref_dir, "data", "goforward.raw"), np.int16)
    ref = refdrv.RefModel(hd)
    scr = np.ascontiguousarray(ref.score(ref.featurize_fresh(pcm)))
    ref.close()
    d_scr = torch.from_numpy(np.concatenate([scr, scr[:90]])).cuda()
    utt_off = np.array([0, len(scr), len(scr) + 90], np.int32)
    ctx = api.HmmContext(tidigits.tp, tidigits.sseq, tidigits.n_sen)
    # grammar search
    from oracle import oracle
    g = refdrv.fsg(hd, dic, os.path.join(ref_dir, "model", "tidigits_lm", "tidigits.fsg"), pcm)
    hist, n = ctx.fsg(d_scr.data_ptr(), utt_off, g, len(g["hist"]) + 64)
    assert n[0] == len(g["hist"]) and np.array_equal(hist[0], g["hist"])
    assert np.array_equal(hist[1], oracle.fsg_run(tidigits.tp, tidigits.sseq, g, scr[:90]))
    # both n-gram passes
    lm = os.path.join(ref_dir, "model", "tidigits_lm", "tidigits.lm.bin")
    first = refdrv.fwdtree(hd, lm, dic, pcm)
    both = refdrv.fwdtree(hd, lm, dic, pcm, fwdflat="yes")
    nc = both["n_ci"]
    cit, cis = tidigits.phone_tmat[:nc], tidigits.phone_ssid[:nc]
    out1 = ctx.ngram_fwdtree(d_scr.data_ptr(), utt_off, both["info"], both["model"], cit, len(first["bp"]) + 64, len(first["bss"]) + 4096)
    assert np.array_equal(out1[0][0], first["bp"]) and np.array_equal(out1[0][1], first["bss"]) and np.array_equal(out1[0][2], first["bp_idx"])
    want1 = oracle.fwdtree_run(tidigits.tp, tidigits.sseq, cit, both["info"], both["model"], scr[:90])
    assert np.array_equal(out1[1][0], want1[0]) and np.array_equal(out1[1][1], want1[1])
    out2 = ctx.ngram_fwdflat(d_scr.data_ptr(), utt_off, both["info"], both["model"], cit, cis, [o[0] for o in out1],
                             len(both["bp"]) + 64, len(both["bss"]) + 4096)
    assert np.array_equal(out2[0][0], both["bp"]) and np.array_equal(out2[0][1], both["bss"]) and np.array_equal(out2[0][2], both["bp_idx"])
    want2 = oracle.fwdflat_run(tidigits.tp, tidigits.sseq, cit, cis, both["info"], both["model"], want1[0], scr[:90])
    assert np.array_equal(out2[1][0], want2[0]) and np.array_equal(out2[1][1], want2[1])
    ctx.close()


@pytest.mark.timeout(600)
def test_default_pipeline_drop_in_through_the_binding(api, en_us):
    """The shipped default configuration (look-ahead, both passes, lattice + bestpath): device tables are
    imported into the reference through integration/ps_search_cuda.c and its own ngram_search_hyp must
    give the hypothesis and score of an undisturbed reference decode."""
    import torch
    from oracle import refdrv
    if not refdrv.available():
        pytest.skip("oracle/_ref/libpsref.so not built")
    rd = os.path.dirname(refdrv.LIB_PATH)
    hd, lm, dic = os.path.join(rd, "model", "en-us"), os.path.join(rd, "data", "turtle.lm.bin"), os.path.join(rd, "data", "turtle.dic")
    pcm = np.fromfile(os.path.join(rd, "data", "goforward.raw"), np.int16)
    kv = dict(fwdflat="yes", bestpath="yes", pl_window="5")
    want = refdrv.fwdtree(hd, lm, dic, pcm, **kv)
    ref = refdrv.RefModel(hd)
    scr = np.ascontiguousarray(ref.score(ref.featurize_fresh(pcm)))
    ref.close()
    ref = refdrv.RefModel(hd)                                   # fresh: the phone loop must start from a fresh CMN state
    pl = ref.phoneloop(pcm)
    ref.close()
    T, nc = len(scr), want["n_ci"]
    d_scr, d_pen = torch.from_numpy(scr).cuda(), torch.from_numpy(np.ascontiguousarray(pl["pen"], np.int32)).cuda()
    utt_off = np.array([0, T], np.int32)
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    cit, cis = en_us.phone_tmat[:nc], en_us.phone_ssid[:nc]
    first = ctx.ngram_fwdtree(d_scr.data_ptr(), utt_off, want["info"], want["model"], cit, 8192, 1 << 18, d_pen.data_ptr(), 5)
    bp, bss, idx = ctx.ngram_fwdflat(d_scr.data_ptr(), utt_off, want["info"], want["model"], cit, cis, [first[0][0]], 8192, 1 << 18)[0]
    ctx.close()
    rt = refdrv.ngram_roundtrip(hd, lm, dic, pcm, bp, bss, idx, **kv)
    assert rt["hyp"] == want["hyp"] == "go forward ten meters" and rt["score"] == want["score"]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("tag", ("flat_default", "flat_wide", "flat_narrow"))
def test_two_pass_chained_on_the_device(api, en_us, tag):
    """psb_ngram_two_pass_batch_device: first-pass tables never leave the device."""
    import torch
    gf = golden("en_us_goforward.npz")
    scr = gf["senscr"]
    c = _case(golden("en_us_fwdtree.npz"), tag)
    n_ci = int(c["info"][6])
    U = 5
    utt_off = (np.arange(U + 1) * len(scr)).astype(np.int32)
    d_scr = torch.from_numpy(np.ascontiguousarray(np.tile(scr, (U, 1)))).cuda()
    d_pen, win = None, 0
    if tag == "flat_default":
        win = int(gf["pl_params"][4])
        d_pen = torch.from_numpy(np.ascontiguousarray(np.tile(gf["pl_pen"].astype(np.int32), (U, 1)))).cuda()
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    out, n_first = ctx.ngram_two_pass(d_scr.data_ptr(), utt_off, c["info"], c["model"], en_us.phone_tmat[:n_ci], en_us.phone_ssid[:n_ci],
                                      len(c["bp"]) + 64, len(c["bss"]) + 4096, d_pen.data_ptr() if d_pen is not None else None, win,
                                      first_cap=8192, first_bss_cap=1 << 18)
    assert (n_first == n_first[0]).all() and n_first[0] > 0
    for u in range(U):
        bp, bss, idx = out[u]
        assert np.array_equal(bp, c["bp"]) and np.array_equal(bss, c["bss"]) and np.array_equal(idx, c["bp_idx"]), u
    ctx.close()


@pytest.mark.timeout(300)
def test_two_pass_with_the_array_lm(api, en_us):
    """LM as arrays on the device (psb_lm_core.h: the reference's interpolation search + float backoff sums),
    model block exported without the dense table."""
    import torch
    gf = golden("en_us_goforward.npz")
    g = golden("en_us_fwdtree.npz")
    scr = gf["senscr"]
    want = _case(g, "flat_default")
    n_ci = int(want["info"][6])
    U = 3
    utt_off = (np.arange(U + 1) * len(scr)).astype(np.int32)
    d_scr = torch.from_numpy(np.ascontiguousarray(np.tile(scr, (U, 1)))).cuda()
    d_pen = torch.from_numpy(np.ascontiguousarray(np.tile(gf["pl_pen"].astype(np.int32), (U, 1)))).cuda()
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    out, _ = ctx.ngram_two_pass(d_scr.data_ptr(), utt_off, g["nodense.info"], g["nodense.model"], en_us.phone_tmat[:n_ci],
                                en_us.phone_ssid[:n_ci], len(want["bp"]) + 64, len(want["bss"]) + 4096, d_pen.data_ptr(),
                                int(gf["pl_params"][4]), first_cap=8192, first_bss_cap=1 << 18, lm_arrays=g["lmarr"])
    for u in range(U):
        assert np.array_equal(out[u][0], want["bp"]) and np.array_equal(out[u][1], want["bss"]) and np.array_equal(out[u][2], want["bp_idx"])
    ctx.close()
