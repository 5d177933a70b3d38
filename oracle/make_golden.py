"""Generate tests/golden/*.npz from the compiled reference (oracle/_ref/libpsref.so).

Run in the build container only (needs /root/reference):  python -m oracle.make_golden
Everything written here is OUTPUT of the unmodified reference run on its own shipped models
and test audio: packed model arrays as its loaders leave them in memory, features from its
fe/feat front end, int16 senone scores from its ps_mgau back-ends, hmm_t states from its
hmm.c / phone_loop_search.c.  The GPU box has no /root/reference; tests there use these files.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import refdrv  # noqa: E402
from pocketsphinx_b200.model import PackedModel, load_npz  # noqa: E402

REF = os.environ.get("PS_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden")


def save_golden(path, limit=950_000, **arrays):
    """np.savez with LZMA members, split into parts (path, name.part1.npz, ...) that each stay under `limit` bytes: an
    array too large for one part is cut along axis 0 (pocketsphinx_b200.model.load_npz concatenates the pieces)."""
    import glob
    import io
    import lzma
    import zipfile

    def npy(a):
        b = io.BytesIO()
        np.lib.format.write_array(b, np.asanyarray(a), allow_pickle=False)
        return b.getvalue()
    pieces = []
    for k, a in arrays.items():
        a = np.asanyarray(a)
        n = 1
        while n < max(1, len(a) if a.ndim else 1) and len(lzma.compress(npy(a[:(len(a) + n - 1) // n]))) > limit * 0.9:
            n *= 2
        step = (len(a) + n - 1) // n if a.ndim else 1
        for i in range(n if a.ndim else 1):
            b = npy(a[i * step:(i + 1) * step] if a.ndim else a)
            pieces.append((k, b, len(lzma.compress(b))))
    stem = path[:-len(".npz")]
    for old in glob.glob(glob.escape(stem) + ".part*.npz"):
        os.remove(old)
    files, size = [[]], 0
    for pc in pieces:
        if files[-1] and size + pc[2] > limit:
            files.append([]); size = 0
        files[-1].append(pc); size += pc[2]
    for i, fl in enumerate(files):
        with zipfile.ZipFile(path if i == 0 else "%s.part%d.npz" % (stem, i), "w", zipfile.ZIP_LZMA) as z:
            for k, b, _ in fl:
                z.writestr(k + ".npy", b)


def save_model(name, pm_dict, keep_phones=None):
    pm = PackedModel.from_dict(pm_dict)
    if keep_phones is not None:          # en-us has 137k triphones; the CI phones are enough
        pm.phone_ssid = pm.phone_ssid[:keep_phones]
        pm.phone_tmat = pm.phone_tmat[:keep_phones]
    path = os.path.join(OUT, name)
    save_golden(path, **pm.to_npz_dict())
    print(name, os.path.getsize(path) // 1024, "KiB")
    return pm


def make_align():
    """en_us_align.npz: the reference's own state_align_search (ps_set_alignment) on goforward.raw
    with its transcript, all senones, no look-ahead: phone chain and state-level alignment."""
    pcm = np.fromfile(os.path.join(REF, "test/data/goforward.raw"), np.int16)
    out = {}
    for tag, words in (("a", "<s> go forward ten meters </s>"), ("b", "go forward ten meters"),
                       ("c", "<s> go forward ten meters </s> <s> go forward </s>")):
        a = refdrv.align(os.path.join(REF, "model/en-us/en-us"), os.path.join(REF, "model/en-us/cmudict-en-us.dict"),
                         words, pcm)
        for k in ("ssid", "tmatid", "start", "dur", "score"):
            out[tag + "_" + k] = a[k]
        print("align", tag, len(a["ssid"]), "phones", a["dur"].sum(), "frames covered")
    save_golden(os.path.join(OUT, "en_us_align.npz"), **out)


def make_kws():
    """en_us_kws.npz: the reference's own kws_search on goforward.raw (all senones, no look-ahead)
    for a single keyphrase and for a four-entry list: configuration as kws_search_reinit built it
    and the final detection list."""
    import tempfile
    pcm = np.fromfile(os.path.join(REF, "test/data/goforward.raw"), np.int16)
    hmm, dic = os.path.join(REF, "model/en-us/en-us"), os.path.join(REF, "model/en-us/cmudict-en-us.dict")
    out = {}
    with tempfile.NamedTemporaryFile("w", suffix=".list", delete=False) as f:
        f.write("forward /1e-20/\nten meters /1e-30/\ngo /1e-10/\nbackward /1e-40/\n")
    for tag, kw in (("a", dict(keyphrase="forward", kws_threshold="1e-20")), ("b", dict(keyfile=f.name))):
        a = refdrv.kws(hmm, dic, pcm, **kw)
        for k in ("pl_ssid", "pl_tmat", "kp_off", "kp_thresh", "kp_ssid", "kp_tmat", "det"):
            out[tag + "_" + k] = a[k]
        out[tag + "_beam"], out[tag + "_plp"] = np.int32(a["beam"]), np.int32(a["plp"])
        print("kws", tag, len(a["kp_off"]) - 1, "keyphrases", len(a["det"]), "detections")
    os.unlink(f.name)
    save_golden(os.path.join(OUT, "en_us_kws.npz"), **out)


def make_allphone():
    """en_us_allphone.npz: the reference's own allphone_search (no phone LM, context-independent
    graph = the default -allphone_ci yes) on goforward.raw: graph, parameters, history count and
    the phone segmentation."""
    pcm = np.fromfile(os.path.join(REF, "test/data/goforward.raw"), np.int16)
    a = refdrv.allphone(os.path.join(REF, "model/en-us/en-us"), pcm)
    out = {k: a[k] for k in ("ci", "ssid", "tmatid", "succ_off", "succ", "segs")}
    for k in ("start", "beam", "pbeam", "inspen", "n_history"):
        out[k] = np.int32(a[k])
    print("allphone", len(a["ci"]), "nodes", len(a["succ"]), "links", a["n_history"], "history entries", len(a["segs"]), "segments")
    # the same search with the shipped phone LM: dense bigram / trigram score tables tabulated
    # through the search's own LM object, and the resulting segmentation
    b = refdrv.allphone(os.path.join(REF, "model/en-us/en-us"), pcm,
                        allphone=os.path.join(REF, "model/en-us/en-us-phone.lm.bin"))
    assert np.array_equal(b["ssid"], a["ssid"]) and np.array_equal(b["succ"], a["succ"])
    out["lm_bg"], out["lm_tg"], out["lm_segs"] = b["bg"], b["tg"], b["segs"]
    out["lm_n_history"] = np.int32(b["n_history"])
    for k in ("beam", "pbeam"):
        assert int(b[k]) == int(a[k])
    print("allphone + phone LM", len(b["segs"]), "segments")
    save_golden(os.path.join(OUT, "en_us_allphone.npz"), **out)


def make_fsg():
    """en_us_fsg.npz: the reference's own fsg_search on goforward.raw for two grammars -- its shipped
    test/data/goforward.fsg and tests/golden/commands.fsg (ours: loops, null transitions out of the
    start state and between states, a single-phone word) -- with the default beams and with -maxhmmpf
    low enough to trigger the beam narrowing: flattened lextree, links, null arcs, parameters, the
    complete history table, hypothesis and score."""
    pcm = np.fromfile(os.path.join(REF, "test/data/goforward.raw"), np.int16)
    hd, dic = os.path.join(REF, "model/en-us/en-us"), os.path.join(REF, "model/en-us/cmudict-en-us.dict")
    out = {}
    for tag, path, kv in (("go", os.path.join(REF, "test/data/goforward.fsg"), {}),
                          ("go_hmmpf", os.path.join(REF, "test/data/goforward.fsg"), dict(maxhmmpf="20")),
                          ("cmd", os.path.join(OUT, "commands.fsg"), {}),
                          ("cmd_wide", os.path.join(OUT, "commands.fsg"), dict(beam="1e-80", pbeam="1e-80", wbeam="1e-60")),
                          ("cmd_hmmpf", os.path.join(OUT, "commands.fsg"), dict(maxhmmpf="100", wip="0.2", pip="0.5"))):
        r = refdrv.fsg(hd, dic, path, pcm, **kv)
        for k, v in r.items():
            out[tag + "." + k] = np.array("\n".join(v)) if k == "vocab" else np.array(v)
        print("fsg", tag, len(r["pnodes"]), "pnodes", len(r["links"]), "links", len(r["hist"]), "history entries:", r["hyp"], r["score"])
    save_golden(os.path.join(OUT, "en_us_fsg.npz"), **out)


def make_fwdtree():
    """en_us_fwdtree.npz: the reference's own first pass (ngram_search_fwdtree, turtle LM + dictionary,
    no fwdflat / bestpath / look-ahead) on goforward.raw: the flattened search (lextree, dictionary and
    dict2pid tables, dense trigram table, parameters) and what it produced -- every backpointer-table
    entry, the right-context score stack, bp_table_idx, hypothesis and score -- for the default
    settings, wide and narrow beams, absolute pruning (-maxwpf, -maxhmmpf) and non-default penalties."""
    pcm = np.fromfile(os.path.join(REF, "test/data/goforward.raw"), np.int16)
    hd = os.path.join(REF, "model/en-us/en-us")
    out = {}
    for tag, kv in (("default", {}),
                    ("wide", dict(beam="1e-80", pbeam="1e-80", wbeam="1e-60", lpbeam="1e-60", lponlybeam="1e-50")),
                    ("narrow", dict(beam="1e-30", pbeam="1e-25", wbeam="1e-15", lpbeam="1e-20", lponlybeam="1e-15")),
                    ("maxwpf", dict(maxwpf="5")),
                    ("abs", dict(maxhmmpf="50", maxwpf="10")),
                    ("pen", dict(nwpen="0.5", pip="0.7", wip="0.3", lw="9.5", silprob="0.01", fillprob="1e-4")),
                    # the shipped default: phone-loop look-ahead on (its penalties are en_us_goforward.npz:pl_pen)
                    ("lookahead", dict(pl_window="5"))):
        r = refdrv.fwdtree(hd, os.path.join(REF, "test/data/turtle.lm.bin"), os.path.join(REF, "test/data/turtle.dic"), pcm, **kv)
        for k in ("info", "model", "bp", "bss", "bp_idx", "words"):
            out[tag + "." + k] = r[k]
        out[tag + ".vocab"] = np.array("\n".join(r["vocab"]))
        out[tag + ".hyp"] = np.array(r["hyp"])
        out[tag + ".score"] = np.int32(r["score"])
        print("fwdtree", tag, r["n_root"], "root", r["n_nonroot"], "non-root channels,", r["bpidx"], "bp entries,",
              r["bss_head"], "rc scores:", r["hyp"], r["score"])
    # second pass (ngram_search_fwdflat) on top of the first: the shipped default pipeline (look-ahead on in
    # the first pass), wide and narrow second-pass beams with other end-frame / start-window limits
    for tag, kv in (("flat_default", dict(pl_window="5")),
                    ("flat_wide", dict(fwdflatbeam="1e-80", fwdflatwbeam="1e-40", fwdflatefwid="1", fwdflatsfwin="60")),
                    ("flat_narrow", dict(fwdflatbeam="1e-30", fwdflatwbeam="1e-10", fwdflatefwid="8", fwdflatsfwin="5",
                                         fwdflatlw="12"))):
        r = refdrv.fwdtree(hd, os.path.join(REF, "test/data/turtle.lm.bin"), os.path.join(REF, "test/data/turtle.dic"), pcm,
                           fwdflat="yes", **kv)
        for k in ("info", "model", "bp", "bss", "bp_idx", "words"):
            out[tag + "." + k] = r[k]
        out[tag + ".vocab"] = np.array("\n".join(r["vocab"]))
        out[tag + ".hyp"] = np.array(r["hyp"])
        out[tag + ".score"] = np.int32(r["score"])
        print("fwdflat", tag, r["bpidx"], "bp entries,", r["bss_head"], "rc scores:", r["hyp"], r["score"])
    # the turtle LM as sorted arrays (integration/ps_search_cuda.c:cuda_ngram_export_lm) for the array-LM mode of
    # the searches, and a sample of the reference's own trigram scores to pin the array scoring without the reference
    nw = int(out["default.info"][1])
    rng = np.random.default_rng(3)
    q = np.stack([rng.integers(0, nw, 20000), rng.integers(-1, nw, 20000), rng.integers(-1, nw, 20000)], 1).astype(np.int32)
    out["lmarr"], out["lmarr_scores"] = refdrv.lm_arrays(hd, os.path.join(REF, "test/data/turtle.lm.bin"),
                                                         os.path.join(REF, "test/data/turtle.dic"), q)
    out["lmarr_queries"] = q
    r = refdrv.fwdtree(hd, os.path.join(REF, "test/data/turtle.lm.bin"), os.path.join(REF, "test/data/turtle.dic"), pcm,
                       dense_lm=False, fwdflat="yes")
    out["nodense.info"], out["nodense.model"] = r["info"], r["model"]          # same search, exported without the dense table
    save_golden(os.path.join(OUT, "en_us_fwdtree.npz"), **out)


def make_fe():
    """tests/golden/fe_reference.npz: the reference front end's tables and outputs for oracle/fe_golden.cases()."""
    from oracle import fe_golden
    go = np.fromfile(os.path.join(REF, "test", "data", "goforward.raw"), np.int16)
    out = {"goforward": go[:23000]}
    hd = os.path.join(os.path.dirname(refdrv.LIB_PATH), "model", "en-us")
    for kv, mf_in, ft_in in fe_golden.cases(go):
        name = fe_golden.config_name(kv)
        ref = refdrv.RefModel(hd, **kv)
        for k, v in ref.fe_desc().items():
            out["desc.%s.%s" % (name, k)] = np.asarray(v)
        for pcm in mf_in:
            out["mfcc.%s.%s" % (name, fe_golden.pcm_key(pcm))] = ref.mfcc(pcm)
        for pcm in ft_in:
            if len(pcm):
                out["feat.%s.%s" % (name, fe_golden.pcm_key(pcm))] = ref.featurize_fresh(pcm)
        ref.close()
    save_golden(fe_golden.GOLDEN, **out)


def make_fixed_point():
    """fx_en_us.npz / fx_tidigits.npz: the reference compiled with -DFIXED_POINT (oracle/_ref/libpsref_fx.so,
    `make -C oracle fx`) on goforward.raw: its Q12 features, every top-N list and its senone scores.  Run as
    `PSREF_LIB=oracle/_ref/libpsref_fx.so python -m oracle.make_golden fx`.  To keep the files small the model's
    int32 means / variance terms and the scores are stored as differences from what the float build's goldens
    give (|d mean| <= 1 after (int32)(mean * 4096), d var in {0, 1}, d senscr within int16): tests/conftest.py
    `fx_case` puts them back together; the determinants are (int32)det exactly."""
    assert "fx" in os.path.basename(refdrv.LIB_PATH), "set PSREF_LIB to the FIXED_POINT build"
    ref_dir = os.path.dirname(refdrv.LIB_PATH)
    pcm = np.fromfile(os.path.join(ref_dir, "data", "goforward.raw"), np.int16)
    for name, mdl, gm, gg in (("en_us", "en-us", "en_us_ptm_model.npz", "en_us_goforward.npz"),
                              ("tidigits", "tidigits_hmm", "tidigits_sc_model.npz", "tidigits_goforward.npz")):
        ref = refdrv.RefModel(os.path.join(ref_dir, "model", mdl))
        feats = ref.featurize(pcm).view(np.int32)          # mfcc_t = int32 (Q12), carried as 4-byte words
        scr, topn = ref.score(feats.view(np.float32), want_topn=True)
        pm = PackedModel.load(os.path.join(OUT, gm))
        mean, var, det = ref.export("mean", np.int32).ravel(), ref.export("var", np.int32).ravel(), ref.export("det", np.int32).ravel()
        dm = mean - (pm.mean.astype(np.float32) * np.float32(4096)).astype(np.int32)
        dv = var - pm.var.astype(np.int32)
        assert np.array_equal(det, pm.det.astype(np.int32)) and np.abs(dm).max() <= 1 and dv.min() >= 0 and dv.max() <= 1
        ds = scr.astype(np.int32) - load_npz(os.path.join(OUT, gg))["senscr"]
        assert np.abs(ds).max() < 32768
        path = os.path.join(OUT, "fx_%s.npz" % name)
        save_golden(path, feats=feats, dmean=dm.astype(np.int8), dvar=dv.astype(np.int8), dsenscr=ds.astype(np.int16),
                            topn=topn.astype(np.int32))
        print(path, os.path.getsize(path) // 1024, "KiB;", "%.0f %% of the scores differ from the float build's" % (100 * (ds != 0).mean()))


def main():
    os.makedirs(OUT, exist_ok=True)
    if len(sys.argv) > 1 and sys.argv[1] == "fe":
        return make_fe()
    if len(sys.argv) > 1 and sys.argv[1] == "fx":
        return make_fixed_point()
    if len(sys.argv) > 1 and sys.argv[1] == "fwdtree":
        return make_fwdtree()
    if len(sys.argv) > 1 and sys.argv[1] == "fsg":
        return make_fsg()
    if len(sys.argv) > 1 and sys.argv[1] == "allphone":
        return make_allphone()
    if len(sys.argv) > 1 and sys.argv[1] == "align":
        return make_align()
    if len(sys.argv) > 1 and sys.argv[1] == "kws":
        return make_kws()
    pcm = np.fromfile(os.path.join(REF, "test/data/goforward.raw"), np.int16)

    # ---- en-us PTM (BASELINE config 1): goforward.raw, 278 frames, all senones ----
    m = refdrv.RefModel(os.path.join(REF, "model/en-us/en-us"))
    save_model("en_us_ptm_model.npz", m.packed(), keep_phones=4096)
    pl = m.phoneloop(pcm)                       # first utterance of a fresh decoder
    feats = pl["feat"]
    scr, topn = m.score(feats, want_topn=True)
    assert (scr == pl["senscr"]).all()
    par = pl["params"]
    save_golden(
        os.path.join(OUT, "en_us_goforward.npz"), feats=feats, senscr=scr,
        topn_last=topn[-1], topn_first=topn[0],
        pl_hmm=pl["hmm"].view(np.uint8).reshape(pl["hmm"].shape + (88,)), pl_best=pl["best"], pl_pen=pl["pen"],
        pl_params=np.array([par["n_phones"], par["beam"], par["pbeam"], par["pip"], par["window"]], np.int32),
        pl_weight=np.float64(par["penalty_weight"]))
    # active-list mode (compallsen = no): random flags with a few wide gaps
    rng = np.random.default_rng(7)
    T = 40
    flags = (rng.random((T, m.n_sen)) < 0.3).astype(np.uint8)
    flags[:, 1000:1700] = 0
    flags[5] = 0
    flags[6, :] = 0
    flags[6, 4000] = 1
    ascr, nact, lists = m.score_active(feats[:T], flags)
    save_golden(os.path.join(OUT, "en_us_active.npz"), flags=np.packbits(flags, axis=1),
                        n_sen=m.n_sen, senscr=ascr, nact=nact)
    m.close()

    # ---- tidigits semi-continuous (4 streams, 256 Gaussians, 4-bit clustered sendump) ----
    m = refdrv.RefModel(os.path.join(REF, "test/data/tidigits/hmm"))
    print("tidigits:", m.kind, m.n_sen, m.n_mgau, m.n_feat, m.n_density, m.featlen, "4bit" if m.mixw_4bit else "8bit")
    save_model("tidigits_sc_model.npz", m.packed())
    f = m.featurize(pcm)
    s, tn = m.score(f, want_topn=True)
    save_golden(os.path.join(OUT, "tidigits_goforward.npz"), feats=f, senscr=s, topn=tn)
    m.close()

    # ---- an4 continuous (ms back-end, 1 Gaussian per senone) ----
    m = refdrv.RefModel(os.path.join(REF, "test/data/an4_ci_cont"))
    print("an4:", m.kind, m.n_sen, m.n_mgau, m.n_feat, m.n_density, m.featlen, "topn", m.topn)
    save_model("an4_cont_model.npz", m.packed())
    f = m.featurize(pcm)
    s = m.score(f)
    save_golden(os.path.join(OUT, "an4_goforward.npz"), feats=f, senscr=s)
    m.close()

    # ---- en-us through the ms back-end too (-senmgau .ptm. forces ms_mgau_init first) ----
    # not shipped: en-us has no mixture_weights file, only a sendump; skipped.

    # ---- hmm_vit_eval: random states through the reference's five specialisations ----
    rng = np.random.default_rng(11)
    cases = {}
    for n_emit in (3, 5, 4, 1):
        n_tmat, n_sseq, n_sen, n = 7, 50, 200, 4096
        tp = np.full((n_tmat, n_emit, n_emit + 1), 255, np.uint8)
        for t in range(n_tmat):
            for i in range(n_emit):
                tp[t, i, i] = rng.integers(0, 60)
                tp[t, i, i + 1] = rng.integers(0, 60)
                if i + 2 <= n_emit and rng.random() < 0.5:
                    tp[t, i, i + 2] = rng.integers(0, 90)
        sseq = rng.integers(0, n_sen, (n_sseq, n_emit)).astype(np.uint16)
        ctx = refdrv.RefHmmCtx(tp, sseq)
        senscr = rng.integers(0, 700, n_sen).astype(np.int16)
        mpx = (rng.random(n) < 0.5).astype(np.int32)
        hm = ctx.init(n, mpx, rng.integers(0, n_sseq, n), rng.integers(0, n_tmat, n))
        # random but plausible path scores, some states dead, some mpx slots empty
        sc = rng.integers(-200000, 0, (n, 5)).astype(np.int32)
        dead = rng.random((n, 5)) < 0.25
        sc[dead] = -0x20000000
        near = rng.random((n, 5)) < 0.03
        sc[near] = -0x20000000 + rng.integers(-300, 300, near.sum())
        hm["score"] = sc
        hm["history"] = rng.integers(-1, 1000, (n, 5))
        hm["out_score"] = rng.integers(-200000, 0, n)
        hm["out_history"] = rng.integers(-1, 1000, n)
        for st in range(1, n_emit):
            sel = (mpx == 1) & (rng.random(n) < 0.7)
            hm["senid"][sel, st] = rng.integers(0, n_sseq, sel.sum())
        # dead states of mpx HMMs keep BAD_SSID like the search leaves them
        badsel = (mpx[:, None] == 1) & dead & (np.arange(5)[None, :] > 0)
        hm["senid"][badsel] = 0xffff
        before = hm.copy()
        best = ctx.vit_eval(hm, senscr)
        before["ctx"] = 0
        hm["ctx"] = 0
        cases["n%d_tp" % n_emit] = tp
        cases["n%d_sseq" % n_emit] = sseq
        cases["n%d_senscr" % n_emit] = senscr
        cases["n%d_before" % n_emit] = before.view(np.uint8).reshape(n, 88)
        cases["n%d_after" % n_emit] = hm.view(np.uint8).reshape(n, 88)
        cases["n%d_best" % n_emit] = np.int32(best)
        ctx.close()
    save_golden(os.path.join(OUT, "hmm_vit_eval.npz"), **cases)
    make_align()
    make_kws()
    make_allphone()
    for fn in sorted(os.listdir(OUT)):
        print("%8d KiB  %s" % (os.path.getsize(os.path.join(OUT, fn)) // 1024, fn))


if __name__ == "__main__":
    main()
