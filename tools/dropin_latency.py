#!/usr/bin/env python
"""Per-frame drop-in latency (VERDICT r1 weak #8): what an unmodified decoder gets from
psb_scorer_frame_eval (one launch chain + a 10 KB D2H + a stream sync per call; twice per frame with
the phone-loop look-ahead) next to the reference's own ptm_mgau_frame_eval on one host core.
  (a) micro: api.Mgau.frame_eval on the en-us golden model, all senones / CI senones only / a 30 % active list;
  (b) inside a real decode: the compiled reference's ps_decode_raw of goforward.raw with its own back-end and
      with the CUDA back-end bound through integration/ps_mgau_cuda.c (wall clock of the whole decode, per frame).
Prints one JSON object; run on the GPU box:  python tools/dropin_latency.py > gpurun_out/dropin_latency.json"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from pocketsphinx_b200 import _lib, api
    from pocketsphinx_b200.model import PackedModel, load_npz
    gd = os.path.join(ROOT, "tests", "golden")
    pm = PackedModel.load(os.path.join(gd, "en_us_ptm_model.npz"))
    g = load_npz(os.path.join(gd, "en_us_goforward.npz"))
    feats = g["feats"]
    out = {"model": "en-us PTM 42x3x128x13, 5126 senones", "frames": int(len(feats))}
    m = api.Model(pm)
    rng = np.random.default_rng(0)
    flags = (rng.random(pm.n_sen) < 0.3).astype(np.uint8)
    ci = np.zeros(pm.n_sen, np.uint8)
    ci[:pm.n_ci_sen] = 1
    try:
        from oracle import oracle
        lists = {"compallsen": None, "ci_only": oracle.flags2list(ci), "active_30pct": oracle.flags2list(flags)}
    except Exception:
        lists = {"compallsen": None}
    micro = {}
    for name, lst in lists.items():
        s = api.Mgau(m, pl_window=0)
        for rep in range(2):                     # first pass warms up
            t0 = time.perf_counter()
            for t in range(len(feats)):
                if lst is None:
                    s.frame_eval(feats[t], t)
                else:
                    s.frame_eval(feats[t], t, lst, compallsen=False)
                s.frame_idx = t + 1
            dt = time.perf_counter() - t0
            s.frame_idx = 0
        micro[name] = {"us_per_call": dt / len(feats) * 1e6}
        s.close()
    out["psb_scorer_frame_eval"] = micro
    m.close()
    try:
        from oracle import refdrv
        ref = os.path.dirname(refdrv.LIB_PATH)
        rm = refdrv.RefModel(os.path.join(ref, "model", "en-us"))
        t0 = time.perf_counter()
        for _ in range(3):
            rm.score(feats)
        out["reference_ptm_mgau_frame_eval_us_per_frame_1core"] = (time.perf_counter() - t0) / (3 * len(feats)) * 1e6
        rm.close()
        pcm = np.fromfile(os.path.join(ref, "data", "goforward.raw"), np.int16)
        args = (os.path.join(ref, "model", "en-us"), os.path.join(ref, "model", "en-us.lm.bin"),
                os.path.join(ref, "model", "cmudict-en-us.dict"), pcm)
        dec = {}
        for name, kv in (("default (pl_window 5: two frame_eval calls per frame)", {}), ("pl_window 0", {"pl_window": "0"})):
            row = {}
            for use_cuda in (False, True):
                r = refdrv.decode(*args, use_cuda=use_cuda, libpath=_lib.LIB_PATH, twice=True, **kv)
                row["cuda" if use_cuda else "host"] = {"utt_ms": r["utt_us"] / 1e3, "us_per_frame": r["utt_us"] / max(1, r["n_frames"]),
                                                       "frames": r["n_frames"], "hyp": r["hyp"], "frame_eval_calls": r.get("cuda_calls")}
            dec[name] = row
        out["ps_decode_raw_en_us_lm_cmudict"] = dec
        out["note"] = ("utt_ms: ps_start_utt .. ps_end_utt of the second of two passes over goforward.raw (front end, GMM, fwdtree, "
                       "fwdflat, bestpath); frame_eval_calls counts both passes; host vs cuda differ only in the GMM back-end")
    except Exception as e:
        out["reference_error"] = str(e)[:200]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
