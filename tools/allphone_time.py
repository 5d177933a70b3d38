"""Times psb_allphone_net_batch_device on the en-us context-dependent PHMM net (-allphone_ci no, 29 324 nodes)
over a batch of real-length utterances (goforward.raw's 278 frames of senone scores, repeated), without and with
the phone LM (test/unit/test_allphone.c's beams), and the context-independent net for comparison: CUDA events
around the call, warm-up, median.  Reports the history bytes per utterance, the card name and power limit, and
the reference's goforward.raw decode with its allphone search on one host core (the compiled reference under
oracle/_ref; CI and CD net without an LM, and the CD net with the phone LM where --phone-lm exists).  Prints
one JSON line per measurement.

    python tools/allphone_time.py [--utts 1,16,64] [--reps 5] [--phone-lm path] [--skip-reference | --reference-only]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", default="1,16,64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--phone-lm", default=os.path.join(os.environ.get("PS_REFERENCE", "/nonexistent"), "model", "en-us",
                                                       "en-us-phone.lm.bin"),
                    help="the reference's en-us-phone.lm.bin, for its phone-LM timing (skipped where absent)")
    ap.add_argument("--skip-reference", action="store_true")
    ap.add_argument("--reference-only", action="store_true")
    args = ap.parse_args()
    if args.reference_only:
        return reference_time(args.phone_lm)
    import torch
    from conftest import golden
    from test_allphone_net_emul import cd_phones
    from pocketsphinx_b200 import allphone_net as A, api
    from pocketsphinx_b200.model import PackedModel
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu)), flush=True)
    pm = PackedModel.load(os.path.join(ROOT, "tests", "golden", "en_us_ptm_model.npz"))
    g = golden("en_us_allphone_cd.npz")
    scr = golden("en_us_goforward.npz")["senscr"]
    ctx = api.HmmContext(pm.tp, pm.sseq, pm.n_sen)
    nets = dict(cd=A.build_net(cd_phones(g), ci_only=False), ci=A.build_net(cd_phones(g), ci_only=True))
    for n_utt in [int(x) for x in args.utts.split(",")]:
        d = torch.from_numpy(np.concatenate([scr] * n_utt)).cuda()
        uo = (np.arange(n_utt + 1) * len(scr)).astype(np.int32)
        for name, net in nets.items():
            for lm in (False, True):
                kw = dict(bg=g["lm_bg"], tg=g["lm_tg"]) if lm else dict(inspen=int(g["inspen"]))
                beams = (int(g["lm_beam"]), int(g["lm_pbeam"])) if lm else (int(g["beam"]), int(g["pbeam"]))
                ms = []
                for r in range(args.reps + 1):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    e0.record()
                    out = ctx.allphone_net(d.data_ptr(), uo, net, *beams, hist_budget=64 << 30, **kw)
                    e1.record()
                    torch.cuda.synchronize()
                    if r:
                        ms.append(e0.elapsed_time(e1))
                assert (out["status"] == 0).all()
                print(json.dumps(dict(net=name, lm=lm, nodes=len(net["ci"]), utts=n_utt, frames=len(scr),
                                      device_ms_median=float(np.median(ms)), device_ms_min=float(min(ms)),
                                      ms_per_utt=float(np.median(ms)) / n_utt, n_hist=int(out["n_hist"][0]),
                                      hist_bytes_per_utt=int(out["n_hist"][0]) * 16,
                                      hist_bytes_reserved_per_utt=len(scr) * len(net["ci"]) * 16)), flush=True)
        del d
    ctx.close()
    if not args.skip_reference:
        reference_time(args.phone_lm)


def reference_time(phone_lm):
    """The reference's whole goforward.raw decode with its allphone search on one host core: the wall time
    of the utterance alone (start_utt .. end_utt, second of two passes; front end and all-senone scoring
    included), median of 3.  Without a loadable -allphone LM, allphone_search_init falls back to the
    unconstrained phone loop (allphone_search.c:578-585): that is the no-LM search."""
    import ctypes as C
    from oracle import refdrv
    if not refdrv.available():
        return
    L = refdrv.lib()
    hmm = os.path.join(ROOT, "oracle", "_ref", "model", "en-us").encode()
    pcm = np.fromfile(os.path.join(ROOT, "oracle", "_ref", "data", "goforward.raw"), np.int16)
    runs = [("ci_no_lm", "allphone=-\nallphone_ci=yes"), ("cd_no_lm", "allphone=-\nallphone_ci=no")]
    if phone_lm and os.path.exists(phone_lm):
        runs.append(("cd_phone_lm", "allphone=%s\nallphone_ci=no\nbeam=1e-20\npbeam=1e-10\nlw=2.0" % phone_lm))
    out = {}
    for name, kv in runs:
        ts = []
        for _ in range(3):
            hyp, seg = C.create_string_buffer(4096), C.create_string_buffer(65536)
            st = np.zeros(4, np.int32)
            st[3] = 1
            n = L.refdrv_decode(hmm, None, None, (kv + "\ncompallsen=yes").encode(), pcm.ctypes.data_as(C.c_void_p), len(pcm),
                                0, None, hyp, 4096, seg, 65536, st.ctypes.data_as(C.c_void_p))
            assert n > 0, name
            ts.append(st[3] / 1e6)
        out[name] = float(np.median(ts))
    print(json.dumps(dict(reference_one_core_goforward_utterance_s=out)), flush=True)


if __name__ == "__main__":
    main()
