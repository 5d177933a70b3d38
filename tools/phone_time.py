"""Times phone decoding from audio (pocketsphinx_b200.phones.PhoneDecoder) with the en-us model: 1000 utterances of
10 s (goforward.raw repeated to length) on the CI net without and with the phone LM
(tests/golden/en-us-phone.lm.bin), and 64 such utterances on the context-dependent net (-allphone_ci no) with the
phone LM.  For each: the device time of the search alone (CUDA events around HmmContext.allphone_net on the scores decode_raw_batch left on the device), the device time
and the wall time of decode_raw_batch (front end, senone scores, search and the host's result rules); the card's name
and power limit; and the reference's allphone search on one host core for one such utterance at the same settings
(the compiled reference under oracle/_ref through its public API: ps_init, ps_decode_raw with -compallsen yes,
ps_get_hyp; model loading included).  One JSON line per measurement.

    python tools/phone_time.py [--utts 1000] [--cd-utts 64] [--secs 10] [--reps 3] [--ref-reps 1] [--configs ci,ci_lm,cd_lm]
                               [--skip-reference]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
REF = os.path.join(ROOT, "oracle", "_ref")
HD, LM = os.path.join(REF, "model", "en-us"), os.path.join(ROOT, "tests", "golden", "en-us-phone.lm.bin")
GO = os.path.join(REF, "data", "goforward.raw")

# name: (phone LM, settings, utterances argument)
CONFIGS = dict(ci=(None, {}, "utts"), ci_lm=(LM, {}, "utts"), cd_lm=(LM, dict(allphone_ci="no"), "cd_utts"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=1000)
    ap.add_argument("--cd-utts", type=int, default=64)
    ap.add_argument("--secs", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-reps", type=int, default=1)
    ap.add_argument("--configs", default="ci,ci_lm,cd_lm")
    ap.add_argument("--skip-reference", action="store_true")
    args = ap.parse_args()
    utt = np.resize(np.fromfile(GO, np.int16), int(args.secs * 16000)).astype(np.int16)
    configs = {k: v for k, v in CONFIGS.items() if k in args.configs.split(",")}
    if not args.skip_reference:
        reference_time(utt, configs, args.ref_reps)
    import torch
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.phones import PhoneDecoder
    if api.device_count() == 0:
        raise SystemExit("phone_time.py measures on a CUDA device; none found")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu)), flush=True)
    for name, (lm, kv, n_arg) in configs.items():
        n = getattr(args, n_arg)
        dec = PhoneDecoder(HD, lm, max_utts=n, max_frames=n * (len(utt) // 160 + 1), **kv)
        p = dec.search
        utts = [utt] * n
        wall, dev, search_ms, res = [], [], [], None
        for r in range(args.reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            res = dec.decode_raw_batch(utts)
            e1.record()
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            off = np.cumsum([0] + [o["n_frames"] for o in res]).astype(np.int32)
            k0, k1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            k0.record()
            dec.ctx.allphone_net(dec.batch.senscr_device_ptr(), off, p["net"], p["beam"], p["pbeam"], p["inspen"],
                                 bg=p["bg"], tg=p["tg"])
            k1.record()
            torch.cuda.synchronize()
            if r:
                wall.append((t1 - t0) * 1e3); dev.append(e0.elapsed_time(e1)); search_ms.append(k0.elapsed_time(k1))
        n_frames = int(off[-1])
        print(json.dumps(dict(config=name, nodes=len(p["net"]["ci"]), phone_lm=lm is not None, utts=n, frames=n_frames,
                              audio_s=n_frames / 100.0, phones=sum(len(o["seg"]) for o in res),
                              failed=sum(o["hyp"] is None for o in res),
                              search_device_ms_median=float(np.median(search_ms)),
                              decode_device_ms_median=float(np.median(dev)),
                              decode_wall_ms_median=float(np.median(wall)), decode_wall_ms_min=float(min(wall)))),
              flush=True)
        dec.close()


def reference_time(utt, configs, reps):
    """The reference's allphone search on one host core: one utterance, front end and all-senone scoring included,
    and ps_init (model and phone LM loading) too."""
    from oracle import refdrv
    if not refdrv.available() or not os.path.exists(LM):
        print(json.dumps(dict(reference="not available (oracle/_ref not built)")), flush=True)
        return
    from phone_cases import ref_phones
    for name, (lm, kv, _) in configs.items():
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            ref_phones(HD, lm, pcm=utt, **kv)
            ts.append((time.perf_counter() - t0) * 1e3)
        print(json.dumps(dict(reference=name, utts=1, audio_s=len(utt) / 16000.0, host_cores=1,
                              wall_ms_median_with_init=float(np.median(ts)))), flush=True)


if __name__ == "__main__":
    main()
