"""Times keyword spotting (pocketsphinx_b200.kws.KeywordSpotter) with the en-us model: a batch of 10-second
utterances (goforward.raw repeated to length) with the reference's goforward.kws list and with a synthetic list of
500 keyphrases drawn from cmudict (well above the 512 HMMs the kernel once kept per utterance), and one 60-minute
stream.  For each: the device time of the kws search alone (CUDA events around HmmContext.kws), the device time of
front end + senone scores + search, and the wall time of spot_raw_batch (host detection rules included); the card's
name and power limit; and the reference's kws search on one host core for one such utterance (the compiled
reference under oracle/_ref, front end and all-senone scoring included, median of --reps).  One JSON line per
measurement.

    python tools/kws_time.py [--utts 1000] [--secs 10] [--stream-min 60] [--reps 3] [--lists goforward,cmudict500]
                             [--shapes batch,stream] [--skip-reference]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
REF = os.path.join(ROOT, "oracle", "_ref")
HD, DIC = os.path.join(REF, "model", "en-us"), os.path.join(REF, "model", "cmudict-en-us.dict")
GO = os.path.join(REF, "data", "goforward.raw")
KWS_FILE = os.path.join(ROOT, "tests", "golden", "goforward.kws")


def synthetic_list(path, n, seed=1):
    """n distinct cmudict words (no alternate pronunciations), one per line: a keyphrase list of n entries."""
    with open(DIC) as f:
        words = [l.split()[0] for l in f if l.strip() and "(" not in l.split()[0]]
    rng = np.random.default_rng(seed)
    pick = rng.choice(len(words), n, replace=False)
    with open(path, "w") as f:
        f.write("".join(words[i] + "\n" for i in sorted(pick)))


def tiled(pcm, n):
    return np.resize(pcm, n).astype(np.int16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=1000)
    ap.add_argument("--secs", type=float, default=10.0)
    ap.add_argument("--stream-min", type=float, default=60.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--lists", default="goforward,cmudict500")
    ap.add_argument("--shapes", default="batch,stream")
    ap.add_argument("--skip-reference", action="store_true")
    args = ap.parse_args()
    go = np.fromfile(GO, np.int16)
    utt = tiled(go, int(args.secs * 16000))
    stream = tiled(go, int(args.stream_min * 60 * 16000))
    tmp = tempfile.mkdtemp(prefix="kws_time_")
    big = os.path.join(tmp, "cmudict500.list")
    synthetic_list(big, 500)
    lists = {k: v for k, v in dict(goforward=KWS_FILE, cmudict500=big).items() if k in args.lists.split(",")}
    if not args.skip_reference:
        reference_time(utt, lists, args.reps)
    import torch
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.kws import KeywordSpotter
    if api.device_count() == 0:
        raise SystemExit("kws_time.py measures on a CUDA device; none found")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu)), flush=True)
    frames_batch = args.utts * (len(utt) // 160 + 1)
    for name, path in lists.items():
        s = KeywordSpotter(HD, DIC, kws=path, max_utts=args.utts, max_frames=max(frames_batch, len(stream) // 160 + 1))
        H = len(s.pl_ssid) + int(s.kp_off[-1])
        for shape, utts in (("batch", [utt] * args.utts), ("stream", [stream])):
            if shape not in args.shapes.split(","):
                continue
            wall, dev, kws_ms, res = [], [], [], None
            for r in range(args.reps + 1):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                res = s.spot_raw_batch(utts)
                e1.record()
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                # the search alone, on the scores spot_raw_batch left on the device
                off = np.cumsum([0] + [o["n_frames"] for o in res]).astype(np.int32)
                k0, k1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                k0.record()
                s.ctx.kws(s.batch.senscr_device_ptr(), off, s.pl_ssid, s.pl_tmat, s.kp_off, s.kp_thresh, s.kp_ssid,
                          s.kp_tmat, s.beam, s.plp)
                k1.record()
                torch.cuda.synchronize()
                if r:
                    wall.append((t1 - t0) * 1e3); dev.append(e0.elapsed_time(e1)); kws_ms.append(k0.elapsed_time(k1))
            n_frames = sum(o["n_frames"] for o in res)
            print(json.dumps(dict(list=name, keyphrases=len(s.keyphrases), hmms=H, shape=shape, utts=len(utts),
                                  frames=n_frames, audio_s=n_frames / 100.0, detections=sum(len(o["detections"]) for o in res),
                                  kws_device_ms_median=float(np.median(kws_ms)), spot_device_ms_median=float(np.median(dev)),
                                  spot_wall_ms_median=float(np.median(wall)), spot_wall_ms_min=float(min(wall)))), flush=True)
        s.close()


def reference_time(utt, lists, reps):
    """The reference's kws search on one host core: one utterance, front end and all-senone scoring included, and
    ps_init (model and dictionary loading) too."""
    from oracle import refdrv
    if not refdrv.available():
        print(json.dumps(dict(reference="not available (oracle/_ref/libpsref.so not built)")), flush=True)
        return
    for name, path in lists.items():
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            refdrv.kws(HD, DIC, utt, keyfile=path)
            ts.append((time.perf_counter() - t0) * 1e3)
        print(json.dumps(dict(reference=name, utts=1, audio_s=len(utt) / 16000.0, host_cores=1,
                              wall_ms_median_with_init=float(np.median(ts)))), flush=True)


if __name__ == "__main__":
    main()
