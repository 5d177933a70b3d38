"""Times device VAD + endpointing (psb_vad_process_device: CUDA events around its kernels, and the host call end
to end; both arms produce flags and segments) against the compiled reference on one host core, for 1000 x 10 s
streams and one 60-minute stream at 10 and 30 ms frames, with the repair count and passes.  The reference has two
arms: `reference_vad_ms` is the ps_vad_classify loop alone, `reference_endpointer_ms` is ps_endpointer_process on
every frame + ps_endpointer_end_stream (which classifies too), the same work as the device arm.  Then
Decoder.decode_stream_batch against decoding the same long stream as one utterance (median of --decode-reps runs
each, after a warm-up decode).  Streams are the reference's test recordings (tests/golden/vad_audio.npz) with random
silence between them.  Prints one JSON line per measurement; --out also writes them all.

    python tools/vad_time.py [--decode-minutes 60] [--decode-reps 2] [--skip-vad] [--out path.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def make_stream(seconds, rng, a):
    parts, n = [], int(seconds * 16000)
    while sum(len(p) for p in parts) < n:
        parts.append(np.zeros(int(rng.integers(0, 2 * 16000)), np.int16))
        parts.append(a[["goforward", "numbers", "libri_0870", "libri_0880"][int(rng.integers(4))]])
    return np.concatenate(parts)[:n]


def device_time(ep, streams, reps=10):
    import torch
    from pocketsphinx_b200._lib import check, lib
    pcm = torch.from_numpy(np.concatenate(streams)).cuda()
    samp_off = np.zeros(len(streams) + 1, np.int64)
    samp_off[1:] = np.cumsum([len(s) for s in streams])
    total = int(sum(len(s) // ep.frame_size for s in streams))
    flags = torch.zeros(total, dtype=torch.int8, device="cuda")
    seg_n = torch.zeros(len(streams), dtype=torch.int32, device="cuda")
    segs = torch.zeros((total, 2), dtype=torch.int64, device="cuda")
    times = torch.zeros((total, 2), dtype=torch.float64, device="cuda")
    frame_off = np.zeros(len(streams) + 1, np.int32)
    ms, out = C.c_float(), []
    for r in range(reps + 2):
        t0 = time.perf_counter()
        check(lib().psb_vad_process_device(ep.h, C.c_void_p(pcm.data_ptr()), samp_off.ctypes.data_as(C.c_void_p), len(streams),
                                           C.c_void_p(flags.data_ptr()), frame_off.ctypes.data_as(C.c_void_p),
                                           C.c_void_p(seg_n.data_ptr()), C.c_void_p(segs.data_ptr()), C.c_void_p(times.data_ptr()),
                                           C.byref(ms)), "psb_vad_process_device")
        if r >= 2:
            out.append((ms.value, (time.perf_counter() - t0) * 1e3))
    k = np.array(out)
    return dict(kernel_ms_median=float(np.median(k[:, 0])), kernel_ms_min=float(k[:, 0].min()),
                call_ms_median=float(np.median(k[:, 1])), repairs=ep.last_repairs, repair_passes=ep.last_passes, frames=total,
                segments=int(seg_n.sum().item()))


def ref_time(streams, fl):
    """(ps_vad_classify loop, ps_endpointer_process + end_stream loop) in ms on one host core, median of 3."""
    import vad_cases as V
    out = []
    for f in (lambda s: V.ref_flags(0, 16000, fl, s), lambda s: V.ref_segments(s, 0, 16000, fl)):
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            for s in streams:
                f(s)
            ts.append((time.perf_counter() - t0) * 1e3)
        out.append(float(np.median(ts)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--decode-minutes", type=float, default=60.0)
    ap.add_argument("--decode-reps", type=int, default=2)
    ap.add_argument("--skip-vad", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import vad_cases as V
    from pocketsphinx_b200 import api
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    a = V.audio()
    rng = np.random.default_rng(0)
    batch = [make_stream(10, rng, a) for _ in range(1000)]
    long = make_stream(3600, rng, a)
    res = dict(gpu=gpu, rows=[])
    for fl in (() if args.skip_vad else (0.01, 0.03)):
        for name, streams in (("1000 x 10 s", batch), ("1 x 60 min", [long])):
            for warmup in (None, 0):
                ep = api.Endpointer(0.3, 0.9, 0, 16000, fl, warmup=warmup)
                row = dict(shape=name, frame_length=fl, warmup=ep.warmup, **device_time(ep, streams, reps=10 if warmup is None else 2))
                ep.close()
                if warmup is None:
                    row["reference_vad_ms"], row["reference_endpointer_ms"] = ref_time(streams, fl)
                print(json.dumps(row), flush=True)
                res["rows"].append(row)
    if args.decode_minutes > 0:
        from pocketsphinx_b200.decoder import Decoder
        ref = os.path.join(ROOT, "oracle", "_ref")
        hd, dic, lm = os.path.join(ref, "model", "en-us"), os.path.join(ref, "data", "turtle.dic"), os.path.join(ref, "data", "turtle.lm.bin")
        s = long[:int(args.decode_minutes * 60 * 16000)]
        dec = Decoder(hd, dic, lm, max_utts=4096, max_frames=len(s) // 160 + 1000)
        dec.decode_stream_batch([s[:16000 * 30]])                  # warm-up
        t_seg, t_one = [], []
        for _ in range(args.decode_reps):
            t0 = time.perf_counter()
            out = dec.decode_stream_batch([s])
            t_seg.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            one = dec.decode_raw_batch([s])
            t_one.append(time.perf_counter() - t0)
        res["decode"] = dict(minutes=args.decode_minutes, reps=args.decode_reps, decode_stream_batch_s=t_seg,
                             segments=len(out[0]), one_utterance_s=t_one, one_utterance_frames=one[0]["n_frames"])
        print(json.dumps(res["decode"]), flush=True)
        dec.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
