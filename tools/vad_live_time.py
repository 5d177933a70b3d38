"""Times live endpointing (psb_vad_feed_device): N slots each fed the next `chunk` ms of its own long stream per call,
with CUDA events around the call's kernels and the host call end to end, next to one whole-stream call
(psb_vad_process_device) over the same audio.  Streams are the reference's test recordings (tests/golden/vad_audio.npz)
with random silence between them, 16 kHz.  Prints one JSON line per measurement.

    python tools/vad_live_time.py [--slots 1000] [--chunk-ms 100] [--seconds 20] [--frame 0.01] [--calls 100]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=1000)
    ap.add_argument("--chunk-ms", type=int, default=100)
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--frame", type=float, default=0.01)
    ap.add_argument("--calls", type=int, default=100)
    args = ap.parse_args()
    import torch
    import vad_cases as V
    from pocketsphinx_b200 import api
    from pocketsphinx_b200._lib import check, lib
    from vad_time import device_time, make_stream

    a = V.audio()
    rng = np.random.default_rng(0)
    n, step = args.slots, args.chunk_ms * 16
    base = make_stream(args.seconds + 10, rng, a)
    # every slot its own stretch of the same long recording
    streams = [np.roll(base, int(rng.integers(len(base))))[:int(args.seconds * 16000)] for _ in range(n)]
    le = api.LiveEndpointer(n, 0.3, 0.9, 0, 16000, args.frame)
    d_pcm = torch.from_numpy(np.stack(streams)).cuda()          # [slot][samples]
    fs = le.frame_size
    cap = n * ((step + fs - 1) // fs)
    d_flags = torch.zeros(max(cap, 1), dtype=torch.int8, device="cuda")
    d_seg_n = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_segs = torch.zeros((cap + n, 2), dtype=torch.int64, device="cuda")
    d_times = torch.zeros((cap + n, 2), dtype=torch.float64, device="cuda")
    d_status = torch.zeros((n, 40), dtype=torch.uint8, device="cuda")
    slots = np.arange(n, dtype=np.int32)
    samp_off = np.arange(n + 1, dtype=np.int64) * step
    frame_off = np.zeros(n + 1, np.int32)
    ms = C.c_float()
    calls = min(args.calls, int(args.seconds * 16000) // step)
    out = []
    for c in range(calls):
        chunk = d_pcm[:, c * step:(c + 1) * step].contiguous()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        check(lib().psb_vad_feed_device(le.h, slots.ctypes.data_as(C.c_void_p), n, C.c_void_p(chunk.data_ptr()),
                                        samp_off.ctypes.data_as(C.c_void_p), None, C.c_void_p(d_flags.data_ptr()),
                                        frame_off.ctypes.data_as(C.c_void_p), C.c_void_p(d_seg_n.data_ptr()),
                                        C.c_void_p(d_segs.data_ptr()), C.c_void_p(d_times.data_ptr()),
                                        C.c_void_p(d_status.data_ptr()), C.byref(ms)), "psb_vad_feed_device")
        wall = (time.perf_counter() - t0) * 1e3
        if c >= 2:
            out.append((ms.value, wall))
    k = np.array(out)
    audio_s = calls * step / 16000
    print(json.dumps(dict(measure="live", slots=n, chunk_ms=args.chunk_ms, frame=args.frame, calls=calls,
                          device_ms_median=float(np.median(k[:, 0])), device_ms_min=float(k[:, 0].min()),
                          wall_ms_median=float(np.median(k[:, 1])), wall_ms_max=float(k[:, 1].max()),
                          audio_s_per_slot=audio_s)))
    whole = device_time(le, [s[:calls * step] for s in streams])
    whole.update(measure="whole_stream", slots=n, frame=args.frame, audio_s_per_slot=audio_s)
    print(json.dumps(whole))
    le.close()


if __name__ == "__main__":
    main()
