"""Times live pitch tracking (psb_pitch_feed_device): N slots, each fed the next `chunk` ms of its own 10 s stream per
call, with CUDA events around the call's kernels and the host call end to end, next to one whole-stream call
(psb_pitch_process_device) over the same 10 s per slot.  16 kHz, the program's defaults.  Streams are the reference's
test recordings (goforward, dhd.2934z) repeated from random offsets.  The card's name and power limit are read in the
same run.  Prints one JSON line per measurement.

    python tools/pitch_live_time.py [--slots 1000] [--chunk-ms 100] [--seconds 10] [--reps 5]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=1000)
    ap.add_argument("--chunk-ms", type=int, default=100)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import pitch_cases as P
    from pocketsphinx_b200 import api
    from pocketsphinx_b200._lib import check, lib
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rec = np.concatenate([P.recording("goforward.raw"), P.recording("dhd.2934z.raw")])
    rng = np.random.default_rng(0)
    n, total = args.slots, int(args.seconds * 16000)
    step = args.chunk_ms * 16
    streams = [np.resize(np.roll(rec, int(rng.integers(len(rec)))), total) for _ in range(n)]
    calls = -(-total // step)
    # per call, every slot's next chunk back to back on the device: [call][slot][step]
    pcm = torch.from_numpy(np.stack([np.pad(s, (0, calls * step - total)).reshape(calls, step) for s in streams], 1)
                           .copy()).cuda()
    L = lib()
    tr = api.LivePitchTracker(n)
    slots = np.arange(n, dtype=np.int32)
    cap = n * (-(-step // tr.frame_shift) + 2 * tr.smooth_window)
    d_per = torch.zeros(cap, dtype=torch.int16, device="cuda")
    d_bd = torch.zeros(cap, dtype=torch.int16, device="cuda")
    out_off = np.zeros(n + 1, np.int32)
    status = np.zeros(n, api.PITCH_LIVE_STATUS)
    ms = C.c_float()
    dev, wall, reads = [], [], 0
    for rep in range(args.reps + 1):                            # the first pass allocates the buffers: not timed
        tr.reset(slots)
        for c in range(calls):
            lens = np.full(n, min(step, total - c * step), np.int64)
            samp_off = np.zeros(n + 1, np.int64)
            samp_off[1:] = np.cumsum(lens)
            fin = np.full(n, int(c == calls - 1), np.int8)
            chunk = pcm[c] if lens[0] == step else pcm[c, :, :lens[0]].contiguous()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            check(L.psb_pitch_feed_device(tr.h, slots.ctypes.data, n, chunk.data_ptr(), samp_off.ctypes.data,
                                          fin.ctypes.data, out_off.ctypes.data, d_per.data_ptr(), d_bd.data_ptr(),
                                          status.ctypes.data, C.byref(ms)), "psb_pitch_feed_device")
            if rep >= 1:
                dev.append(ms.value)
                wall.append((time.perf_counter() - t0) * 1e3)
                reads += int(out_off[-1])
    frames = int(status["frames"].sum())
    print(json.dumps(dict(shape="%d slots x %d ms per call" % (n, args.chunk_ms), gpu=gpu, calls=len(dev),
                          frames_per_slot=frames // n, reads_per_pass=reads // args.reps,
                          device_ms_median=float(np.median(dev)), device_ms_min=float(np.min(dev)),
                          wall_ms_median=float(np.median(wall)),
                          device_ms_per_pass=float(np.sum(dev)) / args.reps)), flush=True)
    # one whole-stream call over the same audio
    whole = torch.from_numpy(np.concatenate(streams)).cuda()
    samp_off = np.zeros(n + 1, np.int64)
    samp_off[1:] = np.cumsum([len(s) for s in streams])
    per = torch.zeros(n * tr.n_frames(total), dtype=torch.int16, device="cuda")
    bd = torch.zeros_like(per)
    wout = np.zeros(n + 1, np.int32)
    wd, ww = [], []
    for r in range(args.reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        check(L.psb_pitch_process_device(tr.h, whole.data_ptr(), samp_off.ctypes.data, n, wout.ctypes.data,
                                         per.data_ptr(), bd.data_ptr(), C.byref(ms)), "psb_pitch_process_device")
        if r >= 1:
            wd.append(ms.value)
            ww.append((time.perf_counter() - t0) * 1e3)
    print(json.dumps(dict(shape="%d streams x %g s, one whole-stream call" % (n, args.seconds), gpu=gpu,
                          reads=int(wout[-1]), device_ms_median=float(np.median(wd)), wall_ms_median=float(np.median(ww)))),
          flush=True)
    # the live reads joined equal the whole-stream reads (the last pass fed every slot through to its end)
    assert reads // args.reps == int(wout[-1])
    tr.close()


if __name__ == "__main__":
    main()
