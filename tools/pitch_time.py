"""Times the device pitch tracker (psb_pitch_process_device: CUDA events around its two kernels, and the host call
end to end; PitchTracker.track_batch wall time including the copies and the Python results) against the compiled
reference's yin_* loop on one host core (extract_pitch's loop, tests/emul/pitch_refdrv.c), for 1000 x 10 s streams
and one 60-minute stream at 16 kHz with the program's defaults.  Streams are the reference's test recordings
(goforward, dhd.2934z) repeated from random offsets.  The card's name and power limit are read in the same run.
Prints one JSON line per measurement; --out also writes them all.

    python tools/pitch_time.py [--reps 5] [--ref-streams N] [--out path.json]"""
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


def device_time(tr, streams, reps):
    import torch
    from pocketsphinx_b200._lib import check, lib
    pcm = torch.from_numpy(np.concatenate(streams)).cuda()
    samp_off = np.zeros(len(streams) + 1, np.int64)
    samp_off[1:] = np.cumsum([len(s) for s in streams])
    frames = int(sum(tr.n_frames(len(s)) for s in streams))
    per = torch.zeros(max(frames, 1), dtype=torch.int16, device="cuda")
    bd = torch.zeros(max(frames, 1), dtype=torch.int16, device="cuda")
    out_off = np.zeros(len(streams) + 1, np.int32)
    ms, out = C.c_float(), []
    for r in range(reps + 1):                                    # the first call allocates the rows: not timed
        t0 = time.perf_counter()
        check(lib().psb_pitch_process_device(tr.h, C.c_void_p(pcm.data_ptr()), samp_off.ctypes.data_as(C.c_void_p),
                                             len(streams), out_off.ctypes.data_as(C.c_void_p), C.c_void_p(per.data_ptr()),
                                             C.c_void_p(bd.data_ptr()), C.byref(ms)), "psb_pitch_process_device")
        if r >= 1:
            out.append((ms.value, (time.perf_counter() - t0) * 1e3))
    wall = []
    for r in range(reps):
        t0 = time.perf_counter()
        tr.track_batch(streams)
        wall.append((time.perf_counter() - t0) * 1e3)
    k = np.array(out)
    return dict(frames=frames, reads=int(out_off[-1]), kernel_ms_median=float(np.median(k[:, 0])),
                kernel_ms_min=float(k[:, 0].min()), call_ms_median=float(np.median(k[:, 1])),
                track_batch_ms_median=float(np.median(wall)), frames_per_s=frames / (np.median(k[:, 0]) * 1e-3))


def ref_time(streams):
    """The reference's yin_* loop over every stream on one host core, ms (one run)."""
    import pitch_cases as P
    P.ref_run(streams[0][:16000], 16000)                          # builds the driver
    t0 = time.perf_counter()
    for s in streams:
        P.ref_run(s, 16000)
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-streams", type=int, default=None, help="time the reference on the first N streams only")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import pitch_cases as P
    from pocketsphinx_b200 import api
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rec = np.concatenate([P.recording("goforward.raw"), P.recording("dhd.2934z.raw")])
    rng = np.random.default_rng(0)
    batch = [np.resize(np.roll(rec, int(rng.integers(len(rec)))), 10 * 16000) for _ in range(1000)]
    long = np.resize(rec, 3600 * 16000)
    tr = api.PitchTracker()
    res = dict(gpu=gpu, rows=[])
    for name, streams in (("1000 x 10 s", batch), ("1 x 60 min", [long])):
        row = dict(shape=name, gpu=gpu, **device_time(tr, streams, args.reps))
        rs = streams[:args.ref_streams] if args.ref_streams else streams
        row["reference_streams"] = len(rs)
        row["reference_ms"] = ref_time(rs)
        print(json.dumps(row), flush=True)
        res["rows"].append(row)
    tr.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
