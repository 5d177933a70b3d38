"""Device time of the whole front end (psb_fe_process_device: every kernel from PCM to features, CUDA events) on
the en-us options (-remove_noise yes, batch CMN) with the noise tracker carried across a session's utterances
(psb_fe_set_stream_starts, fe_noise_kernel), 10 s utterances of seeded noise:
  1000 utterances as 1000 fresh streams, the default path (no stream starts named) and all-ones flags;
  10 sessions x 100 utterances and 1 session x 1000, carried (one stream start per session);
  1 session x 360 utterances (60 minutes), carried;
and, for the serial one-session walks, live CMN over the same 1 x 1000 and 1 x 360 sessions without the carried
tracker.  Prints the GPU, its power limit and SM clocks, then one JSON line per configuration: median / min / max
ms over --reps runs after one warm-up run, the configurations alternating within each round.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=60)
        return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {}


def main():
    import torch
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.fe_tables import make_fe_desc, make_fe_opts
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--secs", type=int, default=10)
    a = ap.parse_args()
    n = 16000 * a.secs
    long_n = 3600 // a.secs
    # name, opts (None: psb_fe_create), utterances, sessions, stream starts: None (not named), "all", "session"
    configs = [("1000 fresh streams (default path)", None, 1000, 1000, None),
               ("1000 fresh streams (all-ones flags)", None, 1000, 1000, "all"),
               ("10 sessions x 100, carried", None, 1000, 10, "session"),
               ("1 session x 1000, carried", None, 1000, 1, "session"),
               ("1 session x %d, carried" % long_n, None, long_n, 1, "session"),
               ("1 session x 1000, live CMN", dict(cmn="live"), 1000, 1, None),
               ("1 session x %d, live CMN" % long_n, dict(cmn="live"), long_n, 1, None)]
    rng = np.random.default_rng(0)
    pcm_all = torch.from_numpy((rng.standard_normal(1000 * n) * 2000).astype(np.int16)).cuda()
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), **gpu_info())))
    d = make_fe_desc()
    runs = []
    for name, opts, n_utt, n_sess, starts in configs:
        fe = api.FrontEnd(d, 0, None if opts is None else make_fe_opts(**opts))
        off = np.arange(n_utt + 1, dtype=np.int64) * n
        sess = np.linspace(0, n_utt, n_sess + 1).astype(np.int32)
        flags = None
        if starts == "all":
            flags = np.ones(n_utt, bool)
        elif starts == "session":
            flags = np.zeros(n_utt, bool)
            flags[sess[:-1]] = True
        total = sum(fe.n_frames(n) for _ in range(n_utt))
        out = torch.empty(total * fe.feat_dim, dtype=torch.float32, device="cuda")
        runs.append(dict(name=name, fe=fe, off=off, sess=sess, flags=flags, opts=opts, out=out, total=total, n_utt=n_utt,
                         n_sess=n_sess, ms=[]))

    def once(r):
        if r["opts"] is not None or r["flags"] is not None:
            r["fe"].set_sessions(r["sess"])
        if r["flags"] is not None:
            r["fe"].set_stream_starts(r["flags"])
        return r["fe"].process_device(pcm_all.data_ptr(), r["off"], r["out"].data_ptr())[1]

    for rep in range(a.reps + 1):
        for r in runs:
            t = once(r)
            if rep:
                r["ms"].append(t)
    for r in runs:
        ms = r["ms"]
        print(json.dumps(dict(config=r["name"], utts=r["n_utt"], sessions=r["n_sess"], frames=r["total"],
                              ms_median=round(float(np.median(ms)), 3), ms_min=round(min(ms), 3), ms_max=round(max(ms), 3))))
        r["fe"].close()


if __name__ == "__main__":
    main()
