"""Device time of the front end (psb_fe_process_device: every kernel from PCM to features) with the options of
psb_fe_create_ex, 10 s utterances of seeded noise: 1000 utterances of tidigits s2_4x + dither (one session
each), 1000 of en-us with live CMN in 1, 10 and 1000 sessions, en-us with batch CMN as the baseline, and one
60-minute session (360 utterances) with live CMN and with dither.  Prints one JSON line per configuration:
median / min / max ms over --reps runs after one warm-up run.  Needs a GPU."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.fe_tables import make_fe_desc, make_fe_opts
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--secs", type=int, default=10)
    a = ap.parse_args()
    tid = dict(wlen=0.025, nfilt=20, lowerf=1, upperf=4000, round_filters=False, remove_dc=True, remove_noise=False,
               lifter=0, transform="dct")
    n = 16000 * a.secs
    rng = np.random.default_rng(0)
    configs = [("en-us batch (baseline)", {}, None, 1000, 1000),
               ("tidigits s2_4x + dither", tid, dict(feat="s2_4x", cmn="batch", dither=True), 1000, 1000),
               ("en-us live, 1000 sessions", {}, dict(cmn="live"), 1000, 1000),
               ("en-us live, 10 sessions", {}, dict(cmn="live"), 1000, 10),
               ("en-us live, 1 session", {}, dict(cmn="live"), 1000, 1),
               ("60-minute session, live CMN", {}, dict(cmn="live"), 3600 // a.secs, 1),
               ("60-minute session, dither", tid, dict(feat="s2_4x", cmn="batch", dither=True), 3600 // a.secs, 1)]
    pcm_all = torch.from_numpy((rng.standard_normal(1000 * n) * 2000).astype(np.int16)).cuda()
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0))))
    for name, desc, opts, n_utt, n_sess in configs:
        fe = api.FrontEnd(make_fe_desc(**desc), 0, None if opts is None else make_fe_opts(**opts))
        off = np.arange(n_utt + 1, dtype=np.int64) * n
        sess = np.linspace(0, n_utt, n_sess + 1).astype(np.int32)
        total = sum(fe.n_frames(n) for _ in range(n_utt))
        out = torch.empty(total * fe.feat_dim, dtype=torch.float32, device="cuda")
        ms = []
        for r in range(a.reps + 1):
            if opts is not None:
                fe.set_sessions(sess)
            _, t = fe.process_device(pcm_all.data_ptr(), off, out.data_ptr())
            if r:
                ms.append(t)
        print(json.dumps(dict(config=name, utts=n_utt, sessions=n_sess, frames=total, ms_median=float(np.median(ms)),
                              ms_min=min(ms), ms_max=max(ms))))
        fe.close()


if __name__ == "__main__":
    main()
