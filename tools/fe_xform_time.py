"""Device time of the front end (psb_fe_process_device: every kernel from PCM to features) on 1000 utterances of
10 s of seeded noise, en-us front end with batch CMN: the plain path, then with -varnorm yes, each -agc mode (one
session per utterance, so emax runs one warp per utterance) and a 29 x 39 LDA transform.  Runs the configurations
in turn, --reps times over (alternating, so clock drift spreads over all of them), after one warm-up run each.
Prints the GPU's name and power limit, then one JSON line per configuration: median / min / max ms.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.fe_tables import make_fe_desc, make_fe_opts
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--secs", type=int, default=10)
    ap.add_argument("--utts", type=int, default=1000)
    a = ap.parse_args()
    q, _ = np.linalg.qr(np.random.default_rng(1).standard_normal((39, 39)))
    lda = q[:29].astype(np.float32)
    configs = [("plain (batch CMN)", None), ("varnorm", dict(varnorm=True)), ("agc max", dict(agc="max")),
               ("agc emax", dict(agc="emax")), ("agc noise", dict(agc="noise")), ("lda 29 x 39", dict(lda=lda))]
    n, n_utt = 16000 * a.secs, a.utts
    pcm = torch.from_numpy((np.random.default_rng(0).standard_normal(n_utt * n) * 2000).astype(np.int16)).cuda()
    off = np.arange(n_utt + 1, dtype=np.int64) * n
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), power_limit=power)))
    fes = [api.FrontEnd(make_fe_desc(), 0, None if o is None else make_fe_opts(cmn="batch", **o)) for _, o in configs]
    total = sum(fes[0].n_frames(n) for _ in range(n_utt))
    out = torch.empty(total * 39, dtype=torch.float32, device="cuda")
    ms = [[] for _ in configs]
    for r in range(a.reps + 1):
        for i, fe in enumerate(fes):
            _, t = fe.process_device(pcm.data_ptr(), off, out.data_ptr())
            if r:
                ms[i].append(t)
    for (name, _), fe, m in zip(configs, fes, ms):
        print(json.dumps(dict(config=name, utts=n_utt, frames=total, feat_dim=fe.feat_dim, ms_median=float(np.median(m)),
                              ms_min=min(m), ms_max=max(m))))
        fe.close()


if __name__ == "__main__":
    main()
