"""Device time of the whole front end (psb_fe_process_device: every kernel from PCM to features, CUDA events) with
per-utterance VTLN filter banks (psb_fe_set_filterbanks), on the en-us options (-remove_noise yes, batch CMN),
1000 utterances of 10 s of seeded noise:
  neutral: no banks named, the handle's own bank (the default path);
  one warped bank: every utterance reads one bank, -warp_params 0.9;
  13 factors: -warp_params 0.88 .. 1.12 spread over the batch (utterance u reads factor u mod 13).
The banks are named before every timed call, as a caller does; the events time the kernels only.  Prints the GPU,
its power limit and SM clocks, then one JSON line per configuration: median / min / max ms over --reps runs after
one warm-up run, the configurations alternating within each round.  Needs a GPU."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fe_noise_time import gpu_info  # noqa: E402  (tools/ is this script's directory)


def main():
    import torch
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.fe_tables import make_fe_desc
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--secs", type=int, default=10)
    ap.add_argument("--utts", type=int, default=1000)
    a = ap.parse_args()
    n, n_utt = 16000 * a.secs, a.utts
    rng = np.random.default_rng(0)
    pcm_all = torch.from_numpy((rng.standard_normal(n_utt * n) * 2000).astype(np.int16)).cuda()
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), **gpu_info())))
    fe = api.FrontEnd(make_fe_desc())
    off = np.arange(n_utt + 1, dtype=np.int64) * n
    total = sum(fe.n_frames(n) for _ in range(n_utt))
    out = torch.empty(total * fe.feat_dim, dtype=torch.float32, device="cuda")
    factors = ["%.2f" % (0.88 + 0.02 * i) for i in range(13)]
    configs = [("neutral", None), ("one warped bank (0.9)", ["0.9"] * n_utt),
               ("13 factors 0.88 .. 1.12", [factors[u % 13] for u in range(n_utt)])]
    ms = {name: [] for name, _ in configs}
    for rep in range(a.reps + 1):
        for name, warps in configs:
            if warps is not None:
                fe.set_warps(warps)
            t = fe.process_device(pcm_all.data_ptr(), off, out.data_ptr())[1]
            if rep:
                ms[name].append(t)
    for name, _ in configs:
        m = ms[name]
        print(json.dumps(dict(config=name, utts=n_utt, frames=total, ms_median=round(float(np.median(m)), 3),
                              ms_min=round(min(m), 3), ms_max=round(max(m), 3))))
    fe.close()


if __name__ == "__main__":
    main()
