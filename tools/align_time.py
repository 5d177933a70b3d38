"""Times forced alignment on the GPU: the Aligner on 1000 x 10 s of goforward with its transcript, the Decoder with and
without state_align on the same audio, and one 5-minute utterance decoded with state_align.  Reports align_kernel's
time (CUDA events), wall time, and the token arena's bytes next to the dense table's (2 x frames x phones x states x
4 B), with the card's name and power limit read in the same run.  Needs a GPU and the reference's model files under
oracle/_ref/ (built by build()).  Prints one JSON object; --out also writes it to a file.

    python tools/align_time.py [--utts 1000] [--decode-utts 64] [--out results/align_time.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.path.join(ROOT, "oracle", "_ref")
HD, DIC, LM = (os.path.join(REF, "model", "en-us"), os.path.join(REF, "model", "cmudict-en-us.dict"),
               os.path.join(REF, "model", "en-us.lm.bin"))
GO = os.path.join(REF, "data", "goforward.raw")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def dense_bytes(frames, phones):
    return 2 * 4 * 3 * int(sum(int(t) * int(h) for t, h in zip(frames, phones)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=1000)
    ap.add_argument("--chunk", type=int, default=125)
    ap.add_argument("--decode-utts", type=int, default=64)
    ap.add_argument("--long-seconds", type=int, default=300)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.align import Aligner
    from pocketsphinx_b200.decoder import Decoder
    if not torch.cuda.is_available():
        raise SystemExit("align_time.py measures on the GPU and found none")
    go = np.fromfile(GO, np.int16)
    rep = int(np.ceil(160000 / len(go)))
    ten = np.tile(go, rep)[:160000]                                     # 10 s of goforward
    text = " ".join(["go forward ten meters"] * rep)
    res = dict(card=card())

    # 1. Aligner, 1000 x 10 s with the transcript, in batches of --chunk
    al = Aligner(HD, DIC, max_utts=a.chunk, max_frames=a.chunk * 1100)
    al.align_raw_batch([ten] * 2, [text] * 2)                          # warm-up
    kern, tok, frames_all, phones_all, ok = 0.0, 0, [], [], 0
    t0 = time.perf_counter()
    for s in range(0, a.utts, a.chunk):
        n = min(a.chunk, a.utts - s)
        out = al.align_raw_batch([ten] * n, [text] * n)
        torch.cuda.synchronize()
        kern += float(api.lib().psb_align_last_kernel_ms(al.ctx.h))
        tok = max(tok, al.last_token_bytes)
        ok += sum(x is not None for x in out)
        frames_all += [out[0].words[-1].start + out[0].words[-1].duration] * n if out[0] else []
        phones_all += [len(out[0].phones)] * n if out[0] else []
    wall = time.perf_counter() - t0
    res["aligner"] = dict(utts=a.utts, seconds_each=10, aligned=ok, wall_s=wall, align_kernel_ms=kern,
                          arena_bytes_per_batch=tok, dense_bytes_per_batch=dense_bytes(frames_all[:a.chunk],
                                                                                        phones_all[:a.chunk]))
    al.close()

    # 2. Decoder without and with state_align on the same audio
    batch = [ten] * a.decode_utts
    for name, kv in (("decoder", {}), ("decoder_state_align", dict(state_align="yes"))):
        dec = Decoder(HD, DIC, LM, max_utts=a.decode_utts, max_frames=a.decode_utts * 1100, **kv)
        dec.decode_raw_batch(batch[:2])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = dec.decode_raw_batch(batch)
        torch.cuda.synchronize()
        r = dict(utts=a.decode_utts, wall_s=time.perf_counter() - t0)
        if kv:
            fr = [d["n_frames"] for d in out]
            ph = [len(d["alignment"].phones) if d["alignment"] else 0 for d in out]
            r.update(align_kernel_ms=float(api.lib().psb_align_last_kernel_ms(dec.ctx.h)),
                     arena_bytes=dec.last_align_token_bytes, dense_bytes=dense_bytes(fr, ph),
                     aligned=sum(d["alignment"] is not None for d in out))
        res[name] = r
        dec.close()

    # 3. one 5-minute utterance decoded whole with state_align
    n = a.long_seconds * 16000
    long = np.tile(go, int(np.ceil(n / len(go))))[:n]
    dec = Decoder(HD, DIC, LM, max_utts=2, max_frames=a.long_seconds * 100 + 1000, state_align="yes")
    t0 = time.perf_counter()
    out = dec.decode_raw_batch([long])
    torch.cuda.synchronize()
    d = out[0]
    ph = len(d["alignment"].phones) if d["alignment"] else 0
    res["long"] = dict(seconds=a.long_seconds, frames=d["n_frames"], words=len(d["seg"]), phones=ph,
                       aligned=d["alignment"] is not None, error=d["alignment_error"], wall_s=time.perf_counter() - t0,
                       align_kernel_ms=float(api.lib().psb_align_last_kernel_ms(dec.ctx.h)),
                       arena_bytes=dec.last_align_token_bytes, dense_bytes=dense_bytes([d["n_frames"]], [ph]))
    dec.close()
    s = json.dumps(res)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
