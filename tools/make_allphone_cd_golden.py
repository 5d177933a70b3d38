"""Writes tests/golden/en_us_allphone_cd.npz from the compiled reference (oracle/_ref/libpsref.so) and its
source tree's en-us model: the reference's allphone_search over the context-dependent PHMM net
(-allphone_ci no) on goforward.raw, without a phone LM (default beams) and with the shipped phone LM at
test/unit/test_allphone.c's settings (beam 1e-20, pbeam 1e-10, lw 2.0); the net it built (exported as
successor lists by refdrv.allphone); and the mdef phone table (ssid, tmat, wpos / base / lc / rc, filler
flags, names) that pocketsphinx_b200/allphone_net.py builds the net from where there is no model.

    python tools/make_allphone_cd_golden.py          (PS_REFERENCE: the reference's source tree)"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refdrv  # noqa: E402
from oracle.make_golden import OUT, REF, save_golden  # noqa: E402
from pocketsphinx_b200 import s3io  # noqa: E402


def main():
    pcm = np.fromfile(os.path.join(REF, "test/data/goforward.raw"), np.int16)
    hmm = os.path.join(REF, "model/en-us/en-us")
    md = s3io.read_mdef(os.path.join(hmm, "mdef"))
    out = dict(ph_ssid=md["phone_ssid"], ph_tmat=md["phone_tmat"].astype(np.int16), ph_ctx=md["phone_ctx"].astype(np.int8),
               ph_filler=md["phone_filler"], ciname=np.array(md["ciname"]), sil=np.int32(md["sil"]))
    a = refdrv.allphone(hmm, pcm, allphone_ci="no")
    for k in ("ci", "ssid", "tmatid", "succ_off", "succ", "segs"):
        out[k] = a[k]
    for k in ("start", "beam", "pbeam", "inspen", "n_history"):
        out[k] = np.int32(a[k])
    print("allphone CD", len(a["ci"]), "nodes", len(a["succ"]), "links", a["n_history"], "history entries", len(a["segs"]), "segments")
    b = refdrv.allphone(hmm, pcm, allphone_ci="no", allphone=os.path.join(REF, "model/en-us/en-us-phone.lm.bin"),
                        beam="1e-20", pbeam="1e-10", lw="2.0")
    assert np.array_equal(b["ssid"], a["ssid"]) and np.array_equal(b["succ"], a["succ"])
    out["lm_bg"], out["lm_tg"], out["lm_segs"] = b["bg"], b["tg"], b["segs"]
    for k in ("beam", "pbeam", "n_history"):
        out["lm_" + k] = np.int32(b[k])
    print("allphone CD + phone LM", b["n_history"], "history entries:", " ".join(md["ciname"][c] for c in b["segs"][:, 0]))
    save_golden(os.path.join(OUT, "en_us_allphone_cd.npz"), **out)


if __name__ == "__main__":
    main()
