"""CPU design experiment (oracle/ps_oracle.c: pso_filter_experiment): is a codeword filter that
is looser than the scan's own running threshold safe for the PTM top-N list?  See DESIGN.md 9."""
import ctypes as C
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle  # noqa: E402
from pocketsphinx_b200.model import PackedModel, load_npz, quantize_for_ties, synth_feats, synth_ptm  # noqa: E402

L = oracle.lib()
L.pso_filter_experiment.restype = C.c_int32


def run(pm, feats, lag):
    om = oracle.OracleModel(pm)
    st = np.zeros(5, np.int64)
    f = np.ascontiguousarray(feats, np.float32).reshape(len(feats), -1)
    L.pso_filter_experiment(C.byref(om.c), C.c_void_p(f.ctypes.data), C.c_int32(f.shape[0]), C.c_int32(lag),
                            C.c_void_p(st.ctypes.data))
    return st


t0 = time.time()
pm = synth_ptm(seed=0)
feats = synth_feats(pm, 4, 300, seed=3)
for lag in (1, 2, 5, 20):
    tot = sum(run(pm, feats[u], lag) for u in range(4))
    print("synthetic 256 Gauss, lag", lag, "lists", tot[0], "differ", tot[1], "scanned %.3f of all" % (tot[3] / tot[4]), flush=True)
pmq, gen = quantize_for_ties(synth_ptm(seed=2, n_density=64, n_sen=400), seed=6)
fq = gen(6, 200, s=9)
for lag in (1, 3, 10):
    tot = sum(run(pmq, fq[u], lag) for u in range(6))
    print("tie stress, lag", lag, "lists", tot[0], "differ", tot[1], "scanned %.3f" % (tot[3] / tot[4]), flush=True)
g = load_npz(os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "en_us_goforward.npz"))
en = PackedModel.load(os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "en_us_ptm_model.npz"))
for lag in (1, 5, 30):
    st = run(en, g["feats"], lag)
    print("en-us goforward, lag", lag, "lists", st[0], "differ", st[1], "scanned %.3f" % (st[3] / st[4]), flush=True)
print("%.1f s" % (time.time() - t0))
