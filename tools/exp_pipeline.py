"""Scratch experiment (GPU): device-resident and host-buffer step times of the BASELINE shape for
the sub-batch counts listed in the environment (PIPES)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pocketsphinx_b200 import api
from pocketsphinx_b200.model import synth_ptm, synth_feats
import bench
pm = synth_ptm(seed=0)
T = 998; U = int(os.environ.get("UTTS", "1000"))
feats = synth_feats(pm, U, T, seed=1234)
model = api.Model(pm)
total = U * T
off = api.Batch.offsets([T] * U)
fp = torch.from_numpy(feats.reshape(total, pm.sumlen)).pin_memory()
d = fp.cuda()
batch = api.Batch(model, U, total)
ctx = api.HmmContext(pm.tp, pm.sseq, pm.n_sen)
H = pm.n_ciphone
PL = bench.PL
pl = api.PhoneLoop(ctx, pm.phone_ssid[:H], pm.phone_tmat[:H], PL["window"], PL["beam"], PL["pbeam"], PL["pip"], PL["weight"])
best = torch.empty(total, dtype=torch.int32).pin_memory()
pen = torch.empty((total, H), dtype=torch.int32).pin_memory()
def run(n):
    batch.event_record(0)
    for _ in range(n): batch.decode_device(pl, d.data_ptr(), off)
    batch.event_record(1)
    return batch.event_elapsed_ms() / n
def runh(n):
    batch.sync(); t0 = time.perf_counter()
    for _ in range(n): batch.decode_host(pl, fp, off, best=best, pen=pen)
    batch.sync(); return (time.perf_counter() - t0) * 1e3 / n
for _ in range(3): batch.decode_device(pl, d.data_ptr(), off)
batch.sync()
for pipe in [int(x) for x in os.environ.get("PIPES", "1,2,3,4").split(",")]:
    batch.set_pipeline(pipe)
    run(1); runh(1)
    print("pipeline", pipe, "device %.2f %.2f" % (run(4), run(4)), "host %.2f %.2f" % (runh(4), runh(4)), flush=True)
