"""Device time of the search-scale Viterbi sweep (hmmset_sweep_kernel, plain instantiation) against the candidates it was
chosen from, in one process on one card.

Inputs are the headline's (bench.py): the BASELINE-shape synthetic PTM, channel_template's 6 081 entered instances per
utterance, 998 frames per utterance, and int16 senone scores written by the library's own GMM stage from seeded
features -- 200 utterances by default, a 2 GB score matrix, far beyond the L2.  The candidates are CTA shapes,
frames per block barrier and steps that exist only in this tool's build of psb_hmm.cu (-DPSB_SWEEP_CANDIDATES, linked against the
library's other objects into a temporary directory or --build-dir); `library` is the kernel the library ships.
`library_lane_sorted` is the library's kernel on the same instances uploaded with every CTA slice sorted by its state-0
senone: what a per-segment lane order would give the score gathers, measured without building one.

Rounds alternate over the variants; CUDA events around the launch.  One JSON line: per variant median / min / max ms
and whether best[t][u] and the downloaded state equal the library kernel's byte for byte, with the card's name and
power limit.  Needs a CUDA device and a built tree (csrc/build/*.o)."""
import argparse
import ctypes as C
import glob
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CSRC = os.path.join(ROOT, "pocketsphinx_b200", "csrc")

# candidate numbers of psb_hmmset_sweep_candidate_device (psb_hmm.cu): threads x instances per thread, frames per barrier;
# no_fast: without the warp-uniform path for frames in which every instance evaluates its exit state; live_test: also with
# padding slots kept out of the frame's maximum by a compare per slot and frame instead of by their transitions
CANDIDATES = [("library", 0), ("256x4_fr2", 1), ("512x4_fr1", 2), ("512x4_fr4_no_fast", 3), ("512x4_fr8", 4),
              ("256x4_fr2_no_fast_live_test", 5), ("512x4_fr2_no_fast_live_test", 6), ("512x4_fr2", 7), ("256x4_fr4", 8)]
SLICE = 512 * 4                                 # instances per CTA of the library's kernel


def build_candidates(build_dir):
    """psb_hmm.cu with the candidate instantiations + the library's other objects -> build_dir/libpsb200_sweep.so"""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    arch = ["-gencode", "arch=compute_90a,code=sm_90a"]
    objs = [o for o in sorted(glob.glob(os.path.join(CSRC, "build", "*.o"))) if os.path.basename(o) != "psb_hmm.o"]
    if not objs:
        raise SystemExit("sweep_time: %s/build/*.o missing: build the library first" % CSRC)
    obj, out = os.path.join(build_dir, "psb_hmm_candidates.o"), os.path.join(build_dir, "libpsb200_sweep.so")
    src = os.path.join(CSRC, "psb_hmm.cu")
    if not (os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(f) for f in glob.glob(os.path.join(CSRC, "psb_hmm.cu*")))):
        subprocess.check_call([nvcc] + arch + ["-O3", "-std=c++17", "-lineinfo", "-fmad=false", "-Xcompiler", "-fPIC",
                                               "-DPSB_SWEEP_CANDIDATES", "-c", src, "-o", obj])
        subprocess.check_call([nvcc] + arch + ["-shared", "-o", out, obj] + objs + ["-lcudart"])
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--utts", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--build-dir", default=None, help="where the candidate library is built and kept (default: a temporary directory)")
    ap.add_argument("--build-only", action="store_true", help="compile the candidate library and stop (no device needed)")
    args = ap.parse_args()

    tmp = None
    if args.build_dir is None:
        tmp = tempfile.TemporaryDirectory(prefix="psb_sweep_time_")
        args.build_dir = tmp.name
    os.makedirs(args.build_dir, exist_ok=True)
    lib_path = build_candidates(args.build_dir)
    if args.build_only:
        print(lib_path)
        return

    import torch
    from pocketsphinx_b200 import _lib
    _lib.LIB_PATH = lib_path                     # every api object below runs this build
    import bench
    from pocketsphinx_b200 import api
    from pocketsphinx_b200.model import synth_feats
    if api.device_count() <= 0:
        raise SystemExit("sweep_time: no CUDA device")
    cand = api.lib().psb_hmmset_sweep_candidate_device
    cand.restype = C.c_int
    cand.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_float)]

    U, T = args.utts, bench.frames_for(10)
    pm, desc, _raw = bench.load_model("baseline")
    model = api.Model(pm, device=0)
    total = U * T
    off = api.Batch.offsets([T] * U)
    d_feats = torch.from_numpy(synth_feats(pm, U, T, seed=1234).reshape(total, pm.sumlen)).cuda()
    batch = api.Batch(model, U, total)
    batch.score_device(d_feats.data_ptr(), off)  # the real GMM stage writes the score matrix
    batch.sync()
    scr = batch.senscr_device_ptr()
    ctx = api.HmmContext(pm.tp, pm.sseq, pm.n_sen, device=0)
    tmpl = bench.channel_template(pm, api.HMM_DTYPE)
    n = len(tmpl)
    # the same instances with every CTA slice ordered by its state-0 senone
    order = np.concatenate([a + np.argsort(tmpl["senid"][a:a + SLICE, 0], kind="stable") for a in range(0, n, SLICE)])
    seg_off = np.arange(U + 1, dtype=np.int64) * n
    d_row0 = torch.from_numpy(np.asarray(off[:U], np.int64)).cuda()
    d_best = torch.empty((T, U), dtype=torch.int32, device="cuda")

    sets = {}
    for name, t in (("upload", tmpl), ("sorted", np.ascontiguousarray(tmpl[order]))):
        hs = api.HmmSet(ctx, U * n + U * 512, U)
        hs.upload(np.tile(t, U), seg_off)
        hs.snapshot()
        sets[name] = hs

    def run(hs, c):
        hs.restore()
        ms = C.c_float()
        api.check(cand(hs.h, C.c_void_p(scr), total, C.c_void_p(d_row0.data_ptr()), None, T, C.c_void_p(d_best.data_ptr()),
                       c, C.byref(ms)), "psb_hmmset_sweep_candidate_device")
        return ms.value

    variants = [(name, sets["upload"], c) for name, c in CANDIDATES] + [("library_lane_sorted", sets["sorted"], 0)]
    times = {name: [] for name, _, _ in variants}
    same = {}
    ref_best = ref_state = None
    for rnd in range(args.rounds + 1):           # round 0 warms every variant up and compares the results
        for name, hs, c in variants:
            ms = run(hs, c)
            if rnd > 0:
                times[name].append(ms)
                continue
            best, state = d_best.cpu().numpy(), hs.download()
            if name == "library_lane_sorted":    # back to upload order
                inv = np.empty_like(state)
                inv.reshape(U, n)[:, order] = state.reshape(U, n)
                state = inv
            if ref_best is None:
                ref_best, ref_state = best, state
            same[name] = {"best_equal": bool(np.array_equal(best, ref_best)),
                          "state_equal": bool(state.tobytes() == ref_state.tobytes())}
    out = {"tool": "sweep_time", "model": desc, "utts": U, "frames": T, "instances_per_utt": n, "n_sen": int(pm.n_sen),
           "score_matrix_gb": total * pm.n_sen * 2 / 1e9, "rounds": args.rounds, "gpu": bench.gpu_info(0), "variants": {}}
    for name, _, _ in variants:
        v = sorted(times[name])
        out["variants"][name] = dict(median_ms=float(np.median(v)), min_ms=v[0], max_ms=v[-1], **same[name])
    print(json.dumps(out))
    for hs in sets.values():
        hs.close()
    ctx.close(); batch.close(); model.close()
    if tmp is not None:
        tmp.cleanup()


if __name__ == "__main__":
    main()
