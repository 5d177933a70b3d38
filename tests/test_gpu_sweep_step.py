"""GPU (-m gpu): the fused search-scale sweep (psb_hmmset_sweep_device, and the beam variant on the same inputs) on the
inputs the sweep's pre-decoded, branch-free step has to get bit-exact and that tests/test_gpu_parity.py does not force:
absent arcs (transition byte 255 at (1,3) and (0,2): the stale-t2 path), scores driven onto the WORST_SCORE floor, exact
ties in every history pick, a frame count that is not a multiple of the frames closed per block barrier, segments
spanning several CTAs with a partial last thread and a segment ending on the score matrix's last row.  Each case is
checked against hmm_vit_eval of the oracle and against the per-frame kernel: the whole state and best[t][segment]."""
import numpy as np
import pytest

from conftest import assert_hmm_equal, golden, hmm_view

pytestmark = pytest.mark.gpu

WORST = -0x20000000


@pytest.fixture(scope="module")
def api():
    from pocketsphinx_b200 import api
    assert api.device_count() > 0, "no CUDA device visible"
    return api


# segments: a single instance, an empty one, one of several CTAs with a partial last thread (2 * 1024 + 37), one
# ending on the matrix's last row, one finishing early; T odd
SEG_LEN = [1, 0, 2 * 1024 + 37, 1500, 700]


def make_case(n_emit, case, T, seed):
    g = golden("hmm_vit_eval.npz")
    tp, sseq = g["n%d_tp" % n_emit].copy(), g["n%d_sseq" % n_emit]
    n_sen = len(g["n%d_senscr" % n_emit])
    n_sen -= n_sen & 1                                                  # the fused kernel's shape
    hm = hmm_view(g["n%d_before" % n_emit]).copy()
    hm = hm[(hm["mpx"] == 0) & (hm["senid"][:, :n_emit] < n_sen).all(1)]
    rng = np.random.default_rng(seed)
    n = sum(SEG_LEN)
    hm = np.ascontiguousarray(hm[rng.integers(0, len(hm), n)])
    hm["history"][:, :n_emit] = rng.integers(0, 1 << 30, (n, n_emit))   # every pick shows in the history
    hm["out_history"] = rng.integers(0, 1 << 30, n)
    n_tmat = tp.shape[0]
    hm["tmatid"] = rng.integers(0, n_tmat, n)
    R = 3 * T
    if case == "absent_arcs":
        # 255 at (1,3) for a third of the matrices, at (0,2) for another third, both for some; state 1 at WORST for a
        # fifth of the instances so the exit state is skipped and t2 stays INT_MIN when (0,2) is absent
        q = np.arange(n_tmat) % 4
        tp[q == 1, 1, 3] = 255
        tp[q == 2, 0, 2] = 255
        tp[q == 3, 1, 3] = 255
        tp[q == 3, 0, 2] = 255
        hm["score"][:, :n_emit] = -rng.integers(0, 3000, (n, n_emit))
        hm["score"][rng.random(n) < 0.2, 1] = WORST
        senscr = rng.integers(0, 900, (R, n_sen)).astype(np.int16)
    elif case == "floor":
        # int16 rows near 32767 from scores near the floor: every state reaches WORST_SCORE and stays there
        hm["score"][:, :n_emit] = WORST + rng.integers(0, 40 * 32767, (n, n_emit))
        hm["out_score"] = WORST + rng.integers(0, 40 * 32767, n)
        senscr = (32767 - rng.integers(0, 64, (R, n_sen))).astype(np.int16)
    else:
        # ties: scores, transitions and (constant) rows on a grid of 10, so the candidates of each pick meet
        hm["score"][:, :n_emit] = -10 * rng.integers(0, 3, (n, n_emit))
        tp[:] = np.where(rng.random(tp.shape) < 0.5, 0, 10).astype(tp.dtype)
        senscr = np.repeat(10 * rng.integers(0, 4, (R, 1)), n_sen, axis=1).astype(np.int16)
    return tp, sseq, hm, n_sen, senscr


@pytest.mark.parametrize("n_emit", [3, 5])
@pytest.mark.parametrize("case,T", [("absent_arcs", 9), ("floor", 301), ("ties", 13)])
def test_sweep_step_matches_oracle_and_per_frame(api, n_emit, case, T):
    import torch
    from oracle import oracle
    tp, sseq, hm0, n_sen, senscr = make_case(n_emit, case, T, seed=100 + 7 * n_emit + T)
    R = len(senscr)
    n = len(hm0)
    seg_off = np.concatenate([[0], np.cumsum(SEG_LEN)]).astype(np.int64)
    n_seg = len(SEG_LEN)
    n_rows = np.array([T, T, T, T, T - 4], np.int32)
    row0 = np.array([2, 0, T + 1, R - T, 5], np.int64)                  # segment 3 ends on the matrix's last row
    ctx = api.HmmContext(tp, sseq, n_sen)
    d_scr = torch.from_numpy(senscr).cuda()
    d_row0, d_nrows = torch.from_numpy(row0).cuda(), torch.from_numpy(n_rows).cuda()
    res = []
    for fused in (False, True):
        hs = api.HmmSet(ctx, n + 8 * 512, 16)
        hs.upload(hm0, seg_off)
        d_best = torch.zeros((T, n_seg), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        if fused:
            hs.sweep_device(d_scr.data_ptr(), R, T, d_best.data_ptr(), d_row0=d_row0.data_ptr(), d_n_rows=d_nrows.data_ptr())
        else:
            hs.eval_frames_device(d_scr.data_ptr(), T, d_best.data_ptr(), d_row0=d_row0.data_ptr(), d_n_rows=d_nrows.data_ptr())
        res.append((hs.download(), d_best.cpu().numpy()))
        hs.close()
    octx = oracle.OracleHmmCtx(tp, sseq)
    want = hm0.copy()
    for s in range(n_seg):
        a, b = seg_off[s], seg_off[s + 1]
        for t in range(T):
            if t >= n_rows[s] or a == b:
                assert res[1][1][t, s] == WORST
                continue
            seg = np.ascontiguousarray(want[a:b])
            wb = octx.vit_eval(seg, senscr[row0[s] + t])
            want[a:b] = seg
            assert res[1][1][t, s] == wb, "segment %d frame %d" % (s, t)
    assert_hmm_equal(res[1][0], want, n_emit, "%s: fused vs oracle" % case)
    assert np.array_equal(res[0][1], res[1][1])
    assert_hmm_equal(res[0][0], res[1][0], n_emit, "%s: per-frame vs fused" % case)
    if case == "floor":
        assert (want["score"][:, :n_emit] == WORST).mean() > 0.3, "the floor must be reached"

    # the beam variant shares the loop: every instance active at frame0, against the oracle's pruned sweep
    frame0, beam = 3, -2000
    hb = hm0.copy()
    hb["frame"] = frame0
    hs = api.HmmSet(ctx, n + 8 * 512, 16)
    hs.upload(hb, seg_off)
    d_best = torch.zeros((T, n_seg), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    hs.sweep_beam_device(d_scr.data_ptr(), R, T, frame0, beam, d_best.data_ptr(), d_row0=d_row0.data_ptr(),
                         d_n_rows=d_nrows.data_ptr())
    got, best = hs.download(), d_best.cpu().numpy()
    hs.close()
    ctx.close()
    want = hb.copy()
    for s in range(n_seg):
        a, b = seg_off[s], seg_off[s + 1]
        Ts = int(min(T, n_rows[s]))
        seg = np.ascontiguousarray(want[a:b])
        wb, _ = oracle.sweep_beam(octx, seg, senscr[row0[s]:row0[s] + Ts], frame0, beam, -1)
        want[a:b] = seg
        assert np.array_equal(best[:Ts, s], wb), "%s: beam segment %d best" % (case, s)
    assert_hmm_equal(got, want, n_emit, "%s: beam sweep" % case)
