"""GPU (-m gpu): how the fused sweep (psb_hmmset_sweep_device) lays a segment out over its CTAs of 512 threads x 4
instances.  Segments whose sizes straddle one CTA (2 048 instances), ragged frame counts and a segment ending on the score
matrix's last row against n_frames launches of the per-frame kernel: best[t][segment] and the whole downloaded state, byte
for byte.  Padding slots: a CTA's slots beyond the segment's end gather senone 0 and are kept out of the frame's maximum by
their transitions alone, so senone 0 scores -32768 in every row here and segment 0's only instance sits on the WORST_SCORE
floor -- any padding slot that rose above the floor would show in best[t][0].  Snapshot / restore / a second sweep give the
bytes of a fresh upload, and the beam sweep on a set the plain sweep has run on is the beam sweep on a fresh one."""
import numpy as np
import pytest

from conftest import assert_hmm_equal, golden, hmm_view

pytestmark = pytest.mark.gpu

WORST = -0x20000000
CTA = 512 * 4
SEG_LEN = [1, CTA - 1, CTA, CTA + 1, 6081, 3 * CTA + 1]
T = 7
N_ROWS = np.array([T, T - 2, T, T, T - 3, T], np.int32)


@pytest.fixture(scope="module")
def api():
    from pocketsphinx_b200 import api
    assert api.device_count() > 0, "no CUDA device visible"
    return api


def make_case(n_emit, seed):
    g = golden("hmm_vit_eval.npz")
    tp, sseq = g["n%d_tp" % n_emit], g["n%d_sseq" % n_emit]
    n_sen = len(g["n%d_senscr" % n_emit])
    n_sen -= n_sen & 1                                                  # the fused kernel's shape
    hm = hmm_view(g["n%d_before" % n_emit]).copy()
    sid = hm["senid"][:, :n_emit]
    hm = hm[(hm["mpx"] == 0) & (sid < n_sen).all(1) & (sid > 0).all(1)]  # senone 0 is the padding slots' alone
    rng = np.random.default_rng(seed)
    n = sum(SEG_LEN)
    hm = np.ascontiguousarray(hm[rng.integers(0, len(hm), n)])
    hm["score"][:, :n_emit] = -rng.integers(0, 3000, (n, n_emit))
    hm["history"][:, :n_emit] = rng.integers(0, 1 << 30, (n, n_emit))
    hm["out_history"] = rng.integers(0, 1 << 30, n)
    hm["tmatid"] = rng.integers(0, tp.shape[0], n)
    hm["score"][0, :n_emit] = WORST                                     # segment 0's instance stays on the floor
    hm["out_score"][0] = WORST
    hm["frame"] = 0                                                     # all active for the beam sweep from frame 0
    R = 4 * T
    senscr = rng.integers(0, 900, (R, n_sen)).astype(np.int16)
    senscr[:, 0] = -32768
    seg_off = np.concatenate([[0], np.cumsum(SEG_LEN)]).astype(np.int64)
    row0 = np.array([2, 0, T + 1, R - T, 5, 3], np.int64)               # segment 3 ends on the matrix's last row
    return tp, sseq, hm, n_sen, senscr, seg_off, row0


def run(api, ctx, hm, seg_off, d_scr, R, d_row0, d_nrows, how, hs=None):
    import torch
    own = hs is None
    if own:
        hs = api.HmmSet(ctx, len(hm) + 8 * 512, 16)
        hs.upload(hm, seg_off)
    d_best = torch.zeros((T, len(seg_off) - 1), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    if how == "fused":
        hs.sweep_device(d_scr.data_ptr(), R, T, d_best.data_ptr(), d_row0=d_row0.data_ptr(), d_n_rows=d_nrows.data_ptr())
    elif how == "per_frame":
        hs.eval_frames_device(d_scr.data_ptr(), T, d_best.data_ptr(), d_row0=d_row0.data_ptr(), d_n_rows=d_nrows.data_ptr())
    else:
        hs.sweep_beam_device(d_scr.data_ptr(), R, T, 0, -2000, d_best.data_ptr(), d_row0=d_row0.data_ptr(), d_n_rows=d_nrows.data_ptr())
    out = hs.download(), d_best.cpu().numpy()
    if own:
        hs.close()
    return out


@pytest.mark.parametrize("n_emit", [3, 5])
def test_sweep_cta_layout_matches_per_frame(api, n_emit):
    import torch
    tp, sseq, hm, n_sen, senscr, seg_off, row0 = make_case(n_emit, 300 + n_emit)
    R = len(senscr)
    ctx = api.HmmContext(tp, sseq, n_sen)
    d_scr = torch.from_numpy(senscr).cuda()
    d_row0, d_nrows = torch.from_numpy(row0).cuda(), torch.from_numpy(N_ROWS).cuda()
    args = (api, ctx, hm, seg_off, d_scr, R, d_row0, d_nrows)
    want, want_best = run(*args, "per_frame")
    got, got_best = run(*args, "fused")
    assert np.array_equal(got_best, want_best)
    assert (want_best[:, 0] == WORST).all(), "segment 0 must stay on the floor for the padding slots to show"
    assert (want_best[:N_ROWS[4], 4] > WORST).all()
    assert_hmm_equal(got, want, n_emit, "fused vs per-frame")
    assert got.tobytes() == want.tobytes()

    # snapshot / restore / a second sweep: the bytes of a fresh upload; then the beam sweep on that set
    hs = api.HmmSet(ctx, len(hm) + 8 * 512, 16)
    hs.upload(hm, seg_off)
    hs.snapshot()
    first, _ = run(*args, "fused", hs=hs)
    hs.restore()
    assert_hmm_equal(hs.download(), hm, n_emit, "restore brings back the uploaded instances, in upload order")
    second, second_best = run(*args, "fused", hs=hs)
    assert first.tobytes() == got.tobytes() and second.tobytes() == got.tobytes()
    assert np.array_equal(second_best, want_best)
    hs.restore()
    beam_after, beam_after_best = run(*args, "beam", hs=hs)
    hs.close()
    beam_fresh, beam_fresh_best = run(*args, "beam")
    assert np.array_equal(beam_after_best, beam_fresh_best)
    assert beam_after.tobytes() == beam_fresh.tobytes()
    ctx.close()
