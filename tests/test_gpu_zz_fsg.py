"""GPU (-m gpu): psb_fsg_batch_device (the grammar search of fsg_search.c on the device) against the
reference's golden history tables and against the oracle on ragged batches.

The phase code is also checked on the host against the reference (tests/test_fsg_emul.py)."""

import numpy as np
import pytest

from conftest import golden

pytestmark = [pytest.mark.gpu]

TAGS = ("go", "go_hmmpf", "cmd", "cmd_wide", "cmd_hmmpf")


def _case(g, tag):
    return {k[len(tag) + 1:]: g[k] for k in g.files if k.startswith(tag + ".")}


@pytest.fixture(scope="module")
def api():
    from pocketsphinx_b200 import api
    assert api.device_count() > 0, "no CUDA device visible"
    return api


@pytest.mark.timeout(300)
@pytest.mark.parametrize("tag", TAGS)
def test_fsg_batch_matches_reference_and_oracle(api, en_us, tag):
    import torch
    from oracle import oracle
    scr = golden("en_us_goforward.npz")["senscr"]
    c = _case(golden("en_us_fsg.npz"), tag)
    # the reference's utterance, prefixes of it (0, 1, 100 frames), a middle piece, and the whole again
    parts = [scr, scr[:0], scr[:1], scr[:100], scr[60:200], scr]
    utt_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int32)
    d_scr = torch.from_numpy(np.ascontiguousarray(np.concatenate(parts))).cuda()
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    cap = len(c["hist"]) + 64
    hist, n = ctx.fsg(d_scr.data_ptr(), utt_off, c, cap)
    assert n[0] == len(c["hist"]) and np.array_equal(hist[0], c["hist"])          # the reference's own table
    assert n[5] == n[0] and np.array_equal(hist[5], hist[0])
    for u in (1, 2, 3, 4):
        want = oracle.fsg_run(en_us.tp, en_us.sseq, c, parts[u])
        assert n[u] == len(want) and np.array_equal(hist[u], want), "utterance %d" % u
    bp, score = oracle.fsg_find_exit(hist[0], c["links"], len(scr), int(c["final_state"]))
    assert bp > 0 and score == int(c["score"])
    h2, n2 = ctx.fsg(d_scr.data_ptr(), utt_off, c, 50)                             # truncated tables, full counts
    assert np.array_equal(n2, n) and all(np.array_equal(a, b[:50]) for a, b in zip(h2, hist))
    ctx.close()


@pytest.mark.timeout(300)
def test_fsg_rejects_bad_graphs(api, en_us):
    import torch
    from pocketsphinx_b200._lib import PsbError
    scr = golden("en_us_goforward.npz")["senscr"][:10]
    c = dict(_case(golden("en_us_fsg.npz"), "go"))
    d_scr = torch.from_numpy(np.ascontiguousarray(scr)).cuda()
    ctx = api.HmmContext(en_us.tp, en_us.sseq, en_us.n_sen)
    pn = c["pnodes"].copy()
    inner = np.nonzero((pn[:, 7] == 0) & (pn[:, 2] >= 0))[0]
    pn[inner[1], 2] = pn[inner[0], 2]
    c["pnodes"] = pn
    with pytest.raises(PsbError):
        ctx.fsg(d_scr.data_ptr(), np.array([0, 10], np.int32), c, 64)
    ctx.close()


def test_block_scan_selftest(api):
    """fsg_exscan on the device against numpy, lengths around the chunk (128) and warp (32) boundaries."""
    import ctypes as C
    from pocketsphinx_b200._lib import check, lib
    rng = np.random.default_rng(2)
    for n in (0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1000, 4097):
        a = rng.integers(0, 5, n).astype(np.int32)
        want = np.concatenate([[0], np.cumsum(a)[:-1]]).astype(np.int32) if n else a.copy()
        got = a.copy()
        total = np.zeros(2, np.int32)
        check(lib().psb_selftest_block_scan(0, got.ctypes.data_as(C.c_void_p), n, total.ctypes.data_as(C.c_void_p)),
              "psb_selftest_block_scan")
        assert np.array_equal(got, want) and total[0] == a.sum() and total[1] == 0, n
