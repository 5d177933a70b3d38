"""CPU: step-by-step simulation of the device scan of psb_fsg_core.h (fsg_exscan: CTA-wide with warp
shuffles + a shared carry) -- the one building block of the search kernels the host emulation replaces
by a plain loop.  Every statement between two barriers is
executed for all "threads" before the next; a shuffle reads the source lane's value from before the
statement.  This checks the algorithm as written (chunking, carries, partial last chunk, empty input),
not the CUDA code itself: that is tests/test_gpu_zz_fsg.py::test_block_scan_selftest."""
import numpy as np
import pytest


def exscan_cta(a, n, nt=128):
    a = a.copy()
    scan = np.zeros(34, np.int64)
    tid = np.arange(nt)
    lane, w = tid & 31, tid >> 5
    base = 0
    while base < n:
        i = base + tid
        v = np.where(i < n, a[np.minimum(i, n - 1)], 0)
        incl = v.copy()
        o = 1
        while o < 32:
            t = np.where(lane >= o, incl[np.maximum(tid - o, 0)], 0)      # __shfl_up_sync(incl, o)
            incl = np.where(lane >= o, incl + t, incl)
            o <<= 1
        scan[w[lane == 31]] = incl[lane == 31]
        carry = scan[33]                                                   # (barrier)
        wbase = np.array([scan[:k].sum() for k in w])
        m = i < n
        a[i[m]] = (carry + wbase + incl - v)[m]
        scan[33] = carry + wbase[nt - 1] + incl[nt - 1]                    # (barrier) thread nt-1 (barrier)
        base += nt
    return a, int(scan[33])


@pytest.mark.parametrize("scan", [exscan_cta])
def test_scan_as_written(scan):
    rng = np.random.default_rng(1)
    for n in (0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1000, 4097):
        x = rng.integers(0, 5, n).astype(np.int64)
        want = np.concatenate([[0], np.cumsum(x)[:-1]]) if n else x
        got, total = scan(x, n)
        assert np.array_equal(got, want) and total == x.sum(), n
