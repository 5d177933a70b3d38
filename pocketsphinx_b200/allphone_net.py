"""The PHMM net of phone decoding (allphone_search.c) in the factored form psb_allphone_net_batch_device
takes, built from the model definition alone, and the integer search parameters allphone_search_init
computes.

phmm_build (allphone_search.c:220-317) makes one node per distinct (CI phone, tmat, senone sequence)
over the CI phones (-allphone_ci yes) or over every phone of the mdef (-allphone_ci no).  New nodes are
prepended to their CI phone's list, and the nodes are numbered ci-major in list order, which is the
order phmm_exit numbers history entries in.  Every CI phone's node gets full context sets; a CD phone
adds its left / right context to its node's lc / rc, a filler context standing for every filler.
phmm_link (:167-215) then links p -> p2 exactly when ci(p2) is in rc(p) and ci(p) is in lc(p2), which
is what the device search evaluates instead of walking links.
"""
import math

import numpy as np

SENSCR_SHIFT = 10


def mdef_phones(md):
    """The slice of s3io.read_mdef's result a net is built from."""
    return dict(n_ciphone=int(md["n_ciphone"]), phone_ssid=md["phone_ssid"], phone_tmat=md["phone_tmat"],
                phone_ctx=md["phone_ctx"], phone_filler=md["phone_filler"], sil=int(md["sil"]))


def build_net(phones, ci_only):
    """phones: mdef_phones(s3io.read_mdef(path)) (or the same keys from a fixture).  Returns a dict:
    ssid, tmatid, ci (int32 [H]), lc, rc (uint64 [H]), n_ci, start (allphone_search_start's silence
    node), pid (the phone that created each node)."""
    n_ci = int(phones["n_ciphone"])
    if n_ci > 64:
        raise ValueError("%d CI phones: the context sets are 64-bit masks" % n_ci)
    ssid = np.asarray(phones["phone_ssid"], np.int64)
    tmat = np.asarray(phones["phone_tmat"], np.int64)
    ctx = np.asarray(phones["phone_ctx"], np.int64)
    filler = np.asarray(phones["phone_filler"], np.int64)[:n_ci]
    sil = int(phones["sil"])
    n_phone = n_ci if ci_only else len(ssid)
    lists = [[] for _ in range(n_ci)]            # creation order; the walk order is the reverse
    key2node, node_of = {}, np.empty(n_phone, np.int64)
    created = []                                  # (ci, position in creation order, pid)
    for pid in range(n_phone):
        ci = pid if pid < n_ci else int(ctx[pid, 1])
        k = (ci, int(tmat[pid]), int(ssid[pid]))   # phmm_lookup (:146-165)
        j = key2node.get(k)
        if j is None:
            j = key2node[k] = len(created)
            created.append((ci, len(lists[ci]), pid))
            lists[ci].append(j)
        node_of[pid] = j
    order = [j for ci in range(n_ci) for j in reversed(lists[ci])]
    rank = np.empty(len(created), np.int64)
    rank[order] = np.arange(len(order))
    full = np.uint64((1 << n_ci) - 1)
    fill_mask = np.uint64(sum(1 << int(c) for c in np.nonzero(filler)[0]))
    lc = np.zeros(len(created), np.uint64)
    rc = np.zeros(len(created), np.uint64)
    lc[node_of[:n_ci]] = full
    rc[node_of[:n_ci]] = full
    if n_phone > n_ci:
        cd = np.arange(n_ci, n_phone)
        one = np.uint64(1)
        for side, col in ((lc, 2), (rc, 3)):
            c = ctx[cd, col]
            bits = np.where(filler[c] != 0, fill_mask, one << c.astype(np.uint64))
            np.bitwise_or.at(side, node_of[cd], bits)
    pid = np.array([created[j][2] for j in order], np.int64)
    ci_arr = np.array([created[j][0] for j in order], np.int32)
    start = int(rank[node_of[sil]]) if 0 <= sil < n_ci else -1
    return dict(ssid=ssid[pid].astype(np.int32), tmatid=tmat[pid].astype(np.int32), ci=ci_arr,
                lc=lc[order], rc=rc[order], n_ci=n_ci, start=start, pid=pid.astype(np.int32))


def expand_links(net):
    """phmm_link's successor lists (CSR, each list in the reference's order: rc ascending, then the
    target's list order, prepended -- i.e. reversed) from the factored form."""
    ci, lc, rc, n_ci = net["ci"], net["lc"], net["rc"], int(net["n_ci"])
    by_ci = [np.nonzero(ci == c)[0] for c in range(n_ci)]
    succ_off, succ = [0], []
    for p in range(len(ci)):
        lst = []
        for b in range(n_ci):
            if (int(rc[p]) >> b) & 1:
                t = by_ci[b]
                lst.extend(t[((lc[t] >> np.uint64(ci[p])) & np.uint64(1)) != 0].tolist())
        succ.extend(reversed(lst))
        succ_off.append(len(succ))
    return np.array(succ_off, np.int32), np.array(succ, np.int32)


def search_params(beam=1e-48, pbeam=1e-48, pip=1.0, lw=6.5, logbase=1.0001):
    """beam, pbeam, inspen as allphone_search_init (:580-601) computes them: logmath_log of the
    probability (log(p) * (1 / log(base)), truncated by the int cast) >> SENSCR_SHIFT; inspen additionally
    weighted by lw before the shift.  The search keeps lw in an int32 field, so -lw 6.5 weighs by 6."""
    inv = 1.0 / math.log(logbase)

    def lm(x):
        if x <= 0:
            return -(1 << 31) >> 2   # logmath_log of zero: the log-math zero (logmath.c:86)
        return int(math.log(x) * inv)
    return lm(beam) >> SENSCR_SHIFT, lm(pbeam) >> SENSCR_SHIFT, (lm(pip) * int(lw)) >> SENSCR_SHIFT
