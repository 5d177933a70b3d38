"""Sphinx-3 acoustic-model files (the data formats on the input side of the hot path): writers, and
readers that turn a model directory into the arrays the device scorers take (read_model_dir, below).

Host-side plumbing for synthetic models: writes the files the reference's loaders read
(`means`, `variances`, `sendump`, `mixture_weights`, `transition_matrices`, text `mdef`,
`feat.params`; formats: SURVEY A.3, src/util/bio.c:188-296, src/ms_gauden.c:159-229,
src/ptm_mgau.c:457-661, src/tmat.c:178-236, src/mdef.c:515-700) and mirrors, in float64 with
the same libm calls, the precomputation those loaders apply, so that a model generated here is
the same model -- bit for bit -- after the unmodified reference has loaded it
(tests/test_s3io_vs_ref.py checks that against oracle/_ref when present).
"""
import math
import os
import re
import struct

import numpy as np

BYTE_ORDER_MAGIC = 0x11223344


def _chksum(data: bytes, s=0):
    """bio.c:266-296 chksum_accum: rotate-left-20 and add, per 32-bit word."""
    w = np.frombuffer(data, "<u4").astype(np.uint64)
    for v in w.tolist():
        s = (((s << 20) | (s >> 12)) + v) & 0xFFFFFFFF
    return s


def _chksum_fast(data: bytes, s=0):
    # same recurrence, vectorised in blocks: s_{k+1} = rotl20(s_k) + w_k  (mod 2^32)
    w = np.frombuffer(data, "<u4")
    s = int(s)
    for v in w.tolist():
        s = (((s << 20) & 0xFFFFFFFF) | (s >> 12)) + v & 0xFFFFFFFF
    return s


def _write_s3(path, header_pairs, payload: bytes):
    with open(path, "wb") as f:
        f.write(b"s3\n")
        for k, v in header_pairs:
            f.write(("%s %s\n" % (k, v)).encode())
        f.write(b"endhdr\n")
        f.write(struct.pack("<I", BYTE_ORDER_MAGIC))
        f.write(payload)
        f.write(struct.pack("<I", _chksum_fast(payload)))


def write_gauden(path, arr, n_mgau, n_feat, n_density, featlen):
    """means / variances: int32 n_mgau, n_feat, n_density, veclen[n_feat], n_floats, then
    float32 [n_mgau][n_feat][n_density][veclen] (ms_gauden.c:159-229)."""
    arr = np.ascontiguousarray(arr, "<f4").ravel()
    hdr = struct.pack("<3i", n_mgau, n_feat, n_density) + struct.pack("<%di" % n_feat, *[int(x) for x in featlen])
    hdr += struct.pack("<i", arr.size)
    _write_s3(path, [("version", "1.0"), ("chksum0", "yes")], hdr + arr.tobytes())


def write_tmat(path, tp_float):
    """transition_matrices: int32 n_tmat, n_src, n_dst, n; float32 [n_tmat][n_src][n_dst]."""
    tp_float = np.ascontiguousarray(tp_float, "<f4")
    n_tmat, n_src, n_dst = tp_float.shape
    hdr = struct.pack("<4i", n_tmat, n_src, n_dst, tp_float.size)
    _write_s3(path, [("version", "1.0"), ("chksum0", "yes")], hdr + tp_float.tobytes())


def write_mixw(path, w):
    """mixture_weights: int32 n_sen, n_feat, n_comp, n; float32 [n_sen][n_feat][n_comp]."""
    w = np.ascontiguousarray(w, "<f4")
    n_sen, n_feat, n_comp = w.shape
    hdr = struct.pack("<4i", n_sen, n_feat, n_comp, w.size)
    _write_s3(path, [("version", "1.0"), ("chksum0", "yes")], hdr + w.tobytes())


def write_sendump(path, mixw, n_feat, n_density, n_sen, mixw_cb=None):
    """sendump (ptm_mgau.c:457-661): length-prefixed title/header strings, key/value strings
    terminated by a zero length, then rows/cols (unclustered) or the 16-byte cluster codebook
    (4-bit), then per feature, per codeword one row of n_sen bytes ((n_sen+1)/2 when 4-bit)."""
    def lps(s):
        b = s.encode() + b"\0"
        return struct.pack("<i", len(b)) + b
    four = mixw_cb is not None and len(mixw_cb) == 16
    out = lps("V6 Senone Probs, Smoothed, Normalized") + lps("synthetic model written by pocketsphinx_b200.s3io")
    out += lps("feature_count %d" % n_feat) + lps("mixture_count %d" % n_density) + lps("model_count %d" % n_sen)
    if four:
        out += lps("cluster_count 16") + lps("cluster_bits 4")
    out += struct.pack("<i", 0)
    if four:
        out += bytes(bytearray(np.asarray(mixw_cb, np.uint8).tolist()))
    else:
        out += struct.pack("<2i", n_density, n_sen)
    out += np.ascontiguousarray(mixw, np.uint8).tobytes()
    with open(path, "wb") as f:
        f.write(out)


def write_mdef_text(path, n_ci, n_emit, sen2ci, n_ci_sen, n_tmat=None):
    """Text model definition (mdef.c:515-700): CI phones P0..P{n-1} (the last is SIL, a filler)
    plus synthetic word-internal triphones that own the remaining senones so that every senone
    maps to its base phone (bin_mdef sen2cimap, needed by the PTM back-end)."""
    n_sen = len(sen2ci)
    n_tmat = n_tmat or n_ci
    names = ["P%03d" % i for i in range(n_ci - 1)] + ["SIL"]
    by_ci = [[] for _ in range(n_ci)]
    for s in range(n_ci_sen, n_sen):
        by_ci[int(sen2ci[s])].append(s)
    tri = []
    for b in range(n_ci):
        own = by_ci[b]
        k = 0
        ctx = 0
        while k < len(own):
            sens = [own[min(k + j, len(own) - 1)] for j in range(n_emit)]
            k += n_emit
            lft, rt = ctx // (n_ci - 1), ctx % (n_ci - 1)      # never SIL as context
            ctx += 1
            tri.append((b, lft, rt, sens))
    lines = ["# synthetic mdef written by pocketsphinx_b200.s3io", "0.3", "%d n_base" % n_ci, "%d n_tri" % len(tri),
             "%d n_state_map" % ((n_ci + len(tri)) * (n_emit + 1)), "%d n_tied_state" % n_sen,
             "%d n_tied_ci_state" % n_ci_sen, "%d n_tied_tmat" % n_tmat, "#",
             "# Columns definitions", "#base lft  rt p attrib tmat      ... state id's ..."]
    for i in range(n_ci):
        attr = "filler" if names[i] == "SIL" else "n/a"
        st = " ".join("%5d" % (i * n_emit + j) for j in range(n_emit))
        lines.append("%5s   -   - - %7s %4d %s    N" % (names[i], attr, i % n_tmat, st))
    for b, lft, rt, sens in tri:
        attr = "filler" if names[b] == "SIL" else "n/a"
        st = " ".join("%5d" % s for s in sens)
        lines.append("%5s %3s %3s i %7s %4d %s    N" % (names[b], names[lft], names[rt], attr, b % n_tmat, st))
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")
    return len(tri)


# ---------------------------------------------------------------------------------------
# mirrors of the loaders' arithmetic (float64 + libm, like the C code)

LOGBASE = 1.0001


def precompute_gaussians(var_raw, n_mgau, n_feat, n_density, featlen, varfloor=1e-4, logbase=LOGBASE):
    """gauden_dist_precompute (ms_gauden.c:264-308): floor the variances, det = sum over
    dims of (float)(int)(log(1/sqrt(2 pi v)) / log b), var = (float)(int)(log-domain 1/(2v))."""
    inv = 1.0 / math.log(logbase)
    v32 = np.ascontiguousarray(var_raw, np.float32).ravel().copy()
    v32[v32 < np.float32(varfloor)] = np.float32(varfloor)
    vals = v32.astype(np.float64).tolist()
    two_pi = 2.0 * math.pi
    dterm = np.array([float(int(math.log(1.0 / math.sqrt(v * two_pi)) * inv)) for v in vals], np.float32)
    pvar = np.array([float(int((1.0 / (v * 2.0)) * inv)) for v in vals], np.float32)
    det = np.zeros((n_mgau, n_feat, n_density), np.float32)
    pos = 0
    for m in range(n_mgau):
        for f in range(n_feat):
            fl = int(featlen[f])
            blk = dterm[pos:pos + n_density * fl].reshape(n_density, fl)
            acc = np.zeros(n_density, np.float32)
            for j in range(fl):                      # float32 accumulation in dimension order
                acc = (acc + blk[:, j]).astype(np.float32)
            det[m, f] = acc
            pos += n_density * fl
    return pvar, det


def quantize_tmat(tp_float, tpfloor=1e-4, logbase=LOGBASE):
    """tmat_init (tmat.c:215-236): normalise each row, floor the non-zero entries, renormalise,
    then tp = min(255, (-(int)(log(p)/log b)) >> 10); zero probabilities become 255."""
    inv = 1.0 / math.log(logbase)
    t = np.ascontiguousarray(tp_float, np.float32).copy()
    out = np.zeros(t.shape, np.uint8)
    zero = -(1 << 31) >> 2                                  # logmath zero for shift 0
    for i in range(t.shape[0]):
        for j in range(t.shape[1]):
            row = t[i, j]
            s = np.float64(0.0)
            for x in row.tolist():                            # vector_sum_norm: float64 sum
                s += x
            if s != 0.0:
                row = (row.astype(np.float64) * (1.0 / s)).astype(np.float32)
            row = np.where((row != 0) & (row.astype(np.float64) < tpfloor), np.float32(tpfloor), row)   # vector_nz_floor
            s = np.float64(0.0)
            for x in row.tolist():
                s += x
            if s != 0.0:
                row = (row.astype(np.float64) * (1.0 / s)).astype(np.float32)
            for k, p in enumerate(row.tolist()):
                lp = zero if p <= 0 else int(math.log(p) * inv)
                ltp = (-lp) >> 10
                out[i, j, k] = 255 if ltp > 255 else ltp
    return out


def quantize_mixw_ms(w, mixwfloor=1e-7, logbase=LOGBASE):
    """senone_mixw_read (ms_senone.c:135-268): per (senone, stream) normalise, floor, renormalise,
    then pdf = min(255, (-(int)(log(p)/log b) + 511) >> 10).  w: float32 [n_sen][n_feat][n_cw]."""
    inv = 1.0 / math.log(logbase)
    w = np.ascontiguousarray(w, np.float32)
    out = np.zeros(w.shape, np.uint8)
    zero = -(1 << 31) >> 2
    for i in range(w.shape[0]):
        for f in range(w.shape[1]):
            row = w[i, f]
            s = 0.0
            for x in row.tolist():
                s += x
            if s != 0.0:
                row = (row.astype(np.float64) * (1.0 / s)).astype(np.float32)
            row = np.where(row.astype(np.float64) < mixwfloor, np.float32(mixwfloor), row)      # vector_floor
            s = 0.0
            for x in row.tolist():
                s += x
            if s != 0.0:
                row = (row.astype(np.float64) * (1.0 / s)).astype(np.float32)
            for c, p in enumerate(row.tolist()):
                lp = zero if p <= 0 else int(math.log(p) * inv)
                q = -lp + 511
                out[i, f, c] = (q >> 10) if q < (255 << 10) else 255
    return out


def write_model_dir(path, *, kind, n_mgau, n_feat, n_density, featlen, mean, var_raw, tp_float, sen2ci, n_ci,
                    n_emit, n_ci_sen, mixw_q=None, mixw_cb=None, mixw_float=None, feat_params=None):
    """Write a complete acoustic-model directory the reference's acmod_init can load."""
    os.makedirs(path, exist_ok=True)
    write_gauden(os.path.join(path, "means"), mean, n_mgau, n_feat, n_density, featlen)
    write_gauden(os.path.join(path, "variances"), var_raw, n_mgau, n_feat, n_density, featlen)
    write_tmat(os.path.join(path, "transition_matrices"), tp_float)
    write_mdef_text(os.path.join(path, "mdef"), n_ci, n_emit, sen2ci, n_ci_sen, n_tmat=tp_float.shape[0])
    if mixw_q is not None:
        write_sendump(os.path.join(path, "sendump"), mixw_q, n_feat, n_density, len(sen2ci), mixw_cb)
    if mixw_float is not None:
        write_mixw(os.path.join(path, "mixture_weights"), mixw_float)
    with open(os.path.join(path, "feat.params"), "w") as f:
        f.write(feat_params or "")


# ---------------------------------------------------------------------------------------
# Readers: an acoustic-model directory -> the arrays psb_model_create takes, without the reference.
# The same files the reference's loaders read, the same arithmetic afterwards (the mirrors above);
# tests/test_s3io_read.py compares every array with what the compiled reference holds after
# acmod_init on its three shipped models (PTM en-us, semi-continuous tidigits, continuous an4).

def _read_s3(path, verify=True):
    """bio_readhdr + payload (bio.c:188-262): "s3\\n", "key value" lines up to "endhdr", the byte-order
    word, data, and (chksum0 yes, verify) the trailing checksum of bio_fread's rotate-and-add (:266-296)."""
    with open(path, "rb") as f:
        raw = f.read()
    if not raw.startswith(b"s3\n"):
        raise ValueError("%s: not an s3 file" % path)
    end = raw.find(b"endhdr\n")
    if end < 0:
        raise ValueError("%s: no endhdr" % path)
    hdr = {}
    for line in raw[3:end].decode("latin-1").split("\n"):
        line = line.strip()
        if line and not line.startswith("#"):
            k, _, v = line.partition(" ")
            hdr[k] = v.strip()
    pos = end + 7
    magic = struct.unpack_from("<I", raw, pos)[0]
    if magic == BYTE_ORDER_MAGIC:
        order = "<"
    elif struct.unpack_from(">I", raw, pos)[0] == BYTE_ORDER_MAGIC:
        order = ">"
    else:
        raise ValueError("%s: bad byte-order word %#x" % (path, magic))
    body = raw[pos + 4:]
    if verify and hdr.get("chksum0", "no") == "yes":
        body, tail = body[:-4], body[-4:]
        data = body if order == "<" else np.frombuffer(body, ">u4").astype("<u4").tobytes()
        if _chksum_fast(data) != struct.unpack(order + "I", tail)[0]:
            raise ValueError("%s: checksum mismatch" % path)
    return hdr, body, order


def read_gauden(path):
    """means / variances (gauden_param_read, ms_gauden.c:140-230) -> (n_mgau, n_feat, n_density,
    featlen, float32 [n_mgau][n_feat][n_density][featlen[f]] flat)."""
    hdr, b, o = _read_s3(path)
    n_mgau, n_feat, n_density = struct.unpack_from(o + "3i", b, 0)
    if n_mgau <= 0 or n_feat <= 0 or n_density <= 0 or n_feat > 64:
        raise ValueError("%s: bad dimensions" % path)
    featlen = np.array(struct.unpack_from(o + "%di" % n_feat, b, 12), np.int32)
    n = struct.unpack_from(o + "i", b, 12 + 4 * n_feat)[0]
    if (featlen <= 0).any() or n != n_mgau * n_density * int(featlen.sum()):
        raise ValueError("%s: %d floats for %d x %d x %s" % (path, n, n_mgau, n_density, featlen.tolist()))
    arr = np.frombuffer(b, o + "f4", n, 16 + 4 * n_feat).astype(np.float32)
    return n_mgau, n_feat, n_density, featlen, arr


def read_tmat(path):
    """transition_matrices (tmat_init, tmat.c:131-205): float32 [n_tmat][n_src][n_src + 1]."""
    hdr, b, o = _read_s3(path)
    n_tmat, n_src, n_dst, n = struct.unpack_from(o + "4i", b, 0)
    if n_tmat <= 0 or n_tmat >= 32767 or n_dst != n_src + 1 or n != n_tmat * n_src * n_dst:
        raise ValueError("%s: unsupported transition matrices %d x %d x %d" % (path, n_tmat, n_src, n_dst))
    return np.frombuffer(b, o + "f4", n, 16).astype(np.float32).reshape(n_tmat, n_src, n_dst)


def read_lda(path):
    """feature_transform / -lda (feat_read_lda, lda.c:61-137): float32 [n_lda][m][n]; the front end uses [0],
    eigenvectors in rows.  The reference computes the checksum but never compares it, so neither does this."""
    hdr, b, o = _read_s3(path, verify=False)
    if len(b) < 16:
        raise ValueError("%s: truncated transform header" % path)
    d1, d2, d3, n = struct.unpack_from(o + "4I", b, 0)
    if n == 0 or n != d1 * d2 * d3 or len(b) < 16 + 4 * n:
        raise ValueError("%s: bad transform dimensions %d x %d x %d (%d values, %d bytes of data)"
                         % (path, d1, d2, d3, n, len(b) - 16))
    return np.frombuffer(b, o + "f4", n, 16).astype(np.float32).reshape(d1, d2, d3)


def write_lda(path, lda):
    """A feature_transform file (bio_fwrite_3d with its checksum) of float32 [n_lda][m][n]."""
    a = np.ascontiguousarray(lda, "<f4")
    assert a.ndim == 3
    payload = struct.pack("<4I", *a.shape, a.size) + a.tobytes()
    _write_s3(path, [("version", "0.1"), ("chksum0", "yes")], payload)


def read_mixw(path):
    """mixture_weights (senone_mixw_read, ms_senone.c:135-200): float32 [n_sen][n_feat][n_cw]."""
    hdr, b, o = _read_s3(path)
    n_sen, n_feat, n_cw, n = struct.unpack_from(o + "4i", b, 0)
    if min(n_sen, n_feat, n_cw) <= 0 or n != n_sen * n_feat * n_cw:
        raise ValueError("%s: bad dimensions" % path)
    return np.frombuffer(b, o + "f4", n, 16).astype(np.float32).reshape(n_sen, n_feat, n_cw)


def read_sendump(path, n_feat, n_density, n_sen):
    """sendump (read_sendump, ptm_mgau.c:457-661 = s2_semi_mgau.c:886-1090): returns (mixw uint8
    [n_feat][n_density][row], cluster codebook (16 bytes) or empty); row = n_sen, or (n_sen + 1) / 2 for
    4-bit cluster ids."""
    with open(path, "rb") as f:
        raw = f.read()
    pos, o = 0, "<"
    n = struct.unpack_from("<i", raw, 0)[0]
    if n < 1 or n > 999:
        o = ">"
        n = struct.unpack_from(">i", raw, 0)[0]
        if n < 1 or n > 999:
            raise ValueError("%s: title length out of range" % path)

    def string():
        nonlocal pos
        k = struct.unpack_from(o + "i", raw, pos)[0]
        pos += 4
        if k == 0:
            return None
        if k < 0 or pos + k > len(raw):
            raise ValueError("%s: bad header string" % path)
        s = raw[pos:pos + k]
        pos += k
        return s
    for what in ("title", "header"):
        s = string()
        if s is None or s[-1:] != b"\0":
            raise ValueError("%s: bad %s" % (path, what))
    kv = dict(feature_count=n_feat, mixture_count=n_density, model_count=n_sen, cluster_count=0, cluster_bits=8)
    while True:
        s = string()
        if s is None:
            break
        key, _, val = s.split(b"\0")[0].decode("latin-1").partition(" ")
        if key in kv:
            m = re.match(r"\s*([+-]?\d+)", val)           # atoi
            kv[key] = int(m.group(1)) if m else 0
    r, c = kv["mixture_count"], kv["model_count"]
    n_clust, n_bits = kv["cluster_count"], kv["cluster_bits"]
    if n_clust == 0:                                      # older files: rows / columns here, columns possibly padded
        r, c = struct.unpack_from(o + "2i", raw, pos)
        pos += 8
    if (kv["feature_count"], kv["mixture_count"], kv["model_count"]) != (n_feat, n_density, n_sen):
        raise ValueError("%s: %d streams x %d densities x %d senones, the model has %d x %d x %d" % (
            path, kv["feature_count"], kv["mixture_count"], kv["model_count"], n_feat, n_density, n_sen))
    if n_clust not in (0, 15, 16) or n_bits not in (4, 8):
        raise ValueError("%s: cluster count %d / bits %d" % (path, n_clust, n_bits))
    if n_clust == 15:
        n_clust = 16
    cb = np.frombuffer(raw, np.uint8, n_clust, pos).copy()
    pos += n_clust
    step = (c + 1) // 2 if n_bits == 4 else c
    row = (n_sen + 1) // 2 if n_clust else n_sen
    if r < n_density or step < row or pos + n_feat * r * step > len(raw):
        raise ValueError("%s: %d rows of %d bytes do not hold the model / the file" % (path, r, step))
    rows = np.frombuffer(raw, np.uint8, n_feat * r * step, pos).reshape(n_feat, r, step)
    return np.ascontiguousarray(rows[:, :n_density, :row]), cb


def read_mdef(path):
    """Model definition: the binary form (bin_mdef_read, bin_mdef.c:323-522) or a text one without
    triphones (mdef.c:515-700; triphones would need bin_mdef_read_text's phone reordering: convert such a
    file with the reference's pocketsphinx_mdef_convert).  Returns a dict: n_ciphone, n_phone,
    n_emit_state, n_ci_sen, n_sen, n_tmat, ciname, sseq [n_sseq][n_emit], phone_ssid, phone_tmat,
    phone_filler, sen2cimap, cd_tree (the triphone lookup tree: ctx, n_down, down / pid; None for a CI-only
    text file), sil (the id of SIL or -1)."""
    with open(path, "rb") as f:
        raw = f.read()
    if raw[:4] in (b"BMDF", b"FDMB"):
        o = "<" if raw[:4] == b"BMDF" else ">"
        version, fmt_len = struct.unpack_from(o + "2i", raw, 4)
        if version > 1:
            raise ValueError("%s: format version %d" % (path, version))
        pos = 12 + fmt_len
        n_ci, n_phone, n_emit, n_ci_sen, n_sen, n_tmat, n_sseq, n_ctx, n_cd_tree, sil = struct.unpack_from(o + "10i", raw, pos)
        pos += 40
        if n_emit <= 0:
            raise ValueError("%s: variable-length topologies are not supported" % path)
        names, p = [], pos
        for _ in range(n_ci):
            e = raw.index(b"\0", p)
            names.append(raw[p:e].decode("latin-1"))
            p = e + 1
        p = pos + ((p - pos + 3) & ~3)
        cd_tree = np.frombuffer(raw, np.dtype([("ctx", o + "i2"), ("n_down", o + "i2"), ("down", o + "i4")]), n_cd_tree, p)
        p += 8 * n_cd_tree                                   # cd_tree_t {int16 ctx, n_down; int32 down / pid}
        ent = np.frombuffer(raw, np.dtype([("ssid", o + "i4"), ("tmat", o + "i4"), ("info", "u1", 4)]), n_phone, p)
        p += 12 * n_phone
        sseq_size = struct.unpack_from(o + "i", raw, p)[0]
        if sseq_size != n_sseq * n_emit:
            raise ValueError("%s: %d senone ids for %d sequences of %d" % (path, sseq_size, n_sseq, n_emit))
        sseq = np.frombuffer(raw, o + "u2", sseq_size, p + 4).astype(np.uint16).reshape(n_sseq, n_emit)
        ssid, tmat = ent["ssid"].astype(np.int32), ent["tmat"].astype(np.int32)
        filler = ent["info"][:n_ci, 0].astype(np.uint8)
        # CD phones: info = {wpos, ctx[3]} with ctx[0] the base phone (bin_mdef.h:86-89)
        base = np.concatenate([np.arange(n_ci), ent["info"][n_ci:, 1].astype(np.int64)])
    else:
        lines = [l.strip() for l in raw.decode("latin-1").split("\n")]
        lines = [l for l in lines if l and not l.startswith("#")]
        if lines[0] != "0.3":
            raise ValueError("%s: text mdef version %s" % (path, lines[0]))
        cnt = {}
        for l in lines[1:7]:
            v, k = l.split()[:2]
            cnt[k] = int(v)
        n_ci, n_tri, n_sen, n_ci_sen, n_tmat = cnt["n_base"], cnt["n_tri"], cnt["n_tied_state"], cnt["n_tied_ci_state"], cnt["n_tied_tmat"]
        if n_tri != 0:
            raise NotImplementedError("%s: text mdef with triphones (bin_mdef_read_text reorders them); convert it to the binary form" % path)
        n_emit = cnt["n_state_map"] // n_ci - 1
        names, filler, tmat, seqs = [], [], [], []
        for l in lines[7:7 + n_ci]:
            t = l.split()
            if len(t) != 6 + n_emit + 1 or t[-1] != "N":
                raise ValueError("%s: bad phone line %r" % (path, l))
            names.append(t[0]); filler.append(1 if t[4] == "filler" else 0); tmat.append(int(t[5]))
            seqs.append(tuple(int(x) for x in t[6:6 + n_emit]))
        uniq = {}
        ssid = []
        for s in seqs:                                       # mdef.c sseq_compress: ids in order of first appearance
            ssid.append(uniq.setdefault(s, len(uniq)))
        sseq = np.array(list(uniq), np.uint16).reshape(len(uniq), n_emit)
        ssid, tmat, filler = np.array(ssid, np.int32), np.array(tmat, np.int32), np.array(filler, np.uint8)
        n_phone, base = n_ci, np.arange(n_ci)
        cd_tree = None
    if sseq.size and int(sseq.max()) >= n_sen:
        raise ValueError("%s: senone id out of range" % path)
    if (ssid < 0).any() or (ssid >= len(sseq)).any() or (tmat < 0).any() or (tmat >= n_tmat).any():
        raise ValueError("%s: phone table out of range" % path)
    sen2ci = np.full(n_sen, -1, np.int32)                     # the first phone (in id order) that uses a senone
    for i in range(n_phone - 1, -1, -1):
        sen2ci[sseq[ssid[i]]] = base[i]
    return dict(n_ciphone=n_ci, n_phone=n_phone, n_emit_state=n_emit, n_ci_sen=n_ci_sen, n_sen=n_sen, n_tmat=n_tmat,
                ciname=names, sseq=sseq, phone_ssid=ssid, phone_tmat=tmat, phone_filler=filler, sen2cimap=sen2ci,
                cd_tree=cd_tree, sil=names.index("SIL") if "SIL" in names else -1)


def read_feat_params(path):
    """feat.params: "-name value" pairs, as acmod_parse_args hands them to the configuration."""
    out = {}
    if not os.path.exists(path):
        return out
    tok = open(path).read().split()
    i = 0
    while i < len(tok):
        if tok[i].startswith("-") and i + 1 < len(tok):
            out[tok[i].lstrip("-")] = tok[i + 1]
            i += 2
        else:
            i += 1
    return out


def read_model_dir(path, **config):
    """An acoustic-model directory (mdef, means, variances, transition_matrices, sendump or
    mixture_weights, feat.params) -> the dict pocketsphinx_b200.model.PackedModel.from_dict takes, choosing
    the back-end as acmod_init_am does (acmod.c:62-130: PTM when there is one codebook per CI phone,
    semi-continuous for a single codebook, the generic multi-stream one otherwise) and applying the
    loaders' arithmetic (variance flooring + log-domain precompute, transition / mixture-weight
    quantisation).  config: overrides of the reference's settings (varfloor, tmatfloor, mixwfloor, topn,
    ds, aw, topn_beam, logbase)."""
    from .model import make_logadd8
    cfg = dict(varfloor="0.0001", tmatfloor="0.0001", mixwfloor="0.0000001", topn="4", ds="1", aw="1", topn_beam="0",
               logbase="1.0001")
    cfg.update(read_feat_params(os.path.join(path, "feat.params")))
    cfg.update({k: str(v) for k, v in config.items()})
    logbase = float(cfg["logbase"])
    md = read_mdef(os.path.join(path, "mdef"))
    tp = quantize_tmat(read_tmat(os.path.join(path, "transition_matrices")), float(cfg["tmatfloor"]), logbase)
    if tp.shape[0] < md["n_tmat"] or tp.shape[1] != md["n_emit_state"]:
        raise ValueError("%s: transition matrices %s do not fit the model definition" % (path, tp.shape))
    n_mgau, n_feat, n_density, featlen, mean = read_gauden(os.path.join(path, "means"))
    v = read_gauden(os.path.join(path, "variances"))
    if (v[0], v[1], v[2]) != (n_mgau, n_feat, n_density) or not np.array_equal(v[3], featlen):
        raise ValueError("%s: means and variances differ in shape" % path)
    var, det = precompute_gaussians(v[4], n_mgau, n_feat, n_density, featlen, float(cfg["varfloor"]), logbase)
    n_sen = md["n_sen"]
    sendump = os.path.join(path, "sendump")
    mixw_file = os.path.join(path, "mixture_weights")
    out = dict(n_sen=n_sen, n_mgau=n_mgau, n_feat=n_feat, n_density=n_density, topn=int(cfg["topn"]), featlen=featlen,
               mean=mean, var=var, det=det.ravel(), logadd8=make_logadd8(logbase), n_emit_state=md["n_emit_state"], tp=tp,
               sseq=md["sseq"], phone_ssid=md["phone_ssid"], phone_tmat=md["phone_tmat"], n_ciphone=md["n_ciphone"],
               n_ci_sen=md["n_ci_sen"], ds_ratio=int(cfg["ds"]), aw=int(cfg["aw"]), mixw_cb=np.zeros(0, np.uint8))
    if n_mgau == md["n_ciphone"] and n_mgau <= 256:
        kind = "ptm"
    elif n_mgau == 1:
        kind = "s2_semi"
    else:
        kind = "ms"
    out["kind"] = kind
    if kind in ("ptm", "s2_semi"):
        if not os.path.exists(sendump):
            raise NotImplementedError("%s: %s model without a sendump file (float mixture weights for this back-end are not read here)" % (path, kind))
        out["mixw"], out["mixw_cb"] = read_sendump(sendump, n_feat, n_density, n_sen)
        out["sen2cb"] = md["sen2cimap"].copy() if kind == "ptm" else np.zeros(n_sen, np.int32)
        if kind == "s2_semi":
            tb = [int(x) for x in cfg["topn_beam"].split(",") if x != ""][:n_feat]
            out["topn_beam"] = np.array(tb + [max(tb + [0])] * (n_feat - len(tb)), np.uint8)       # split_topn, s2_semi_mgau.c:1206
    else:
        w = read_mixw(mixw_file)
        if w.shape != (n_sen, n_feat, n_density):
            raise ValueError("%s: mixture weights %s do not fit the model" % (path, w.shape))
        pdf = quantize_mixw_ms(w, float(cfg["mixwfloor"]), logbase)                                 # [sen][feat][cw]
        out["mixw"] = pdf.transpose(1, 2, 0).copy() if n_mgau == 1 else pdf                        # ms_senone.c:224-262
        out["sen2cb"] = np.arange(n_sen, dtype=np.int32)                                            # ".cont." (ms_senone.c:313-325)
        if n_mgau != n_sen:
            raise NotImplementedError("%s: %d codebooks for %d senones needs a -senmgau map" % (path, n_mgau, n_sen))
        if out["topn"] == 0 or out["topn"] > n_density:                                             # ms_mgau.c:142-149
            out["topn"] = n_density
        out["logadd_ms"] = make_logadd8(logbase).astype(np.uint32)                                  # senone_init: shift 10 table
        out["logadd_ms_zero"] = -(1 << 31) >> 12
    return out
