"""TEST INFRASTRUCTURE: the front-end shapes beyond the en-us default (16 kHz, 410-sample frames, 160-sample shift,
512-point FFT, 13 cepstra), shared by tests/test_fe_port_shapes.py (CPU: oracle/fe_port.py against the compiled
reference) and tests/test_gpu_fe_shapes.py (the device against both).

Each entry of GRID is one configuration: the reference's settings on top of a model's feat.params (`kv`, strings as
on its command line), the same settings for fe_tables.make_fe_desc (`mk`), and the frame size / shift / FFT size
they give.  Entries with `ncep` run on a synthetic continuous model whose feature length is 3 * ncep (the reference's
acmod_init refuses a -ncep that does not match the model), written to a temporary directory at test time."""
import os

import numpy as np

from oracle import refdrv

REF = os.path.dirname(refdrv.LIB_PATH)
EN_US = os.path.join(REF, "model", "en-us")

# model/en-us/en-us/feat.params without -svspec / -model, which name the en-us model's own streams
EN_US_FEAT_PARAMS = ("-lowerf 130\n-upperf 6800\n-nfilt 25\n-transform dct\n-lifter 22\n-feat 1s_c_d_dd\n-agc none\n"
                     "-cmn batch\n-varnorm no\n-remove_noise yes\n")


def _e(name, shape, kv=None, mk=None, ncep=None):
    kv = dict(kv or {})
    mk = dict(mk or {})
    if ncep is not None:
        kv.update(ncep=str(ncep), ceplen=str(ncep))
        mk.update(ncep=ncep)
    return dict(id=name, shape=shape, kv=kv, mk=mk, ncep=ncep)


GRID = [
    _e("8k", (205, 80, 256), dict(samprate="8000", upperf="3500"), dict(samprate=8000, upperf=3500)),
    _e("8k_nfft512", (205, 80, 512), dict(samprate="8000", upperf="3500", nfft="512"),
       dict(samprate=8000, upperf=3500, nfft=512)),
    _e("11k", (283, 110, 512), dict(samprate="11025", upperf="5000"), dict(samprate=11025, upperf=5000)),
    _e("22k", (565, 221, 1024), dict(samprate="22050"), dict(samprate=22050)),
    _e("32k_dc", (820, 320, 1024), dict(samprate="32000", remove_dc="yes"), dict(samprate=32000, remove_dc=True)),
    _e("nfft1024", (410, 160, 1024), dict(nfft="1024"), dict(nfft=1024)),
    _e("frate200", (410, 80, 512), dict(frate="200"), dict(frate=200)),
    _e("frate50", (800, 320, 1024), dict(frate="50", wlen="0.05"), dict(frate=50, wlen=0.05)),
    _e("short_win", (160, 100, 256), dict(wlen="0.01", nfft="256", frate="160"), dict(wlen=0.01, nfft=256, frate=160)),
    _e("alpha0", (410, 160, 512), dict(alpha="0"), dict(alpha=0.0)),
    _e("nfilt64", (410, 160, 512), dict(nfilt="64"), dict(nfilt=64)),
    _e("nfilt64_legacy", (410, 160, 512), dict(nfilt="64", transform="legacy", remove_noise="no"),
       dict(nfilt=64, transform="legacy", remove_noise=False)),
    _e("ncep1", (410, 160, 512), ncep=1),
    _e("ncep20", (410, 160, 512), ncep=20),
    _e("ncep32", (410, 160, 512), dict(nfilt="40"), dict(nfilt=40), ncep=32),
]
BY_ID = {e["id"]: e for e in GRID}


def model_dir(entry, tmp):
    """The model directory of a grid entry: en-us, or a synthetic continuous model with 3 * ncep-dimensional
    features written under tmp (a directory path) once."""
    if entry["ncep"] is None:
        return EN_US
    from pocketsphinx_b200 import s3io
    from pocketsphinx_b200.model import synth_ms
    d = os.path.join(str(tmp), "ncep%d" % entry["ncep"])
    if not os.path.exists(os.path.join(d, "feat.params")):
        pm, raw = synth_ms(seed=entry["ncep"], n_sen=40, n_density=2, featlens=(3 * entry["ncep"],), topn=2, return_raw=True)
        sen2ci = np.concatenate([np.repeat(np.arange(10), 3), np.arange(pm.n_sen - 30) % 10]).astype(np.int32)
        s3io.write_model_dir(d, kind=pm.kind, n_mgau=pm.n_mgau, n_feat=pm.n_feat, n_density=pm.n_density,
                             featlen=pm.featlen, mean=raw["mean"], var_raw=raw["var_raw"], tp_float=raw["tp_float"],
                             sen2ci=sen2ci, n_ci=10, n_emit=3, n_ci_sen=30, mixw_float=raw.get("mixw_float"),
                             mixw_q=raw.get("mixw_q"), mixw_cb=raw.get("mixw_cb"), feat_params=EN_US_FEAT_PARAMS)
    return d


def ref_model(entry, tmp, **extra):
    """refdrv.RefModel of a grid entry (extra: more reference settings, strings)."""
    kv = dict(entry["kv"], **extra)
    if entry["ncep"] is not None:
        kv.update(senmgau=".cont.", topn="2")
    return refdrv.RefModel(model_dir(entry, tmp), **kv)


def goforward():
    from oracle import fe_golden
    return fe_golden.goforward()


def boundary_lengths(frame_size, frame_shift):
    """Lengths around the first frame boundaries of a shape: no sample, one, one frame +- 1, two frames +- 1."""
    fs, sh = frame_size, frame_shift
    return [0, 1, fs - 1, fs, fs + 1, fs + sh - 1, fs + sh, fs + sh + 1]


def utterances(entry):
    """The inputs of a grid entry: goforward slices at the boundary lengths, a few thousand samples of goforward
    and of seeded noise (loud enough to clip now and then), and silence (every mel energy at the log floor)."""
    fs, sh, _ = entry["shape"]
    go = goforward()
    rng = np.random.default_rng(sum(map(ord, entry["id"])))
    noise = np.clip(rng.normal(0, 6000, 3000), -32768, 32767).astype(np.int16)
    utts = [go[7000:7000 + n] for n in boundary_lengths(fs, sh)]
    return utts + [go[12000:16000], noise, np.zeros(fs + 3 * sh, np.int16)]
