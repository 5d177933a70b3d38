"""The compiled reference's front end recorded in tests/golden/fe_reference.npz -- TEST INFRASTRUCTURE ONLY.

`python -m oracle.make_golden fe` runs oracle/_ref/libpsref.so on the inputs defined here (slices of its test
utterance goforward.raw and seeded noise) and stores fe_desc / mfcc / featurize_fresh; Recorded replays them for
the front-end tests, which so run where the reference is not built.
"""
import hashlib
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "fe_reference.npz")

# reference options on top of the en-us model's feat.params
PORT_CONFIGS = [dict(), dict(transform="legacy", remove_noise="no", lifter="0"), dict(transform="htk", remove_dc="yes"),
                dict(cmn="none")]


def config_name(kv):
    return ",".join("%s=%s" % (k, kv[k]) for k in sorted(kv)) or "default"


def pcm_key(pcm):
    return hashlib.sha1(np.ascontiguousarray(pcm, np.int16).tobytes()).hexdigest()[:16]


def port_inputs(go):
    rng = np.random.default_rng(3)
    noise = np.clip(rng.normal(0, 3000, 5000), -32768, 32767).astype(np.int16)
    return [go[:6000], go[20000:23000], noise, go[:411], go[:100], np.zeros(1500, np.int16)]


def frame_count_inputs():
    return [np.zeros(n, np.int16) for n in (0, 1, 100, 409, 410, 411, 569, 570, 571, 2000)]


def cases(go):
    """(configuration, mfcc inputs, featurize_fresh inputs) for every configuration the tests replay."""
    return [(kv, port_inputs(go) + (frame_count_inputs() if not kv else []), port_inputs(go)) for kv in PORT_CONFIGS]


_store = None


def _load():
    global _store
    if _store is None:
        from pocketsphinx_b200.model import load_npz
        _store = load_npz(GOLDEN)
    return _store


def goforward():
    """The reference's test utterance (test/data/goforward.raw), int16 PCM."""
    return _load()["goforward"]


class Recorded:
    """fe_desc / mfcc / featurize_fresh of the reference in configuration `kv`, for the recorded inputs."""

    def __init__(self, **kv):
        self.name = config_name(kv)
        self.g = _load()
        if "desc.%s.n_cep" % self.name not in self.g:
            raise KeyError("configuration %s not recorded in %s" % (self.name, GOLDEN))

    def fe_desc(self):
        p = "desc.%s." % self.name
        d = {}
        for k, v in self.g.items():
            if k.startswith(p):
                key = k[len(p):]
                d[key] = v if v.ndim else (v.dtype.type(v) if v.dtype == np.float32 else v.item())
        return d

    def _get(self, what, pcm):
        k = "%s.%s.%s" % (what, self.name, pcm_key(pcm))
        if k not in self.g:
            raise KeyError("%s of this input (%d samples) not recorded for %s" % (what, len(pcm), self.name))
        return self.g[k]

    def mfcc(self, pcm):
        return self._get("mfcc", pcm)

    def featurize_fresh(self, pcm):
        return self._get("feat", pcm)

    def close(self):
        pass
