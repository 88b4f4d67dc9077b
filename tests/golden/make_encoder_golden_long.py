"""Writes tests/golden/encoder_golden_long.json: size + SHA-256 of what OUR encoder emits in long mode (K-C1h with zk_ldm.inc's index of
the input) for a few (input, frame size, checksum, prefix) cases -- from the CPU emulation build of the sources (tests/emul), like
make_encoder_golden_ldm.py.  tests/test_long_mode.py asserts that both builds reproduce these bytes and takes its inputs from here.
Re-run after any intended change of the matcher's output:
    python tests/golden/make_encoder_golden_long.py"""
import hashlib
import importlib.util
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE))); sys.path.insert(0, os.path.dirname(HERE))
import numpy as np
from zeekstd_b200 import _native, corpus
from zeekstd_b200.build import build_emul
from util import make_ctx

_spec = importlib.util.spec_from_file_location("make_encoder_golden_ldm", os.path.join(HERE, "make_encoder_golden_ldm.py"))
_ldm = importlib.util.module_from_spec(_spec); _spec.loader.exec_module(_ldm)
edited_copy = _ldm.edited_copy


def mix(n: int, seed: int) -> np.ndarray:
    return corpus.as_numpy(corpus.make_mix(n, seed=seed, segment=16 << 10)).copy()


def skewed(n: int, seed: int) -> np.ndarray:
    """random bytes skewed towards zero bits: compressible, but nothing 64 bytes long repeats"""
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, n, dtype=np.uint8) & rng.integers(0, 256, n, dtype=np.uint8)


def far_repeats(n: int, seed: int) -> np.ndarray:
    """A (n bytes of the mix), B (n skewed random bytes), an edited copy of A, an edited copy of B: each copy 2n bytes after its original"""
    a, b = mix(n, seed), skewed(n, seed + 1)
    return np.concatenate([a, b, edited_copy(a, seed + 2, max(2, n >> 14)), edited_copy(b, seed + 3, max(2, n >> 14))])


def inputs():
    """name -> (input, frame size, checksum, prefix or None)"""
    d = np.frombuffer(open(os.path.join(HERE, "dickens.txt"), "rb").read(), dtype=np.uint8)
    rep = far_repeats(20 << 10, 5)
    return {"dickens": (d[:120_000], 120_000, True, None),
            "far_repeats": (rep, 50_000, False, None),
            "far_repeats_odd_frames": (rep, 32769, True, None),
            "prefix": (edited_copy(d[:60_000], 6, 5), 1 << 20, True, d[:50_000])}


if __name__ == "__main__":
    ctx = make_ctx(_native.load(build_emul()))
    out = {}
    for name, (x, fs, ck, prefix) in inputs().items():
        comp, cs, ds = ctx.compress_frames(x, fs, 19, ck, prefix=prefix, long_mode=True)
        out[name] = {"size": int(comp.size), "sha256": hashlib.sha256(comp.tobytes()).hexdigest()}
    json.dump(out, open(os.path.join(HERE, "encoder_golden_long.json"), "w"), indent=1)
    print(json.dumps(out, indent=1))
