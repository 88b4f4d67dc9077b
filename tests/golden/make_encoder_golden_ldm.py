"""Writes tests/golden/encoder_golden_ldm.json: size + SHA-256 of what OUR encoder emits with long-distance matching on (patch mode, K-C1h
with zk_ldm.inc) for a few (OLD, NEW, frame size) cases: OLD is a slice of tests/golden/dickens.txt or of the bench's class mix, NEW its
edited copy (edited_copy below) -- from the CPU emulation build of the sources (tests/emul), like make_encoder_golden_hc.py.
tests/test_patch_ldm.py asserts that both builds reproduce these bytes.  Re-run after any intended change of the matcher's output:
    python tests/golden/make_encoder_golden_ldm.py"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE))); sys.path.insert(0, os.path.dirname(HERE))
import numpy as np
from zeekstd_b200 import _native, corpus
from zeekstd_b200.build import build_emul
from util import make_ctx


def edited_copy(old: np.ndarray, seed: int, edits: int, span: int = 48) -> np.ndarray:
    """NEW from OLD: `edits` seeded insertions, deletions and overwritten spans of 1..span bytes, and one region of 1/16 of the input
    moved elsewhere, so that content shifts by amounts that are multiples of nothing"""
    rng = np.random.default_rng(seed)
    b = bytearray(old.tobytes())
    for k in range(edits):
        p = int(rng.integers(0, max(1, len(b) - span)))
        m = int(rng.integers(1, span + 1))
        fresh = rng.integers(0, 256, m, dtype=np.uint8).tobytes()
        if k % 3 == 0:
            b[p:p] = fresh
        elif k % 3 == 1:
            del b[p:p + m]
        else:
            b[p:p + m] = fresh
    m = len(b) // 16
    if m:
        p = int(rng.integers(0, len(b) - m)); region = bytes(b[p:p + m]); del b[p:p + m]
        q = int(rng.integers(0, len(b))); b[q:q] = region
    return np.frombuffer(bytes(b), dtype=np.uint8)


def inputs():
    """name -> (OLD, NEW, frame size, checksum)"""
    d = np.frombuffer(open(os.path.join(HERE, "dickens.txt"), "rb").read(), dtype=np.uint8)
    mix = corpus.as_numpy(corpus.make_mix(160 << 10, seed=7, segment=16 << 10))
    return {"dickens": (d[:150_000], edited_copy(d[:150_000], 1, 9), 40_000, True),
            "mix": (mix, edited_copy(mix, 2, 12), 100_000, False),
            "mix_short_prefix": (mix[:50], mix[:70_000], 1 << 20, True)}


if __name__ == "__main__":
    ctx = make_ctx(_native.load(build_emul()))
    out = {}
    for name, (old, new, fs, ck) in inputs().items():
        comp, cs, ds = ctx.compress_frames(new, fs, 19, ck, prefix=old, long_distance=True)
        out[name] = {"size": int(comp.size), "sha256": hashlib.sha256(comp.tobytes()).hexdigest()}
    json.dump(out, open(os.path.join(HERE, "encoder_golden_ldm.json"), "w"), indent=1)
    print(json.dumps(out, indent=1))
