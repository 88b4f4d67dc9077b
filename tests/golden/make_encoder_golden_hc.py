"""Writes tests/golden/encoder_golden_hc.json: size + SHA-256 of what OUR encoder emits at level 19 (the high-level tier, K-C1h; levels 16-22
give the same bytes), for tests/golden/dickens_96k.txt (40 000-byte frames, checksum on) and for a 256 KiB slice of the bench's class mix
(corpus.make_mix, 100 000-byte frames, no checksum) -- from the CPU emulation build of the sources (tests/emul), like make_encoder_golden.py.
tests/test_high_levels.py asserts that both builds reproduce these bytes.  Re-run after any intended change of the tier's output:
    python tests/golden/make_encoder_golden_hc.py"""
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

LEVELS = (19,)


def inputs():
    """name -> (data, frame size, checksum)"""
    d = np.frombuffer(open(os.path.join(HERE, "dickens_96k.txt"), "rb").read(), dtype=np.uint8)
    return {"dickens": (d, 40_000, True), "mix": (corpus.as_numpy(corpus.make_mix(256 << 10, seed=7)), 100_000, False)}


if __name__ == "__main__":
    ctx = make_ctx(_native.load(build_emul()))
    out = {}
    for name, (data, fs, ck) in inputs().items():
        for lvl in LEVELS:
            comp, cs, ds = ctx.compress_frames(data, fs, lvl, ck)
            out[f"{name}:{lvl}"] = {"size": int(comp.size), "sha256": hashlib.sha256(comp.tobytes()).hexdigest()}
    json.dump(out, open(os.path.join(HERE, "encoder_golden_hc.json"), "w"), indent=1)
    print(json.dumps(out, indent=1))
