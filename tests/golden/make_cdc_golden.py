"""Writes tests/golden/cdc_golden.json: frame sizes, size and SHA-256 of what OUR encoder emits with content-defined frames
(FrameSizePolicy::ContentDefined, zk_compress_frames_cdc) for a few (input, s, level) cases, from the CPU emulation build of the sources
(tests/emul), like make_encoder_golden_ldm.py.  tests/test_content_frames.py asserts that both builds reproduce these bytes.  Re-run after
any intended change of the cut or of the encoder's output:
    python tests/golden/make_cdc_golden.py"""
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


def inputs():
    """name -> (input, s, level, checksum)"""
    d = np.frombuffer(open(os.path.join(HERE, "dickens.txt"), "rb").read(), dtype=np.uint8)
    mix = corpus.as_numpy(corpus.make_mix(200 << 10, seed=11, segment=16 << 10))
    return {"dickens_s4096_l3": (d[:150_000], 4096, 3, True),
            "mix_s16k_l1": (mix, 16 << 10, 1, False),
            "mix_s5000_l-3": (mix[:90_000], 5000, -3, True),
            "dickens_s8192_l19": (d[:60_000], 8192, 19, False)}


if __name__ == "__main__":
    ctx = make_ctx(_native.load(build_emul()))
    out = {}
    for name, (x, s, level, ck) in inputs().items():
        comp, cs, ds, used = ctx.compress_frames_cdc(x, s, level, ck)
        out[name] = {"d_sizes": [int(v) for v in ds], "size": int(comp.size), "sha256": hashlib.sha256(comp.tobytes()).hexdigest()}
    json.dump(out, open(os.path.join(HERE, "cdc_golden.json"), "w"), indent=1)
    print(json.dumps(out, indent=1))
