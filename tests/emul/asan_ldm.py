"""TEST INFRASTRUCTURE: long-distance matching (patch mode, zk_ldm.inc) on the CPU emulation build compiled with
-fsanitize=address,undefined, the way asan_check.py drives the rest of the kernels: fixed edge cases, then random
(prefix, edited copy, frame size) cases with the switch on; libzstd (refPrefix) and the decode kernels must restore every frame.

  ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0 \\
  LD_PRELOAD=/usr/lib/x86_64-linux-gnu/libasan.so.8:/usr/lib/x86_64-linux-gnu/libubsan.so.1 \\
  CXX=/usr/bin/g++ python tests/emul/asan_ldm.py [seconds of random cases]
"""
import importlib.util, os, sys, time
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE))); sys.path.insert(0, os.path.dirname(HERE))
import zeekstd_b200 as zk
from zeekstd_b200 import _native as N, corpus
from zeekstd_b200.build import build_emul
from oracle import oracle as O
from util import offsets

spec = importlib.util.spec_from_file_location("mk", os.path.join(os.path.dirname(HERE), "golden", "make_encoder_golden_ldm.py"))
mk = importlib.util.module_from_spec(spec); spec.loader.exec_module(mk)
lib = N.load(build_emul(sanitize=True)); ctx = zk.Context(0, lib)


def check(new, fs, pf, ck=True):
    comp, cs, ds = ctx.compress_frames(new, fs, 3, ck, prefix=pf, long_distance=True)
    pad = np.concatenate([comp, np.zeros(64, np.uint8)])
    out, sizes = O.ref_decompress_frames(pad, offsets(cs), offsets(ds), prefix=pf)
    assert list(sizes) == [int(d) for d in ds] and out.tobytes() == new.tobytes(), ("libzstd does not restore", new.size, fs, pf.size)
    back, st, rc = ctx.decompress_frames(pad, offsets(cs), offsets(ds), True, prefix=pf)
    assert rc == 0 and back[: new.size].tobytes() == new.tobytes(), ("own decode", rc, new.size, fs, pf.size)


x = corpus.make_class("text", 70_000, 9).numpy()
old = corpus.make_mix(100_000, seed=4, segment=16 << 10).numpy()
new = np.concatenate([old[:40_000], x[:333], old[39_000:], old[:5]])          # a shifted middle, a match that ends with the prefix
for fs, pf in ((30_000, old), (1, old[:400]), (1 << 20, old[:63]), (1 << 20, old[:64]), (1 << 20, old[:5000]), (32_769, old[-70:])):
    check(new[:300] if fs == 1 else new, fs, pf)
z = np.full(50_000, 7, np.uint8)
check(z, 1 << 20, z)                                                          # every position hashes alike
kinds = ["text", "structured", "lowent", "random", "runs"]
rng = np.random.default_rng(5)
t0 = time.time(); it = 0
while time.time() - t0 < (float(sys.argv[1]) if len(sys.argv) > 1 else 30):
    pf = corpus.make_class(kinds[rng.integers(5)], int(rng.integers(1, 120_000)), int(rng.integers(1 << 30))).numpy()
    d = mk.edited_copy(pf, int(rng.integers(1 << 30)), int(rng.integers(0, 12)))[: int(rng.integers(1, 150_000))]
    check(d, int(rng.choice([100, 4096, 32767, 32768, 32769, 100_000, 1 << 20])), pf, bool(rng.integers(2))); it += 1
print("asan/ubsan clean with long-distance matching;", it, "random cases")
