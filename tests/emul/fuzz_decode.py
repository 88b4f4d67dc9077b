"""TEST INFRASTRUCTURE: mutation fuzzing of the DECODE kernels on the sanitized CPU emulation build (see asan_check.py for the
environment).  Seeds are libzstd-written frames of every corpus class at several levels; each case mutates one (bit flips, byte
stores, truncation, splices, length-field edits) and decodes it under three contexts -- default routing of segments,
CTAs only (ZK_EXEC_SHORT=0), single warps only (ZK_EXEC_SHORT=2^30) -- beside libzstd; seeds with a prefix decode in
prefix mode under all three:
  * libzstd restores the mutated frame  -> our output must be identical (checksum verification off on both sides when the
    mutation may have hit the checksum itself);
  * libzstd rejects it                  -> we must reject it too, with a zstd error code;
  * never an ASan/UBSan report, never a hang.
usage: python tests/emul/fuzz_decode.py [seconds=120] [seed=1]
"""
import os, sys, time
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE))); sys.path.insert(0, os.path.dirname(HERE))
import zeekstd_b200 as zk
from zeekstd_b200 import _native as N, corpus
from zeekstd_b200.build import build_emul
from oracle import oracle as O
from util import decode_frames

secs = float(sys.argv[1]) if len(sys.argv) > 1 else 120.0
rng = np.random.default_rng(int(sys.argv[2]) if len(sys.argv) > 2 else 1)
# ZK_FUZZ_LIB=product: the nvcc build on a real GPU (optionally under compute-sanitizer) instead of the emulation build
lib = N.load() if os.environ.get("ZK_FUZZ_LIB") == "product" else N.load(build_emul(sanitize=os.environ.get("ZK_FUZZ_SANITIZE", "1") == "1"))
ctxs = {"default": zk.Context(0, lib)}
for name, short in (("cta", "0"), ("warp_all", str(1 << 30))):
    os.environ["ZK_EXEC_SHORT"] = short; ctxs[name] = zk.Context(0, lib); del os.environ["ZK_EXEC_SHORT"]

kinds = ["text", "structured", "lowent", "random", "runs"]
seeds = []
for i in range(40):
    parts = []; left = int(rng.integers(200, 60_000))
    while left > 0:
        m = min(left, int(rng.integers(100, 40_000))); parts.append(corpus.make_class(kinds[rng.integers(5)], m, int(rng.integers(1 << 30))).numpy()); left -= m
    d = np.concatenate(parts)
    lvl = int(rng.choice([1, 3, 7, 19])); ck = bool(rng.integers(2))
    pfx = corpus.make_class("text", int(rng.integers(100, 30_000)), int(rng.integers(1 << 30))).numpy() if i % 4 == 3 else None
    if pfx is not None:
        d = np.concatenate([pfx[len(pfx) // 3:], d])[: len(d)]            # something to find in the prefix
    frames, cs, ds = O.ref_compress_frames(d, 1 << 30, lvl, ck, prefix=pfx)
    seeds.append((frames[0], len(d), d.tobytes(), pfx))


def mutate(b: bytes) -> bytes:
    a = bytearray(b)
    for _ in range(int(rng.choice([1, 1, 1, 2, 3, 8]))):
        k = int(rng.integers(7)); n = len(a)
        if n < 8: break
        p = int(rng.integers(n))
        if k == 0: a[p] ^= 1 << int(rng.integers(8))
        elif k == 1: a[p] = int(rng.integers(256))
        elif k == 2: a[p] = int(rng.choice([0, 1, 0x7F, 0x80, 0xFF]))
        elif k == 3: del a[p: p + int(rng.integers(1, 9))]
        elif k == 4: a[p:p] = bytes(rng.integers(0, 256, int(rng.integers(1, 9)), dtype=np.uint8))
        elif k == 5:
            q = int(rng.integers(n)); ln = int(rng.integers(1, 64)); a[p: p + ln] = a[q: q + ln]
        else: a = a[: max(5, p)]
    # bias towards the headers: the first 24 bytes and block headers decide the structure
    if rng.integers(3) == 0 and len(a) > 24:
        a[int(rng.integers(4, 24))] ^= 1 << int(rng.integers(8))
    return bytes(a)


t0 = time.time(); cases_run = agree_ok = agree_err = stricter = 0
while time.time() - t0 < secs:
    frame, dlen, plain, pfx = seeds[int(rng.integers(len(seeds)))]
    bad = mutate(frame)
    cap = dlen
    ref_out, ref_sizes = O.ref_decompress_frames(np.frombuffer(bad, dtype=np.uint8) if bad else np.zeros(0, np.uint8), [0, len(bad)], [0, cap], prefix=pfx)
    ref_ok = ref_sizes[0] >= 0
    for name in ctxs:
        ctx = ctxs[name]
        comp = np.frombuffer(bad, dtype=np.uint8)
        out, st, rc = ctx.decompress_frames(comp, np.array([0, len(bad)], dtype=np.uint64), np.array([0, cap], dtype=np.uint64), True, prefix=pfx)
        strict = False
        if ref_ok and ref_sizes[0] == cap and rc == -20:
            # libzstd 1.5.5's fast 4-stream Huffman path (table log 11) does not check that a stream is consumed exactly
            # (huf_decompress.c, "finish bit streams one by one"); its portable path, the format specification (RFC 8878 4.2.2:
            # "the bitstream must be fully consumed"), the C restatement and these kernels do.  Tolerated when the restatement agrees.
            try:
                O.oracle_decompress_ex(comp, cap, prefix=pfx)
            except O.ZstdError as e:
                strict = e.code == 20
        if strict:
            stricter += 1
            continue
        fail = (ref_ok and ref_sizes[0] == cap and (rc != 0 or bytes(out[:cap]) != bytes(ref_out[:cap]))) or (not ref_ok and not (rc != 0 and zk.Error(rc, lib).is_zstd()))
        if fail:
            import pickle
            pickle.dump({"bad": bad, "good": frame, "cap": cap, "pfx": None if pfx is None else pfx.tobytes(), "ctx": name, "rc": rc, "ref": ref_sizes[0]}, open(os.environ.get("ZK_FUZZ_DUMP", "/tmp/fuzz_fail.pkl"), "wb"))
        if ref_ok and ref_sizes[0] == cap:
            assert rc == 0, (name, "libzstd restores this frame, we fail", rc, bad.hex()[:200], len(bad))
            assert bytes(out[:cap]) == bytes(ref_out[:cap]), (name, "output differs", len(bad))
        elif not ref_ok:
            assert rc != 0 and zk.Error(rc, lib).is_zstd(), (name, "libzstd rejects this frame", ref_sizes[0], rc, bad.hex()[:200], len(bad))
        # (a frame that ends early -- fewer bytes than its seek-table entry promises -- is an error of the ARCHIVE, not of zstd:
        #  the reference's Decoder would run into the next frame; here the entry fails or succeeds, but never crashes)
    cases_run += 1; agree_ok += ref_ok; agree_err += not ref_ok
print(f"fuzz clean: {cases_run} mutated frames ({agree_ok} still valid, {agree_err} rejected by both; {stricter} decodes stricter than libzstd 1.5.5 on an inexact Huffman stream end), contexts {list(ctxs)}")
