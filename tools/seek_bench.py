"""BASELINE config 5 on the GPU box: random 64 KiB reads from a seekable archive written by the reference path (libzstd)."""
import json, os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zeekstd_b200 as zk
from zeekstd_b200 import corpus, seek
from oracle import oracle as O
ctx = zk.Context(0)
n = int(os.environ.get("ZK_SEEK_BYTES", str(4 << 30))); FS = 2 << 20; R = 65536
x = corpus.make_mix(n, seed=20260924, device="cuda").cpu().numpy()
a, st = O.ref_seekable_archive(x, FS, 1, False, threads=os.cpu_count())
arch_t = torch.frombuffer(bytearray(a + b"\0" * 64), dtype=torch.uint8).pin_memory(); arch = arch_t.numpy()
scratch_t = torch.empty((1 << 30) + (4 << 20), dtype=torch.uint8).pin_memory(); scratch = scratch_t.numpy()
rng = np.random.default_rng(7)
offs = rng.integers(0, n - R, 10_000)
# (1) one read at a time through the Decoder API (latency)
dec = zk.Decoder(zk.DecodeOptions(a))
lat = []
k1 = int(os.environ.get("ZK_SEEK_SINGLE", "300"))
for o in offs[:k1]:
    t = time.perf_counter(); dec.set_offset(int(o)); dec.set_offset_limit(int(o) + R); got = dec.read_all(); lat.append(time.perf_counter() - t)
    assert got == x[o:o + R].tobytes()
    dec.set_offset_limit(n)
lat = np.array(lat) * 1e3
# (2) all 10k reads batched
t = time.perf_counter(); seek.read_ranges(ctx, arch, np.array(st.c), np.array(st.d), offs[:64], R, scratch=scratch)   # warm-up
t = time.perf_counter(); outs, nfr = seek.read_ranges(ctx, arch, np.array(st.c), np.array(st.d), offs, R, scratch=scratch); tb = time.perf_counter() - t
assert all(outs[i] == x[offs[i]:offs[i] + R].tobytes() for i in range(0, len(offs), 97))
# bytes that had to be decoded: per touched frame, up to the end of the furthest read in it
ends = {}
for o in offs:
    o = int(o); f_lo, f_hi = o // FS, (o + R - 1) // FS
    for f in range(f_lo, f_hi):
        ends[f] = FS
    ends[f_hi] = max(ends.get(f_hi, 0), o + R - f_hi * FS)
needed = sum(ends.values())
# reference: libzstd, one thread, decode from the frame start to the end of the read (what Decoder does, decode.rs:228-266)
import ctypes
tl = []
for o in offs[:200]:
    f = st.frame_index_decomp(int(o)); t = time.perf_counter()
    fr = a[st.c[f]: st.c[f + 2] if f + 2 < len(st.c) else st.c[-1]]
    out = O.ref_decompress_any(fr, 2 * FS + 1); tl.append(time.perf_counter() - t)
tl = np.array(tl) * 1e3
res = dict(archive_bytes=len(a), frames=st.num_frames(), reads=len(offs), read_bytes=R,
           single_read_ms=dict(p50=round(float(np.percentile(lat, 50)), 3), p99=round(float(np.percentile(lat, 99)), 3), n=k1),
           batched=dict(seconds=round(tb, 3), returned_GiBps=round(len(offs) * R / 2**30 / tb, 2), frames_decoded=nfr,
                        needed_GiB=round(needed / 2**30, 3), decoded_needed_GiBps=round(needed / 2**30 / tb, 2),
                        note="every touched frame is decoded once and only as far as the last byte some read wants of it"),
           reference_cpu_single_read_ms=dict(p50=round(float(np.percentile(tl, 50)), 3), p99=round(float(np.percentile(tl, 99)), 3), note="libzstd 1 thread, whole frame(s) decoded"))
print(json.dumps(res), flush=True)
os.makedirs("tools_out", exist_ok=True); json.dump(res, open("tools_out/seek.json", "w"), indent=1)
