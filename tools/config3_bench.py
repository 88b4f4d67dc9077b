"""GPU-box measurement of BASELINE configs[2]: 8 GiB of text (dickens.txt slices), 512 KiB frames (16 384 frames), archive
written by libzstd through the reference's Encoder sequence (level 3, checksums on -- the reference's defaults,
encode.rs:176-180), DECOMPRESS-ONLY on one H100, output compared bit for bit with the input and timed beside libzstd.
usage: python tools/config3_bench.py [GiB=8] > config3.json"""
import ctypes, json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import bench
from oracle import oracle as O
from zeekstd_b200 import corpus

FRAME = 512 << 10
gib = float(sys.argv[1]) if len(sys.argv) > 1 else 8.0
nb = int(gib * 2**30)
rig = bench.Rig(0)
lib, ctx, N, dev = rig.lib, rig.ctx, rig.N, rig.dev
ncores = os.cpu_count() or 1

PIECE = 1 << 30
x = torch.empty(nb, dtype=torch.uint8, device=dev)
arc, cs_all, ds_all = [], [], []
t_cpu_c = 0.0
for p0 in range(0, nb, PIECE):
    n = min(PIECE, nb - p0)
    x[p0:p0 + n] = corpus.make_text(n, seed=7 + p0 // PIECE, device=dev)
    host = x[p0:p0 + n].cpu().numpy()
    t0 = time.perf_counter()
    frames, cs, ds = O.ref_compress_frames(host, FRAME, 3, True, threads=ncores)
    t_cpu_c += time.perf_counter() - t0
    arc.append(np.frombuffer(b"".join(frames), dtype=np.uint8)); cs_all += cs; ds_all += ds
    if p0 == 0:
        first = (arc[0], list(cs), list(ds), host)
archive = np.concatenate(arc); del arc
k = len(cs_all)
co = np.zeros(k + 1, dtype=np.uint64); co[1:] = np.cumsum(np.asarray(cs_all, dtype=np.uint64))
do = np.zeros(k + 1, dtype=np.uint64); do[1:] = np.cumsum(np.asarray(ds_all, dtype=np.uint64))
assert int(do[-1]) == nb

# libzstd decompress beside it: all threads on the first GiB, one thread on its first 128 MiB
a0, cs0, ds0, host0 = first
c0 = np.zeros(len(cs0) + 1, dtype=np.uint64); c0[1:] = np.cumsum(cs0); d0 = np.zeros(len(ds0) + 1, dtype=np.uint64); d0[1:] = np.cumsum(ds0)
best_all = 1e9
for _ in range(3):
    t0 = time.perf_counter(); out, sizes = O.ref_decompress_frames(a0, c0, d0, threads=ncores); best_all = min(best_all, time.perf_counter() - t0)
assert np.array_equal(out, host0)
kk = (128 << 20) // FRAME
t0 = time.perf_counter(); O.ref_decompress_frames(a0[: int(c0[kk])], c0[: kk + 1], d0[: kk + 1], threads=1); one = time.perf_counter() - t0

# device-resident
d_arc = torch.from_numpy(archive).to(dev)
back = torch.zeros(nb + 64, dtype=torch.uint8, device=dev)
torch.cuda.synchronize()
ms = []
for it in range(6):
    rig.flush.fill_(1); torch.cuda.synchronize()
    rc = lib.zk_decompress_frames_dev(ctx._h, d_arc.data_ptr(), co.ctypes.data_as(N.u64p), do.ctypes.data_as(N.u64p), k, back.data_ptr(), 1, None, None)
    assert rc == 0, rc
    if it >= 3:
        ms.append(ctx.last_device_ms)
torch.cuda.synchronize()
exact = bool(torch.equal(back[:nb], x))
lib.zk_ctx_profile(ctx._h, 1)                      # per-kernel split from two extra passes (event pairs around every launch)
for it in range(2):
    rc = lib.zk_decompress_frames_dev(ctx._h, d_arc.data_ptr(), co.ctypes.data_as(N.u64p), do.ctypes.data_as(N.u64p), k, back.data_ptr(), 1, None, None)
    assert rc == 0, rc
kms = (ctypes.c_float * 8)(); kcnt = (ctypes.c_uint32 * 8)(); lib.zk_ctx_profile_read(ctx._h, kms, kcnt)
lib.zk_ctx_profile(ctx._h, 0)
del back

# host pointers (pinned): H2D of the archive and D2H of the 8 GiB inside the timed region
h_arc = torch.empty(archive.size, dtype=torch.uint8).pin_memory(); h_arc.copy_(torch.from_numpy(archive))
h_out = torch.empty(nb + 64, dtype=torch.uint8).pin_memory()
e2e = []
for it in range(4):
    t0 = time.perf_counter()
    rc = lib.zk_decompress_frames(ctx._h, h_arc.data_ptr(), co.ctypes.data_as(N.u64p), do.ctypes.data_as(N.u64p), k, h_out.data_ptr(), 1, None)
    assert rc == 0, rc
    if it:
        e2e.append(time.perf_counter() - t0)
exact_host = bool(torch.equal(h_out[:nb], x.cpu()))
g = nb / 2**30
print(json.dumps({
    "config": f"configs[2]: {g:g} GiB text (dickens.txt slices, {corpus.text_source()}), 512 KiB frames, libzstd level 3 + checksum archive, decompress only",
    "frames": k, "ratio": round(nb / archive.size, 4), "bit_exact_device": exact, "bit_exact_host": exact_host,
    "device_GiBps": round(g / (sum(ms) / len(ms) / 1e3), 2), "device_ms": [round(m, 2) for m in ms],
    "e2e_host_GiBps": round(g / (sum(e2e) / len(e2e)), 2), "e2e_s": [round(t, 4) for t in e2e],
    "kernel_ms_per_GiB": {bench.KERNEL_NAMES[i]: round(float(kms[i]) / 2 / g, 2) for i in range(8) if kcnt[i]},
    "libzstd_all_threads_GiBps": round(1.0 / best_all * (len(host0) / 2**30), 2), "libzstd_threads": ncores,
    "libzstd_one_thread_GiBps": round((128 / 1024) / one, 3),
    "libzstd_compress_all_threads_GiBps": round(g / t_cpu_c, 2)}), flush=True)
