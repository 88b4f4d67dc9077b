"""Ad-hoc GPU check (run on a GPU machine): compress on the GPU, verify with libzstd + our GPU decoder, rough timing."""
import ctypes, json, os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle as O
from zeekstd_b200 import corpus, _native as N
lib = N.load(require_all=False)
ctx = ctypes.c_void_p(); assert lib.zk_ctx_create(0, 0, ctypes.byref(ctx)) == 0
print(lib.zk_version(), torch.cuda.get_device_name(0), flush=True)

def run(name, x_dev, fs, lvl, ck, reps=3, verify_cpu=True):
    n = x_dev.numel()
    src = torch.cat([x_dev, torch.zeros(64, dtype=torch.uint8, device="cuda")])
    cap = lib.zk_compress_bound(n, fs)
    dst = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    nfmax = n // fs + 2
    cs = np.zeros(nfmax, dtype=np.uint32); ds = np.zeros(nfmax, dtype=np.uint32)
    nf = ctypes.c_uint32(); dl = ctypes.c_size_t()
    best = 1e9
    for r in range(reps):
        rc = lib.zk_compress_frames_dev(ctx, src.data_ptr(), n, fs, lvl, ck, dst.data_ptr(), cap, cs.ctypes.data_as(N.u32p),
                                        ds.ctypes.data_as(N.u32p), nfmax, ctypes.byref(nf), ctypes.byref(dl), None)
        assert rc == 0, rc
        best = min(best, lib.zk_ctx_last_device_ms(ctx))
    nfr = nf.value; clen = dl.value
    x = x_dev.cpu().numpy()
    comp = dst[:clen].cpu().numpy()
    co = np.zeros(nfr + 1, dtype=np.uint64); co[1:] = np.cumsum(cs[:nfr]); do = np.zeros(nfr + 1, dtype=np.uint64); do[1:] = np.cumsum(ds[:nfr])
    ok_cpu = None
    if verify_cpu:
        out, sizes = O.ref_decompress_frames(comp, co, do, threads=os.cpu_count())
        ok_cpu = bool((out == x).all()) and all(s == d for s, d in zip(sizes, ds[:nfr]))
    # our own decoder
    d_out = torch.zeros(n + 64, dtype=torch.uint8, device="cuda"); st = np.zeros(nfr, dtype=np.int32)
    rc = lib.zk_decompress_frames_dev(ctx, dst.data_ptr(), co.ctypes.data_as(N.u64p), do.ctypes.data_as(N.u64p), nfr, d_out.data_ptr(), ck, st.ctypes.data_as(N.i32p), None)
    dec_ms = lib.zk_ctx_last_device_ms(ctx)
    ok_gpu = rc == 0 and bool(torch.equal(d_out[:n], x_dev))
    ref_c = None
    if n <= (256 << 20):
        _, rcs, _ = O.ref_compress_frames(x, fs, lvl, bool(ck), threads=os.cpu_count()); ref_c = sum(rcs)
    res = dict(name=name, bytes=n, frames=nfr, level=lvl, ck=ck, ratio=round(n / clen, 3), libzstd_ratio=round(n / ref_c, 3) if ref_c else None,
               ok_libzstd=ok_cpu, ok_gpu_dec=ok_gpu, comp_ms=round(best, 3), comp_GiBps=round(n / 2**30 / (best / 1e3), 2), dec_ms=round(dec_ms, 3),
               dec_GiBps=round(n / 2**30 / (dec_ms / 1e3), 2))
    print(json.dumps(res), flush=True)
    return res

out = []
for kind in ["text", "structured", "lowent", "random", "runs"]:
    out.append(run(kind + "-8M", corpus.make_class(kind, 8 << 20, 3, device="cuda"), 1 << 20, 3, 1))
out.append(run("empty", torch.zeros(0, dtype=torch.uint8, device="cuda"), 1 << 20, 3, 1))
out.append(run("mix-256M-2M-L1", corpus.make_mix(256 << 20, device="cuda"), 2 << 20, 1, 0))
out.append(run("mix-256M-2M-L3ck", corpus.make_mix(256 << 20, device="cuda"), 2 << 20, 3, 1))
if os.environ.get("ZK_CHECK_BIG"):
    out.append(run("mix-1G-2M-L1", corpus.make_mix(1 << 30, device="cuda"), 2 << 20, 1, 0, verify_cpu=True))
os.makedirs("tools_out", exist_ok=True)
json.dump(out, open("tools_out/check_encode.json", "w"), indent=1)
