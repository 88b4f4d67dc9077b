"""Ad-hoc GPU check (run on a GPU machine): parity + rough timing of the device-resident decode path."""
import ctypes, json, os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle as O
from zeekstd_b200 import corpus, _native as N

lib = N.load(require_all=False)
ctx = ctypes.c_void_p()
rc = lib.zk_ctx_create(0, 0, ctypes.byref(ctx)); assert rc == 0, rc
print(lib.zk_version(), torch.cuda.get_device_name(0), "cpus", os.cpu_count(), flush=True)

def run(name, x, fs, lvl, ck, reps=5):
    t0 = time.time()
    frames, cs, ds = O.ref_compress_frames(x, fs, lvl, ck, threads=os.cpu_count())
    t_c = time.time() - t0
    n = len(frames)
    comp = np.frombuffer(b"".join(frames) + b"\0" * 64, dtype=np.uint8)
    co = np.zeros(n + 1, dtype=np.uint64); co[1:] = np.cumsum(cs)
    do = np.zeros(n + 1, dtype=np.uint64); do[1:] = np.cumsum(ds)
    d_comp = torch.from_numpy(comp.copy()).cuda()
    d_out = torch.zeros(int(do[-1]) + 64, dtype=torch.uint8, device="cuda")
    st = np.zeros(n, dtype=np.int32)
    best = 1e9
    for r in range(reps):
        d_out.zero_(); torch.cuda.synchronize()
        rc = lib.zk_decompress_frames_dev(ctx, d_comp.data_ptr(), co.ctypes.data_as(N.u64p), do.ctypes.data_as(N.u64p), n,
                                          d_out.data_ptr(), 1 if ck else 0, st.ctypes.data_as(N.i32p), None)
        ms = lib.zk_ctx_last_device_ms(ctx)
        best = min(best, ms)
    ok = bool((d_out[: x.size].cpu().numpy() == x).all())
    res = dict(name=name, bytes=int(x.size), frames=n, level=lvl, checksum=ck, ratio=round(x.size / sum(cs), 3), rc=rc, ok=ok,
               bad=int((st != 0).sum()), best_ms=round(best, 3), GiBps=round(x.size / 2**30 / (best / 1e3), 2), cpu_compress_s=round(t_c, 2))
    print(json.dumps(res), flush=True)
    return res

out = []
sz = int(os.environ.get("ZK_CHECK_MB", "256")) << 20
for kind in ["text", "structured", "lowent", "random", "runs"]:
    out.append(run(kind + "-small", corpus.make_class(kind, 3 << 20, 3).numpy(), 1 << 20, 1, True, reps=2))
mix = corpus.make_mix(sz, device="cuda").cpu().numpy()
out.append(run("mix-2M-L1", mix, 2 << 20, 1, False))
out.append(run("mix-2M-L3ck", mix, 2 << 20, 3, True))
if os.environ.get("ZK_CHECK_BIG"):
    big = corpus.make_mix(1 << 30, device="cuda").cpu().numpy()
    out.append(run("mix-1GiB-2M-L1", big, 2 << 20, 1, False, reps=3))
    out.append(run("mix-1GiB-512K-L1", big, 512 << 10, 1, False, reps=3))
    del big
txt = corpus.make_text(sz, device="cuda").cpu().numpy()
out.append(run("text-2M-L1", txt, 2 << 20, 1, False))
out.append(run("text-512K-L1", txt, 512 << 10, 1, False))
os.makedirs("tools_out", exist_ok=True)
json.dump(out, open("tools_out/check_decode.json", "w"), indent=1)
