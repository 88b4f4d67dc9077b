"""Profile target (run under a profiler on a GPU machine): one warm-up + N timed device-resident decodes of a text/mix batch."""
import ctypes, os, sys, json
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle as O
from zeekstd_b200 import corpus, _native as N
lib = N.load(require_all=False)
ctx = ctypes.c_void_p(); assert lib.zk_ctx_create(0, 0, ctypes.byref(ctx)) == 0
kind = os.environ.get("ZK_PROF_KIND", "mix"); mb = int(os.environ.get("ZK_PROF_MB", "256")); fs = int(os.environ.get("ZK_PROF_FS", str(2 << 20)))
lvl = int(os.environ.get("ZK_PROF_LEVEL", "1")); reps = int(os.environ.get("ZK_PROF_REPS", "2"))
x = (corpus.make_mix(mb << 20, device="cuda") if kind == "mix" else corpus.make_class(kind, mb << 20, 7, device="cuda")).cpu().numpy()
frames, cs, ds = O.ref_compress_frames(x, fs, lvl, False, threads=os.cpu_count())
n = len(frames)
comp = np.frombuffer(b"".join(frames) + b"\0" * 64, dtype=np.uint8)
co = np.zeros(n + 1, dtype=np.uint64); co[1:] = np.cumsum(cs)
do = np.zeros(n + 1, dtype=np.uint64); do[1:] = np.cumsum(ds)
d_comp = torch.from_numpy(comp.copy()).cuda(); d_out = torch.zeros(int(do[-1]) + 64, dtype=torch.uint8, device="cuda")
st = np.zeros(n, dtype=np.int32)
for r in range(reps):
    rc = lib.zk_decompress_frames_dev(ctx, d_comp.data_ptr(), co.ctypes.data_as(N.u64p), do.ctypes.data_as(N.u64p), n, d_out.data_ptr(), 0, st.ctypes.data_as(N.i32p), None)
    print(json.dumps(dict(kind=kind, mb=mb, rc=rc, ms=lib.zk_ctx_last_device_ms(ctx))), flush=True)
