"""Profile target (run under a profiler on a GPU machine): device-resident compress + decompress of the bench workload (1 GiB mix, 2 MiB frames)."""
import ctypes, os, sys, json
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zeekstd_b200 as zk
from zeekstd_b200 import corpus, _native as N, parallel as P
lib = N.load(); ctx = zk.Context(0, lib); codec = P.DeviceCodec(ctx)
mb = int(os.environ.get("ZK_PROF_MB", "1024")); FRAME = 2 << 20
x = corpus.make_mix(mb << 20, seed=20260924, device="cuda")
lvl, ck = int(os.environ.get("LVL", "1")), os.environ.get("CK", "0") == "1"
for r in range(int(os.environ.get("ZK_PROF_REPS", "2"))):
    comp, cs, ds = codec.compress(x, FRAME, lvl, ck); t_c = lib.zk_ctx_last_device_ms(ctx._h)
    co = np.concatenate([[0], np.cumsum(cs)]); do = np.concatenate([[0], np.cumsum(ds)])
    out = codec.decompress(comp, co, do, ck); t_d = lib.zk_ctx_last_device_ms(ctx._h)
    print(json.dumps(dict(mb=mb, comp_ms=round(t_c, 2), dec_ms=round(t_d, 2), ratio=round(x.numel() / comp.numel(), 4), ok=bool(torch.equal(out, x)))), flush=True)
