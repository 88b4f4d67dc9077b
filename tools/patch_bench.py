"""Patch mode with and without long-distance matching (zk_ldm.inc) on one GPU.

OLD = the first --mib MiB of the bench's class mix, NEW = its edited copy (seeded insertions, deletions, overwritten spans and one moved
region), 2 MiB frames, level 16.  The two variants alternate within one call; each step flushes L2 first, times the call and checks the
round trip.  Patch mode has host-pointer entry points only, so the time is a host clock around the synchronous call: it includes the
copies of the prefix and the input to the device and of the archive back (zk_ctx_last_device_ms covers device-pointer calls only).
Reports the patch size beside libzstd's (windowLog + long-distance matching + refPrefix, the reference CLI's sequence), GiB/s of NEW for
both variants, and the card with its power limit and SM clock.  --profile runs one more call of each variant under torch.profiler and
prints the summed device time of its kernels and the time of every kernel (the index is zk_ldm_index_kernel, zk_ldm_check_kernel and
the sort kernels launched between them).

    python tools/patch_bench.py --mib 64 --steps 3 --warmup 1 [--profile]
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
import torch


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=64)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--profile", action="store_true")
    ns = ap.parse_args()
    assert torch.cuda.is_available(), "patch_bench needs a GPU"
    import bench
    import zeekstd_b200 as zk
    spec = importlib.util.spec_from_file_location("mk", os.path.join(ROOT, "tests", "golden", "make_encoder_golden_ldm.py"))
    mk = importlib.util.module_from_spec(spec); spec.loader.exec_module(mk)
    from test_patch_ldm import _libzstd_patch_size
    from util import offsets

    fs, level = 2 << 20, 16
    old = bench.gen_mix(ns.mib << 20, bench.SEED, device="cuda").cpu().numpy()
    new = mk.edited_copy(old, 1, 40 * ns.mib)
    ctx = zk.Context(0)
    flush = torch.empty(128 << 20, dtype=torch.uint8, device="cuda")
    ms = {False: [], True: []}
    size = {}
    for step in range(ns.warmup + ns.steps):
        for ldm in (False, True):
            flush.zero_(); torch.cuda.synchronize()
            t0 = time.perf_counter()
            comp, cs, ds = ctx.compress_frames(new, fs, level, True, prefix=old, long_distance=ldm)
            t = (time.perf_counter() - t0) * 1e3
            pad = np.concatenate([comp, np.zeros(64, np.uint8)])
            back, st, rc = ctx.decompress_frames(pad, offsets(cs), offsets(ds), True, prefix=old)
            assert rc == 0 and back[: new.size].tobytes() == new.tobytes()
            size[ldm] = int(comp.size)
            if step >= ns.warmup:
                ms[ldm].append(t)
    gib = new.size / 2**30
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"card": q.stdout.strip(), "new_bytes": int(new.size), "prefix_bytes": int(old.size), "frame_size": fs, "level": level,
           "patch_bytes_ldm": size[True], "bytes_without_ldm": size[False], "libzstd_patch_bytes": _libzstd_patch_size(new, old, fs, level, True),
           "call_ms_ldm": ms[True], "call_ms_without": ms[False],
           "gib_s_ldm": gib / (min(ms[True]) / 1e3), "gib_s_without": gib / (min(ms[False]) / 1e3)}
    if ns.profile:
        from torch.profiler import ProfilerActivity, profile
        for ldm in (False, True):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ctx.compress_frames(new, fs, level, True, prefix=old, long_distance=ldm)
                torch.cuda.synchronize()
            rows = sorted(((e.key, e.count, e.device_time_total / 1e3) for e in prof.key_averages() if e.device_time_total and "zk_" in e.key),
                          key=lambda r: -r[2])
            res["kernels_ms_ldm" if ldm else "kernels_ms_without"] = {"sum": round(sum(r[2] for r in rows), 3),
                                                                      **{k: {"launches": c, "ms": round(t, 3)} for k, c, t in rows[:16]}}
    print(json.dumps(res))
    ctx.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
