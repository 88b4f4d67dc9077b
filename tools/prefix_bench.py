"""Prefix (patch) mode decode on the H100: device time of the decode kernels per GiB for an archive of the bench's mix in 2 MiB frames at
levels 1 and 3, every frame compressed against the same raw-content prefix, which shares content with the input (a slice of the mix made
with another seed: the same text source and record generators).  Prefix mode is reachable through the host-pointer calls only
(zk_compress_frames_prefix / zk_decompress_frames_prefix), so each step is one such call; `kern_ms_per_GiB` is the sum of the decode
kernels' durations (torch.profiler, CUDA activities) and `exec_ms_per_GiB` that of the plan kernel and the sequence executors, the part of
the decode that prefix mode changes; `wall_ms_per_GiB` is the whole call, copies included.  The L2 is flushed before every step and the
output is compared with the input after every step.  Restated-decoder statistics of the first frames show how many matches reach into the
prefix.  The card's name, power limit and SM clock are read (read-only nvidia-smi queries) in the same call.

--lib times another build on the same card: every round runs each build in a process of its own, the builds alternated, on the same
archives (written once by the in-tree build).  Prints one JSON line per (round, build, level) and one JSON object with the medians at the end.

usage: python tools/prefix_bench.py [--lib PATH] [--levels 1,3] [--mb 256] [--prefix-kib 512] [--rounds 3] [--steps 3] [--warmup 2] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GIB = 1 << 30
FRAME = 2 << 20
EXEC = ("zk_plan_kernel", "zk_exec")


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def child(args):
    """one build, one level: decode the archive in args.archive, print one JSON line"""
    import torch
    import zeekstd_b200 as zk
    from zeekstd_b200 import _native as N
    lib = N.load(args.lib)
    z = np.load(args.archive)
    comp, co, do, prefix, x = z["comp"], z["co"], z["do"], z["prefix"], z["data"]
    n = x.size
    ctx = zk.Context(0, lib)
    out = np.empty(n + 64, dtype=np.uint8)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")          # larger than the 50 MB L2: written before every step
    ok = True

    def step():
        nonlocal ok
        flush.fill_(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, st, rc = ctx.decompress_frames(comp, co, do, False, out=out, prefix=prefix)
        wall = (time.perf_counter() - t0) * 1e3
        ok = ok and rc == 0 and not st.any() and np.array_equal(out[:n], x)
        return wall

    for _ in range(args.warmup):
        step()
    l0, s0 = ctx.kernel_launches, ctx.decode_segments
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        wall = [step() for _ in range(args.steps)]
        torch.cuda.synchronize()
    launches, segs = ctx.kernel_launches - l0, ctx.decode_segments - s0
    ctx.close()
    kern = exe = 0.0
    for e in prof.events():
        name = e.name[5:] if e.name.startswith("void ") else e.name      # (template kernels carry their return type)
        if e.device_type == torch.autograd.DeviceType.CUDA and name.startswith("zk_"):
            d = (e.time_range.end - e.time_range.start) / 1e3
            kern += d
            exe += d if name.startswith(EXEC) else 0.0
    per = args.steps * n / GIB
    print(json.dumps({"lib": os.path.abspath(args.lib), "level": args.level, "ok": bool(ok),
                      "kern_ms_per_GiB": round(kern / per, 3), "exec_ms_per_GiB": round(exe / per, 3),
                      "wall_ms_per_GiB": round(float(np.sum(wall)) / per, 3),
                      "gpu_launches_per_decode": launches / args.steps, "segments_per_decode": segs / args.steps}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="another build to time beside the in-tree one")
    ap.add_argument("--levels", default="1,3")
    ap.add_argument("--mb", type=int, default=256)
    ap.add_argument("--prefix-kib", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--archive", help=argparse.SUPPRESS)
    ap.add_argument("--level", type=int, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    import torch
    import bench
    import zeekstd_b200 as zk
    from oracle import oracle as O
    from zeekstd_b200 import _native as N
    assert torch.cuda.is_available(), "prefix_bench measures the GPU: no CUDA device"
    for k in ("ZK_EXEC_SHORT", "ZK_EXEC_WARPS", "ZK_RING_BYTES"):
        os.environ.pop(k, None)
    n = args.mb << 20
    x = bench.gen_mix(n, bench.SEED).numpy()
    prefix = bench.gen_mix(args.prefix_kib << 10, bench.SEED + 1).numpy()
    libs = [os.path.abspath(N.PRODUCT_SO)] + ([os.path.abspath(args.lib)] if args.lib else [])
    res = {"card": card(), "bytes": n, "frame": FRAME, "prefix_bytes": prefix.size, "steps": args.steps, "archives": {}, "runs": []}
    tmp = tempfile.mkdtemp(prefix="zk_prefix_bench_")
    try:
        ctx = zk.Context(0, N.load(libs[0]))
        for lv in [int(v) for v in args.levels.split(",")]:
            comp, cs, ds = ctx.compress_frames(x, FRAME, lv, False, prefix=prefix)
            co = np.concatenate([[0], np.cumsum(cs, dtype=np.uint64)]).astype(np.uint64)
            do = np.concatenate([[0], np.cumsum(ds, dtype=np.uint64)]).astype(np.uint64)
            stats = [O.oracle_decompress_ex(comp[int(co[i]): int(co[i + 1])], int(ds[i]), prefix=prefix)[1] for i in range(min(4, len(cs)))]
            res["archives"][lv] = {"ratio": round(n / comp.size, 4), "frames": len(cs),
                                   "prefix_matches_first_frames": [s["prefix_matches"] for s in stats]}
            np.savez(os.path.join(tmp, f"l{lv}.npz"), comp=np.concatenate([comp, np.zeros(64, np.uint8)]), co=co, do=do, prefix=prefix, data=x)
        ctx.close()
        print(json.dumps({"card": res["card"], "archives": res["archives"]}), flush=True)
        for r in range(args.rounds):
            for lib in libs:
                for lv in [int(v) for v in args.levels.split(",")]:
                    cmd = [sys.executable, os.path.abspath(__file__), "--child", "--lib", lib, "--archive", os.path.join(tmp, f"l{lv}.npz"),
                           "--level", str(lv), "--steps", str(args.steps), "--warmup", str(args.warmup)]
                    p = subprocess.run(cmd, capture_output=True, text=True)
                    if p.returncode:
                        sys.stderr.write(p.stdout + p.stderr)
                        raise SystemExit(f"child failed: {' '.join(cmd)}")
                    row = dict(json.loads(p.stdout.strip().splitlines()[-1]), round=r)
                    res["runs"].append(row)
                    print(json.dumps(row), flush=True)
    finally:
        for f in os.listdir(tmp):
            os.remove(os.path.join(tmp, f))
        os.rmdir(tmp)
    res["median"] = {f"{lib}|L{lv}": {k: float(np.median([q[k] for q in res["runs"] if q["lib"] == lib and q["level"] == lv]))
                                      for k in ("kern_ms_per_GiB", "exec_ms_per_GiB", "wall_ms_per_GiB", "gpu_launches_per_decode")}
                     for lib in libs for lv in [int(v) for v in args.levels.split(",")]}
    res["all_ok"] = all(q["ok"] for q in res["runs"])
    res["card_after"] = card()
    txt = json.dumps(res)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(txt + "\n")


if __name__ == "__main__":
    main()
