"""Content-defined frames (FrameSizePolicy::ContentDefined) on the H100: device-resident zk_compress_frames_cdc_dev on the bench's 1 GiB mix
against zk_compress_frames_sized_dev with the sizes it chose (the difference is the cost of the cut) and the uniform call at s, alternating
in one process (CUDA events, L2 flushed before every call, every output restored); the cut kernels' ms per GiB from zk_ctx_profile; the
frame-size distribution; the share of an edited copy's frames that its archive has in common with the original's.  Prints one JSON line
per case, with the card's name and power limit read in the same call.

usage: python tools/cdc_bench.py [--bytes N] [--sizes 65536,2097152] [--levels 1,3] [--runs R] [--edit-bytes N] [--out FILE]"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import zeekstd_b200 as zk  # noqa: E402
from golden.make_encoder_golden_ldm import edited_copy  # noqa: E402
from sized_bench import PAD, Runner, bench_offsets, card  # noqa: E402
from zeekstd_b200 import _native  # noqa: E402


def cdc(r: Runner, n: int, s: int, level: int):
    def go(stream):
        nfmax = n // 1024 + 1
        cs = np.zeros(nfmax, np.uint32); ds = np.zeros(nfmax, np.uint32); k = ctypes.c_uint32(); dl = ctypes.c_size_t(); used = ctypes.c_size_t()
        rc = r.lib.zk_compress_frames_cdc_dev(r.ctx._h, r.x.data_ptr(), n, s, level, 0, 1, r.dst.data_ptr(), r.dst.numel(),
                                              cs.ctypes.data_as(_native.u32p), ds.ctypes.data_as(_native.u32p), nfmax, ctypes.byref(k),
                                              ctypes.byref(dl), ctypes.byref(used), stream)
        assert rc == 0 and used.value == n, rc
        return cs[: k.value], ds[: k.value], int(dl.value)
    return r._timed(go)


def cut_ms_per_gib(r: Runner, n: int, s: int, level: int, reps: int = 3) -> float:
    """profile slot 0 of the encoder: the cut kernels (count, scan, emit, next, walk) of every pass"""
    ms = (ctypes.c_float * 8)(); cnt = (ctypes.c_uint32 * 8)()
    r.lib.zk_ctx_profile(r.ctx._h, 1)
    for _ in range(reps):
        cdc(r, n, s, level)
    r.lib.zk_ctx_profile_read(r.ctx._h, ms, cnt)
    r.lib.zk_ctx_profile(r.ctx._h, 0)
    return ms[0] / reps / (n / (1 << 30))


def shared_fraction(ctx, n: int, s: int, level: int, edits: int) -> dict:
    old = bench.gen_mix(n, bench.SEED + 1, device="cpu").numpy()
    new = edited_copy(old, 5, edits)
    out = {}
    for policy in ("content", "uncompressed"):
        def frames(x):
            if policy == "content":
                comp, cs, _, _ = ctx.compress_frames_cdc(x, s, level, True)
            else:
                comp, cs, _ = ctx.compress_frames(x, s, level, True)
            co = bench_offsets(cs)
            return [comp[int(co[i]):int(co[i + 1])].tobytes() for i in range(len(cs))]
        old_set = set(frames(old))
        nf = frames(new)
        shared = sum(f in old_set for f in nf)
        out[policy] = {"frames": len(nf), "shared": shared, "fraction": round(shared / len(nf), 4)}
    return {"edit_bytes": n, "edits": edits, "s": s, **out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=1 << 30)
    ap.add_argument("--sizes", default=f"{64 << 10},{2 << 20}")
    ap.add_argument("--levels", default="1,3")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--edit-bytes", type=int, default=256 << 20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = zk.Context(0)
    n = args.bytes
    x = torch.cat([bench.gen_mix(n, bench.SEED, device="cuda"), torch.zeros(PAD, dtype=torch.uint8, device="cuda")])
    r = Runner(ctx, x)
    results = []
    for s in (int(v) for v in args.sizes.split(",")):
        for level in (int(v) for v in args.levels.split(",")):
            t = {"cdc": [], "sized": [], "uniform": []}
            for _ in range(args.runs):
                ms, (cs, ds, tot) = cdc(r, n, s, level); t["cdc"].append(ms)
                r.check(0, n, cs, ds, tot)
                ms, (scs, stot) = r.sized(0, ds.astype(np.uint32), level); t["sized"].append(ms)
                assert stot == tot and np.array_equal(scs, cs), "cdc frames differ from the sized call's"
                ms, (ucs, uds, utot) = r.uniform(0, n, s, level); t["uniform"].append(ms)
                r.check(0, n, ucs, uds, utot)
            q = np.percentile(ds, [1, 10, 50, 90, 99]).astype(int).tolist()
            mx = min(4 * s, 1 << 30)
            case = {"s": s, "level": level, "bytes": n, "frames": int(ds.size), "mean_frame": int(n // ds.size),
                    "frame_percentiles_1_10_50_90_99": q, "forced_at_mx": round(float(np.mean(ds[:-1] == mx)), 5),
                    "ratio_cdc": round(n / tot, 4), "ratio_uniform": round(n / utot, 4),
                    **{f"{k}_ms": [round(v, 3) for v in vs] for k, vs in t.items()},
                    **{f"{k}_gibs": round(n / (1 << 30) / (min(vs) / 1e3), 2) for k, vs in t.items()},
                    "cut_ms_per_gib": round(cut_ms_per_gib(r, n, s, level), 3), "card": card()}
            print(json.dumps(case), flush=True)
            results.append(case)
    edit = {**shared_fraction(ctx, args.edit_bytes, 64 << 10, 1, 64), "card": card()}
    print(json.dumps(edit), flush=True)
    results.append(edit)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
