"""Seekable patches against the whole-prefix patch and plain compression on one NEW / OLD pair.

    python tools/patch_slices_bench.py [--mib 384] [--frame-mib 2] [--reps 3] [--out DIR]

OLD is --mib MiB of the bench's mix; NEW is OLD with 64 small edits and its first 8 MiB moved to the end.  Reports the three archive sizes
(plain level 16, whole-prefix --long, slices), the time of Context.patch_ranges per GiB of OLD + NEW, compress and decompress GiB/s of the
slice patch against the whole-prefix patch (host pointers, best of --reps after one warm-up, host clock around synchronous calls), and the
prefix bytes one single-frame read uploads.  Prints one JSON line and writes it to DIR/patch_slices_bench.json when --out is given.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import zeekstd_b200 as zk  # noqa: E402
from zeekstd_b200 import corpus  # noqa: E402


def _best(fn, reps):
    fn()
    best, out = None, None
    for _ in range(reps):
        t = time.perf_counter()
        out = fn()
        dt = time.perf_counter() - t
        best = dt if best is None else min(best, dt)
    return best, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=384)
    ap.add_argument("--frame-mib", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    ctx = zk.Context(0)
    n = a.mib << 20
    old = corpus.make_mix(n, seed=1, segment=64 << 10).numpy()
    new = old.copy()
    rng = np.random.default_rng(9)
    for at in rng.integers(0, n - 64, 64):
        new[at:at + 32] = rng.integers(0, 256, 32, dtype=np.uint8)
    new = np.concatenate([new[8 << 20:], new[:8 << 20]])
    fs = a.frame_mib << 20
    sizes = np.array([min(fs, new.size - s) for s in range(0, new.size, fs)], dtype=np.uint32)
    gib = 1 << 30

    plain = ctx.compress_frames_sized(new, sizes, 16, True)[0].size
    t_ranges, rg = _best(lambda: ctx.patch_ranges(new, sizes, old, fs), a.reps)
    t_slices, res = _best(lambda: ctx.compress_frames_patch(new, sizes, old, rg, 16, True), a.reps)
    comp, cs, ds = res
    head = zk.patch_slices_write(old.size, rg)
    t_whole, wres = _best(lambda: ctx.compress_frames(new, fs, 16, True, prefix=old, long_distance=True), a.reps)
    wcomp, wcs, wds = wres
    pad = np.concatenate([comp, np.zeros(64, np.uint8)])
    wpad = np.concatenate([wcomp, np.zeros(64, np.uint8)])
    co = np.concatenate([[0], np.cumsum(cs, dtype=np.uint64)]).astype(np.uint64)
    do = np.concatenate([[0], np.cumsum(ds, dtype=np.uint64)]).astype(np.uint64)
    wco = np.concatenate([[0], np.cumsum(wcs, dtype=np.uint64)]).astype(np.uint64)
    wdo = np.concatenate([[0], np.cumsum(wds, dtype=np.uint64)]).astype(np.uint64)
    out = np.empty(new.size + 64, np.uint8)
    t_dslices, r1 = _best(lambda: ctx.decompress_frames(pad, co, do, True, out=out, prefix=old, prefix_ranges=rg)[2], a.reps)
    ok_slices = r1 == 0 and out[: new.size].tobytes() == new.tobytes()
    t_dwhole, r2 = _best(lambda: ctx.decompress_frames(wpad, wco, wdo, True, out=out, prefix=old)[2], a.reps)
    ok_whole = r2 == 0 and out[: new.size].tobytes() == new.tobytes()
    f = len(sizes) // 2
    before = ctx.prefix_bytes_uploaded
    one = np.concatenate([comp[int(co[f]):int(co[f + 1])], np.zeros(64, np.uint8)])
    back, st, rc = ctx.decompress_frames(one, [0, int(cs[f])], [0, int(ds[f])], True, prefix=old, prefix_ranges=rg[f:f + 1])
    one_frame_upload = ctx.prefix_bytes_uploaded - before
    r = {
        "gpu": gpu, "old_mib": a.mib, "frame_mib": a.frame_mib, "frames": int(len(sizes)),
        "bytes_plain": int(plain), "bytes_whole_prefix_long": int(wcomp.size), "bytes_slices": int(comp.size + len(head)),
        "ranges_ms": round(t_ranges * 1e3, 2), "ranges_ms_per_gib_old_plus_new": round(t_ranges * 1e3 / ((old.size + new.size) / gib), 2),
        "compress_gibps_slices": round(new.size / gib / t_slices, 3), "compress_gibps_whole_prefix": round(new.size / gib / t_whole, 3),
        "decompress_gibps_slices": round(new.size / gib / t_dslices, 3), "decompress_gibps_whole_prefix": round(new.size / gib / t_dwhole, 3),
        "one_frame_prefix_bytes_uploaded": int(one_frame_upload), "one_frame_range_bytes": int(rg[f][1] - rg[f][0]),
        "restored": bool(ok_slices and ok_whole and rc == 0 and back[: int(ds[f])].tobytes() == new[int(do[f]):int(do[f + 1])].tobytes()),
    }
    line = json.dumps(r)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "patch_slices_bench.json"), "w") as fh:
            fh.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
