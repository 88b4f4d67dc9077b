"""Negative (fast) compression levels on the H100: compress and decompress rates, ratio and per-kernel device time of the device-resident
entry points (zk_compress_frames_dev / zk_decompress_frames_dev) on the bench's 1 GiB mix in 2 MiB frames, against level 1.  The levels are
alternated round-robin, every step starts with an L2 flush and is timed by the context's CUDA events, and every step's round trip is checked.
The card's name, power limit and SM clock are read (read-only nvidia-smi queries) in the same call.  Prints one JSON object; --out also writes it.

usage: python tools/fast_levels_bench.py [--bytes N] [--levels 1,-1,-3,-7,-31] [--steps 5] [--warmup 2] [--out FILE]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import zeekstd_b200 as zk  # noqa: E402
from zeekstd_b200 import _native as N  # noqa: E402

GIB = 1 << 30
FRAME = bench.FRAME
SLOTS = ["scan", "seq", "huf", "exec", "xxh64", "match", "entropy_enc", "frame_assembly"]     # zk_ctx_profile slots (zeekstd_b200.h)


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


class Step:
    """one device-resident compress + decompress of x at one level; -> (compress ms, decompress ms, compressed bytes)"""

    def __init__(self, lib, ctx, x):
        self.lib, self.ctx, self.x, self.n = lib, ctx, x, x.numel()
        self.src = torch.cat([x, torch.zeros(64, dtype=torch.uint8, device=x.device)])
        self.cap = lib.zk_compress_bound(self.n, FRAME)
        self.comp = torch.zeros(self.cap + 64, dtype=torch.uint8, device=x.device)
        self.back = torch.zeros(self.n + 64, dtype=torch.uint8, device=x.device)
        self.nfmax = self.n // FRAME + 2
        self.cs = np.zeros(self.nfmax, dtype=np.uint32); self.ds = np.zeros(self.nfmax, dtype=np.uint32)
        torch.cuda.synchronize()

    def __call__(self, level: int):
        lib, ctx = self.lib, self.ctx
        nf, dl = ctypes.c_uint32(), ctypes.c_size_t()
        rc = lib.zk_compress_frames_dev(ctx._h, self.src.data_ptr(), self.n, FRAME, level, 0, self.comp.data_ptr(), self.cap,
                                        self.cs.ctypes.data_as(N.u32p), self.ds.ctypes.data_as(N.u32p), self.nfmax, ctypes.byref(nf),
                                        ctypes.byref(dl), None)
        assert rc == 0, rc
        t_c = ctx.last_device_ms
        k = nf.value
        co = np.zeros(k + 1, dtype=np.uint64); co[1:] = np.cumsum(self.cs[:k])
        do = np.zeros(k + 1, dtype=np.uint64); do[1:] = np.cumsum(self.ds[:k])
        rc = lib.zk_decompress_frames_dev(ctx._h, self.comp.data_ptr(), co.ctypes.data_as(N.u64p), do.ctypes.data_as(N.u64p), k,
                                          self.back.data_ptr(), 0, None, None)
        assert rc == 0, rc
        t_d = ctx.last_device_ms
        assert torch.equal(self.back[: self.n], self.x), f"round trip mismatch at level {level}"
        return t_c, t_d, int(co[-1])


def profile(lib, ctx, step, level: int) -> dict:
    """per-kernel device ms of one step (a run of its own: the profiler's events are not in the timed steps)"""
    def read():
        ms = (ctypes.c_float * 8)(); cnt = (ctypes.c_uint32 * 8)()
        lib.zk_ctx_profile_read(ctx._h, ms, cnt)
        return np.array(ms[:], dtype=np.float64)
    lib.zk_ctx_profile(ctx._h, 1)
    before = read()
    step(level)
    d = read() - before
    lib.zk_ctx_profile(ctx._h, 0)
    return {SLOTS[i]: round(float(d[i]), 3) for i in range(8) if d[i] > 0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=bench.WORKLOAD_BYTES)
    ap.add_argument("--levels", default="1,-1,-3,-7,-31")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fast_levels_bench measures the GPU: no CUDA device"
    levels = [int(v) for v in args.levels.split(",")]
    lib = N.load()
    ctx = zk.Context(0, lib)
    x = bench.gen_mix(args.bytes, bench.SEED, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")          # larger than the 50 MB L2: written before every step
    step = Step(lib, ctx, x)
    res = {"card": card(), "bytes": args.bytes, "frame": FRAME, "steps": args.steps, "levels": {}}
    t = {lv: ([], []) for lv in levels}
    clen = {}
    for it in range(args.warmup + args.steps):
        for lv in levels:
            flush.fill_(1); torch.cuda.synchronize()
            tc, td, clen[lv] = step(lv)
            if it >= args.warmup:
                t[lv][0].append(tc); t[lv][1].append(td)
    res["card_during"] = card()
    for lv in levels:
        tc, td = np.array(t[lv][0]), np.array(t[lv][1])
        gib = args.bytes / GIB
        res["levels"][str(lv)] = {
            "ratio": round(args.bytes / clen[lv], 4),
            "compress_GiBps": {"mean": round(gib / (tc.mean() / 1e3), 2), "min": round(gib / (tc.max() / 1e3), 2), "max": round(gib / (tc.min() / 1e3), 2)},
            "decompress_GiBps": {"mean": round(gib / (td.mean() / 1e3), 2), "min": round(gib / (td.max() / 1e3), 2), "max": round(gib / (td.min() / 1e3), 2)},
            "kernel_ms": profile(lib, ctx, step, lv)}
        print(json.dumps({lv: res["levels"][str(lv)]}), flush=True)
    res["card_after"] = card()
    txt = json.dumps(res)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(txt + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
