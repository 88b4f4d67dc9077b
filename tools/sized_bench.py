"""Frames of caller-chosen sizes on the H100: one zk_compress_frames_sized_dev call against the uniform call at the same mean frame size and
against one zk_compress_frames_dev call per frame (what a caller had to do before), alternating in one process.  Input: the bench's mix cut
by seeded log-uniform sizes in [1 KiB, 4 MiB]; device-resident, CUDA events, the L2 flushed before every call; every output is restored
and compared.  Prints one JSON line per case; --out also writes the list.

usage: python tools/sized_bench.py [--bytes N] [--levels 1,3,-3] [--hc-bytes N] [--per-frame K] [--runs R] [--out FILE]"""
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
from zeekstd_b200 import _native, parallel  # noqa: E402

PAD = 64


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def cut(n: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    out, tot = [], 0
    while tot < n:
        d = min(int(np.exp(rng.uniform(np.log(1 << 10), np.log(4 << 20)))), n - tot)
        out.append(d); tot += d
    return np.asarray(out, np.uint32)


class Runner:
    def __init__(self, ctx, x: torch.Tensor):
        self.ctx, self.lib, self.x = ctx, ctx.lib, x
        self.flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        self.dst = torch.empty(x.numel() + x.numel() // 8 + (64 << 20), dtype=torch.uint8, device="cuda")

    def _timed(self, fn):
        self.flush_buf.fill_(1)                       # evict the L2 (50 MiB on the H100)
        st = torch.cuda.current_stream()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st); r = fn(st.cuda_stream); b.record(st)
        b.synchronize()
        return a.elapsed_time(b), r

    def sized(self, off: int, sizes: np.ndarray, level: int):
        def go(stream):
            cs = np.zeros(sizes.size, np.uint32); dl = ctypes.c_size_t()
            rc = self.lib.zk_compress_frames_sized_dev(self.ctx._h, self.x.data_ptr() + off, sizes.ctypes.data_as(_native.u32p), sizes.size, level, 0,
                                                      self.dst.data_ptr(), self.dst.numel(), cs.ctypes.data_as(_native.u32p), ctypes.byref(dl), stream)
            assert rc == 0, rc
            return cs, int(dl.value)
        return self._timed(go)

    def uniform(self, off: int, n: int, fs: int, level: int):
        def go(stream):
            nf = n // fs + 2
            cs = np.zeros(nf, np.uint32); ds = np.zeros(nf, np.uint32); k = ctypes.c_uint32(); dl = ctypes.c_size_t()
            rc = self.lib.zk_compress_frames_dev(self.ctx._h, self.x.data_ptr() + off, n, fs, level, 0, self.dst.data_ptr(), self.dst.numel(),
                                                 cs.ctypes.data_as(_native.u32p), ds.ctypes.data_as(_native.u32p), nf, ctypes.byref(k),
                                                 ctypes.byref(dl), stream)
            assert rc == 0, rc
            return cs[: k.value], ds[: k.value], int(dl.value)
        return self._timed(go)

    def per_frame(self, sizes: np.ndarray, level: int):
        def go(stream):
            pos, out, cs = 0, 0, []
            one = np.zeros(1, np.uint32); k = ctypes.c_uint32(); dl = ctypes.c_size_t()
            for d in sizes:
                rc = self.lib.zk_compress_frames_dev(self.ctx._h, self.x.data_ptr() + pos, int(d), max(int(d), 1), level, 0, self.dst.data_ptr() + out,
                                                     self.dst.numel() - out, one.ctypes.data_as(_native.u32p), None, 1, ctypes.byref(k),
                                                     ctypes.byref(dl), stream)
                assert rc == 0, rc
                pos += int(d); out += int(dl.value); cs.append(int(one[0]))
            return np.asarray(cs, np.uint32), out
        return self._timed(go)

    def check(self, off: int, n: int, cs, ds, total: int):
        dev = parallel.DeviceCodec(self.ctx)
        back = dev.decompress(self.dst[:total], bench_offsets(cs), bench_offsets(ds), False)
        assert torch.equal(back, self.x[off:off + n]), "round trip"


def bench_offsets(sizes):
    o = np.zeros(len(sizes) + 1, np.uint64); o[1:] = np.cumsum(np.asarray(sizes, np.uint64)); return o


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=1 << 30)
    ap.add_argument("--levels", default="1,3,-3")
    ap.add_argument("--hc-bytes", type=int, default=64 << 20, help="input of the level-19 case")
    ap.add_argument("--per-frame", type=int, default=2000, help="frames of the one-call-per-frame comparison")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = zk.Context(0)
    x = torch.cat([bench.gen_mix(args.bytes, bench.SEED, device="cuda"), torch.zeros(PAD, dtype=torch.uint8, device="cuda")])
    r = Runner(ctx, x)
    info = card()
    results = []
    cases = [(int(lv), args.bytes) for lv in args.levels.split(",")] + [(19, args.hc_bytes)]
    for level, n in cases:
        sizes = cut(n, 20261016)
        head = sizes[: args.per_frame]
        mean = max(1, n // sizes.size)
        t = {"sized": [], "uniform": [], "sized_head": [], "per_frame_head": []}
        for _ in range(args.runs):
            ms, (cs, tot) = r.sized(0, sizes, level); t["sized"].append(ms)
            r.check(0, n, cs, sizes, tot)
            ms, (ucs, uds, utot) = r.uniform(0, n, mean, level); t["uniform"].append(ms)
            r.check(0, n, ucs, uds, utot)
            ms, (hcs, htot) = r.sized(0, head, level); t["sized_head"].append(ms)
            ms, (pcs, ptot) = r.per_frame(head, level); t["per_frame_head"].append(ms)
            r.check(0, int(head.sum(dtype=np.uint64)), pcs, head, ptot)
            # frames whose size differs from their one-call-per-frame encoding, with their first block and block count
            fb = np.concatenate([[0], np.cumsum(np.maximum(1, (head.astype(np.int64) + 32767) // 32768))])
            differ = [(int(f), int(fb[f]), int(fb[f + 1] - fb[f])) for f in np.nonzero(pcs != hcs)[0]]
        case = {"level": level, "bytes": n, "frames": int(sizes.size), "mean_frame": mean, "head_frames": int(head.size),
                "head_bytes": int(head.sum(dtype=np.uint64)), "ratio_sized": round(n / tot, 4), "ratio_uniform": round(n / utot, 4),
                **{f"{k}_ms": [round(v, 3) for v in vs] for k, vs in t.items()},
                "sized_gbs": round(n / min(t["sized"]) / 1e6, 2), "uniform_gbs": round(n / min(t["uniform"]) / 1e6, 2),
                "per_frame_over_sized_head": round(min(t["per_frame_head"]) / min(t["sized_head"]), 1),
                "frames_differing_from_per_frame_calls": differ, "card": info}
        print(json.dumps(case), flush=True)
        results.append(case)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
