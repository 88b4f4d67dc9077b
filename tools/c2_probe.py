"""Per-kernel device time of compression on the H100: K-C1 `zk_match_kernel` (`zk_match_wide_kernel` from level 13,
`zk_match_fast_kernel` below 0), K-C2s `zk_seq_enc_kernel`, K-C2l `zk_lit_enc_kernel` and K-C2f `zk_block_finish_kernel`, per GiB, for
device-resident compression (zk_compress_frames_dev) of the bench's 1 GiB mix in 2 MiB frames at levels 1, 3 and -1 (the level -1 literal kernel does no Huffman work, so its K-C2s time is the sequence side alone).  K-C2s and K-C2l
run side by side on two streams; the longer of the two ends the K-C2 profile slot.  Every step starts with an L2 flush, as in bench.py.
Kernel durations come from torch.profiler with CUDA activities, in a run of its own; the card's name, power limit and SM clock are read
(read-only nvidia-smi queries) in the same call.  --lib compares another build of the library on the same card.  Prints one JSON object.

usage: python tools/c2_probe.py [--levels 1,3,-1] [--steps 3] [--warmup 2] [--lib PATH] [--out FILE]"""
import argparse
import ctypes
import json
import os
import re
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
KERNELS = ["zk_match_kernel", "zk_match_wide_kernel", "zk_match_fast_kernel", "zk_seq_enc_kernel", "zk_lit_enc_kernel", "zk_block_finish_kernel"]


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", default="1,3,-1")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lib", default=None, help="library to load (default: the in-tree build)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "c2_probe measures the GPU: no CUDA device"
    levels = [int(v) for v in args.levels.split(",")]
    lib = N.load(args.lib)
    ctx = zk.Context(0, lib)
    n, frame = bench.WORKLOAD_BYTES, bench.FRAME
    x = bench.gen_mix(n, bench.SEED, device="cuda")
    src = torch.cat([x, torch.zeros(64, dtype=torch.uint8, device="cuda")])
    cap = lib.zk_compress_bound(n, frame)
    comp = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    nfmax = n // frame + 2
    cs = np.zeros(nfmax, dtype=np.uint32); ds = np.zeros(nfmax, dtype=np.uint32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")          # larger than the 50 MB L2: written before every step

    def step(level):
        flush.fill_(1)
        nf, dl = ctypes.c_uint32(), ctypes.c_size_t()
        rc = lib.zk_compress_frames_dev(ctx._h, src.data_ptr(), n, frame, level, 0, comp.data_ptr(), cap, cs.ctypes.data_as(N.u32p),
                                        ds.ctypes.data_as(N.u32p), nfmax, ctypes.byref(nf), ctypes.byref(dl), None)
        assert rc == 0, rc
        return int(dl.value)

    res = {"card": card(), "lib": os.path.abspath(args.lib or N.PRODUCT_SO), "bytes": n, "frame": frame, "steps": args.steps, "levels": {}}
    for lv in levels:
        for _ in range(args.warmup):
            step(lv)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                clen = step(lv)
            torch.cuda.synchronize()
        us = {k: 0.0 for k in KERNELS}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            for k in KERNELS:
                if re.search(rf"\b{k}[<(]", ev.name):
                    us[k] += ev.time_range.elapsed_us()
        per_gib = args.steps * n / GIB
        res["levels"][str(lv)] = {"ratio": round(n / clen, 4),
                                  "kernel_ms_per_GiB": {k: round(v / 1e3 / per_gib, 3) for k, v in us.items() if v > 0}}
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
