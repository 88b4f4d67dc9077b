"""High compression levels (K-C1h, levels >= 16) on the H100, in one call:
  * ratio of levels 13 / 16 / 19 on tests/golden/dickens.txt and on the bench's mix, in 2 MiB frames, next to libzstd (1.5.5, the oracle's
    reference library) at the same levels -- libzstd's high levels take minutes per GiB on the CPU, so the mix's libzstd column and the codec's
    column beside it are measured on the first --ref-bytes of the mix;
  * device-resident compress and decompress GiB/s at levels 13 and 19 on the --bytes mix (tools/fast_levels_bench.py's steps: L2 flushed
    before every step, CUDA events of the context, levels alternated, every round trip checked);
  * device ms per GiB of each K-C1h kernel group (stage, hash, sort, link, search, parse) at level 19, from torch.profiler in a run of its own.
The card's name, power limit and SM clock are read (read-only nvidia-smi queries) in the same call.  Prints one JSON object; --out also writes it.

usage: python tools/hc_bench.py [--bytes N] [--ref-bytes N] [--steps 3] [--warmup 1] [--out FILE]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import zeekstd_b200 as zk  # noqa: E402
from fast_levels_bench import Step, card, profile  # noqa: E402
from oracle import oracle as O  # noqa: E402
from zeekstd_b200 import _native as N  # noqa: E402

GIB = 1 << 30
FRAME = 2 << 20
LEVELS = (13, 16, 19)
GROUPS = {"zk_hc_stage": "stage", "zk_hc_hash": "hash", "zk_hc_hist": "sort", "zk_hc_scan": "sort", "zk_hc_scatter": "sort",
          "zk_hc_link": "link", "zk_hc_search": "search", "zk_hc_parse": "parse"}


def ratios(ctx, x: np.ndarray) -> dict:
    ours = {lv: round(x.size / ctx.compress_frames(x, FRAME, lv, False)[0].size, 4) for lv in LEVELS}
    ref = {lv: round(x.size / sum(O.ref_compress_frames(x, FRAME, lv, False, threads=os.cpu_count() or 1)[1]), 4) for lv in LEVELS}
    return {"codec": ours, "libzstd": ref}


def kernel_ms_per_gib(step, n: int) -> dict:
    from torch.profiler import ProfilerActivity, profile as tprofile
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        step(19)
        torch.cuda.synchronize()
    tot = {}
    for ev in prof.key_averages():
        for pre, g in GROUPS.items():
            if ev.key.startswith(pre) or ev.key.startswith("void " + pre):
                tot[g] = tot.get(g, 0.0) + ev.device_time_total / 1e3
    return {g: round(ms / (n / GIB), 2) for g, ms in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=bench.WORKLOAD_BYTES)
    ap.add_argument("--ref-bytes", type=int, default=64 << 20)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "hc_bench measures the GPU: no CUDA device"
    lib = N.load()
    ctx = zk.Context(0, lib)
    res = {"card": card(), "bytes": args.bytes, "frame": FRAME, "steps": args.steps}
    dickens = np.frombuffer(open(os.path.join(ROOT, "tests", "golden", "dickens.txt"), "rb").read(), dtype=np.uint8)
    res["ratio_dickens"] = ratios(ctx, dickens)
    x = bench.gen_mix(args.bytes, bench.SEED, device="cuda")
    res["ratio_mix_head"] = dict(ratios(ctx, x[: args.ref_bytes].cpu().numpy()), bytes=args.ref_bytes)
    print(json.dumps({k: res[k] for k in ("ratio_dickens", "ratio_mix_head")}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")          # larger than the 50 MB L2: written before every step
    step = Step(lib, ctx, x)
    t = {lv: ([], []) for lv in (13, 19)}
    clen = {}
    for it in range(args.warmup + args.steps):
        for lv in (13, 19):
            flush.fill_(1); torch.cuda.synchronize()
            tc, td, clen[lv] = step(lv)
            if it >= args.warmup:
                t[lv][0].append(tc); t[lv][1].append(td)
    res["card_during"] = card()
    gib = args.bytes / GIB
    res["device"] = {}
    for lv in (13, 19):
        tc, td = np.array(t[lv][0]), np.array(t[lv][1])
        res["device"][str(lv)] = {
            "ratio": round(args.bytes / clen[lv], 4),
            "compress_GiBps": {"mean": round(gib / (tc.mean() / 1e3), 3), "min": round(gib / (tc.max() / 1e3), 3), "max": round(gib / (tc.min() / 1e3), 3)},
            "decompress_GiBps": {"mean": round(gib / (td.mean() / 1e3), 2), "min": round(gib / (td.max() / 1e3), 2), "max": round(gib / (td.min() / 1e3), 2)},
            "slot_ms": profile(lib, ctx, step, lv)}
    res["hc_kernel_ms_per_GiB"] = kernel_ms_per_gib(step, args.bytes)
    res["card_after"] = card()
    txt = json.dumps(res)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(txt + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
