"""Per-kernel device time of the decode entropy stage on the H100: K-D1h `zk_huf_kernel`, K-D1s `zk_seq2_kernel` and the entropy slot
(first start to last end of the two), per GiB, for device-resident decompression (zk_decompress_frames_dev) of the bench's 1 GiB mix in
2 MiB frames at levels 1 and 3 (no checksum).  The archive of each level is written once; every decode step starts with an L2 flush, as in
bench.py, and its output is compared with the input.  Each setting gets a context of its own (`ZK_HUF_CTAS` / `ZK_HUF_PAD` are read when a
context is created, as is `ZK_SEQ2_CTAS`, swept by --seq2) and is decoded with the Huffman kernel on the side stream (`ZK_DEV_SIDE=1`, the default: the two entropy kernels run
side by side) and without it (`ZK_DEV_SIDE=0`: one after the other, so each kernel's time is its own).  Kernel durations and the slot come
from torch.profiler with CUDA activities; `dec_ms_per_GiB` is the whole decompress call (the context's CUDA events) over separate,
unprofiled steps.  The card's name, power limit and SM clock are read (read-only nvidia-smi queries) in the same call.  --lib profiles
another build of the library on the same card.  Prints one JSON line per setting and one JSON object at the end.

usage: python tools/huf_probe.py [--levels 1,3] [--ctas default,4,6,8,9] [--seq2 default] [--pads 0] [--side 0,1] [--steps 3] [--warmup 2]
                                [--lib PATH] [--out FILE]
       (a --ctas / --seq2 entry `default` leaves ZK_HUF_CTAS / ZK_SEQ2_CTAS unset; every --pads entry is swept at every --ctas entry,
       every --ctas entry at every --seq2 entry)"""
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
HUF, SEQ = "zk_huf_kernel", "zk_seq2_kernel"


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", default="1,3")
    ap.add_argument("--ctas", default="default,4,6,8,9")
    ap.add_argument("--seq2", default="default")
    ap.add_argument("--pads", default="0")
    ap.add_argument("--side", default="0,1")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lib", default=None, help="library to load (default: the in-tree build)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "huf_probe measures the GPU: no CUDA device"
    for k in ("ZK_HUF_CTAS", "ZK_SEQ2_CTAS", "ZK_HUF_PAD", "ZK_DEV_SIDE"):
        os.environ.pop(k, None)
    lib = N.load(args.lib)
    n, frame = bench.WORKLOAD_BYTES, bench.FRAME
    x = bench.gen_mix(n, bench.SEED, device="cuda")
    src = torch.cat([x, torch.zeros(64, dtype=torch.uint8, device="cuda")])
    cap = lib.zk_compress_bound(n, frame)
    comp = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    back = torch.zeros(n + 64, dtype=torch.uint8, device="cuda")
    nfmax = n // frame + 2
    cs = np.zeros(nfmax, dtype=np.uint32); ds = np.zeros(nfmax, dtype=np.uint32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")          # larger than the 50 MB L2: written before every step
    per_gib = n / GIB

    res = {"card": card(), "lib": os.path.abspath(args.lib or N.PRODUCT_SO), "bytes": n, "frame": frame, "steps": args.steps, "runs": []}
    for lv in [int(v) for v in args.levels.split(",")]:
        ctx = zk.Context(0, lib)
        nf, dl = ctypes.c_uint32(), ctypes.c_size_t()
        rc = lib.zk_compress_frames_dev(ctx._h, src.data_ptr(), n, frame, lv, 0, comp.data_ptr(), cap, cs.ctypes.data_as(N.u32p),
                                        ds.ctypes.data_as(N.u32p), nfmax, ctypes.byref(nf), ctypes.byref(dl), None)
        assert rc == 0, rc
        ctx.close()
        k = nf.value
        co = np.concatenate([[0], np.cumsum(cs[:k], dtype=np.uint64)]).astype(np.uint64)
        do = np.concatenate([[0], np.cumsum(ds[:k], dtype=np.uint64)]).astype(np.uint64)
        for s2, c, pad in [(s2, c, pad) for s2 in args.seq2.split(",") for c in args.ctas.split(",") for pad in args.pads.split(",")]:
            for var, v in (("ZK_SEQ2_CTAS", s2), ("ZK_HUF_CTAS", c)):
                if v == "default":
                    os.environ.pop(var, None)
                else:
                    os.environ[var] = v
            os.environ["ZK_HUF_PAD"] = pad
            ctx = zk.Context(0, lib)
            for side in args.side.split(","):
                os.environ["ZK_DEV_SIDE"] = side

                def step():
                    flush.fill_(1)
                    rc = lib.zk_decompress_frames_dev(ctx._h, comp.data_ptr(), co.ctypes.data_as(N.u64p), do.ctypes.data_as(N.u64p), k,
                                                      back.data_ptr(), 0, None, None)
                    assert rc == 0, rc
                    return ctx.last_device_ms

                for _ in range(args.warmup):
                    step()
                ok = bool(torch.equal(back[:n], x))
                dec = [step() for _ in range(args.steps)]
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.steps):
                        step()
                    torch.cuda.synchronize()
                ev = {HUF: [], SEQ: []}
                for e in prof.events():
                    if e.device_type != torch.autograd.DeviceType.CUDA:
                        continue
                    for kn in ev:
                        if e.name.startswith(kn):
                            ev[kn].append((e.time_range.start, e.time_range.end))
                assert len(ev[HUF]) == len(ev[SEQ]) == args.steps, {kn: len(v) for kn, v in ev.items()}
                h, s = sorted(ev[HUF]), sorted(ev[SEQ])
                slot = [max(a[1], b[1]) - min(a[0], b[0]) for a, b in zip(h, s)]

                def ms(spans):
                    return round(sum(spans) / len(spans) / 1e3 / per_gib, 3)

                r = {"level": lv, "seq2_ctas": s2, "huf_ctas": c, "huf_pad": int(pad), "side": int(side), "ok": ok,
                     "ms_per_GiB": {"K-D1h": ms([b - a for a, b in h]), "K-D1s": ms([b - a for a, b in s]), "slot": ms(slot)},
                     "dec_ms_per_GiB": round(float(np.mean(dec)) / per_gib, 3)}
                res["runs"].append(r)
                print(json.dumps(r), flush=True)
            ctx.close()
    for k in ("ZK_HUF_CTAS", "ZK_SEQ2_CTAS", "ZK_HUF_PAD", "ZK_DEV_SIDE"):
        os.environ.pop(k, None)
    res["card_after"] = card()
    txt = json.dumps(res)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(txt + "\n")


if __name__ == "__main__":
    main()
