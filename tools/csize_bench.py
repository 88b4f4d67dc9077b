"""FrameSizePolicy::Compressed(target) on the H100: the batch path (zk_compress_frames_csize[_dev]) against the uniform policy at the
same mean frame size, its per-kernel split, and the host Encoder<W> against the per-frame trial loop it replaced (driven here through
RawEncoder, which keeps that loop).  Input: the bench's mix (corpus.make_mix).  Prints one JSON object; --out also writes it.

usage: python tools/csize_bench.py [--bytes N] [--levels 1,3,13] [--targets 1048576,65536] [--host-bytes N] [--runs R] [--out FILE]"""
import argparse
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import zeekstd_b200 as zk  # noqa: E402
from zeekstd_b200 import corpus, parallel  # noqa: E402

GIB = 1 << 30


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def timed(fn, runs: int):
    """-> (best seconds, last result); fn ends in a device synchronisation (the entry points are synchronous)"""
    fn()
    best, r = float("inf"), None
    for _ in range(runs):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t)
    return best, r


PHASES = (("variants", ("zk_match", "zk_seq_enc", "zk_lit_enc", "zk_block_finish", "zk_prefix_stage")),
          ("cut", ("zk_csize_psum", "zk_csize_next", "zk_csize_walk")),
          ("assembly", ("zk_geo_starts", "zk_geo_block", "zk_frame_")))


def kernel_split(fn) -> dict:
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ms = {k: 0.0 for k, _ in PHASES}
    for ev in prof.key_averages():
        for k, names in PHASES:
            if any(ev.key.startswith(n) or n in ev.key for n in names):
                ms[k] += ev.device_time_total / 1e3
    return {k: round(v, 3) for k, v in ms.items()}


def trial_loop(ctx, data: bytes, target: int, level: int) -> bytes:
    """the per-frame trial compression the Encoder used before: RawEncoder with the Encoder's 128 KiB staging buffer"""
    enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Compressed(target)).compression_level(level).into_raw_encoder()
    out, st = io.BytesIO(), bytearray(131591)
    pos = 0
    while pos < len(data):
        p = enc.compress(memoryview(data)[pos:], st)
        out.write(st[: p.out_progress]); pos += p.in_progress
    while True:
        p = enc.end_frame(st)
        out.write(st[: p.out_progress])
        if p.data_left == 0:
            return out.getvalue()


def batch_encoder(ctx, data: bytes, target: int, level: int) -> bytes:
    sink = io.BytesIO()
    enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Compressed(target)).compression_level(level).into_encoder(sink)
    for p in range(0, len(data), 1 << 20):
        enc.compress(data[p: p + (1 << 20)])
    enc.end_frame()
    return sink.getvalue()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=GIB)
    ap.add_argument("--levels", default="1,3,13")
    ap.add_argument("--targets", default=f"{1 << 20},{64 << 10}")
    ap.add_argument("--host-bytes", type=int, default=32 << 20, help="input of the host Encoder comparison (the trial loop is slow)")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "csize_bench measures the GPU: no CUDA device"
    res = {"card": card(), "bytes": args.bytes, "cases": []}
    ctx = zk.Context(0)
    dev = parallel.DeviceCodec(ctx)
    x = corpus.make_mix(args.bytes, device="cuda")
    host = corpus.as_numpy(x[: args.host_bytes].cpu()).tobytes()
    for level in [int(v) for v in args.levels.split(",")]:
        for target in [int(v) for v in args.targets.split(",")]:
            t_cs, (comp, cs, ds, _) = timed(lambda: dev.compress_csize(x, target, level, False), args.runs)
            fs = max(1, int(round(float(np.mean(ds)))))
            t_un, _ = timed(lambda: dev.compress(x, fs, level, False), args.runs)
            split = kernel_split(lambda: dev.compress_csize(x, target, level, False))
            r = np.asarray(cs, dtype=np.float64) / target
            case = {"level": level, "target": target, "frames": int(len(cs)), "mean_d_size": fs,
                    "csize_dev_gibs": round(args.bytes / GIB / t_cs, 3), "uniform_dev_gibs": round(args.bytes / GIB / t_un, 3),
                    "csize_over_uniform": round(t_un / t_cs, 3), "kernel_ms": split,
                    "c_size_over_target": {"min": round(float(r.min()), 4), "p50": round(float(np.median(r)), 4),
                                           "p99": round(float(np.percentile(r, 99)), 4), "max": round(float(r.max()), 4),
                                           "below_1": int((r[:-1] < 1).sum())}}
            # host Encoder<W>: trial loop (the previous path) and the batch path, alternated
            tt, tb = [], []
            for _ in range(2):
                t = time.perf_counter(); a = trial_loop(ctx, host, target, level); tt.append(time.perf_counter() - t)
                t = time.perf_counter(); b = batch_encoder(ctx, host, target, level); tb.append(time.perf_counter() - t)
            case["host_bytes"] = len(host)
            case["host_trial_loop_gibs"] = round(len(host) / GIB / min(tt), 4)
            case["host_batch_encoder_gibs"] = round(len(host) / GIB / min(tb), 4)
            case["host_trial_loop_bytes"], case["host_batch_encoder_bytes"] = len(a), len(b)
            res["cases"].append(case)
            print(json.dumps(case), flush=True)
    res["card_after"] = card()
    txt = json.dumps(res)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(txt + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
