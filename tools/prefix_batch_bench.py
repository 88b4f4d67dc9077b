"""Per-frame prefixes on the H100: N objects, each compressed against its own old version, in one batch call against N single-frame calls.

Object i is a 1 MiB slice of the bench's mix; its old version is the same slice with a few in-place edits of the same length.  The batch call
is zk_compress_frames_sized_prefixes / zk_decompress_frames_prefixes with the old versions back to back as the prefix buffer and object i's
range over its own old version; the single calls are zk_compress_frames_sized(_ldm) / zk_decompress_frames_prefix with that old version as
the prefix, which is how such a batch is made without per-frame prefixes (one upload of the prefix per call).  Compression runs at level 3
and at level 16 with long-distance matching; the batch call's frames are byte-equal to the single calls' (checked every round).

Timing: host-pointer calls (the prefix paths have no device entry points) with a host clock around each synchronous call; the L2 is flushed
before every call, outside the clock; the variants alternate within each round; every round trip is checked.  The card's name and power
limit are read (read-only nvidia-smi query) in the same call.  Prints one JSON line per round and one with the medians.

usage: python tools/prefix_batch_bench.py [--objects 256] [--kib 1024] [--rounds 3] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--objects", type=int, default=256)
    ap.add_argument("--kib", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import zeekstd_b200 as zk
    from zeekstd_b200 import corpus
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the H100 only")
    ctx = zk.Context(0)
    n_obj, size = args.objects, args.kib << 10
    new = corpus.as_numpy(corpus.make_mix(n_obj * size, seed=51, segment=16 << 10)).copy()
    old = new.copy()
    rng = np.random.default_rng(52)
    for at in rng.integers(0, old.size - 64, n_obj * 8):
        old[at:at + 32] = rng.integers(0, 256, 32, dtype=np.uint8)
    sizes = [size] * n_obj
    ranges = np.array([(i * size, (i + 1) * size) for i in range(n_obj)], dtype=np.uint64)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")          # larger than the 50 MB L2

    def timed(fn):
        flush.fill_(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        return (time.perf_counter() - t0) * 1e3, r

    def compress_batch(level, ldm):
        return timed(lambda: ctx.compress_frames_sized(new, sizes, level, True, prefix=old, long_distance=ldm, prefix_ranges=ranges))

    def compress_single(level, ldm):
        ms, parts = 0.0, []
        for i in range(n_obj):
            t, r = timed(lambda: ctx.compress_frames_sized(new[i * size:(i + 1) * size], [size], level, True, prefix=old[i * size:(i + 1) * size],
                                                           long_distance=ldm))
            ms += t; parts.append(r[0])
        return ms, parts

    def offsets(cs):
        o = np.zeros(len(cs) + 1, np.uint64); o[1:] = np.cumsum(np.asarray(cs, np.uint64)); return o

    info = card()
    rows = []
    out = np.empty(new.size + 64, np.uint8)
    for rnd in range(args.rounds):
        row = {"round": rnd}
        for level, ldm in ((3, False), (16, True)):
            tag = f"L{level}{'_ldm' if ldm else ''}"
            order = ("batch", "single") if rnd % 2 == 0 else ("single", "batch")
            res = {}
            for v in order:
                res[v] = compress_batch(level, ldm) if v == "batch" else compress_single(level, ldm)
            ms_b, (comp, cs, ds) = res["batch"]
            ms_s, parts = res["single"]
            co = offsets(cs)
            assert all(comp[int(co[i]):int(co[i + 1])].tobytes() == parts[i].tobytes() for i in range(n_obj)), tag
            row[f"compress_{tag}_batch_ms"] = round(ms_b, 2); row[f"compress_{tag}_single_ms"] = round(ms_s, 2)
            row[f"ratio_{tag}"] = round(new.size / comp.size, 2)
            # decompress: one batch call against one call per object with its old version as the prefix
            pad = np.concatenate([comp, np.zeros(64, np.uint8)])
            do = offsets(ds)
            dres = {}
            for v in order:
                if v == "batch":
                    t, (back, st, rc) = timed(lambda: ctx.decompress_frames(pad, co, do, True, out=out, prefix=old, prefix_ranges=ranges))
                    assert rc == 0 and np.array_equal(back[: new.size], new), tag
                    dres[v] = t
                else:
                    t_all = 0.0
                    for i in range(n_obj):
                        one = np.concatenate([parts[i], np.zeros(64, np.uint8)])
                        t, (back, st, rc) = timed(lambda: ctx.decompress_frames(one, [0, parts[i].size], [0, size], True,
                                                                                 prefix=old[i * size:(i + 1) * size]))
                        assert rc == 0 and np.array_equal(back[:size], new[i * size:(i + 1) * size]), (tag, i)
                        t_all += t
                    dres[v] = t_all
            row[f"decompress_{tag}_batch_ms"] = round(dres["batch"], 2); row[f"decompress_{tag}_single_ms"] = round(dres["single"], 2)
        print(json.dumps(row), flush=True)
        rows.append(row)
    med = {k: float(np.median([r[k] for r in rows])) for k in rows[0] if k != "round"}
    summary = {"card": info, "objects": n_obj, "object_bytes": size, "rounds": args.rounds, "median": med}
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"rounds": rows, **summary}, f, indent=1)


if __name__ == "__main__":
    main()
