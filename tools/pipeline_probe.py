"""How much of each device-resident stage is fill and drain: the bench's 1 GiB mix in 2 MiB frames, compressed and decompressed through
zk_compress_frames_dev / zk_decompress_frames_dev at level 1 and at level 3 with checksum, with ZK_DEV_SUB_BYTES swept over 64 MiB ... 1 GiB
(the sub-batches of one call run as the build runs them).  Every call starts with an L2 flush and is timed by the context's CUDA events
(zk_ctx_last_device_ms); its per-stage times come from zk_ctx_profile.  The settings are alternated round-robin and every round trip is
checked.

For each stage the median times are fitted as  t = a * bytes + b * sub_batches  (bytes is the same for every setting, so a * bytes is the
intercept of a line in the sub-batch count): b is what each sub-batch's stage pays whatever its size -- its fill and drain.  The sum of the
b's over a direction's chain is the most that overlapping the sub-batches of a call can win at that count.  The card's name, power limit and
SM clock are read (read-only nvidia-smi queries) in the same call.  Prints one JSON object; --out also writes it.

--slots sweeps the pipelined calls as well (ZK_DEV_SLOTS sub-batches in flight); the fits are made of the one-slot rows, where the
sub-batches run one after another.

usage: python tools/pipeline_probe.py [--bytes N] [--subs 64,128,256,512,1024] [--slots 1] [--levels 1,3c] [--reps 5] [--out FILE]"""
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

MIB = 1 << 20
FRAME = bench.FRAME
SLOTS = ["K-D0 scan", "K-D1s seq", "K-D1h huf", "K-D1p+K-D2 exec", "xxh64", "K-C1 match", "K-C2 entropy", "K-C3 frame"]   # zk_ctx_profile
COMPRESS, DECOMPRESS = (5, 6, 7), (0, 1, 2, 3, 4)


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def subs_of(n: int, sub: int) -> int:
    """sub-batches zk_next_sub / ZkFrames::next_sub cut n bytes of whole 2 MiB frames into"""
    per = max(1, sub // FRAME)
    return -(-(-(-n // FRAME)) // per)


class Call:
    def __init__(self, lib, ctx, x, flush):
        self.lib, self.ctx, self.x, self.n, self.flush = lib, ctx, x, x.numel(), flush
        self.src = torch.cat([x, torch.zeros(64, dtype=torch.uint8, device=x.device)])
        self.cap = lib.zk_compress_bound(self.n, FRAME)
        self.comp = torch.zeros(self.cap + 64, dtype=torch.uint8, device=x.device)
        self.back = torch.zeros(self.n + 64, dtype=torch.uint8, device=x.device)
        self.nfmax = self.n // FRAME + 2
        self.cs = np.zeros(self.nfmax, dtype=np.uint32); self.ds = np.zeros(self.nfmax, dtype=np.uint32)
        torch.cuda.synchronize()

    def prof(self):
        ms = (ctypes.c_float * 8)(); cnt = (ctypes.c_uint32 * 8)()
        self.lib.zk_ctx_profile_read(self.ctx._h, ms, cnt)
        self.lib.zk_ctx_profile(self.ctx._h, 1)
        return [float(v) for v in ms]

    def __call__(self, level: int, checksum: bool):
        """-> (compress ms, compress stage ms, decompress ms, decompress stage ms, compressed bytes)"""
        lib, ctx = self.lib, self.ctx
        nf, dl = ctypes.c_uint32(), ctypes.c_size_t()
        self.flush.fill_(1); torch.cuda.synchronize(); self.prof()
        rc = lib.zk_compress_frames_dev(ctx._h, self.src.data_ptr(), self.n, FRAME, level, int(checksum), self.comp.data_ptr(), self.cap,
                                        self.cs.ctypes.data_as(N.u32p), self.ds.ctypes.data_as(N.u32p), self.nfmax, ctypes.byref(nf),
                                        ctypes.byref(dl), None)
        assert rc == 0, rc
        tc, pc = ctx.last_device_ms, self.prof()
        k = nf.value
        co = np.zeros(k + 1, dtype=np.uint64); co[1:] = np.cumsum(self.cs[:k])
        do = np.zeros(k + 1, dtype=np.uint64); do[1:] = np.cumsum(self.ds[:k])
        self.flush.fill_(1); torch.cuda.synchronize(); self.prof()
        rc = lib.zk_decompress_frames_dev(ctx._h, self.comp.data_ptr(), co.ctypes.data_as(N.u64p), do.ctypes.data_as(N.u64p), k,
                                          self.back.data_ptr(), int(checksum), None, None)
        assert rc == 0, rc
        td, pd = ctx.last_device_ms, self.prof()
        assert torch.equal(self.back[: self.n], self.x), "round trip mismatch"
        return tc, pc, td, pd, int(co[-1])


def fit(ks, ts):
    """least squares t = c + b * k -> (c, b)"""
    b, c = np.polyfit(np.asarray(ks, float), np.asarray(ts, float), 1)
    return float(c), float(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=bench.WORKLOAD_BYTES)
    ap.add_argument("--subs", default="64,128,256,512,1024", help="ZK_DEV_SUB_BYTES settings in MiB")
    ap.add_argument("--slots", default="1", help="ZK_DEV_SLOTS settings")
    ap.add_argument("--levels", default="1,3c", help="levels; a trailing c: with checksum")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    settings = sorted({(int(s) * MIB, int(k)) for k in args.slots.split(",") for s in args.subs.split(",")}, key=lambda t: (t[1], t[0]))
    dev = torch.device("cuda", 0)
    lib = N.load()
    ctx = zk.Context(0, lib)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    x = bench.gen_mix(args.bytes, bench.SEED, device=dev)
    call = Call(lib, ctx, x, flush)
    lib.zk_ctx_profile(ctx._h, 1)
    res = {"card": card(), "bytes": args.bytes, "frame": FRAME, "reps": args.reps, "configs": {}}
    def use(st):
        os.environ["ZK_DEV_SUB_BYTES"], os.environ["ZK_DEV_SLOTS"] = (str(v) for v in st)

    for lv in args.levels.split(","):
        level, ck = int(lv.rstrip("c")), lv.endswith("c")
        rows = {st: [] for st in settings}
        for st in settings:                                 # warm every setting (workspaces grow to the largest)
            use(st)
            call(level, ck)
        for _ in range(args.reps):
            for st in settings:
                use(st)
                rows[st].append(call(level, ck))
        table = []
        for st in settings:
            r = rows[st]
            table.append({"sub_MiB": st[0] // MIB, "slots": st[1], "sub_batches": subs_of(args.bytes, st[0]),
                          "compress_ms": float(np.median([v[0] for v in r])), "decompress_ms": float(np.median([v[2] for v in r])),
                          "compress_ms_range": [min(v[0] for v in r), max(v[0] for v in r)],
                          "decompress_ms_range": [min(v[2] for v in r), max(v[2] for v in r)],
                          "stage_ms": {SLOTS[i]: float(np.median([(v[1][i] if i in COMPRESS else v[3][i]) for v in r])) for i in range(8)},
                          "compressed_bytes": r[-1][4]})
        serial = [t for t in table if t["slots"] == 1]
        best = {d: min(table, key=lambda t: t[f"{d}_ms"]) for d in ("compress", "decompress")}
        cfg = res["configs"][f"level {level}" + (" + checksum" if ck else "")] = {
            "table": table, "best": {d: {k: best[d][k] for k in ("sub_MiB", "slots", f"{d}_ms")} for d in best}}
        ks = [t["sub_batches"] for t in serial]
        if len(set(ks)) < 2 or 1 not in ks:
            continue
        fits = {}
        for name in SLOTS:
            c, b = fit(ks, [t["stage_ms"][name] for t in serial])
            fits[name] = {"a_bytes_ms": round(c, 3), "b_per_sub_ms": round(b, 4)}
        for d in ("compress", "decompress"):
            c, b = fit(ks, [t[f"{d}_ms"] for t in serial])
            fits[f"{d} call"] = {"a_bytes_ms": round(c, 3), "b_per_sub_ms": round(b, 4)}
        one = next(t for t in serial if t["sub_batches"] == 1)
        step = one["compress_ms"] + one["decompress_ms"]
        chain_c = sum(fits[SLOTS[i]]["b_per_sub_ms"] for i in COMPRESS)
        chain_d = sum(fits[SLOTS[i]]["b_per_sub_ms"] for i in (0, 1, 3, 4) if not (i == 4 and not ck))   # K-D1h runs beside K-D1s
        cfg.update({
            "fits": fits,
            "sum_b_compress_ms": round(chain_c, 4), "sum_b_decompress_ms": round(chain_d, 4),
            "step_ms_one_sub": round(step, 3), "sum_b_share_of_step": round((chain_c + chain_d) / step, 4)})
    res["card_after"] = card()
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
