"""Long mode (zk_compress_frames_long_dev) against level 16 (zk_compress_frames_dev) on one H100: device-resident calls alternated in one
process (CUDA events, L2 flushed before every call, every output restored), on
  mix       the bench's 1 GiB class mix, in 64 MiB frames;
  backup    256 MiB of the mix followed by an edited copy of it, in 64 MiB, 256 MiB and 1 GiB frames;
  near      64 MiB of the mix followed by an edited copy of it, in 128 MiB frames (a repeat within the 2^27 window).
Per case: ratio, GiB/s (best of --runs) and, from a separate torch.profiler run, the device time of every kernel, so that the input index
(zk_ldm_index_input_kernel, zk_ldm_check_kernel and the extra sort rounds), zk_ldm_find_kernel and zk_hc_parse_kernel can be read off.
Prints one JSON line per case, with the card's name, power limit and SM clock read in the same call.

--libzstd (CPU only, no GPU needed): libzstd's size at level 16 with windowLog 27 and long-distance matching (`zstd --long=27 -16`), one
frame at a time on the same frames, single-threaded (nbWorkers = 0: multithreaded libzstd cuts a large frame into overlapping jobs and
writes other bytes), for reference.

usage: python tools/long_bench.py [--cases mix,backup,near] [--runs R] [--libzstd] [--out FILE]"""
import argparse
import ctypes
import json
import os
import sys
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
from golden.make_encoder_golden_ldm import edited_copy  # noqa: E402
from oracle import oracle as O  # noqa: E402

LEVEL = 16


def inputs(name: str):
    """-> [(label, input as np.uint8, frame size)]"""
    if name == "mix":
        return [("mix_1GiB_f64M", bench.gen_mix(1 << 30, bench.SEED, device="cpu").numpy(), 64 << 20)]
    if name == "backup":
        a = bench.gen_mix(256 << 20, bench.SEED + 2, device="cpu").numpy()
        x = np.concatenate([a, edited_copy(a, 3, 1000)])
        return [(f"backup_512MiB_f{fs >> 20}M", x, fs) for fs in (64 << 20, 256 << 20, 1 << 30)]
    if name == "near":
        a = bench.gen_mix(64 << 20, bench.SEED + 4, device="cpu").numpy()
        return [("near_128MiB_f128M", np.concatenate([a, edited_copy(a, 5, 300)]), 128 << 20)]
    raise ValueError(name)


def libzstd_size(x: np.ndarray, fs: int) -> int:
    z = ctypes.CDLL(os.environ.get("ZK_LIBZSTD", O.SYSTEM_LIBZSTD))
    z.ZSTD_createCCtx.restype = ctypes.c_void_p
    z.ZSTD_CCtx_setParameter.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]; z.ZSTD_CCtx_setParameter.restype = ctypes.c_size_t
    z.ZSTD_compress2.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t]; z.ZSTD_compress2.restype = ctypes.c_size_t
    z.ZSTD_compressBound.argtypes = [ctypes.c_size_t]; z.ZSTD_compressBound.restype = ctypes.c_size_t
    z.ZSTD_isError.argtypes = [ctypes.c_size_t]
    c = z.ZSTD_createCCtx()
    for param, v in ((100, LEVEL), (101, 27), (160, 1), (400, 0)):   # level, windowLog, LDM, nbWorkers (0: single-threaded)
        assert not z.ZSTD_isError(z.ZSTD_CCtx_setParameter(c, param, v)), param
    dst = np.empty(z.ZSTD_compressBound(fs) + 64, np.uint8)
    total = 0
    for lo in range(0, x.size, fs):
        fr = np.ascontiguousarray(x[lo:lo + fs])
        r = z.ZSTD_compress2(c, dst.ctypes.data, dst.size, fr.ctypes.data, fr.size)
        assert not z.ZSTD_isError(r)
        total += r
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="mix,backup,near")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--libzstd", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    outf = open(args.out, "a") if args.out else None

    def emit(d):
        print(json.dumps(d), flush=True)
        if outf:
            outf.write(json.dumps(d) + "\n"); outf.flush()

    if args.libzstd:
        for name in args.cases.split(","):
            for label, x, fs in inputs(name):
                emit({"case": label, "bytes": int(x.size), "libzstd_long27_l16_bytes": libzstd_size(x, fs)})
        return

    import zeekstd_b200 as zk
    from sized_bench import Runner, bench_offsets, card
    from zeekstd_b200 import _native
    assert torch.cuda.is_available(), "long_bench measures the GPU: no CPU fallback"
    ctx = zk.Context(0)
    lib = ctx.lib
    dev_card = card()
    for name in args.cases.split(","):
        for label, xh, fs in inputs(name):
            n = xh.size
            x = torch.cat([torch.from_numpy(xh), torch.zeros(64, dtype=torch.uint8)]).cuda()
            r = Runner(ctx, x)

            def call(long_mode):
                fn = lib.zk_compress_frames_long_dev if long_mode else lib.zk_compress_frames_dev

                def go(stream):
                    nfmax = n // fs + 2
                    cs = np.zeros(nfmax, np.uint32); ds = np.zeros(nfmax, np.uint32); k = ctypes.c_uint32(); dl = ctypes.c_size_t()
                    rc = fn(ctx._h, x.data_ptr(), n, fs, LEVEL, 0, r.dst.data_ptr(), r.dst.numel(), cs.ctypes.data_as(_native.u32p),
                            ds.ctypes.data_as(_native.u32p), nfmax, ctypes.byref(k), ctypes.byref(dl), stream)
                    assert rc == 0, rc
                    return cs[: k.value], ds[: k.value], int(dl.value)
                return r._timed(go)

            res = {"case": label, "bytes": n, "frame_size": fs, "level": LEVEL, "card": dev_card}
            ms = {False: [], True: []}
            size = {}
            for _ in range(args.runs):
                for lm in (False, True):
                    t, (cs, ds, total) = call(lm)
                    ms[lm].append(round(t, 3)); size[lm] = total
                    r.check(0, n, cs, ds, total)
            for lm, key in ((False, "level16"), (True, "long_mode")):
                res[key] = {"bytes": size[lm], "ratio": round(n / size[lm], 4), "ms": ms[lm], "gib_s": round(n / (1 << 30) / (min(ms[lm]) / 1e3), 2)}
            # the kernels of one call of each, in a run of their own
            for lm, key in ((False, "level16"), (True, "long_mode")):
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    call(lm)
                    torch.cuda.synchronize()
                k = defaultdict(float)
                for ev in prof.key_averages():
                    if ev.device_time_total > 0:
                        k[ev.key.split("(")[0].split("<")[0]] += ev.device_time_total / 1e3
                res[key]["kernels_ms"] = {kk: round(v, 3) for kk, v in sorted(k.items(), key=lambda kv: -kv[1]) if v >= 0.05}
            emit(res)
            del r, x
            torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
