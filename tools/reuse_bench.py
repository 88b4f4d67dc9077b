"""Compressing a new version against the previous archive (zk_compress_frames_sized_reuse) on the H100: the bench's 1 GiB mix as OLD, its
edited copy as NEW, content-defined frames.  Per case, the host-pointer reuse call and the full sized call on NEW's frames alternate in one
process (wall time, L2 flushed before each call, best of --runs); every reuse output is compared with the full call's.  Also the reused
fraction and the split of one reuse call into its phases (ZK_E2E_TRACE: index = pass A, match = NEW's upload, keys, candidate decode and
compare, compress = gather and compress of the changed frames, assemble = assembly and copy down).  Prints one JSON line per case, with
the card's name, power limit and SM clock read in the same call.

usage: python tools/reuse_bench.py [--bytes N] [--sizes 65536,2097152] [--modes 3,19,long] [--edits K] [--runs R] [--out FILE]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import zeekstd_b200 as zk  # noqa: E402
from golden.make_encoder_golden_ldm import edited_copy  # noqa: E402
from sized_bench import card  # noqa: E402


def seekable(comp, cs, ds) -> np.ndarray:
    st = zk.SeekTable()
    for c, d in zip(cs.tolist(), ds.tolist()):
        st.log_frame(int(c), int(d))
    return np.concatenate([comp, np.frombuffer(st.into_serializer().to_bytes(), np.uint8)])


def timed(flush: torch.Tensor, fn):
    flush.fill_(1)                                  # evict the L2 (50 MiB on the H100)
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t) * 1e3, r


def phases(fn) -> dict:
    """one call with ZK_E2E_TRACE set; its phase line read from the C library's stderr"""
    with tempfile.TemporaryFile() as f:
        saved = os.dup(2)
        sys.stderr.flush(); os.dup2(f.fileno(), 2)
        os.environ["ZK_E2E_TRACE"] = "1"
        try:
            fn()
        finally:
            del os.environ["ZK_E2E_TRACE"]
            os.dup2(saved, 2); os.close(saved)
        f.seek(0)
        line = [ln for ln in f.read().decode().splitlines() if ln.startswith("reuse ")][-1].split()
    return {line[i]: float(line[i + 1]) for i in range(1, len(line) - 1, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=1 << 30)
    ap.add_argument("--sizes", default="65536,2097152")
    ap.add_argument("--modes", default="3,19,long")
    ap.add_argument("--edits", type=int, default=64)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = zk.Context(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    old = bench.gen_mix(a.bytes, bench.SEED + 1, device="cpu").numpy()
    new = edited_copy(old, 5, a.edits)
    rows = []
    for s in [int(v) for v in a.sizes.split(",")]:
        osz, nsz = ctx.cut_frames_cdc(old, s)[0], ctx.cut_frames_cdc(new, s)[0]
        for mode in a.modes.split(","):
            level, lm = (16, True) if mode == "long" else (int(mode), False)
            comp, cs, _ = ctx.compress_frames_sized(old, osz, level, True, long_mode=lm)
            arch = seekable(comp, cs, osz)
            full_ms, reuse_ms = [], []
            for _ in range(a.runs):
                t, (fc, fcs, _) = timed(flush, lambda: ctx.compress_frames_sized(new, nsz, level, True, long_mode=lm))
                full_ms.append(t)
                t, (rc_, rcs, ru) = timed(flush, lambda: ctx.compress_frames_reuse(new, nsz, arch, level, True, lm))
                reuse_ms.append(t)
                assert rc_.tobytes() == fc.tobytes() and rcs.tolist() == fcs.tolist()
            ph = phases(lambda: ctx.compress_frames_reuse(new, nsz, arch, level, True, lm))
            row = {"frame_size": s, "mode": mode, "frames": int(nsz.size), "reused": int((ru != 0xFFFFFFFF).sum()),
                   "reused_fraction": round(float((ru != 0xFFFFFFFF).mean()), 4), "full_ms": round(min(full_ms), 1),
                   "reuse_ms": round(min(reuse_ms), 1), "phases_ms": {k: round(v, 1) for k, v in ph.items()}, "bytes": int(new.size),
                   "card": card()}
            print(json.dumps(row), flush=True)
            rows.append(row)
    if a.out:
        json.dump(rows, open(a.out, "w"), indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
