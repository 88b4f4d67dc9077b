"""Seekable patch chains: patches made and applied against v1.zst <- v2.patch <- ... <- v_d.patch, at depths 1 to 4.

    python tools/patch_chain_bench.py [--mib 384] [--frame-mib 2] [--reps 3] [--max-depth 4] [--out DIR]

v1 and v2 are tools/patch_archive_bench.py's OLD and NEW (--mib MiB of the bench's mix; NEW = OLD with 64 small edits and its first 8 MiB
moved to the end), and every further version is the same kind of edit of the one before.  v1.zst is v1 at level 3 in --frame-mib MiB
frames with checksums; v_{k+1}.patch is made against the chain under it (level 16 with checksums, --frame-mib MiB frames) and checked
byte-identical to the patch made against raw v_k.  At depth d (the chain ending at v_d.patch, or v1.zst for d = 1) it times, host clock
around synchronous calls, best of --reps after one warm-up:
  - create: Context.patch_ranges + Context.compress_frames_patch of v_{d+1} against the chain;
  - full apply: Context.decompress_frames of v_{d+1}.patch with its slices, through the chain;
  - one-frame read: the middle entry of v_{d+1}.patch alone, through the chain.
For the one-frame read it reports the entries decoded at each level (Need, DESIGN §3.4.3, restated here and checked against
Context.reference_entries_decoded) and the compressed bytes of those entries sent to the device; for the full apply the entries decoded.
Reads the card's name, power limit and SM clock in the same run.  Prints one JSON line and writes it to DIR/patch_chain_bench.json when
--out is given.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from bisect import bisect_right

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import zeekstd_b200 as zk  # noqa: E402
from zeekstd_b200 import corpus  # noqa: E402

GROUP = 1 << 30                                             # ZK_PATCH_GROUP_BYTES' default


def _best(fn, reps):
    """one warm-up, then the best of reps timed calls -> (seconds, last result)"""
    out = fn()
    best = None
    for _ in range(reps):
        t = time.perf_counter()
        out = fn()
        dt = time.perf_counter() - t
        best = dt if best is None else min(best, dt)
    return best, out


def _edit(v, seed):
    """64 overwritten 32-byte spans, then the first 8 MiB moved to the end"""
    out = v.copy()
    rng = np.random.default_rng(seed)
    for at in rng.integers(0, out.size - 64, 64):
        out[at:at + 32] = rng.integers(0, 256, 32, dtype=np.uint8)
    return np.concatenate([out[8 << 20:], out[:8 << 20]])


def _hull_groups(ranges):
    out, f0, n = [], 0, len(ranges)
    while f0 < n:
        lo = hi = 0
        any_, f = False, f0
        while f < n:
            a, b = ranges[f]
            if a == b:
                f += 1
                continue
            nlo, nhi = (min(lo, a), max(hi, b)) if any_ else (a, b)
            if f > f0 and any_ and nhi - nlo > GROUP:
                break
            lo, hi, any_ = nlo, nhi, True
            f += 1
        out.append((f0, f, lo, hi))
        f0 = f
    return out


def _need(levels, i, lo, hi, per_level):
    """Need(i, [lo, hi)): adds the entries decoded at every level to per_level[level] (a list of entry indices)"""
    r, slices = levels[i]
    d = r.d_off
    g = bisect_right(d.tolist(), lo) - 1
    lst = []
    while g < r.n_entries and int(d[g]) < hi:
        if d[g + 1] > d[g]:
            lst.append(g)
        g += 1
    if slices is not None:
        for _, _, hlo, hhi in _hull_groups([slices[g] for g in lst]):
            if hhi > hlo:
                _need(levels, i - 1, hlo, hhi, per_level)
    per_level[i] += lst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=384)
    ap.add_argument("--frame-mib", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-depth", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    ctx = zk.Context(0)
    fs = a.frame_mib << 20
    versions = [corpus.make_mix(a.mib << 20, seed=1, segment=64 << 10).numpy()]
    for k in range(a.max_depth):
        versions.append(_edit(versions[-1], 9 + k))

    def sizes_of(v):
        return np.array([min(fs, v.size - s) for s in range(0, v.size, fs)], dtype=np.uint32)

    comp1, cs1, ds1 = ctx.compress_frames(versions[0], fs, 3, True)
    table = zk.SeekTable()
    for c, d in zip(cs1.tolist(), ds1.tolist()):
        table.log_frame(c, d)
    chain = zk.ReferenceArchive(comp1.tobytes() + table.into_serializer().to_bytes())
    rows = []
    for depth in range(1, a.max_depth + 1):
        new, sizes = versions[depth], sizes_of(versions[depth])

        def make():
            rg = ctx.patch_ranges(new, sizes, chain, fs)
            return rg, ctx.compress_frames_patch(new, sizes, chain, rg, 16, True)

        t_make, (rg, (comp, cs, ds)) = _best(make, a.reps)
        patch = zk.patch_slices_write(chain.old_len, rg)
        st = zk.SeekTable()
        for f, (c, d) in enumerate(zip(cs.tolist(), ds.tolist())):
            st.log_frame(c + (len(patch) if f == 0 else 0), d)
        patch_bytes = patch + comp.tobytes() + st.into_serializer().to_bytes()
        identical = patch_bytes == ctx.compress_patch_slices(new, sizes, versions[depth - 1], 16, True, fs)
        pad = np.concatenate([comp, np.zeros(64, np.uint8)])
        co = np.concatenate([[0], np.cumsum(cs, dtype=np.uint64)]).astype(np.uint64)
        do = np.concatenate([[0], np.cumsum(ds, dtype=np.uint64)]).astype(np.uint64)
        out = np.empty(new.size + 64, np.uint8)
        dec0 = ctx.reference_entries_decoded
        t_apply, rc = _best(lambda: ctx.decompress_frames(pad, co, do, True, out=out, prefix=chain, prefix_ranges=rg)[2], a.reps)
        apply_entries = (ctx.reference_entries_decoded - dec0) // (a.reps + 1)
        restored = rc == 0 and out[:new.size].tobytes() == new.tobytes()

        f = len(sizes) // 2
        lo, hi = (int(v) for v in rg[f])
        one = np.concatenate([comp[int(co[f]):int(co[f + 1])], np.zeros(64, np.uint8)])
        dec0 = ctx.reference_entries_decoded
        t_one, (back, _, rc1) = _best(lambda: ctx.decompress_frames(one, [0, int(cs[f])], [0, int(ds[f])], True, prefix=chain,
                                                                    prefix_ranges=rg[f:f + 1]), a.reps)
        one_entries = (ctx.reference_entries_decoded - dec0) // (a.reps + 1)
        levels = [(r, None if r.base is None else zk.patch_slices_read(r._keep[0] if isinstance(r._keep, tuple) else r._keep,
                                                                        r.n_entries)[1].tolist()) for r in chain.chain]
        per_level = [[] for _ in levels]
        if hi > lo:
            _need(levels, depth - 1, lo, hi, per_level)
        restored = restored and rc1 == 0 and back[:int(ds[f])].tobytes() == new[int(do[f]):int(do[f + 1])].tobytes()
        rows.append({
            "depth": depth, "patch_bytes": len(patch_bytes), "patch_identical_to_raw": bool(identical), "restored": bool(restored),
            "create_ms": round(t_make * 1e3, 1), "apply_ms": round(t_apply * 1e3, 1), "one_frame_ms": round(t_one * 1e3, 2),
            "apply_entries_decoded": int(apply_entries),
            "one_frame_entries_decoded": int(one_entries),
            "one_frame_entries_per_level": [len(x) for x in per_level],
            "one_frame_model_matches": sum(len(x) for x in per_level) == one_entries,
            "one_frame_reference_bytes_to_device": int(sum(int(r.c_off[g + 1] - r.c_off[g]) for (r, _), lst in zip(levels, per_level)
                                                           for g in lst)),
            "one_frame_slice_bytes": hi - lo,
        })
        chain = zk.ReferenceArchive(patch_bytes, base=chain)
    r = {"gpu": gpu, "version_mib": a.mib, "frame_mib": a.frame_mib, "entries_per_version": int(len(cs1)), "depths": rows}
    line = json.dumps(r)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "patch_chain_bench.json"), "w") as fh:
            fh.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
