"""Seekable patches against the reference as raw bytes (v1) and as a seekable archive (v1.zst) on one NEW / OLD pair.

    python tools/patch_archive_bench.py [--mib 384] [--frame-mib 2] [--reps 3] [--out DIR]

OLD is --mib MiB of the bench's mix, NEW is OLD with 64 small edits and its first 8 MiB moved to the end (tools/patch_slices_bench.py's
pair), and v1.zst is OLD written by this codec at level 3 in --frame-mib MiB frames with checksums.  For each reference it times patch
creation (Context.patch_ranges + Context.compress_frames_patch, level 16 with checksums) and a full apply (Context.decompress_frames with
the slices), host clock around synchronous calls, best of --reps after one warm-up, the two references alternated rep by rep.  For a
one-frame read it reports the reference bytes sent to the device (raw: the prefix bytes uploaded; archive: the compressed bytes of the
entries decoded) and the entries of v1.zst decoded.  It checks that both patches are the same bytes and that every apply is exact.
Prints one JSON line and writes it to DIR/patch_archive_bench.json when --out is given.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import zeekstd_b200 as zk  # noqa: E402
from zeekstd_b200 import corpus  # noqa: E402


def _timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def _alternate(fns, reps):
    """one warm-up of each, then reps rounds of every fn in turn -> (best seconds per fn, last result per fn)"""
    outs = [fn() for fn in fns]
    best = [None] * len(fns)
    for _ in range(reps):
        for i, fn in enumerate(fns):
            dt, outs[i] = _timed(fn)
            best[i] = dt if best[i] is None else min(best[i], dt)
    return best, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=384)
    ap.add_argument("--frame-mib", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    ctx = zk.Context(0)
    n = a.mib << 20
    old = corpus.make_mix(n, seed=1, segment=64 << 10).numpy()
    new = old.copy()
    rng = np.random.default_rng(9)
    for at in rng.integers(0, n - 64, 64):
        new[at:at + 32] = rng.integers(0, 256, 32, dtype=np.uint8)
    new = np.concatenate([new[8 << 20:], new[:8 << 20]])
    fs = a.frame_mib << 20
    sizes = np.array([min(fs, new.size - s) for s in range(0, new.size, fs)], dtype=np.uint32)
    gib = 1 << 30

    comp1, cs1, ds1 = ctx.compress_frames(old, fs, 3, True)
    table = zk.SeekTable()
    for c, d in zip(cs1.tolist(), ds1.tolist()):
        table.log_frame(c, d)
    v1zst = comp1.tobytes() + table.into_serializer().to_bytes()
    ref = zk.ReferenceArchive(v1zst)

    def make(reference):
        rg = ctx.patch_ranges(new, sizes, reference, fs)
        return rg, ctx.compress_frames_patch(new, sizes, reference, rg, 16, True)

    (t_make_raw, t_make_arc), ((rg, (comp, cs, ds)), (rg_a, (comp_a, cs_a, _))) = _alternate([lambda: make(old), lambda: make(ref)], a.reps)
    identical = rg.tolist() == rg_a.tolist() and comp.tobytes() == comp_a.tobytes() and cs.tolist() == cs_a.tolist()
    pad = np.concatenate([comp, np.zeros(64, np.uint8)])
    co = np.concatenate([[0], np.cumsum(cs, dtype=np.uint64)]).astype(np.uint64)
    do = np.concatenate([[0], np.cumsum(ds, dtype=np.uint64)]).astype(np.uint64)
    out_r, out_a = np.empty(new.size + 64, np.uint8), np.empty(new.size + 64, np.uint8)
    (t_apply_raw, t_apply_arc), (rc_r, rc_a) = _alternate(
        [lambda: ctx.decompress_frames(pad, co, do, True, out=out_r, prefix=old, prefix_ranges=rg)[2],
         lambda: ctx.decompress_frames(pad, co, do, True, out=out_a, prefix=ref, prefix_ranges=rg)[2]], a.reps)
    applied = rc_r == 0 and rc_a == 0 and out_r[: new.size].tobytes() == new.tobytes() and out_a[: new.size].tobytes() == new.tobytes()

    f = len(sizes) // 2
    lo, hi = (int(v) for v in rg[f])
    one = np.concatenate([comp[int(co[f]):int(co[f + 1])], np.zeros(64, np.uint8)])
    before = ctx.prefix_bytes_uploaded
    back_r, _, rc1 = ctx.decompress_frames(one, [0, int(cs[f])], [0, int(ds[f])], True, prefix=old, prefix_ranges=rg[f:f + 1])
    raw_upload = ctx.prefix_bytes_uploaded - before
    before, dec0 = ctx.prefix_bytes_uploaded, ctx.reference_entries_decoded
    back_a, _, rc2 = ctx.decompress_frames(one, [0, int(cs[f])], [0, int(ds[f])], True, prefix=ref, prefix_ranges=rg[f:f + 1])
    decoded = ctx.reference_entries_decoded - dec0
    under = [g for g in range(ref.n_entries) if ref.d_off[g] < hi and ref.d_off[g + 1] > lo and ref.d_off[g + 1] > ref.d_off[g]]
    arc_upload = int(sum(int(ref.c_off[g + 1] - ref.c_off[g]) for g in under))
    want = new[int(do[f]):int(do[f + 1])].tobytes()
    r = {
        "gpu": gpu, "old_mib": a.mib, "frame_mib": a.frame_mib, "frames": int(len(sizes)), "v1_zst_bytes": len(v1zst),
        "v1_ratio": round(old.size / comp1.size, 3), "patch_bytes": int(comp.size + zk.patch_slices_size(len(sizes))),
        "create_ms_raw": round(t_make_raw * 1e3, 1), "create_ms_archive": round(t_make_arc * 1e3, 1),
        "create_gibps_raw": round(new.size / gib / t_make_raw, 3), "create_gibps_archive": round(new.size / gib / t_make_arc, 3),
        "apply_ms_raw": round(t_apply_raw * 1e3, 1), "apply_ms_archive": round(t_apply_arc * 1e3, 1),
        "apply_gibps_raw": round(new.size / gib / t_apply_raw, 3), "apply_gibps_archive": round(new.size / gib / t_apply_arc, 3),
        "one_frame_slice_bytes": hi - lo, "one_frame_upload_bytes_raw": int(raw_upload), "one_frame_upload_bytes_archive": arc_upload,
        "one_frame_prefix_bytes_uploaded_archive": int(ctx.prefix_bytes_uploaded - before),
        "one_frame_entries_decoded": int(decoded), "one_frame_entries_under_slice": len(under),
        "patches_identical": bool(identical), "restored": bool(applied and rc1 == 0 and rc2 == 0 and back_r[: len(want)].tobytes() == want
                                                                 and back_a[: len(want)].tobytes() == want),
    }
    line = json.dumps(r)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "patch_archive_bench.json"), "w") as fh:
            fh.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
