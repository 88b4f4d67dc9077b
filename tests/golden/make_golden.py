"""Generates the committed golden fixtures from the reference's own corpus (assets/dickens.txt) and the real
libzstd of the system (oracle/libzstd_driver.c replaying the reference's call sequence), from the corpus as committed
next to this script:   python tests/golden/make_golden.py
"""
import hashlib, json, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
d = np.fromfile(os.path.join(HERE, "dickens.txt"), dtype=np.uint8)
meta = {"libzstd": O.libzstd_version(), "dickens_bytes": int(d.size), "dickens_sha256": hashlib.sha256(d.tobytes()).hexdigest()}

# known answers on the full corpus (BASELINE config 1): frame sizes per level / frame size
for name, fs, lvl, ck in [("l1_2m", 0x200000, 1, False), ("l3_2m_ck", 0x200000, 3, True), ("l1_512k", 512 << 10, 1, False)]:
    frames, cs, ds = O.ref_compress_frames(d, fs, lvl, ck)
    meta[name] = {"c_sizes": cs, "d_sizes": ds, "sha256_frames": hashlib.sha256(b"".join(frames)).hexdigest(),
                  "stats": O.frame_stats(b"".join(frames))}

# small committed fixtures: a 96 KiB slice and archives of it
sl = d[1_000_000: 1_000_000 + 96 * 1024]
sl.tofile(os.path.join(HERE, "dickens_96k.txt"))
meta["slice"] = {"offset": 1_000_000, "bytes": int(sl.size), "sha256": hashlib.sha256(sl.tobytes()).hexdigest()}
arch = {}
for name, fs, lvl, ck in [("dickens_96k_l1_f32k", 32 << 10, 1, False), ("dickens_96k_l3_f96k_ck", 96 << 10, 3, True),
                          ("dickens_96k_l9_f20000_ck", 20000, 9, True), ("dickens_96k_l19_f96k", 96 << 10, 19, False),
                          ("dickens_4k_l3_f100", 100, 3, False)]:
    src = sl[:4096] if "4k" in name else sl
    a, st = O.ref_seekable_archive(src, fs, lvl, ck)
    open(os.path.join(HERE, name + ".zst"), "wb").write(a)
    arch[name] = {"frame_size": fs, "level": lvl, "checksum": ck, "bytes": len(a), "src_bytes": int(src.size), "num_frames": st.num_frames(),
                  "sha256": hashlib.sha256(a).hexdigest(), "stats": O.frame_stats(a[: st.c[-1]])}
meta["archives"] = arch
# XXH64 known answers
meta["xxh64"] = {"empty": O.oracle_xxh64(b""), "a": O.oracle_xxh64(b"a"), "slice": O.oracle_xxh64(sl), "slice_1000": O.oracle_xxh64(sl[:1000])}
json.dump(meta, open(os.path.join(HERE, "golden.json"), "w"), indent=1)
print(json.dumps({k: v for k, v in meta.items() if k not in ("archives",)}, indent=1)[:1500])
print({k: (v["bytes"], v["num_frames"]) for k, v in arch.items()})
