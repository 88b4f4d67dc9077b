"""Shared helpers for the parity tests (both the emulated CPU build and the real sm_90a build)."""
from __future__ import annotations

import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def golden_meta():
    return json.load(open(os.path.join(GOLDEN, "golden.json")))


def golden_bytes(name: str) -> bytes:
    return open(os.path.join(GOLDEN, name), "rb").read()


def make_ctx(lib):
    import zeekstd_b200 as zk
    from zeekstd_b200 import _native
    _native.set_default_lib(lib)
    return zk.Context(0, lib)


def offsets(sizes):
    o = np.zeros(len(sizes) + 1, dtype=np.uint64)
    o[1:] = np.cumsum(np.asarray(sizes, dtype=np.uint64))
    return o


def decode_frames(ctx, frames, d_sizes, verify=True):
    """decode a list of compressed frames with the codec under test -> (bytes, statuses, rc)"""
    comp = np.frombuffer(b"".join(frames) + b"\0" * 64, dtype=np.uint8)
    out, st, rc = ctx.decompress_frames(comp, offsets([len(f) for f in frames]), offsets(d_sizes), verify)
    return out.tobytes(), st, rc


def split_frames(comp: bytes, c_sizes):
    out, pos = [], 0
    for c in c_sizes:
        out.append(comp[pos:pos + int(c)]); pos += int(c)
    return out
