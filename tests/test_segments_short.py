"""Short execution segments run on one warp each (zk_exec_warp_kernel), long ones on CTAs (zk_exec_kernel); ZK_EXEC_SHORT
is the output size up to which a segment counts as short.  Under a threshold that splits the batch between both kernels,
under 0 (CTAs only) and under one that makes every segment short, the output, the per-entry status and the number of
segments must be those of the serial walk (the in-order kernel, ZK_EXEC_V2=1) and of each other.  Every case runs on the
emulation build (`-m "not gpu"`) and on the H100 (`-m gpu`)."""
import os

import numpy as np
import pytest

import zeekstd_b200 as zk
from util import decode_frames, split_frames
from zeekstd_b200 import corpus

MIX_SEED, MIX_BYTES, MIX_FRAME = 20260924, 1 << 20, 256 << 10
# 32 KiB: the level-1 mix has segments on both sides of it (one 32 KiB block, or several blocks); 1 GiB: all short
SETTINGS = {"both": 32 << 10, "cta_only": 0, "all_short": 1 << 30}


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    return request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib")


def _context(lib, env: dict):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return zk.Context(0, lib)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def ctxs(lib):
    c = {name: _context(lib, {"ZK_EXEC_SHORT": str(v)}) for name, v in SETTINGS.items()}
    c["serial"] = _context(lib, {"ZK_EXEC_V2": "1"})
    yield c
    for x in c.values():
        x.close()


@pytest.fixture(scope="module")
def archive(ctxs):
    mix = corpus.as_numpy(corpus.make_mix(MIX_BYTES, seed=MIX_SEED, segment=64 << 10))
    comp, cs, ds = ctxs["serial"].compress_frames(mix, MIX_FRAME, 1, False)
    return mix, split_frames(comp.tobytes(), cs), [int(d) for d in ds]


def _decode(ctx, frames, sizes, verify=True):
    s0 = ctx.decode_segments
    out, st, rc = decode_frames(ctx, frames, sizes, verify)
    return out, list(st), rc, ctx.decode_segments - s0


def test_every_threshold_decodes_like_the_serial_walk(ctxs, archive):
    mix, frames, sizes = archive
    segs = {}
    for name in SETTINGS:
        out, st, rc, segs[name] = _decode(ctxs[name], frames, sizes)
        assert rc == 0 and not any(st) and out == mix.tobytes(), name
    assert len(set(segs.values())) == 1 and segs["both"] > len(frames), segs     # the threshold routes segments, it never changes them


def test_failures_keep_serial_order_under_every_threshold(ctxs, archive):
    """corruption in a later segment, alone or with an earlier one too, sometimes with a wrong entry size as well"""
    _, frames, ds = archive
    rng = np.random.default_rng(11)
    checked = 0
    for trial in range(8):
        e = trial % len(frames)
        f = bytearray(frames[e])
        n = len(f)
        hits = [int(rng.integers(n // 2, n - 1))]
        if trial % 2:
            hits.append(int(rng.integers(16, n // 2)))
        for h in hits:
            f[h] ^= 1 << int(rng.integers(8))
        fr = list(frames); fr[e] = bytes(f)
        sizes = list(ds)
        if trial % 3 == 0:
            sizes[e] += 1
        _, st_ref, _, _ = _decode(ctxs["serial"], fr, sizes, False)
        for name in SETTINGS:
            _, st, _, _ = _decode(ctxs[name], fr, sizes, False)
            assert st == st_ref, (name, trial, st, st_ref)
        checked += st_ref[e] != 0
    assert checked >= 4
