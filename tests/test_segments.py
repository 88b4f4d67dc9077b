"""Execution segments (K-D1p / K-D2): a seek-table entry is run as several independent runs of blocks when its sequences
allow it.  Every case runs on the emulation build (`-m "not gpu"`) and on the H100 (`-m gpu`); `ctx.decode_segments`
counts the segments the decoder ran, so splitting is asserted, not hoped for."""
import os

import numpy as np
import pytest

import zeekstd_b200 as zk
from oracle import oracle as O
from util import decode_frames, make_ctx, offsets, split_frames
from zeekstd_b200 import _native, corpus

# A level-1 archive of the bench generator (64 KiB class pieces, 256 KiB frames).  This seed's archive has blocks whose
# matches read into the block before them (they cannot start a segment) beside blocks that read nothing before their own
# first byte, so it splits into more segments than entries but fewer than blocks.
MIX_SEED, MIX_BYTES, MIX_FRAME = 20260924, 1 << 20, 256 << 10


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def ctx(request):
    lib = request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib")
    c = make_ctx(lib)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx_serial(ctx):
    """the same build with the in-order exec kernel, which walks every entry serially as one unit"""
    os.environ["ZK_EXEC_V2"] = "1"
    try:
        c = zk.Context(0, ctx.lib)
    finally:
        del os.environ["ZK_EXEC_V2"]
    yield c
    c.close()


@pytest.fixture(scope="module")
def mix():
    return corpus.as_numpy(corpus.make_mix(MIX_BYTES, seed=MIX_SEED, segment=64 << 10))


def _decode(ctx, frames, ds, verify=True):
    s0 = ctx.decode_segments
    out, st, rc = decode_frames(ctx, frames, ds, verify)
    return out, st, rc, ctx.decode_segments - s0


def _blocks(frames) -> int:
    return sum(sum(O.frame_stats(f)[k] for k in ("n_raw", "n_rle", "n_comp")) for f in frames)


def test_level1_mix_splits(ctx, mix):
    comp, cs, ds = ctx.compress_frames(mix, MIX_FRAME, 1, False)
    frames = split_frames(comp.tobytes(), cs)
    out, st, rc, segs = _decode(ctx, frames, ds)
    assert rc == 0 and not st.any() and out == mix.tobytes()
    assert len(frames) < segs < _blocks(frames), (len(frames), segs)


def test_level3_and_libzstd_archives(ctx, mix):
    text = corpus.make_class("text", MIX_BYTES, seed=3).numpy()
    comp, cs, ds = ctx.compress_frames(text, MIX_FRAME, 3, True)
    frames = split_frames(comp.tobytes(), cs)
    out, st, rc, segs = _decode(ctx, frames, ds)
    assert rc == 0 and out == text.tobytes()
    assert segs == len(frames)                     # from level 2 on the encoder's blocks search the block before them: text always finds matches there
    comp, cs, ds = ctx.compress_frames(mix, MIX_FRAME, 3, True)
    out, st, rc, segs = _decode(ctx, split_frames(comp.tobytes(), cs), ds)
    assert rc == 0 and out == mix.tobytes() and segs >= len(cs)                 # blocks after random or run pieces may still split
    frames, cs, ds = O.ref_compress_frames(mix, MIX_FRAME, 3, True)
    out, st, rc, segs = _decode(ctx, frames, ds)
    assert rc == 0 and out == mix.tobytes() and segs >= len(frames)


def test_entry_of_several_zstd_frames(ctx, mix):
    """one seek-table entry made of three level-1 zstd frames with checksums: split, and every checksum verified"""
    comp, cs, ds = ctx.compress_frames(mix, MIX_FRAME, 1, True)
    fr = split_frames(comp.tobytes(), cs)
    entries = [b"".join(fr[:3]), fr[3]]
    sizes = [int(sum(ds[:3])), int(ds[3])]
    out, st, rc, segs = _decode(ctx, entries, sizes)
    assert rc == 0 and out == mix.tobytes() and segs > 3
    bad = bytearray(entries[0]); bad[len(fr[0]) + len(fr[1]) - 1] ^= 0x55         # the second frame's checksum
    _, st, rc, _ = _decode(ctx, [bytes(bad), entries[1]], sizes)
    assert st[0] == -22 and st[1] == 0                                            # ZSTD_error_checksum_wrong


def test_range_read_inside_split_entry(ctx, mix):
    """zk_decompress_frames_upto: the walk stops at the first block boundary at or after the wanted prefix, inside a split entry"""
    comp, cs, ds = ctx.compress_frames(mix, MIX_FRAME, 1, True)
    co, do = offsets(cs), offsets(ds)
    buf = np.concatenate([comp[: int(co[-1])], np.zeros(64, np.uint8)])
    for want in (0, 1, 40_000, 100_003, int(ds[0]) - 1, int(ds[0])):
        need = np.full(len(cs), want, dtype=np.uint32)
        out = np.zeros(int(do[-1]) + 64, dtype=np.uint8); st = np.zeros(len(cs), dtype=np.int32)
        rc = ctx.lib.zk_decompress_frames_upto(ctx._h, buf.ctypes.data, co.ctypes.data_as(_native.u64p), do.ctypes.data_as(_native.u64p), len(cs),
                                               out.ctypes.data, need.ctypes.data_as(_native.u32p), 1, st.ctypes.data_as(_native.i32p))
        assert rc == 0 and not st.any()
        for i in range(len(cs)):
            a0 = int(do[i])
            assert out[a0:a0 + want].tobytes() == mix[a0:a0 + want].tobytes()


def test_failures_keep_serial_order(ctx, ctx_serial, mix):
    """corruption in a later segment of an entry, alone or while an earlier segment fails too (and with the entry's
    output size also wrong): the same per-entry status as the serial walk"""
    comp, cs, ds = ctx.compress_frames(mix, MIX_FRAME, 1, False)
    frames = split_frames(comp.tobytes(), cs)
    rng = np.random.default_rng(7)
    checked = 0
    for trial in range(24):
        e = trial % len(frames)
        f = bytearray(frames[e])
        n = len(f)
        hits = [int(rng.integers(n // 2, n - 1))]                                     # a later segment
        if trial % 2:
            hits.append(int(rng.integers(16, n // 2)))                                # ... and an earlier one
        for h in hits:
            f[h] ^= 1 << int(rng.integers(8))
        fr = list(frames); fr[e] = bytes(f)
        sizes = [int(d) for d in ds]
        if trial % 3 == 0:
            sizes[e] += 1                                                             # the final size check fails as well
        _, st, _, _ = _decode(ctx, fr, sizes, False)
        _, st_ref, _, _ = _decode(ctx_serial, fr, sizes, False)
        assert list(st) == list(st_ref), (trial, list(st), list(st_ref))
        checked += st[e] != 0
    assert checked > 12
