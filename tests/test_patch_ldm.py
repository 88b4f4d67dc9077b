"""Long-distance matching against the whole prefix (patch mode, zk_ldm.inc): with the switch on, a frame that repeats the prefix with a few
edits shrinks to the edits; the archive restores through libzstd refPrefix, the plain-C restatement and the codec's decoder (both
executors); the Window_Descriptor follows content + prefix and covers every offset; every level writes level 16's bytes; the switch
reaches the sized call, Encoder, RawEncoder and the CLI; and with the switch off nothing changes.  Every case runs on the emulation
build (`-m "not gpu"`, small inputs) and on the H100 (`-m gpu`, MiB scale)."""
import ctypes
import hashlib
import importlib.util
import io
import json
import os

import numpy as np
import pytest

import cases
import zeekstd_b200 as zk
from oracle import oracle as O
from test_segments_short import _context
from util import GOLDEN, golden_bytes, offsets
from zeekstd_b200 import _native, corpus

BLOCK = 32 << 10
M = 64                                   # bytes hashed = shortest long-distance match
WMAX = 1 << 27

_spec = importlib.util.spec_from_file_location("make_encoder_golden_ldm", os.path.join(GOLDEN, "make_encoder_golden_ldm.py"))
mk = importlib.util.module_from_spec(_spec); _spec.loader.exec_module(mk)
edited_copy = mk.edited_copy


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    return request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib")


@pytest.fixture(scope="module")
def ctx(lib):
    _native.set_default_lib(lib)
    c = zk.Context(0, lib)
    yield c
    c.close()


def _emul(ctx) -> bool:
    return "emul" in ctx.lib._name


def _scale(ctx, emul: int, gpu: int) -> int:
    return emul if _emul(ctx) else gpu


def _mix(n: int, seed: int) -> np.ndarray:
    return corpus.as_numpy(corpus.make_mix(n, seed=seed, segment=16 << 10)).copy()


def _window_size(wd: int) -> int:
    e, m = wd >> 3, wd & 7
    return (1 << (10 + e)) + ((1 << (10 + e)) >> 3) * m


def _window_descriptor(content: int, prefix_len: int) -> int:
    """the smallest Window_Descriptor >= max(128 KiB, min(content + prefix_len, 2^27))"""
    want = max(128 << 10, min(content + prefix_len, WMAX))
    return next(wd for wd in range(256) if _window_size(wd) >= want)


def _libzstd_patch_size(new: np.ndarray, old: np.ndarray, frame_size: int, level: int, checksum: bool) -> int:
    """the reference CLI's call sequence for --patch-from (cli/src/compress.rs:31-37, encode.rs:332-338): windowLog = ilog2(len(OLD)) + 1
    and enableLongDistanceMatching on the CCtx, refPrefix at the start of every frame -> total compressed size"""
    z = ctypes.CDLL(os.environ.get("ZK_LIBZSTD", O.SYSTEM_LIBZSTD))
    z.ZSTD_createCCtx.restype = ctypes.c_void_p
    z.ZSTD_CCtx_setParameter.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]; z.ZSTD_CCtx_setParameter.restype = ctypes.c_size_t
    z.ZSTD_CCtx_refPrefix.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]; z.ZSTD_CCtx_refPrefix.restype = ctypes.c_size_t
    z.ZSTD_compress2.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t]; z.ZSTD_compress2.restype = ctypes.c_size_t
    z.ZSTD_compressBound.argtypes = [ctypes.c_size_t]; z.ZSTD_compressBound.restype = ctypes.c_size_t
    z.ZSTD_isError.argtypes = [ctypes.c_size_t]
    z.ZSTD_freeCCtx.argtypes = [ctypes.c_void_p]
    c = z.ZSTD_createCCtx()
    for param, v in ((100, level), (201, int(checksum)), (101, max(10, old.size.bit_length())), (160, 1)):   # level, checksum, windowLog, LDM
        assert not z.ZSTD_isError(z.ZSTD_CCtx_setParameter(c, param, v)), param
    dst = np.empty(z.ZSTD_compressBound(frame_size) + 64, np.uint8)
    total = 0
    for lo in range(0, new.size, frame_size):
        fr = np.ascontiguousarray(new[lo:lo + frame_size])
        assert not z.ZSTD_isError(z.ZSTD_CCtx_refPrefix(c, old.ctypes.data, old.size))
        r = z.ZSTD_compress2(c, dst.ctypes.data, dst.size, fr.ctypes.data, fr.size)
        assert not z.ZSTD_isError(r)
        total += r
    z.ZSTD_freeCCtx(c)
    return total


def _restores(ctx, comp, cs, ds, new, old, decoders=()):
    """the archive restores through libzstd refPrefix, the plain-C restatement and the codec's decoder(s); every offset stays within the
    announced window -> merged sequence statistics of the restatement"""
    pad = np.concatenate([comp, np.zeros(64, np.uint8)])
    co, do = offsets(cs), offsets(ds)
    out, sizes = O.ref_decompress_frames(pad, co, do, prefix=old)
    assert out.tobytes() == new.tobytes() and sizes == [int(d) for d in ds]
    for c in (ctx,) + tuple(decoders):
        back, st, rc = c.decompress_frames(pad, co, do, True, prefix=old)
        assert rc == 0 and not any(st) and back[: new.size].tobytes() == new.tobytes()
    total = {"prefix_matches": 0, "max_offset": 0, "explicit_offsets": 0, "reps": 0}
    for f in range(len(cs)):
        fr = comp[int(co[f]):int(co[f + 1])]
        got, st = O.oracle_decompress_ex(fr, int(ds[f]), prefix=old)
        assert got == new[int(do[f]):int(do[f + 1])].tobytes()
        assert fr[5] == _window_descriptor(int(ds[f]), old.size if ds[f] else 0), f
        assert st["max_offset"] <= _window_size(int(fr[5])), (f, st)
        total["prefix_matches"] += st["prefix_matches"]; total["explicit_offsets"] += st["explicit_offsets"]
        total["reps"] += st["rep1"] + st["rep2"] + st["rep3"] + st["rep1_minus_1"]
        total["max_offset"] = max(total["max_offset"], st["max_offset"])
    return total


def test_it_is_a_patch(ctx, lib):
    """< 1 % of NEW differs from OLD: with long-distance matching the archive is a few percent of NEW's plain archive and within 3x of
    libzstd's patch; without it the prefix call stays close to the plain size (the prefix's last 32 KiB is all it sees)"""
    n = _scale(ctx, 256 << 10, 8 << 20)
    fs = _scale(ctx, 100_000, 2 << 20)
    old = _mix(n, 3)
    new = edited_copy(old, 11, _scale(ctx, 8, 200))
    plain = ctx.compress_frames(new, fs, 16, True)[0]
    tail_only = ctx.compress_frames(new, fs, 16, True, prefix=old)[0]
    comp, cs, ds = ctx.compress_frames(new, fs, 16, True, prefix=old, long_distance=True)
    ref = _libzstd_patch_size(new, old, fs, 16, True)
    print(f"patch sizes ({'emulation' if _emul(ctx) else 'H100'}, NEW {new.size} B): plain {plain.size}, prefix without LDM {tail_only.size}, "
          f"LDM {comp.size}, libzstd windowLog+LDM+refPrefix {ref}")
    assert comp.size <= 0.05 * plain.size
    assert comp.size <= 3 * ref
    assert tail_only.size >= 0.9 * plain.size
    short = {name: _context(lib, {"ZK_EXEC_SHORT": v}) for name, v in (("cta", "0"), ("warp", str(1 << 30)))}
    st = _restores(ctx, comp, cs, ds, new, old, tuple(short.values()))
    assert st["prefix_matches"] > 0
    if not _emul(ctx):
        assert st["max_offset"] > 2 << 20
    # the wrong prefix or none: a checksum or offset error, never a fault
    pad = np.concatenate([comp, np.zeros(64, np.uint8)])
    other = _mix(n, 4)
    for wrong in (other, None, old[: n // 2]):
        _, status, rc = ctx.decompress_frames(pad, offsets(cs), offsets(ds), True, prefix=wrong)
        assert rc in (-22, -20) and all(s in (0, -22, -20) for s in status), (rc, status)
    for c in short.values():
        c.close()


@pytest.mark.parametrize("content,prefix_len", [(1, 100), (100, 63), (1000, 64), (5000, 200_000), (BLOCK + 1, 70_000), (150_000, 150_000), (70_000, 5)])
def test_window(ctx, content, prefix_len):
    src = _mix(max(content, prefix_len) + 4096, 5)
    old = src[:prefix_len]
    new = np.concatenate([src[100:100 + content // 2], src[: content - content // 2]])
    comp, cs, ds = ctx.compress_frames(new, 1 << 20, 3, True, prefix=old, long_distance=True)
    assert comp[5] == _window_descriptor(content, prefix_len)
    _restores(ctx, comp, cs, ds, new, old)


def test_edges(ctx):
    n = _scale(ctx, 96 << 10, 3 << 20)
    old = _mix(n, 6)
    new = edited_copy(old, 7, 5)
    # no prefix, or an empty one: the plain call at the same level, flag or not
    for lvl in (3, 16):
        plain = ctx.compress_frames(new, 50_000, lvl, True)[0].tobytes()
        assert ctx.compress_frames(new, 50_000, lvl, True, prefix=None, long_distance=True)[0].tobytes() == plain
        assert ctx.compress_frames(new, 50_000, lvl, True, prefix=b"", long_distance=True)[0].tobytes() == plain
    # a prefix shorter than the hashed span: nothing to index; the tier's own search still sees it
    comp, cs, ds = ctx.compress_frames(new, 50_000, 16, True, prefix=old[:M - 1], long_distance=True)
    _restores(ctx, comp, cs, ds, new, old[:M - 1])
    # NEW identical to OLD: a handful of sequences per block
    comp, cs, ds = ctx.compress_frames(old, 1 << 20, 16, True, prefix=old, long_distance=True)
    st = _restores(ctx, comp, cs, ds, old, old)
    blocks = -(-old.size // BLOCK)
    assert comp.size < 40 * blocks and st["explicit_offsets"] + st["reps"] <= 2 * blocks
    # NEW unrelated to OLD (skewed random bytes: nothing 64 bytes long repeats): what the call without the switch writes, to within 1 %
    other = (np.random.default_rng(8).integers(0, 256, n, dtype=np.uint8) & np.random.default_rng(9).integers(0, 256, n, dtype=np.uint8))
    a = ctx.compress_frames(other, 1 << 20, 16, True, prefix=old)[0].size
    comp, cs, ds = ctx.compress_frames(other, 1 << 20, 16, True, prefix=old, long_distance=True)
    assert abs(int(comp.size) - int(a)) <= 0.01 * a
    _restores(ctx, comp, cs, ds, other, old)
    # frame sizes that cut blocks everywhere
    for fs, m in ((1, 150), (100, 3000), (BLOCK - 1, new.size), (BLOCK + 1, new.size)):
        comp, cs, ds = ctx.compress_frames(new[:m], fs, 16, True, prefix=old, long_distance=True)
        _restores(ctx, comp, cs, ds, new[:m], old)
    # caller-chosen sizes with empty frames: each frame is what the uniform call makes of its bytes alone
    sizes = [0, 70_000, 0, 1, new.size - 70_001, 0]
    comp, cs, ds = ctx.compress_frames_sized(new, sizes, 16, True, prefix=old, long_distance=True)
    _restores(ctx, comp, cs, ds, new, old)
    co, do = offsets(cs), offsets(ds)
    for f, d in enumerate(sizes):
        alone = ctx.compress_frames(new[int(do[f]):int(do[f + 1])], max(d, 1), 16, True, prefix=old, long_distance=True)[0]
        assert comp[int(co[f]):int(co[f + 1])].tobytes() == alone.tobytes(), f
    assert ctx.compress_frames_sized(new, sizes, 16, True, prefix=old)[0].tobytes() != comp.tobytes()
    # all-equal bytes on both sides: every position hashes alike; the work stays bounded
    z = np.full(n, 0x41, np.uint8)
    comp, cs, ds = ctx.compress_frames(z, 1 << 20, 16, True, prefix=z, long_distance=True)
    _restores(ctx, comp, cs, ds, z, z)


def test_levels_and_options(ctx):
    n = _scale(ctx, 80 << 10, 2 << 20)
    fs = 50_000
    old = _mix(n, 9)
    new = edited_copy(old, 10, 6)
    want, cs, ds = ctx.compress_frames(new, fs, 16, True, prefix=old, long_distance=True)
    for lvl in (-5, 1, 3, 13, 19):
        assert ctx.compress_frames(new, fs, lvl, True, prefix=old, long_distance=True)[0].tobytes() == want.tobytes(), lvl
    assert ctx.compress_frames(new, fs, 16, True, prefix=old)[0].tobytes() != want.tobytes()
    # Encoder: the batch call, frame for frame
    sink = io.BytesIO()
    opts = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Uncompressed(fs)).checksum_flag(True).compression_level(3)
    enc = opts.long_distance_matching(True).into_encoder(sink)
    data, pos = new.tobytes(), 0
    while pos < len(data):
        pos += enc.compress_with_prefix(memoryview(data)[pos:pos + 30_000], old)
    enc.end_frame(); enc.flush()
    assert sink.getvalue() == want.tobytes()
    # RawEncoder: one frame
    raw = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Uncompressed(fs)).checksum_flag(True).long_distance_matching(True).into_raw_encoder()
    out, st, pos = io.BytesIO(), bytearray(1 << 18), 0
    while pos < fs:
        pr = raw.compress_with_prefix(memoryview(data)[pos:min(pos + 20_000, fs)], st, old)
        out.write(st[: pr.out_progress]); pos += pr.in_progress
    while True:
        pr = raw.end_frame(st)
        out.write(st[: pr.out_progress])
        if pr.data_left == 0:
            break
    assert out.getvalue() == want.tobytes()[: int(cs[0])]
    # Compressed(n) has no long-distance matching: the Encoder refuses the combination
    bad = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Compressed(10_000)).long_distance_matching(True)
    with pytest.raises(zk.Error) as e:
        bad.into_encoder(io.BytesIO())
    assert e.value.rc == -1006
    for name in ("zk_compress_frames_ldm", "zk_compress_frames_sized_ldm", "zk_encode_options_long_distance_matching"):
        assert hasattr(ctx.lib, name)
    assert _native._SIGS["zk_compress_frames_ldm"] == _native._SIGS["zk_compress_frames_prefix"]
    assert _native._SIGS["zk_compress_frames_sized_ldm"] == _native._SIGS["zk_compress_frames_sized"]


def test_encoder_golden(ctx):
    """the matcher's bytes are the same on every build: tests/golden/encoder_golden_ldm.json was written from the emulation build"""
    gold = json.loads(golden_bytes("encoder_golden_ldm.json"))
    got = {}
    for name, (old, new, fs, ck) in mk.inputs().items():
        comp = ctx.compress_frames(new, fs, 19, ck, prefix=old, long_distance=True)[0]
        got[name] = {"size": int(comp.size), "sha256": hashlib.sha256(comp.tobytes()).hexdigest()}
    assert got == gold


def test_cli(ctx, tmp_path):
    old = _mix(_scale(ctx, 100 << 10, 3 << 20), 12)
    new = edited_copy(old, 13, 6)
    po = tmp_path / "old.bin"; po.write_bytes(old.tobytes())
    pn = tmp_path / "new.bin"; pn.write_bytes(new.tobytes())
    a, b, back = tmp_path / "a.zst", tmp_path / "b.zst", tmp_path / "back.bin"
    rc, _, err = cases._cli(ctx, ["compress", "-q", "-s", "64K", "--patch-from", po, "--long", "-o", a, pn])
    assert rc == 0, err
    rc, _, err = cases._cli(ctx, ["compress", "-q", "-s", "64K", "--patch-from", po, "-o", b, pn])
    assert rc == 0, err
    assert a.stat().st_size < b.stat().st_size / 4
    # --patch-from alone: the bytes of the Encoder without the option
    sink = io.BytesIO()
    enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Uncompressed(64 << 10)).checksum_flag(True).compression_level(3).into_encoder(sink)
    data, pos = new.tobytes(), 0
    while pos < len(data):
        pos += enc.compress_with_prefix(memoryview(data)[pos:pos + (1 << 17)], old)
    enc.finish()
    assert b.read_bytes() == sink.getvalue()
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "--patch-apply", po, "-o", back, a])
    assert rc == 0 and back.read_bytes() == new.tobytes(), err
    rc, _, err = cases._cli(ctx, ["compress", "-q", "--long", "-o", tmp_path / "c.zst", pn])
    assert rc != 0 and "--patch-from" in err and not (tmp_path / "c.zst").exists()
    rc, _, err = cases._cli(ctx, ["compress", "-q", "--long", "--patch-from", po, "--frame-size-policy", "compressed", "-o", tmp_path / "d.zst", pn])
    assert rc != 0 and not (tmp_path / "d.zst").exists()


@pytest.mark.gpu
def test_long_span_and_pass_boundary(gpu_lib):
    """a 1 MiB span identical to the prefix is a few sequences per block; 4 MiB frames over more than one internal pass (64 MiB) restore"""
    ctx = zk.Context(0, gpu_lib)
    old = _mix(72 << 20, 14)
    span = old[5_000_001:5_000_001 + (1 << 20)].copy()
    comp, cs, ds = ctx.compress_frames(span, 1 << 20, 16, True, prefix=old, long_distance=True)
    st = _restores(ctx, comp, cs, ds, span, old)
    assert st["explicit_offsets"] + st["reps"] <= 2 * 32 and st["max_offset"] > 60 << 20
    new = edited_copy(old, 15, 300)
    comp, cs, ds = ctx.compress_frames(new, 4 << 20, 16, True, prefix=old, long_distance=True)
    assert comp.size < new.size // 100
    pad = np.concatenate([comp, np.zeros(64, np.uint8)])
    out, sizes = O.ref_decompress_frames(pad, offsets(cs), offsets(ds), prefix=old)
    assert out.tobytes() == new.tobytes()
    back, status, rc = ctx.decompress_frames(pad, offsets(cs), offsets(ds), True, prefix=old)
    assert rc == 0 and back[: new.size].tobytes() == new.tobytes()
    ctx.close()
