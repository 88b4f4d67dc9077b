"""Per-frame prefixes (zk_compress_frames_sized_prefixes, zk_decompress_frames_prefixes): every frame of one batch matched against its own
range of one prefix buffer.  Each frame is byte-equal to the single-prefix call for that frame alone with its range as the prefix, at every
tier, plain, with long-distance matching and in long mode; ranges == NULL is the single-prefix call; the archive restores through the
codec's decoder (both executors, range reads, checksums), libzstd refPrefix and the plain-C restatement, and decodes exactly as the
single-prefix decoder does entry by entry; seekable patches restore one frame from its slice alone; bad ranges are refused.  Every case
runs on the emulation build (`-m "not gpu"`, small inputs) and on the H100 (`-m gpu`, MiB scale)."""
import ctypes

import numpy as np
import pytest

import zeekstd_b200 as zk
from oracle import oracle as O
from test_patch_ldm import _mix, edited_copy
from test_segments_short import _context
from util import offsets
from zeekstd_b200 import _native

BLOCK = 32 << 10
MODES = {"plain": (False, False), "ldm": (True, False), "long": (False, True)}
LEVELS = (-3, 1, 3, 7, 10, 13, 19)


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


def _raw(ctx, data, sizes, level, ck, prefix, ranges, ldm=False, lm=False, dst_cap=None):
    """zk_compress_frames_sized_prefixes as called from C (ranges may be None) -> (rc, comp, c_sizes)"""
    ds = np.ascontiguousarray(sizes, dtype=np.uint32)
    src = np.ascontiguousarray(data, dtype=np.uint8)
    pfx = None if prefix is None else np.ascontiguousarray(prefix, dtype=np.uint8)
    rg = None if ranges is None else np.ascontiguousarray(ranges, dtype=np.uint64).reshape(-1, 2)
    cap = ctx.lib.zk_compress_bound_sized(ds.ctypes.data_as(_native.u32p), ds.size) if dst_cap is None else dst_cap
    dst = np.empty(cap + 64, np.uint8)
    cs = np.zeros(max(ds.size, 1), np.uint32)
    dl = ctypes.c_size_t(12345)
    rc = ctx.lib.zk_compress_frames_sized_prefixes(ctx._h, src.ctypes.data if src.size else None, ds.ctypes.data_as(_native.u32p), ds.size,
                                                   level, int(ck), None if pfx is None else pfx.ctypes.data, 0 if pfx is None else pfx.size,
                                                   None if rg is None else rg.ctypes.data_as(_native.u64p), int(ldm), int(lm),
                                                   dst.ctypes.data, cap, cs.ctypes.data_as(_native.u32p), ctypes.byref(dl))
    return rc, dst[: dl.value], cs[: ds.size]


def _alone(ctx, frame, level, ck, prefix, mode):
    """what the single-prefix sized call writes for one frame alone with `prefix` (None: no prefix)"""
    ldm, lm = MODES[mode]
    return ctx.compress_frames_sized(frame, [frame.size], level, ck, prefix=prefix, long_distance=ldm, long_mode=lm)[0].tobytes()


def _expected(ctx, frame, level, ck, old, lo, hi, mode):
    if mode == "ldm" and (lo == hi or frame.size == 0):
        return _alone(ctx, frame, 16, ck, None, "plain")          # level 16's frame without a prefix
    return _alone(ctx, frame, level, ck, old[lo:hi] if hi > lo else None, mode)


def _case(ctx, seed):
    """OLD, NEW and frames whose ranges cover every shape: empty, short of mixed lengths, overlapping, identical, whole, an empty frame with
    a non-empty range"""
    n = _scale(ctx, 128 << 10, 6 << 20)
    old = _mix(n, seed)
    new = edited_copy(old, seed + 1, 8)
    sizes = [7000, 0, 20_000, 1, 40_000, 3000, 0, 25_000, 9000]
    sizes.append(new.size - sum(sizes))
    ranges = [(0, 0), (10, 20_000), (100, 3100), (5, 5), (1000, 21_000), (0, 40_000), (0, 40_000), (20_000, 60_000), (0, n), (BLOCK, n)]
    return old, new, sizes, ranges


@pytest.mark.parametrize("mode", list(MODES))
def test_frames_equal_single_calls(ctx, mode):
    old, new, sizes, ranges = _case(ctx, 21)
    do = offsets(sizes)
    levels = LEVELS if mode == "plain" or not _emul(ctx) else (-3, 13, 19)    # every level runs level 16 under the flags
    ldm, lm = MODES[mode]
    for level in levels:
        for ck in (False, True):
            comp, cs, ds = ctx.compress_frames_sized(new, sizes, level, ck, prefix=old, long_distance=ldm, long_mode=lm, prefix_ranges=ranges)
            co = offsets(cs)
            for f, (lo, hi) in enumerate(ranges):
                got = comp[int(co[f]):int(co[f + 1])].tobytes()
                assert got == _expected(ctx, new[int(do[f]):int(do[f + 1])], level, ck, old, lo, hi, mode), (mode, level, ck, f)


@pytest.mark.parametrize("mode", list(MODES))
def test_ranges_null_is_the_single_prefix_call(ctx, mode):
    old, new, sizes, _ = _case(ctx, 23)
    ldm, lm = MODES[mode]
    for level in (1, 19):
        rc, comp, cs = _raw(ctx, new, sizes, level, True, old, None, ldm, lm)
        assert rc == 0
        want = ctx.compress_frames_sized(new, sizes, level, True, prefix=old, long_distance=ldm, long_mode=lm)[0]
        assert comp.tobytes() == want.tobytes(), level
    # the whole buffer as every frame's range: the same bytes again
    rc, comp2, _ = _raw(ctx, new, sizes, 19, True, old, [(0, old.size)] * len(sizes), ldm, lm)
    assert rc == 0 and comp2.tobytes() == want.tobytes()


@pytest.mark.parametrize("mode", list(MODES))
def test_small_sub_batches(ctx, lib, mode):
    """frames cut into host sub-batches of a few frames each: the same bytes"""
    old, new, sizes, ranges = _case(ctx, 25)
    ldm, lm = MODES[mode]
    want = ctx.compress_frames_sized(new, sizes, 3, True, prefix=old, long_distance=ldm, long_mode=lm, prefix_ranges=ranges)[0]
    small = _context(lib, {"ZK_HOST_SUB_BYTES_ENC": "30000"})
    got = small.compress_frames_sized(new, sizes, 3, True, prefix=old, long_distance=ldm, long_mode=lm, prefix_ranges=ranges)[0]
    small.close()
    assert got.tobytes() == want.tobytes()


def test_decode(ctx, lib):
    old, new, sizes, ranges = _case(ctx, 27)
    # frame 2 is its own range's bytes: its first match reaches the range's first byte
    lo, hi = ranges[2]
    new = new.copy()
    s2 = int(offsets(sizes)[2])
    new[s2:s2 + sizes[2]] = old[lo:lo + sizes[2]]
    comp, cs, ds = ctx.compress_frames_sized(new, sizes, 3, True, prefix=old, prefix_ranges=ranges)
    pad = np.concatenate([comp, np.zeros(64, np.uint8)])
    co, do = offsets(cs), offsets(ds)
    execs = [ctx] + [_context(lib, {"ZK_EXEC_SHORT": v}) for v in ("0", str(1 << 30))]
    for c in execs:
        back, st, rc = c.decompress_frames(pad, co, do, True, prefix=old, prefix_ranges=ranges)
        assert rc == 0 and not any(st) and back[: new.size].tobytes() == new.tobytes()
        need = [max(0, d // 2) for d in sizes]
        part, st, rc = c.decompress_frames(pad, co, do, True, need=need, prefix=old, prefix_ranges=ranges)
        assert rc == 0
        for f in range(len(sizes)):
            assert part[int(do[f]):int(do[f]) + need[f]].tobytes() == new[int(do[f]):int(do[f]) + need[f]].tobytes()
    for c in execs[1:]:
        c.close()
    for f, (lo, hi) in enumerate(ranges):
        fr = comp[int(co[f]):int(co[f + 1])]
        want = new[int(do[f]):int(do[f + 1])]
        one = np.concatenate([fr, np.zeros(64, np.uint8)])
        slice_ = old[lo:hi] if hi > lo else None
        back, st, rc = ctx.decompress_frames(one, [0, fr.size], [0, want.size], True, prefix=slice_)
        assert rc == 0 and back[: want.size].tobytes() == want.tobytes(), f
        out, _ = O.ref_decompress_frames(one, [0, fr.size], [0, want.size], prefix=slice_)         # libzstd refPrefix
        assert out.tobytes() == want.tobytes(), f
        got, _ = O.oracle_decompress_ex(fr, want.size, prefix=slice_)                            # the plain-C restatement
        assert got == want.tobytes(), f
    # a range one byte shorter at the front: what the single-prefix decoder returns for that shorter prefix, corruption_detected
    lo, hi = ranges[2]
    short = list(ranges); short[2] = (lo + 1, hi)
    _, st, rc = ctx.decompress_frames(pad, co, do, True, prefix=old, prefix_ranges=short)
    one = np.concatenate([comp[int(co[2]):int(co[3])], np.zeros(64, np.uint8)])
    _, st1, rc1 = ctx.decompress_frames(one, [0, int(cs[2])], [0, sizes[2]], True, prefix=old[lo + 1:hi])
    assert rc == -20 and st[2] == -20 and rc1 == -20 and [s for i, s in enumerate(st) if i != 2] == [0] * (len(st) - 1)


def test_seekable_patch(ctx):
    """NEW is OLD with in-place edits of the same length; frame f covers [a, b) and is matched against OLD[a - m, b + m) only: the archive is
    a patch, and one frame restores from its slice of OLD alone"""
    n = _scale(ctx, 256 << 10, 16 << 20)
    fs, m = _scale(ctx, 64 << 10, 1 << 20), _scale(ctx, 4 << 10, 64 << 10)
    old = _mix(n, 31)
    new = old.copy()
    rng = np.random.default_rng(32)
    for at in rng.integers(0, n - 100, _scale(ctx, 8, 64)):
        new[at:at + 40] = rng.integers(0, 256, 40, dtype=np.uint8)
    sizes = [min(fs, n - a) for a in range(0, n, fs)]
    ranges = [(max(0, a - m), min(n, a + fs + m)) for a in range(0, n, fs)]
    plain = ctx.compress_frames_sized(new, sizes, 16, True)[0]
    comp, cs, ds = ctx.compress_frames_sized(new, sizes, 16, True, prefix=old, long_distance=True, prefix_ranges=ranges)
    assert comp.size <= 0.05 * plain.size, (comp.size, plain.size)
    co, do = offsets(cs), offsets(ds)
    f = len(sizes) // 2
    lo, hi = ranges[f]
    one = np.concatenate([comp[int(co[f]):int(co[f + 1])], np.zeros(64, np.uint8)])
    back, st, rc = ctx.decompress_frames(one, [0, int(cs[f])], [0, sizes[f]], True, prefix=old[lo:hi].copy(), prefix_ranges=[(0, hi - lo)])
    assert rc == 0 and back[: sizes[f]].tobytes() == new[int(do[f]):int(do[f + 1])].tobytes()


def test_argument_errors(ctx):
    old, new, sizes, ranges = _case(ctx, 33)
    assert _raw(ctx, new, sizes, 3, False, old, [(0, old.size + 1)] + ranges[1:])[0] == -1006
    assert _raw(ctx, new, sizes, 3, False, old, [(10, 9)] + ranges[1:])[0] == -1006
    rc, comp, _ = _raw(ctx, np.zeros(0, np.uint8), [], 3, False, old, [])
    assert rc == 0 and comp.size == 0
    assert _raw(ctx, new, sizes, 3, False, old, ranges, dst_cap=100)[0] == -70
    with pytest.raises(ValueError):
        ctx.compress_frames_sized(new, sizes, 3, False, prefix=old, prefix_ranges=ranges[1:])
    co = np.zeros(len(sizes) + 1, np.uint64)
    _, _, rc = ctx.decompress_frames(np.zeros(64, np.uint8), co, co, True, prefix=old, prefix_ranges=[(0, old.size + 1)] * len(sizes))
    assert rc == -1006


@pytest.mark.gpu
def test_long_range_and_pass_boundary(gpu_lib):
    """a range above 2^27 bytes next to short ones under long-distance matching, and a level-19 batch across K-C1h's 2048-block pass
    boundary with a tail in front of every frame: each frame equals its single-prefix call"""
    ctx = zk.Context(0, gpu_lib)
    old = _mix((1 << 27) + (3 << 20), 41)
    new = edited_copy(old[(1 << 27):], 42, 50)
    sizes = [1 << 20, 1 << 20, new.size - (2 << 20)]
    ranges = [(0, old.size), (1000, 30_000), ((1 << 27), old.size)]
    comp, cs, _ = ctx.compress_frames_sized(new, sizes, 19, True, prefix=old, long_distance=True, prefix_ranges=ranges)
    co, do = offsets(cs), offsets(sizes)
    for f, (lo, hi) in enumerate(ranges):
        assert comp[int(co[f]):int(co[f + 1])].tobytes() == _expected(ctx, new[int(do[f]):int(do[f + 1])], 19, True, old, lo, hi, "ldm"), f
    back, st, rc = ctx.decompress_frames(np.concatenate([comp, np.zeros(64, np.uint8)]), co, do, True, prefix=old, prefix_ranges=ranges)
    assert rc == 0 and back[: new.size].tobytes() == new.tobytes()
    # 70 frames of 1 MiB: blocks past 2048 run in the second pass
    big = _mix(70 << 20, 43)
    sizes = [1 << 20] * 70
    ranges = [((7 * f) << 10, ((7 * f) << 10) + (f % 5) * 9000) for f in range(70)]
    comp, cs, _ = ctx.compress_frames_sized(big, sizes, 19, False, prefix=old, prefix_ranges=ranges)
    co, do = offsets(cs), offsets(sizes)
    for f in (0, 1, 62, 63, 64, 65, 69):
        lo, hi = ranges[f]
        assert comp[int(co[f]):int(co[f + 1])].tobytes() == _expected(ctx, big[int(do[f]):int(do[f + 1])], 19, False, old, lo, hi, "plain"), f
    ctx.close()
