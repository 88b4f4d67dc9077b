"""Frames of caller-chosen sizes in one batch (zk_compress_frames_sized[_dev], Context.compress_frames_sized): frame f must be exactly what
compress_frames makes of its bytes alone (frame_size = max(size, 1)), at every tier, with and without checksum and prefix; uniform sizes
give compress_frames' bytes; archives restore through libzstd, the codec's decoder and a seek table; sub-batch limits do not change the
output; the contract's errors.  Every case runs on the emulation build (`-m "not gpu"`, small inputs) and on the H100 (`-m gpu`, MiB-scale)."""
import ctypes

import numpy as np
import pytest

import zeekstd_b200 as zk
from oracle import oracle as O
from test_high_levels import _data, _window_descriptor
from util import offsets
from zeekstd_b200 import _native

BLOCK = 32 << 10
LEVELS = [-5, -1, 1, 3, 5, 8, 11, 13, 19]


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


def _sizes(ctx, seed: int) -> list[int]:
    """the block-boundary sizes, runs of 1-byte frames and a seeded log-uniform mix (on the H100 also a frame over 2 MiB)"""
    rng = np.random.default_rng(seed)
    if _emul(ctx):
        edge = [0, 1, 31, 32767, 1, 1, 1, 32769, 0, 32768]
        mix = np.exp(rng.uniform(0, np.log(20_000), 4)).astype(int).tolist()
    else:
        edge = [0, 1, 31, 32767, 32768, 32769, 65536, (2 << 20) + 12345] + [1] * 40 + [0, 0]
        mix = np.exp(rng.uniform(0, np.log(4 << 20), 60)).astype(int).tolist()
    out = edge + mix
    rng.shuffle(out)
    return out


def _reference(ctx, x, sizes, level, checksum, prefix):
    """one compress_frames call per frame -> (concatenated bytes, c_sizes)"""
    parts, cs, pos = [], [], 0
    for d in sizes:
        comp, c, ds = ctx.compress_frames(x[pos:pos + d], max(d, 1), level, checksum, prefix)
        assert len(c) == 1 and int(ds[0]) == d
        parts.append(comp.tobytes()); cs.append(int(c[0])); pos += d
    return b"".join(parts), cs


def _restores(ctx, x, comp, cs, ds, prefix=None):
    pad = np.concatenate([comp, np.zeros(64, np.uint8)])
    out, got = O.ref_decompress_frames(pad, offsets(cs), offsets(ds), prefix=prefix)
    assert out.tobytes() == x.tobytes() and got == [int(d) for d in ds]
    back, st, rc = ctx.decompress_frames(pad, offsets(cs), offsets(ds), True, prefix=prefix)
    assert rc == 0 and not any(st) and back[: x.size].tobytes() == x.tobytes()


@pytest.mark.parametrize("level", LEVELS)
def test_equivalence(ctx, level):
    sizes = _sizes(ctx, 100 + level)
    x = _data("text", sum(sizes), level & 0xFF)
    prefix = _data("text", 50_000, 77)
    combos = [(False, None), (True, prefix)] if _emul(ctx) else [(False, None), (True, None), (False, prefix), (True, prefix)]
    for checksum, pf in combos:
        comp, cs, ds = ctx.compress_frames_sized(x, sizes, level, checksum, pf)
        ref, rcs = _reference(ctx, x, sizes, level, checksum, pf)
        assert list(ds) == sizes and list(cs) == rcs, (level, checksum, pf is None)
        assert comp.tobytes() == ref, (level, checksum, pf is None)
        _restores(ctx, x, comp, cs, ds, pf)


@pytest.mark.parametrize("level", [-1, 1, 3, 13, 19])
def test_uniform_sizes_give_compress_frames_bytes(ctx, level):
    n = 3 * BLOCK + 5000 if _emul(ctx) else 40 << 20
    x = _data("dickens", n)
    for fs in ((40_000, 1000) if _emul(ctx) else (1 << 20, 100_000)):
        sizes = [fs] * (n // fs) + ([n % fs] if n % fs else [])
        comp, cs, ds = ctx.compress_frames(x, fs, level, True)
        got, gcs, gds = ctx.compress_frames_sized(x, sizes, level, True)
        assert got.tobytes() == comp.tobytes() and list(gcs) == list(cs) and list(gds) == list(ds), (level, fs)


def test_seek_table_reads_cross_frames(ctx):
    sizes = _sizes(ctx, 7)
    x = _data("structured", sum(sizes), 7)
    comp, cs, ds = ctx.compress_frames_sized(x, sizes, 3, True)
    _restores(ctx, x, comp, cs, ds)
    st = zk.SeekTable(lib=ctx.lib)
    for c, d in zip(cs, ds):
        st.log_frame(int(c), int(d))
    data = x.tobytes()
    starts = offsets(ds)
    rng = np.random.default_rng(3)
    for f in rng.integers(1, len(sizes) - 1, 6):
        lo = max(0, int(starts[f]) - 700)
        hi = min(len(data), int(starts[f + 1]) + 900)          # from the frame before f to the frame after it
        dec = zk.DecodeOptions(comp.tobytes(), ctx).seek_table(st.clone()).into_decoder()
        dec.set_offset(lo); dec.set_offset_limit(hi)
        assert dec.read_all() == data[lo:hi], (int(f), lo, hi)


@pytest.mark.parametrize("level", [1, 19])
def test_sub_batches_do_not_change_the_output(ctx, monkeypatch, level):
    sizes = _sizes(ctx, 11)
    x = _data("text", sum(sizes), 11)
    prefix = _data("text", 4000, 12)
    comp, cs, _ = ctx.compress_frames_sized(x, sizes, level, True, prefix)
    # sub-batches smaller than the largest frame: frames straddle the limit and one exceeds a sub-batch on its own
    monkeypatch.setenv("ZK_HOST_SUB_BYTES_ENC", str(max(sizes) // 3))
    small, scs, _ = ctx.compress_frames_sized(x, sizes, level, True, prefix)
    assert small.tobytes() == comp.tobytes() and list(scs) == list(cs)
    # the uniform call shares the splitter
    fs = 1000
    ref = ctx.compress_frames(x[:20 * fs + 7], fs, level, False)[0]
    monkeypatch.setenv("ZK_HOST_SUB_BYTES_ENC", str(3 * fs + 500))
    assert ctx.compress_frames(x[:20 * fs + 7], fs, level, False)[0].tobytes() == ref.tobytes()


@pytest.mark.parametrize("level", [13, 19])
def test_window_descriptors_follow_each_frame(ctx, level):
    sizes = [1000, 0, 100_000, 5, 300_000 if not _emul(ctx) else 70_000, 2 << 20 if not _emul(ctx) else 40_000]
    x = _data("text", sum(sizes), 4)
    prefix = _data("text", 50_000, 4)
    for pf in (None, prefix):
        comp, cs, ds = ctx.compress_frames_sized(x, sizes, level, False, pf)
        ptail = 0 if pf is None else BLOCK
        co = offsets(cs)
        for f, d in enumerate(sizes):
            want = _window_descriptor(d, ptail if d else 0) if level >= 16 else 0x40      # the wide tier: 256 KiB
            assert comp[int(co[f]) + 5] == want, (level, f, d, pf is None)
        _restores(ctx, x, comp, cs, ds, pf)


def test_errors(ctx):
    lib = ctx.lib
    dst = np.zeros(1 << 16, np.uint8)
    cs = np.zeros(4, np.uint32)
    dl = ctypes.c_size_t(123)

    def call(sizes, n_frames=None, src=None, cap=dst.size):
        arr = np.asarray(sizes, dtype=np.uint32)
        return lib.zk_compress_frames_sized(ctx._h, src, arr.ctypes.data_as(_native.u32p), len(arr) if n_frames is None else n_frames, 3, 0,
                                            None, 0, dst.ctypes.data, cap, cs.ctypes.data_as(_native.u32p), ctypes.byref(dl))

    assert call([], 0) == 0 and dl.value == 0                                 # no frames: nothing written
    assert call([(1 << 30) + 1]) == -42                                       # parameter_outOfBound
    assert call([0], 0x08000000 + 1) == -1003                                 # ZK_ERR_FRAME_INDEX_TOO_LARGE
    x = _data("random", 5000, 1)
    assert lib.zk_compress_frames_sized(ctx._h, x.ctypes.data, np.array([2000, 3000], np.uint32).ctypes.data_as(_native.u32p), 2, 3, 0,
                                        None, 0, dst.ctypes.data, 100, cs.ctypes.data_as(_native.u32p), ctypes.byref(dl)) == -70
    # one empty frame: the bytes of compress_frames on no input
    comp, c, d = ctx.compress_frames_sized(x[:0], [0], 3, True)
    assert comp.tobytes() == ctx.compress_frames(x[:0], 1, 3, True)[0].tobytes() and list(d) == [0]
    with pytest.raises(ValueError):
        ctx.compress_frames_sized(x, [100, 200], 3)
    assert lib.zk_compress_bound_sized(np.array([5000], np.uint32).ctypes.data_as(_native.u32p), 1) >= 5000 + 14


@pytest.mark.gpu
def test_device_call_matches_host(gpu_lib):
    import torch
    ctx = zk.Context(0, gpu_lib)
    rng = np.random.default_rng(9)
    sizes = [0, 1, 32769] + np.exp(rng.uniform(np.log(1 << 10), np.log(4 << 20), 40)).astype(int).tolist()
    x = _data("text", sum(sizes), 9)
    xd = torch.from_numpy(np.concatenate([x, np.zeros(64, np.uint8)])).cuda()     # the entry points read up to 16 bytes past the input
    ds = np.asarray(sizes, np.uint32)
    for level in (-3, 1, 3, 19):
        comp, cs, _ = ctx.compress_frames_sized(x, sizes, level, True)
        cap = gpu_lib.zk_compress_bound_sized(ds.ctypes.data_as(_native.u32p), len(sizes))
        out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        dcs = np.zeros(len(sizes), np.uint32); dl = ctypes.c_size_t()
        rc = gpu_lib.zk_compress_frames_sized_dev(ctx._h, xd.data_ptr(), ds.ctypes.data_as(_native.u32p), len(sizes), level, 1,
                                                  out.data_ptr(), cap, dcs.ctypes.data_as(_native.u32p), ctypes.byref(dl), None)
        torch.cuda.synchronize()
        assert rc == 0 and out[: dl.value].cpu().numpy().tobytes() == comp.tobytes() and list(dcs) == list(cs), level
    ctx.close()
