"""FrameSizePolicy::Compressed(target) on the batch path (zk_compress_frames_csize): a frame closes after the first 32 KiB block at
which its header + blocks reach `target`, or at 1 GiB of input.  Every archive is checked from its bytes alone (the rule), against
Context.compress_frames of each frame's input range as one frame (byte parity: a block's bytes depend only on its input, its history
depth in the frame and whether it opens the frame), through libzstd and the codec's own decoder, and for independence from how the
input is chunked.  Every case runs on the emulation build (`-m "not gpu"`, small inputs) and on the H100 (`-m gpu`, MiB-scale)."""
import io

import numpy as np
import pytest

import cases
import zeekstd_b200 as zk
from oracle import oracle as O
from util import decode_frames, split_frames
from zeekstd_b200 import _native, corpus

BLOCK = 32 << 10
HUGE = 1 << 31


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


def _data(kind: str, n: int, seed: int = 5) -> np.ndarray:
    return corpus.as_numpy(corpus.make_class(kind, n, seed))


def parse_frame(fr: bytes):
    """-> (block sizes incl. their 3-byte headers, content-size field, checksum flag); asserts the frame is well formed"""
    assert fr[:4] == b"\x28\xb5\x2f\xfd" and len(fr) >= 10
    ck = bool(fr[4] & 4)
    fcs = int.from_bytes(fr[6:10], "little")
    pos, sizes = 10, []
    while True:
        h = int.from_bytes(fr[pos:pos + 3], "little")
        last, typ, size = h & 1, (h >> 1) & 3, h >> 3
        n = 3 + (1 if typ == 1 else size)
        sizes.append(n)
        pos += n
        if last:
            break
    assert pos + (4 if ck else 0) == len(fr)
    return sizes, fcs, ck


def check_rule(comp: np.ndarray, cs, ds, n: int, target: int):
    """every frame obeys the cut rule, read from the archive's bytes"""
    target = max(target, 1)
    frames = split_frames(comp.tobytes(), cs)
    assert sum(int(d) for d in ds) == n and len(frames) == len(ds)
    for i, (fr, d) in enumerate(zip(frames, ds)):
        blocks, fcs, _ = parse_frame(fr)
        assert fcs == d and len(blocks) == max(1, -(-int(d) // BLOCK))
        total = 10 + sum(blocks)
        assert len(blocks) == 1 or total - blocks[-1] < target, (i, total, blocks[-1], target)     # it did not close a block earlier
        if i + 1 < len(frames):
            assert d % BLOCK == 0
            assert total >= target or d == zk.SEEKABLE_MAX_FRAME_SIZE, (i, total, target)
    return frames


def check_parity(ctx, x: np.ndarray, frames, ds, level: int, checksum: bool, prefix=None):
    """every frame is what the uniform path makes of its input range as a single frame"""
    off = 0
    for i, (fr, d) in enumerate(zip(frames, ds)):
        d = int(d)
        ref, _, _ = ctx.compress_frames(x[off:off + d], max(d, 1), level, checksum, prefix)
        assert ref.tobytes() == fr, (i, off, d)
        off += d


def check_restores(ctx, x: np.ndarray, frames, ds, prefix=None):
    comp = b"".join(frames)
    if prefix is None:
        assert O.ref_decompress_any(comp, x.size + 1) == x.tobytes()
    else:
        c_off = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.uint64)
        d_off = np.concatenate([[0], np.cumsum(ds)]).astype(np.uint64)
        out, _ = O.ref_decompress_frames(np.frombuffer(comp + b"\0" * 64, dtype=np.uint8), c_off, d_off, prefix=prefix)
        assert out.tobytes() == x.tobytes()
    if prefix is None:
        out, st, rc = decode_frames(ctx, frames, [int(d) for d in ds], True)
        assert rc == 0 and not any(st) and out == x.tobytes()


@pytest.mark.parametrize("kind", ["text", "random", "runs"])
@pytest.mark.parametrize("level", [1, 3, 5, 8, 11, 13])
def test_rule_parity_and_interop(ctx, level, kind):
    wide = level >= 13
    n = _scale(ctx, 2 * BLOCK + 5000 if wide else 4 * BLOCK + 5000, 6 << 20)
    x = _data(kind, n, level)
    targets = [1, 700, 64 << 10, 1 << 20, HUGE]
    for j, target in enumerate(targets):
        for checksum in (False, True):
            if wide and (j + checksum) % 2 and _emul(ctx):
                continue                           # the wide tier is slow on the emulator: half of the combinations there
            comp, cs, ds, used = ctx.compress_frames_csize(x, target, level, checksum)
            assert used == n
            frames = check_rule(comp, cs, ds, n, target)
            if target == HUGE:
                assert len(frames) == 1
            check_parity(ctx, x, frames, ds, level, checksum)
            check_restores(ctx, x, frames, ds)


def test_wide_tier_history_depths(ctx):
    """frames of more than ZKC_WIDE_HIST + 1 blocks at level 13: every history depth 0..7 is taken from its own variant"""
    n = _scale(ctx, 10 * BLOCK + 333, 24 << 20)
    x = _data("text", n, 3)
    for target in (_scale(ctx, 60_000, 2 << 20), HUGE):
        comp, cs, ds, _ = ctx.compress_frames_csize(x, target, 13, True)
        frames = check_rule(comp, cs, ds, n, target)
        assert max(int(d) for d in ds) > 8 * BLOCK or target != HUGE
        check_parity(ctx, x, frames, ds, 13, True)
        check_restores(ctx, x, frames, ds)


def test_prefix(ctx):
    n = _scale(ctx, 5 * BLOCK + 77, 4 << 20)
    x = _data("text", n, 8)
    prefix = _data("text", 50_000, 8)                                      # the same generator: the prefix helps
    for level in (1, 3):
        comp, cs, ds, _ = ctx.compress_frames_csize(x, 20_000, level, True, prefix)
        frames = check_rule(comp, cs, ds, n, 20_000)
        check_parity(ctx, x, frames, ds, level, True, prefix)
        check_restores(ctx, x, frames, ds, prefix)


def test_chunked_calls_give_the_same_frames(ctx):
    n = _scale(ctx, 9 * BLOCK + 1234, 12 << 20)
    x = _data("text", n, 4)
    target = _scale(ctx, 25_000, 1 << 20)
    whole, cs0, ds0, _ = ctx.compress_frames_csize(x, target, 3, True)
    rng = np.random.default_rng(7)
    parts, cs, ds = [], [], []
    rest, pos = x[:0], 0
    while pos < n:
        k = int(rng.integers(1, max(2, n // 4)))
        buf = np.concatenate([rest, x[pos:pos + k]]); pos += k
        comp, c, d, used = ctx.compress_frames_csize(buf, target, 3, True, final=False)
        assert used < buf.size and used % BLOCK == 0 and int(np.sum(d)) == used
        parts.append(comp.tobytes()); cs += list(c); ds += list(d)
        rest = buf[used:]
    comp, c, d, used = ctx.compress_frames_csize(rest, target, 3, True)
    assert used == rest.size
    parts.append(comp.tobytes()); cs += list(c); ds += list(d)
    assert b"".join(parts) == whole.tobytes() and cs == list(cs0) and ds == list(ds0)


def _encoder_archive(ctx, x: np.ndarray, target: int, level: int, checksum: bool, write: int) -> bytes:
    sink = io.BytesIO()
    enc = (zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Compressed(target)).checksum_flag(checksum)
           .compression_level(level).into_encoder(sink))
    data = x.tobytes()
    for p in range(0, len(data), write or len(data) or 1):
        enc.compress(data[p:p + (write or len(data))])
    enc.finish()
    return sink.getvalue()


def test_encoder_write_sizes_do_not_matter(ctx, tmp_path):
    n = _scale(ctx, 6 * BLOCK + 999, 3 << 20)
    x = _data("text", n, 6)
    target = _scale(ctx, 30_000, 256 << 10)
    comp, cs, ds, _ = ctx.compress_frames_csize(x, target, 3, True)
    archives = {w: _encoder_archive(ctx, x, target, 3, True, w) for w in (1024, 4096, 0)}
    assert len(set(archives.values())) == 1
    arch = archives[0]
    assert arch[:comp.size] == comp.tobytes()
    st = zk.SeekTable.from_bytes(arch)
    assert st.num_frames() == len(cs) and [st.frame_size_comp(i) for i in range(len(cs))] == list(cs)
    assert zk.Decoder(zk.DecodeOptions(arch, ctx)).read_all() == x.tobytes()
    # the CLI reaches the same path through Encoder<W>
    src = tmp_path / "in.bin"; src.write_bytes(x.tobytes())
    out = tmp_path / "in.bin.zst"; back = tmp_path / "back.bin"
    rc, _, err = cases._cli(ctx, ["compress", "-q", "-l", 3, "--frame-size-policy", "compressed", "-s", target, "-o", out, src])
    assert rc == 0, err
    assert out.read_bytes() == arch
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "-o", back, out])
    assert rc == 0 and back.read_bytes() == x.tobytes(), err


def test_edges(ctx):
    # no input: one empty frame, from the entry point and from Encoder.finish()
    comp, cs, ds, used = ctx.compress_frames_csize(np.zeros(0, dtype=np.uint8), 1000, 3, True)
    ref, rcs, _ = ctx.compress_frames(np.zeros(0, dtype=np.uint8), 1, 3, True)
    assert comp.tobytes() == ref.tobytes() and list(ds) == [0] and len(cs) == 1 and used == 0
    assert _encoder_archive(ctx, np.zeros(0, dtype=np.uint8), 1000, 3, True, 0)[:comp.size] == comp.tobytes()
    comp, cs, ds, used = ctx.compress_frames_csize(np.zeros(0, dtype=np.uint8), 1000, 3, True, final=False)
    assert comp.size == 0 and len(cs) == 0 and used == 0
    x = _data("text", _scale(ctx, 4 * BLOCK, 8 << 20), 2)
    # shorter than one block: one frame
    comp, cs, ds, _ = ctx.compress_frames_csize(x[:1000], 1, 1, False)
    assert list(ds) == [1000]
    # final = 0 on input that ends exactly where a frame closes: that frame stays open
    whole, cs0, ds0, _ = ctx.compress_frames_csize(x, 1, 1, False)
    assert list(ds0) == [BLOCK] * (x.size // BLOCK)
    comp, cs, ds, used = ctx.compress_frames_csize(x, 1, 1, False, final=False)
    assert used == x.size - BLOCK and list(ds) == list(ds0[:-1])
    # target beyond the output: one frame; target 0 behaves like 1
    comp, cs, ds, _ = ctx.compress_frames_csize(x, HUGE, 1, False)
    assert list(ds) == [x.size]
    a = ctx.compress_frames_csize(x, 0, 1, False)
    b = ctx.compress_frames_csize(x, 1, 1, False)
    assert a[0].tobytes() == b[0].tobytes() and list(a[1]) == list(b[1])


def test_undersized_buffers_are_refused(ctx):
    import ctypes
    lib = ctx.lib
    x = _data("random", 3 * BLOCK + 10, 1)
    full, cs, ds, _ = ctx.compress_frames_csize(x, 1, 1, False)
    assert len(cs) == 4
    for frames_cap, dst_cap in ((3, full.size), (4, full.size - 1)):
        guard = 4096
        dst = np.full(dst_cap + guard, 0xA5, dtype=np.uint8)
        c = np.full(frames_cap + 16, 0xFFFFFFFF, dtype=np.uint32); d = c.copy()
        nf = ctypes.c_uint32(); dl = ctypes.c_size_t(); used = ctypes.c_size_t()
        rc = lib.zk_compress_frames_csize(ctx._h, x.ctypes.data, x.size, 1, 1, 0, None, 0, 1, dst.ctypes.data, dst_cap,
                                          c.ctypes.data_as(_native.u32p), d.ctypes.data_as(_native.u32p), frames_cap,
                                          ctypes.byref(nf), ctypes.byref(dl), ctypes.byref(used))
        assert rc == -70
        assert (dst[dst_cap:] == 0xA5).all() and (c[frames_cap:] == 0xFFFFFFFF).all() and (d[frames_cap:] == 0xFFFFFFFF).all()


@pytest.mark.gpu
def test_device_entry_point_matches_host(gpu_lib):
    import torch
    from zeekstd_b200 import parallel
    ctx = zk.Context(0, gpu_lib)
    x = _data("text", 5 << 20, 12)
    dev = parallel.DeviceCodec(ctx)
    for level, target in ((1, 1 << 20), (3, 64 << 10), (13, 1 << 20)):
        for final in (True, False):
            comp, cs, ds, used = ctx.compress_frames_csize(x, target, level, True, final=final)
            dcomp, dcs, dds, dused = dev.compress_csize(torch.from_numpy(x).cuda(), target, level, True, final=final)
            assert dcomp.cpu().numpy().tobytes() == comp.tobytes() and list(dcs) == list(cs) and list(dds) == list(ds) and dused == used
    ctx.close()


@pytest.mark.gpu
def test_first_frame_closes_at_one_gib(gpu_lib):
    import torch
    from zeekstd_b200 import parallel
    ctx = zk.Context(0, gpu_lib)
    n = (1 << 30) + (1 << 20)
    comp, cs, ds, used = parallel.DeviceCodec(ctx).compress_csize(torch.zeros(n, dtype=torch.uint8, device="cuda"), HUGE, 1, False)
    assert list(ds) == [1 << 30, 1 << 20] and used == n
    blocks, fcs, _ = parse_frame(comp[: int(cs[0])].cpu().numpy().tobytes())
    assert fcs == 1 << 30 and len(blocks) == (1 << 30) // BLOCK
    ctx.close()
