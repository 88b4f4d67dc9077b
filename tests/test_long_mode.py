"""Long mode (zk_compress_frames_long[_dev], zk_compress_frames_sized_long[_dev], long_mode=True, --long-mode; zk_ldm.inc's index of the
input): every frame also copies from its own bytes up to zkc_ldm_window back, so a large frame finds the repeats that lie beyond the 2 MiB
that level 16 searches.  The archive restores through libzstd, the codec's decoder and the plain-C restatement; the Window_Descriptor follows
the long-distance rule and covers every offset; a frame's bytes depend on its own bytes alone (not on the batch, the sub-batch size, the
entry point or the Encoder's write sizes); with a prefix it is a superset of the long-distance switch; Compressed(n) and ContentDefined(s)
refuse it.  Every case runs on the emulation build (`-m "not gpu"`, small inputs: the repeats there lie within level 16's window) and on
the H100 (`-m gpu`, MiB scale, repeats beyond it)."""
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
from util import GOLDEN, golden_bytes, offsets
from zeekstd_b200 import _native

BLOCK = 32 << 10
HC_WINDOW = 2 << 20

_spec = importlib.util.spec_from_file_location("make_encoder_golden_long", os.path.join(GOLDEN, "make_encoder_golden_long.py"))
mk = importlib.util.module_from_spec(_spec); _spec.loader.exec_module(mk)
edited_copy, mix, skewed, far_repeats = mk.edited_copy, mk.mix, mk.skewed, mk.far_repeats


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


def _window_size(wd: int) -> int:
    e, m = wd >> 3, wd & 7
    return (1 << (10 + e)) + ((1 << (10 + e)) >> 3) * m


def _window_descriptor(content: int, prefix_len: int) -> int:
    """the long-distance rule: the smallest Window_Descriptor >= max(128 KiB, min(content + prefix_len, 2^27))"""
    want = max(128 << 10, min(content + prefix_len, 1 << 27))
    return next(wd for wd in range(256) if _window_size(wd) >= want)


def _restores(ctx, comp, cs, ds, x, prefix=None):
    """the archive restores through libzstd (default DCtx, refPrefix with a prefix), the codec's decoder and the plain-C restatement; every
    frame announces the long-distance window and no offset exceeds it -> merged sequence statistics of the restatement"""
    pad = np.concatenate([comp, np.zeros(64, np.uint8)])
    co, do = offsets(cs), offsets(ds)
    out, sizes = O.ref_decompress_frames(pad, co, do, prefix=prefix)
    assert out.tobytes() == x.tobytes() and sizes == [int(d) for d in ds]
    back, st, rc = ctx.decompress_frames(pad, co, do, True, prefix=prefix)
    assert rc == 0 and not any(st) and back[: x.size].tobytes() == x.tobytes()
    plen = 0 if prefix is None else len(prefix)
    total = {"seqs": 0, "max_offset": 0, "prefix_matches": 0}
    for f in range(len(cs)):
        fr = comp[int(co[f]):int(co[f + 1])]
        got, s = O.oracle_decompress_ex(fr, int(ds[f]), prefix=prefix)
        assert got == x[int(do[f]):int(do[f + 1])].tobytes()
        assert fr[5] == _window_descriptor(int(ds[f]), plen if ds[f] else 0), f
        assert s["max_offset"] <= _window_size(int(fr[5])), (f, s)
        total["seqs"] += s["explicit_offsets"] + s["rep1"] + s["rep2"] + s["rep3"] + s["rep1_minus_1"]
        total["prefix_matches"] += s["prefix_matches"]
        total["max_offset"] = max(total["max_offset"], s["max_offset"])
    return total


def test_finds_what_the_window_cannot(ctx):
    """A (mix), B (skewed random), an edited A, an edited B in one frame: on the H100 the copies lie 6 MiB after their originals, beyond
    level 16's window, and long mode writes a fraction of level 16's archive"""
    x = far_repeats(_scale(ctx, 24 << 10, 3 << 20), 1)
    l16 = ctx.compress_frames(x, x.size, 16, True)[0]
    comp, cs, ds = ctx.compress_frames(x, x.size, 16, True, long_mode=True)
    print(f"one frame of {x.size} B ({'emulation' if _emul(ctx) else 'H100'}): level 16 {l16.size} B, long mode {comp.size} B")
    st = _restores(ctx, comp, cs, ds, x)
    if _emul(ctx):
        assert comp.size <= 1.01 * l16.size
    else:
        assert comp.size < 0.6 * l16.size
        assert st["max_offset"] > HC_WINDOW
    # skewed random bytes: nothing 64 bytes long repeats, so level 16's size to within 1 %
    y = skewed(_scale(ctx, 64 << 10, 8 << 20), 2)
    a = ctx.compress_frames(y, y.size, 16, True)[0].size
    comp, cs, ds = ctx.compress_frames(y, y.size, 16, True, long_mode=True)
    assert abs(int(comp.size) - int(a)) <= 0.01 * a
    _restores(ctx, comp, cs, ds, y)
    # all-equal bytes: every position hashes alike; the call ends and writes a few sequences per block
    z = np.full(_scale(ctx, 96 << 10, 8 << 20), 0x41, np.uint8)
    comp, cs, ds = ctx.compress_frames(z, z.size, 16, True, long_mode=True)
    st = _restores(ctx, comp, cs, ds, z)
    assert st["seqs"] <= 4 * -(-z.size // BLOCK)


def test_frames_stand_alone(ctx, monkeypatch):
    """uniform call == sized call at the same sizes == one call per frame, at frames placed at odd offsets, at small sub-batches, through
    the Encoder at odd write sizes and the RawEncoder; every level writes level 16's bytes"""
    x = far_repeats(_scale(ctx, 24 << 10, 1 << 20), 3)
    fs = _scale(ctx, 40_000, 3 << 20)
    n = x.size
    uniform, ucs, uds = ctx.compress_frames(x, fs, 16, True, long_mode=True)
    sizes = [fs] * (n // fs) + ([n % fs] if n % fs else [])
    assert ctx.compress_frames_sized(x, sizes, 16, True, long_mode=True)[0].tobytes() == uniform.tobytes()
    _restores(ctx, uniform, ucs, uds, x)
    for lvl in (-5, 3, 19):
        assert ctx.compress_frames(x, fs, lvl, True, long_mode=True)[0].tobytes() == uniform.tobytes(), lvl
    # frames at odd offsets of the batch, empty ones included: each is what a call for its bytes alone writes
    odd = [BLOCK + 1, 1, 0, BLOCK - 1, n - 2 * BLOCK - 1, 0]
    comp, cs, ds = ctx.compress_frames_sized(x, odd, 16, True, long_mode=True)
    _restores(ctx, comp, cs, ds, x)
    co, do = offsets(cs), offsets(ds)
    for f, d in enumerate(odd):
        alone = ctx.compress_frames(x[int(do[f]):int(do[f + 1])], max(d, 1), 16, True, long_mode=True)[0]
        assert comp[int(co[f]):int(co[f + 1])].tobytes() == alone.tobytes(), f
    # sub-batches of a frame or two
    monkeypatch.setenv("ZK_HOST_SUB_BYTES_ENC", str(BLOCK + 2))
    assert ctx.compress_frames_sized(x, odd, 16, True, long_mode=True)[0].tobytes() == comp.tobytes()
    assert ctx.compress_frames(x, fs, 16, True, long_mode=True)[0].tobytes() == uniform.tobytes()
    monkeypatch.delenv("ZK_HOST_SUB_BYTES_ENC")
    # Encoder at odd write sizes: the batch call, frame for frame
    sink = io.BytesIO()
    enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Uncompressed(fs)).checksum_flag(True).long_mode(True).into_encoder(sink)
    data, pos, step = x.tobytes(), 0, 7777
    while pos < len(data):
        pos += enc.compress(memoryview(data)[pos:pos + step]); step = step * 3 % 50_021 + 1
    enc.finish()
    assert sink.getvalue()[: uniform.size] == uniform.tobytes()
    # RawEncoder, under both of its policies: its first frame
    for policy, end in ((zk.FrameSizePolicy.Uncompressed(fs), fs), (zk.FrameSizePolicy.Compressed(1 << 30), n)):
        raw = zk.EncodeOptions(ctx).frame_size_policy(policy).checksum_flag(True).long_mode(True).into_raw_encoder()
        out, buf, pos = io.BytesIO(), bytearray(1 << 20), 0
        while pos < end:
            pr = raw.compress(memoryview(data)[pos:min(pos + 20_000, end)], buf)
            out.write(buf[: pr.out_progress]); pos += pr.in_progress
        while True:
            pr = raw.end_frame(buf)
            out.write(buf[: pr.out_progress])
            if pr.data_left == 0:
                break
        want = uniform.tobytes()[: int(ucs[0])] if end == fs else ctx.compress_frames(x, n, 16, True, long_mode=True)[0].tobytes()
        assert out.getvalue() == want


def test_with_a_prefix(ctx):
    """NEW = an edited OLD followed by an edited copy of its own first half: long mode restores with the prefix, is no larger than the
    long-distance switch alone, and writes level 16's bytes at every level"""
    n = _scale(ctx, 48 << 10, 4 << 20)
    old = mix(n, 4)
    first = edited_copy(old, 5, _scale(ctx, 4, 40))
    new = np.concatenate([first, edited_copy(first[: first.size // 2], 6, _scale(ctx, 3, 30))])
    fs = _scale(ctx, 1 << 20, 8 << 20)
    comp, cs, ds = ctx.compress_frames(new, fs, 16, True, prefix=old, long_mode=True)
    ldm = ctx.compress_frames(new, fs, 16, True, prefix=old, long_distance=True)[0]
    print(f"NEW {new.size} B after OLD {old.size} B: long-distance switch {ldm.size} B, long mode {comp.size} B")
    st = _restores(ctx, comp, cs, ds, new, old)
    assert st["prefix_matches"] > 0
    assert comp.size <= ldm.size
    for lvl in (-5, 3, 19):
        assert ctx.compress_frames(new, fs, lvl, True, prefix=old, long_mode=True)[0].tobytes() == comp.tobytes(), lvl
    # both switches: long mode
    assert ctx.compress_frames(new, fs, 16, True, prefix=old, long_distance=True, long_mode=True)[0].tobytes() == comp.tobytes()


@pytest.mark.parametrize("content,prefix_len", [(1, 0), (100, 0), (5000, 0), (BLOCK + 1, 0), (150_000, 0), (1000, 64), (70_000, 5),
                                                (150_000, 150_000), (5000, 200_000)])
def test_window(ctx, content, prefix_len):
    src = mix(max(content, prefix_len) + 4096, 7)
    old = src[:prefix_len] if prefix_len else None
    x = np.concatenate([src[100:100 + content // 2], src[: content - content // 2]])
    comp, cs, ds = ctx.compress_frames(x, 1 << 20, 3, True, prefix=old, long_mode=True)
    assert comp[5] == _window_descriptor(content, prefix_len)
    _restores(ctx, comp, cs, ds, x, old)


def test_refusals(ctx, lib, tmp_path):
    """Compressed(n) and ContentDefined(s) have no long mode: into_encoder refuses it (-1006) and leaves the options with the caller, and the
    CLI says so and writes nothing"""
    sink = _native.WRITE_FN(lambda user, p, n: 0)
    for kind, size in ((zk.FrameSizePolicy.Compressed(1).kind, 10_000), (zk.FrameSizePolicy.ContentDefined(1 << 16).kind, 1 << 16)):
        o = ctypes.c_void_p(lib.zk_encode_options_new(ctx._h))
        lib.zk_encode_options_frame_size_policy(o, kind, size)
        lib.zk_encode_options_long_mode(o, 1)
        e = ctypes.c_void_p()
        assert lib.zk_encode_options_into_encoder(o, sink, _native.FLUSH_FN(0), None, ctypes.byref(e)) == -1006
        lib.zk_encode_options_long_mode(o, 0)                  # still the caller's: usable once the option is off
        assert lib.zk_encode_options_into_encoder(o, sink, _native.FLUSH_FN(0), None, ctypes.byref(e)) == 0
        lib.zk_encoder_free(e)
    for policy in (zk.FrameSizePolicy.Compressed(10_000), zk.FrameSizePolicy.ContentDefined(1 << 16)):
        with pytest.raises(zk.Error) as err:
            zk.EncodeOptions(ctx).frame_size_policy(policy).long_mode(True).into_encoder(io.BytesIO())
        assert err.value.rc == -1006
    src = tmp_path / "in.bin"; src.write_bytes(mix(10_000, 8).tobytes())
    for policy in ("compressed", "content"):
        out = tmp_path / f"{policy}.zst"
        rc, _, err = cases._cli(ctx, ["compress", "-q", "--long-mode", "--frame-size-policy", policy, "-o", out, src])
        assert rc != 0 and "--long-mode" in err and not out.exists()
    assert _native._SIGS["zk_compress_frames_long"] == _native._SIGS["zk_compress_frames_prefix"]
    assert _native._SIGS["zk_compress_frames_sized_long"] == _native._SIGS["zk_compress_frames_sized"]
    assert _native._SIGS["zk_compress_frames_long_dev"] == _native._SIGS["zk_compress_frames_dev"]
    assert _native._SIGS["zk_compress_frames_sized_long_dev"] == _native._SIGS["zk_compress_frames_sized_dev"]


def test_cli(ctx, tmp_path):
    x = far_repeats(_scale(ctx, 16 << 10, 2 << 20), 9)
    src = tmp_path / "in.bin"; src.write_bytes(x.tobytes())
    a, back = tmp_path / "a.zst", tmp_path / "back.bin"
    rc, _, err = cases._cli(ctx, ["compress", "-q", "--long-mode", "-s", "8M", "-o", a, src])
    assert rc == 0, err
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "-o", back, a])
    assert rc == 0 and back.read_bytes() == x.tobytes(), err
    sink = io.BytesIO()
    enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Uncompressed(8 << 20)).checksum_flag(True).compression_level(3)
    enc = enc.long_mode(True).into_encoder(sink)
    data, pos = x.tobytes(), 0
    while pos < len(data):
        pos += enc.compress(memoryview(data)[pos:pos + (1 << 17)])
    enc.finish()
    assert a.read_bytes() == sink.getvalue()
    # with --patch-from: the reference file as well
    old = tmp_path / "old.bin"; old.write_bytes(x[: x.size // 2].tobytes())
    b = tmp_path / "b.zst"
    rc, _, err = cases._cli(ctx, ["compress", "-q", "--long-mode", "--patch-from", old, "-o", b, src])
    assert rc == 0, err
    back2 = tmp_path / "back2.bin"
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "--patch-apply", old, "-o", back2, b])
    assert rc == 0 and back2.read_bytes() == x.tobytes(), err


def test_encoder_golden(ctx):
    """the matcher's bytes are the same on every build: tests/golden/encoder_golden_long.json was written from the emulation build"""
    gold = json.loads(golden_bytes("encoder_golden_long.json"))
    got = {}
    for name, (x, fs, ck, prefix) in mk.inputs().items():
        comp = ctx.compress_frames(x, fs, 19, ck, prefix=prefix, long_mode=True)[0]
        got[name] = {"size": int(comp.size), "sha256": hashlib.sha256(comp.tobytes()).hexdigest()}
    assert got == gold


@pytest.mark.gpu
def test_device_calls_match_host(gpu_lib, monkeypatch):
    """the _dev pair writes the host calls' bytes, at the default and at a small device sub-batch"""
    import torch
    ctx = zk.Context(0, gpu_lib)
    x = far_repeats(3 << 20, 10)
    sizes = [BLOCK + 1, 1, 0, (5 << 20) - 7, x.size - BLOCK - (5 << 20) + 5]
    want = ctx.compress_frames(x, 6 << 20, 16, True, long_mode=True)[0].tobytes()
    want_sized, wcs, _ = ctx.compress_frames_sized(x, sizes, 16, True, long_mode=True)
    xd = torch.from_numpy(np.concatenate([x, np.zeros(64, np.uint8)])).cuda()
    ds = np.asarray(sizes, np.uint32)
    from zeekstd_b200.parallel import DeviceCodec
    dev = DeviceCodec(ctx)
    for sub in (None, 6 << 20):
        if sub:
            monkeypatch.setenv("ZK_DEV_SUB_BYTES", str(sub))
        got = dev.compress(xd[: x.size], 6 << 20, 16, True, long_mode=True)[0]
        torch.cuda.synchronize()
        assert got.cpu().numpy().tobytes() == want
        cap = gpu_lib.zk_compress_bound_sized(ds.ctypes.data_as(_native.u32p), len(sizes))
        out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        dcs = np.zeros(len(sizes), np.uint32); dl = ctypes.c_size_t()
        rc = gpu_lib.zk_compress_frames_sized_long_dev(ctx._h, xd.data_ptr(), ds.ctypes.data_as(_native.u32p), len(sizes), 16, 1,
                                                       out.data_ptr(), cap, dcs.ctypes.data_as(_native.u32p), ctypes.byref(dl), None)
        torch.cuda.synchronize()
        assert rc == 0 and out[: dl.value].cpu().numpy().tobytes() == want_sized.tobytes() and list(dcs) == list(wcs)
    ctx.close()


@pytest.mark.gpu
def test_repeat_in_an_earlier_internal_pass(gpu_lib):
    """a 72 MiB frame whose second copy of A lies more than 64 MiB after the first, in K-C1h's next internal pass"""
    ctx = zk.Context(0, gpu_lib)
    a = mix(4 << 20, 11)
    x = np.concatenate([a, skewed(64 << 20, 12), edited_copy(a, 13, 20)])
    comp, cs, ds = ctx.compress_frames(x, x.size, 16, True, long_mode=True)
    st = _restores(ctx, comp, cs, ds, x)
    assert st["max_offset"] > 64 << 20
    ctx.close()


def pass_cut_input() -> np.ndarray:
    """72 MiB: A (8 MiB of the mix), 52 MiB of skewed random bytes, A with a byte changed every 100-400 bytes, 4 MiB of skewed random bytes.
    The second A lies 60 MiB after the first and straddles 64 MiB, where K-C1h cuts its first internal pass when the frame starts the
    batch: its far repeat offsets are tested on both sides of the cut"""
    a = mix(8 << 20, 16)
    b = a.copy()
    idx = np.cumsum(np.random.default_rng(17).integers(100, 400, b.size // 100))
    b[idx[idx < b.size]] ^= 0x5A
    return np.concatenate([a, skewed(52 << 20, 18), b, skewed(4 << 20, 19)])


@pytest.mark.gpu
def test_pass_cuts_do_not_change_a_frame(gpu_lib):
    """the frame above, alone and behind other frames in one sized batch (so that the batch's 64 MiB passes cut it elsewhere), is the same
    bytes"""
    ctx = zk.Context(0, gpu_lib)
    x = pass_cut_input()
    alone = ctx.compress_frames(x, x.size, 16, True, long_mode=True)[0]
    for lead in ([1], [BLOCK - 1, 5 * BLOCK + 3]):
        data = np.concatenate([mix(sum(lead), 20), x])
        comp, cs, ds = ctx.compress_frames_sized(data, lead + [x.size], 16, True, long_mode=True)
        assert comp[int(offsets(cs)[-2]):].tobytes() == alone.tobytes(), lead
    _restores(ctx, comp, cs, ds, data)
    ctx.close()


@pytest.mark.gpu
def test_one_gib_device_call(gpu_lib):
    """one 1 GiB frame of sixteen copies of 64 MiB through zk_compress_frames_long_dev: every copy after the first is a few long matches"""
    import torch
    from zeekstd_b200 import corpus
    from zeekstd_b200.parallel import DeviceCodec
    ctx = zk.Context(0, gpu_lib)
    dev = DeviceCodec(ctx)
    x = torch.cat([corpus.make_mix(64 << 20, seed=14).cuda()] * 16)
    comp, cs, ds = dev.compress(x, 1 << 30, 16, True, long_mode=True)
    l16 = dev.compress(x, 1 << 30, 16, True)[0]
    torch.cuda.synchronize()
    print(f"1 GiB of 16 x 64 MiB: level 16 {l16.numel()} B, long mode {comp.numel()} B")
    assert comp.numel() < 0.25 * l16.numel()
    back = dev.decompress(comp, offsets(cs), offsets(ds), True)
    torch.cuda.synchronize()
    assert torch.equal(back, x)
    ctx.close()
