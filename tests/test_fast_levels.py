"""Negative compression levels (zstd's fast mode, acceleration = -level): the fast tier of K-C1 (sparse probing, backward extension) with
literals stored Raw or RLE.  Archives must restore through libzstd and the codec's decoder, carry no Huffman literals, keep the expected ratio
order, clamp below -131072 as libzstd does, follow prefix mode and the Compressed(n) rule, and reach the host layer and the CLI.  Every case
runs on the emulation build (`-m "not gpu"`, small inputs) and on the H100 (`-m gpu`, MiB-scale)."""
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
from test_csize_policy import check_parity, check_restores, check_rule
from util import GOLDEN, golden_bytes, offsets
from zeekstd_b200 import _native, corpus

BLOCK = 32 << 10
FAST = [-1, -2, -5, -31, -1000, -131072]
KINDS = ["dickens", "text", "structured", "lowent", "random", "runs"]


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
    if kind == "dickens":
        d = np.frombuffer(golden_bytes("dickens.txt"), dtype=np.uint8)
        return np.resize(d, n) if n > d.size else d[:n].copy()
    return corpus.as_numpy(corpus.make_class(kind, n, seed))


def _roundtrip(ctx, x: np.ndarray, frame_size: int, level: int, checksum: bool, prefix=None) -> np.ndarray:
    """compress, restore through libzstd and through the codec's decoder, check the literals form; -> the archive"""
    comp, cs, ds = ctx.compress_frames(x, frame_size, level, checksum, prefix)
    assert len(cs) == max(1, -(-x.size // frame_size)) and int(np.sum(ds)) == x.size
    out, sizes = O.ref_decompress_frames(np.concatenate([comp, np.zeros(64, np.uint8)]), offsets(cs), offsets(ds), prefix=prefix)
    assert out.tobytes() == x.tobytes() and sizes == [int(d) for d in ds], (frame_size, level, checksum)
    back, st, rc = ctx.decompress_frames(np.concatenate([comp, np.zeros(64, np.uint8)]), offsets(cs), offsets(ds), True, prefix=prefix)
    assert rc == 0 and not any(st) and back[: x.size].tobytes() == x.tobytes(), (frame_size, level, checksum)
    fs = O.frame_stats(comp)
    assert fs["lit_huf"] == 0 and fs["lit_treeless"] == 0, fs
    return comp


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("level", FAST)
def test_round_trip(ctx, level, kind):
    n = _scale(ctx, 3 * BLOCK + 1111, 5 << 20)
    x = _data(kind, n, 11)
    # frame sizes 1 and 100 on a prefix of the input: one frame per byte / per 100 bytes
    sizes = {1: _scale(ctx, 300, 20_000), 100: _scale(ctx, 20_000, 1 << 20), BLOCK - 1: n, BLOCK + 1: n, 2 << 20: n}
    for fs, m in sizes.items():
        for checksum in (False, True):
            _roundtrip(ctx, x[:m], fs, level, checksum)
    comp, cs, ds = ctx.compress_frames(x[:0], 1 << 20, level, True)
    assert list(ds) == [0] and O.ref_decompress_any(comp, 1) == b""


def test_levels_below_the_minimum_clamp(ctx):
    x = _data("dickens", _scale(ctx, 2 * BLOCK + 500, 4 << 20))
    want = ctx.compress_frames(x, 40_000, -131072, True)[0].tobytes()
    for level in (-131073, -(1 << 31)):
        assert ctx.compress_frames(x, 40_000, level, True)[0].tobytes() == want


def test_level_0_is_level_3(ctx):
    x = _data("text", _scale(ctx, 2 * BLOCK + 500, 4 << 20))
    assert ctx.compress_frames(x, 40_000, 0, True)[0].tobytes() == ctx.compress_frames(x, 40_000, 3, True)[0].tobytes()


def test_ratio_order_on_dickens(ctx):
    x = _data("dickens", _scale(ctx, 1 << 20, 10 << 20))
    ratio = {lv: x.size / ctx.compress_frames(x, 2 << 20, lv, False)[0].size for lv in (1, -1, -3, -7, -131072)}
    assert ratio[1] > ratio[-1] >= ratio[-3] >= ratio[-7] >= ratio[-131072], ratio


def test_prefix(ctx):
    x = _data("text", _scale(ctx, 3 * BLOCK + 77, 4 << 20), 8)
    prefix = _data("text", 50_000, 8)                                      # the same generator: the prefix helps
    comp = _roundtrip(ctx, x, 40_000, -1, True, prefix)
    cs = ctx.compress_frames(x, 40_000, -1, True, prefix)[1]
    _, st = O.oracle_decompress_ex(comp[: int(cs[0])].tobytes(), 40_000, prefix=prefix)
    assert st["prefix_matches"] > 0, st


@pytest.mark.parametrize("level", [-1, -7])
def test_compressed_policy(ctx, level):
    n = _scale(ctx, 4 * BLOCK + 5000, 6 << 20)
    for kind in ("text", "random"):
        x = _data(kind, n, 3)
        for target, checksum in ((700, False), (_scale(ctx, 40_000, 1 << 20), True), (1 << 31, False)):
            comp, cs, ds, used = ctx.compress_frames_csize(x, target, level, checksum)
            assert used == n
            frames = check_rule(comp, cs, ds, n, target)
            check_parity(ctx, x, frames, ds, level, checksum)
            check_restores(ctx, x, frames, ds)
    prefix = _data("text", 50_000, 3)
    x = _data("text", n, 3)
    comp, cs, ds, _ = ctx.compress_frames_csize(x, 20_000, level, True, prefix)
    frames = check_rule(comp, cs, ds, n, 20_000)
    check_parity(ctx, x, frames, ds, level, True, prefix)
    check_restores(ctx, x, frames, ds, prefix)


def test_encoders(ctx):
    x = _data("text", _scale(ctx, 3 * BLOCK + 999, 3 << 20), 6)
    data = x.tobytes()
    for policy in (zk.FrameSizePolicy.Uncompressed(40_000), zk.FrameSizePolicy.Compressed(20_000)):
        sink = io.BytesIO()
        enc = zk.EncodeOptions(ctx).frame_size_policy(policy).compression_level(-3).into_encoder(sink)
        for p in range(0, len(data), 4096):
            enc.compress(data[p:p + 4096])
        enc.finish()
        arch = sink.getvalue()
        assert zk.Decoder(zk.DecodeOptions(arch, ctx)).read_all() == data
        assert O.ref_decompress_any(arch, len(data) + 1) == data
        # RawEncoder, including the trial path of Compressed(n)
        raw = zk.EncodeOptions(ctx).frame_size_policy(policy).compression_level(-3).into_raw_encoder()
        out, st, pos = io.BytesIO(), bytearray(1 << 18), 0
        while pos < len(data):
            pr = raw.compress(memoryview(data)[pos:pos + 50_000], st)
            out.write(st[: pr.out_progress]); pos += pr.in_progress
        while True:
            pr = raw.end_frame(st)
            out.write(st[: pr.out_progress])
            if pr.data_left == 0:
                break
        assert O.ref_decompress_any(out.getvalue(), len(data) + 1) == data


def test_cli(ctx, tmp_path):
    x = _data("text", _scale(ctx, 2 * BLOCK + 321, 3 << 20), 9)
    src = tmp_path / "in.bin"; src.write_bytes(x.tobytes())
    for i, flag in enumerate((["-l", "-3"], ["--compression-level=-3"])):
        out = tmp_path / f"in{i}.zst"; back = tmp_path / f"back{i}.bin"
        rc, _, err = cases._cli(ctx, ["compress", "-q", *flag, "-o", out, src])
        assert rc == 0, err
        arch = out.read_bytes()
        assert O.frame_stats(arch)["lit_huf"] == 0
        assert O.ref_decompress_any(arch, x.size + 1) == x.tobytes()
        rc, _, err = cases._cli(ctx, ["decompress", "-q", "-o", back, out])
        assert rc == 0 and back.read_bytes() == x.tobytes(), err
    for bad in ("0", "20"):
        rc, _, _ = cases._cli(ctx, ["compress", "-q", "-l", bad, "-o", tmp_path / "bad.zst", src])
        assert rc != 0 and not (tmp_path / "bad.zst").exists()


def test_encoder_golden(ctx):
    """the fast tier's bytes are the same on every build: tests/golden/encoder_golden_fast.json was written from the emulation build"""
    spec = importlib.util.spec_from_file_location("make_encoder_golden_fast", os.path.join(GOLDEN, "make_encoder_golden_fast.py"))
    mk = importlib.util.module_from_spec(spec); spec.loader.exec_module(mk)
    gold = json.loads(golden_bytes("encoder_golden_fast.json"))
    got = {}
    for name, (data, fs, ck) in mk.inputs().items():
        for lvl in mk.LEVELS:
            comp = ctx.compress_frames(data, fs, lvl, ck)[0]
            got[f"{name}:{lvl}"] = {"size": int(comp.size), "sha256": hashlib.sha256(comp.tobytes()).hexdigest()}
    assert got == gold


@pytest.mark.gpu
def test_bench_mix_device_round_trip(gpu_lib):
    import torch
    import bench
    from zeekstd_b200 import parallel
    ctx = zk.Context(0, gpu_lib)
    dev = parallel.DeviceCodec(ctx)
    x = bench.gen_mix(1 << 30, bench.SEED, device="cuda")
    comp, cs, ds = dev.compress(x, 2 << 20, -1, True)
    back = dev.decompress(comp, offsets(cs), offsets(ds), True)
    assert torch.equal(back, x)
    del comp, back, x
    ctx.close()


@pytest.mark.gpu
def test_device_entry_points_match_host(gpu_lib):
    import torch
    from zeekstd_b200 import parallel
    ctx = zk.Context(0, gpu_lib)
    dev = parallel.DeviceCodec(ctx)
    x = _data("text", 5 << 20, 12)
    xd = torch.from_numpy(x).cuda()
    for level in (-1, -7, -131072):
        comp, cs, ds = ctx.compress_frames(x, 1 << 20, level, True)
        dcomp, dcs, dds = dev.compress(xd, 1 << 20, level, True)
        assert dcomp.cpu().numpy().tobytes() == comp.tobytes() and list(dcs) == list(cs) and list(dds) == list(ds)
        comp, cs, ds, used = ctx.compress_frames_csize(x, 256 << 10, level, True)
        dcomp, dcs, dds, dused = dev.compress_csize(xd, 256 << 10, level, True)
        assert dcomp.cpu().numpy().tobytes() == comp.tobytes() and list(dcs) == list(cs) and list(dds) == list(ds) and dused == used
    ctx.close()
