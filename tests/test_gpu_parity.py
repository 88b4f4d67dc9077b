"""`-m gpu`: the parity tests proper, through the C ABI of the real sm_90a library on an H100.
Same bodies as the emulated suite (tests/cases.py) at realistic sizes, the committed golden fixtures, and -- at
BASELINE.json's full sizes -- size-independent properties (round trips, libzstd cross-decoding).
The oracle is the image's libzstd (1.5.5; the reference pins 1.5.7 through zstd-sys -- same format, same decoder
output by construction: a valid frame has exactly one decoding).  The last test of this file asserts that every cell of
the decoder coverage matrix (SURVEY.md 8a) was actually decoded on the GPU during this run."""
import hashlib
import os

import numpy as np
import pytest

import cases
import zeekstd_b200 as zk
from oracle import oracle as O
from util import decode_frames, golden_meta, make_ctx, offsets, split_frames
from zeekstd_b200 import corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(gpu_lib):
    c = make_ctx(gpu_lib)
    yield c
    c.close()


def test_native_library_is_the_one_running(ctx, gpu_lib):
    assert b"sm_90a" in gpu_lib.zk_version()
    before = ctx.kernel_launches
    cases.check_compress_roundtrip(ctx, corpus.make_class("text", 100_000, 1).numpy(), 50_000, 3, True)
    assert ctx.kernel_launches > before


@pytest.mark.parametrize("kind", ["text", "structured", "lowent", "random", "runs"])
@pytest.mark.parametrize("level,fs,ck", [(1, 2 << 20, False), (3, 512 << 10, True), (7, 1 << 20, True), (19, 300_000, False)])
def test_decode_matches_libzstd(ctx, kind, level, fs, ck):
    n = (6 << 20) if level < 19 else (1 << 20)
    cases.check_decode_matches_libzstd(ctx, corpus.make_class(kind, n, seed=level).numpy(), fs, level, ck)


def test_decode_frame_size_sweep(ctx):
    x = corpus.make_mix(1 << 20, seed=5, segment=32 << 10).numpy()
    for fs in (1, 10, 123, 3_000, 100_000, 1 << 20):              # cli/tests/integration/main.rs:10,146-179 frame sizes
        n = min(x.size, fs * 300)
        cases.check_decode_matches_libzstd(ctx, x[:n], fs, 3, fs % 2 == 0)


@pytest.mark.parametrize("kind", ["text", "structured", "lowent", "random", "runs"])
@pytest.mark.parametrize("level,fs,ck", [(1, 2 << 20, False), (3, 512 << 10, True), (7, 1 << 20, True)])
def test_compress_roundtrip(ctx, kind, level, fs, ck):
    r = cases.check_compress_roundtrip(ctx, corpus.make_class(kind, 6 << 20, seed=7).numpy(), fs, level, ck)
    assert r >= 0.99


def test_compression_levels_are_tiers(ctx):
    """EncodeOptions::compression_level (encode.rs:176): tiers 1, 2-3, 4-6 -- each denser than the one below on the reference's corpus
    (tiers 7-9, 10-12 and >= 13: the last tests of this file)"""
    d = corpus.dickens()[: 8 << 20]
    sizes = [ctx.compress_frames(d, 2 << 20, lvl, False)[0].size for lvl in (1, 3, 4)]
    assert sizes[0] > sizes[1] > sizes[2], sizes


def test_compress_edge_sizes(ctx):
    x = corpus.make_class("text", 300_000, 9).numpy()
    for n, fs in ((0, 100), (1, 100), (15, 100), (16, 16), (31, 100), (100, 100), (101, 100), (32_767, 1 << 20), (32_768, 32_768), (32_769, 65_536),
                  (65_537, 1 << 20), (300_000, 1), (300_000, 7), (300_000, 99_999)):
        if fs < 8:
            n = min(n, 3_000)
        cases.check_compress_roundtrip(ctx, x[:n], fs, 3, n % 2 == 0)


def test_compress_high_entropy_literals(ctx):
    """literal-heavy blocks: Huffman streams longer than the encoder's shared-memory buffer take the tiled packer,
    and the decoder sees 11-bit two-level tables with many long codes"""
    rng = np.random.default_rng(5)
    for k, level in ((64, 1), (128, 3), (200, 1), (250, 3)):
        cases.check_compress_roundtrip(ctx, rng.integers(0, k, 3 << 20, dtype=np.uint8), 1 << 20, level, k % 3 == 0)
    # skewed: a few very frequent symbols and a long tail of rare ones (deep trees, length-limited to 11 bits)
    p = 1.0 / np.arange(1, 257) ** 1.3; p /= p.sum()
    x = rng.choice(256, size=3 << 20, p=p).astype(np.uint8)
    cases.check_compress_roundtrip(ctx, x, 1 << 20, 1, True)
    cases.check_decode_matches_libzstd(ctx, x, 1 << 20, 3, True)


def test_compress_is_deterministic(ctx):
    x = corpus.make_mix(8 << 20, seed=3).numpy()
    a = ctx.compress_frames(x, 1 << 20, 1, True)[0].tobytes()
    b = ctx.compress_frames(x, 1 << 20, 1, True)[0].tobytes()
    assert hashlib.sha256(a).digest() == hashlib.sha256(b).digest()


def test_golden_archives(ctx):
    cases.check_golden_archives(ctx)


def test_corruption_detected(ctx):
    cases.check_corruption_is_detected(ctx, trials=60)


def test_special_entries(ctx):
    cases.check_special_entries(ctx)


def test_patch_cycle(ctx):
    """lib.rs:289-300 patch_cycle (+ the two frame-size-policy variants of lib.rs:302-313)"""
    cases.check_patch_cycle(ctx)
    cases.check_patch_cycle(ctx, zk.FrameSizePolicy.Uncompressed(3000))
    cases.check_patch_cycle(ctx, zk.FrameSizePolicy.Compressed(700))


def test_prefix_batches(ctx):
    cases.check_prefix_batches(ctx)


def test_level3_2mib_frames_checksum(ctx):
    """config-4 shape: level 3 (2 MiB window: offsets reach back to the frame start), 2 MiB frames, checksum on"""
    x = corpus.make_mix(24 << 20, seed=20260925, mix=corpus.CLASS_MIX_MIXED).numpy()
    cases.check_decode_matches_libzstd(ctx, x, 2 << 20, 3, True)
    cases.check_compress_roundtrip(ctx, x, 2 << 20, 3, True)
    # text only: long-range matches across the whole 2 MiB window
    cases.check_decode_matches_libzstd(ctx, corpus.make_class("text", 8 << 20, 4).numpy(), 2 << 20, 3, True)


@pytest.mark.parametrize("level", [1, 3])
def test_huge_single_frame(ctx, level):
    """frames up to 1 GiB are legal (lib.rs:58; cli/tests/integration/main.rs:10 uses "1G"): one 64 MiB frame, both ways"""
    x = corpus.make_mix(64 << 20, seed=77).numpy()
    cases.check_decode_matches_libzstd(ctx, x, 1 << 30, level, True)
    comp, cs, ds = ctx.compress_frames(x, 1 << 30, level, True)
    assert len(cs) == 1 and int(ds[0]) == x.size
    out, sizes = O.ref_decompress_frames(comp, offsets(cs), offsets(ds))
    assert sizes == [x.size] and out.tobytes() == x.tobytes()
    back, st, rc = ctx.decompress_frames(comp, offsets(cs), offsets(ds), True)
    assert rc == 0 and np.array_equal(back, x)


def test_config1_dickens(ctx):
    """BASELINE configs[0]: assets/dickens.txt (committed fixture), level 1, 2 MiB frames -- the libzstd side must reproduce the
    known-answer sizes recorded in golden.json, the GPU must decode that archive bit-exactly, and the GPU's own archive must
    be restored by libzstd; level 3 + checksum as well (lib/benches/compress.rs:24-40, decompress.rs:27-41 shapes)"""
    d = corpus.dickens()
    assert d is not None and d.size == 10_192_446 and hashlib.sha256(d.tobytes()).hexdigest() == golden_meta()["dickens_sha256"]
    for key, level, ck in (("l1_2m", 1, False), ("l3_2m_ck", 3, True)):
        frames, cs, ds = O.ref_compress_frames(d, 2 << 20, level, ck, threads=os.cpu_count())
        assert cs == golden_meta()[key]["c_sizes"] and ds == golden_meta()[key]["d_sizes"]
        out, st, rc = decode_frames(ctx, frames, ds, verify=True)
        assert rc == 0 and out == d.tobytes()
        cases.cover(frames, d.size)
        r = cases.check_compress_roundtrip(ctx, d, 2 << 20, level, ck)
        assert r > 2.0


def test_cli_front_end(ctx, tmp_path):
    """cli/tests/integration/main.rs: the reference's FRAME_SIZES ("10", "123", "3K", "2M", "1G") -- the whole corpus for the
    sizes that give a sane frame count, a 200 000-byte slice for the two tiny ones; plus a subprocess run of `python -m`"""
    d = corpus.dickens().tobytes()
    cases.check_cli(ctx, tmp_path, d, ["3K", "2M", "1G"], tag="full")
    with_p, without = cases.check_cli(ctx, tmp_path, d[1_000_000:1_200_000], ["10", "123"], tag="small")
    assert with_p < without * 0.7      # --patch-from: 3/4 of the new version is in the prefix
    import subprocess
    import sys
    src, z = tmp_path / "sub.txt", tmp_path / "sub.txt.zst"
    src.write_bytes(d[:3_000_000])
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "zeekstd_b200", str(src), "-q"], cwd=root, capture_output=True, timeout=600)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([sys.executable, "-m", "zeekstd_b200", "decompress", str(z), "-c", "--from", str(1 << 20), "--to", "2M"], cwd=root, capture_output=True, timeout=600)
    assert r.returncode == 0 and r.stdout == d[1 << 20: 2 << 20], r.stderr
    arc = np.frombuffer(z.read_bytes(), dtype=np.uint8)
    st = zk.SeekTable.from_bytes(arc)
    cs, ds = _table_sizes(st)
    out, sizes = O.ref_decompress_frames(arc[: st.size_comp()], offsets(cs), offsets(ds), threads=8)     # libzstd reads what the CLI wrote
    assert list(sizes) == ds and out[: 3_000_000].tobytes() == d[:3_000_000]


def _table_sizes(st):
    n = st.num_frames()
    return [st.frame_size_comp(i) for i in range(n)], [st.frame_size_decomp(i) for i in range(n)]


def test_window_limit(ctx):
    """Window_Size above the streaming default and blocks above Block_Maximum_Size = min(Window_Size, 128 KiB) are refused as by libzstd"""
    cases.check_window_limit(ctx)


def test_host_state_machines_random_ops(ctx):
    """randomised differential tests of Decoder (offsets / limits / frames / seeks / resets) and Encoder (framing, lazy close, manual
    end_frame, prefix) against models of the reference's contracts, larger than the emulator can afford"""
    cases.check_decoder_random_ops(ctx, ops=600, seed=31, n=3_000_000, frame_size=100_000)
    cases.check_decoder_random_ops(ctx, ops=300, seed=32, n=60_000, frame_size=1_700)
    assert cases.check_encoder_random_ops(ctx, ops=200, seed=33, frame_size=40_000) > 20
    cases.check_encoder_random_ops(ctx, ops=80, seed=36, frame_size=777, prefix=True)


def test_api_encode_side(ctx):
    cases.check_cycle_tiny_buffers(ctx)
    cases.check_cycle_tiny_buffers(ctx, zk.FrameSizePolicy.Uncompressed(777))
    cases.check_standalone_seek_table(ctx)
    assert cases.check_encoder_decoder_io(ctx) == 1
    assert cases.check_encoder_decoder_io(ctx, zk.FrameSizePolicy.Uncompressed(1000), chunk=333) == 13
    cases.check_frame_counts_match_reference(ctx)
    cases.check_raw_encoder_reset(ctx)
    cases.check_checksum_flag(ctx)


@pytest.mark.parametrize("n", [1, 2, 3, 17, 100, 511, 1023])
def test_frame_size_policies_property(ctx, n):
    cases.check_encoder_decoder_io(ctx, zk.FrameSizePolicy.Uncompressed(n), chunk=997)
    cases.check_encoder_decoder_io(ctx, zk.FrameSizePolicy.Compressed(n), chunk=4096)


def test_api_decode_side(ctx):
    cases.check_decoder_options(ctx)
    cases.check_decoder_state_machine(ctx)
    cases.check_libzstd_archive_through_decoder(ctx)


@pytest.mark.gpu
def test_range_reads_stop_early(ctx):
    cases.check_range_reads_stop_early(ctx, n=9_000_000, frame_size=2 << 20, reads=40)



def test_seek_table(gpu_lib):
    cases.check_seek_table(gpu_lib)


def test_encoder_batches_many_frames(ctx):
    """Encoder<W> hands whole batches of frames to the GPU; archive must equal frame-by-frame semantics"""
    import io
    x = corpus.make_mix(40 << 20, seed=2).numpy()
    sink = io.BytesIO()
    enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Uncompressed(256 << 10)).checksum_flag(True).into_encoder(sink)
    for i in range(0, x.size, 1 << 20):
        enc.write(x[i:i + (1 << 20)])
    total = enc.finish()
    a = sink.getvalue()
    assert total == len(a)
    st = O.OracleSeekTable.parse(a, "foot")
    assert st.num_frames() == 160 and st.d[-1] == x.size
    out, sizes = O.ref_decompress_frames(np.frombuffer(a, dtype=np.uint8), st.c, st.d, threads=os.cpu_count())
    assert out.tobytes() == x.tobytes()
    dec = zk.Decoder(zk.DecodeOptions(a, ctx))
    dec.set_offset(13 << 20); dec.set_offset_limit((13 << 20) + 65536)
    assert dec.read_all() == x[13 << 20: (13 << 20) + 65536].tobytes()


def test_full_size_roundtrip_properties(ctx):
    """BASELINE configs[1] size: 1 GiB, 2 MiB frames, level 1 -- compress on the GPU, decode with libzstd on all cores AND on
    the GPU; plus libzstd-compressed frames decoded on the GPU (bit-exact vs the reference decoder's output == the input)"""
    import torch
    n = int(os.environ.get("ZK_TEST_FULL_BYTES", str(1 << 30)))
    x = corpus.make_mix(n, seed=20260924, device="cuda").cpu().numpy()
    comp, cs, ds = ctx.compress_frames(x, 2 << 20, 1, False)
    assert len(cs) == n // (2 << 20) and int(ds.sum()) == n
    out, sizes = O.ref_decompress_frames(comp, offsets(cs), offsets(ds), threads=os.cpu_count())
    assert sizes == [int(d) for d in ds] and hashlib.sha256(out.tobytes()).digest() == hashlib.sha256(x.tobytes()).digest()
    back, st, rc = ctx.decompress_frames(comp, offsets(cs), offsets(ds), True)
    assert rc == 0 and np.array_equal(back, x)
    frames, rcs, rds = O.ref_compress_frames(x, 2 << 20, 1, False, threads=os.cpu_count())
    back, st, rc = ctx.decompress_frames(np.frombuffer(b"".join(frames) + b"\0" * 64, dtype=np.uint8), offsets(rcs), offsets(rds), True)
    assert rc == 0 and np.array_equal(back, x)


def test_many_small_frames(ctx):
    """config-3-like: high frame count (512 KiB frames of text), libzstd-compressed, GPU decode bit-exact"""
    x = corpus.make_text(256 << 20, seed=7, device="cuda").cpu().numpy()
    frames, cs, ds = O.ref_compress_frames(x, 512 << 10, 1, False, threads=os.cpu_count())
    back, st, rc = ctx.decompress_frames(np.frombuffer(b"".join(frames) + b"\0" * 64, dtype=np.uint8), offsets(cs), offsets(ds), False)
    assert rc == 0 and np.array_equal(back, x)


def test_random_offset_reads(ctx):
    """config-5-like: random 64 KiB reads through set_offset / set_offset_limit on a libzstd-written archive"""
    x = corpus.make_mix(128 << 20, seed=9, device="cuda").cpu().numpy()
    a, st = O.ref_seekable_archive(x, 2 << 20, 1, False, threads=os.cpu_count())
    dec = zk.Decoder(zk.DecodeOptions(a, ctx))
    rng = np.random.default_rng(7)
    for _ in range(40):
        o = int(rng.integers(0, x.size - 65536))
        dec.set_offset(o); dec.set_offset_limit(o + 65536)
        assert dec.read_all() == x[o:o + 65536].tobytes()
        dec.set_offset_limit(x.size)


def test_batched_range_reads(ctx):
    """seek.read_ranges == per-request Decoder semantics, including reads that straddle frames and batch boundaries"""
    from zeekstd_b200 import seek
    x = corpus.make_mix(24 << 20, seed=11, device="cuda").cpu().numpy()
    a, st = O.ref_seekable_archive(x, 1 << 20, 1, False, threads=os.cpu_count())
    arch = np.frombuffer(a + b"\0" * 64, dtype=np.uint8)
    rng = np.random.default_rng(1)
    offs = np.concatenate([rng.integers(0, x.size - 70_000, 200), np.arange(1, 20) * (1 << 20) - 1000])   # some cross frame borders
    outs, nfr = seek.read_ranges(ctx, arch, np.array(st.c), np.array(st.d), offs, 70_000, max_batch_bytes=3 << 20)
    for o, got in zip(offs, outs):
        assert got == x[int(o): int(o) + 70_000].tobytes()


def test_zz_decoder_coverage_matrix(ctx):
    """runs last: every cell of SURVEY.md 8a's decoder coverage matrix was decoded ON THE GPU by the tests above
    (block types, literal kinds, weight encodings, table modes, repeat-offset cases, header variants, skippable and multiple
    frames per entry, frames > 2 MiB, offsets > 1 MiB)"""
    totals = cases.check_coverage_matrix()
    print("coverage matrix:", totals)


def test_zzx_c_example_through_the_c_abi(tmp_path):
    """examples/roundtrip.c compiled as C99 against include/zeekstd_b200.h and run against the product library: no Python between the caller
    and the C ABI"""
    import subprocess
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_abi import _build_c_example
    from zeekstd_b200 import _native
    exe = _build_c_example(tmp_path, _native.PRODUCT_SO)
    r = subprocess.run([str(exe)], capture_output=True, timeout=300)
    assert r.returncode == 0 and r.stdout.startswith(b"ok: 100000 bytes"), (r.stdout, r.stderr)


def test_zzy_level_tiers_7_to_12(ctx):
    """levels 7-9 (8192-entry double table) and 10-12 (16384-entry table), one warp per CTA: denser than the tier below on the reference's
    corpus, every frame restored by libzstd (ragged tail, checksum, prefix).  The tests from here on cover what was added after the round's
    last GPU minutes (first run on a GPU: the driver's) -- they sit after the coverage-matrix assertion, least proven last."""
    d = corpus.dickens()[: 8 << 20]
    sizes = [ctx.compress_frames(d, 2 << 20, lvl, False)[0].size for lvl in (4, 7, 10)]
    assert sizes[0] > sizes[1] > sizes[2], sizes
    for lvl in (7, 9, 10, 12):
        for kind in ("text", "structured", "lowent", "random", "runs"):
            cases.check_compress_roundtrip(ctx, corpus.make_class(kind, 300_001, seed=lvl).numpy(), 131_072, lvl, lvl % 2 == 1)
    cases.check_prefix_batches(ctx, n=400_000, levels=(7, 10))


def test_zzz_encoder_bytes_are_pinned(ctx):
    """the nvcc build reproduces, byte for byte, the compressed output the CPU emulation build of the same sources wrote into
    tests/golden/encoder_golden.json (level tiers 1 ... 10-12 and prefix mode)"""
    cases.check_encoder_golden(ctx, skip=("13",))


def test_zzzz_wide_window_tier(ctx):
    """level >= 13: 256 KiB history, 32-bit positions, 32768-entry table in 128 KiB of dynamic shared memory, Window_Descriptor 256 KiB:
    denser than the tier below, offsets beyond 64 KiB really used, libzstd restores every frame (ragged tail, checksum, prefix), bytes equal to
    the emulation build's"""
    d = corpus.dickens()[: 8 << 20]
    c10, c13 = (ctx.compress_frames(d, 2 << 20, lvl, False)[0] for lvl in (10, 13))
    assert c13.size < c10.size and c13[5] == 0x40
    _, ss = O.oracle_decompress_ex(c13.tobytes(), d.size)
    assert ss["max_offset"] > 65_536
    for lvl in (13, 19):
        for kind in ("text", "structured", "lowent", "random", "runs"):
            cases.check_compress_roundtrip(ctx, corpus.make_class(kind, 600_001, seed=lvl).numpy(), 300_000, lvl, lvl % 2 == 1)
    cases.check_prefix_batches(ctx, n=400_000, levels=(13,))
    cases.check_encoder_golden(ctx, only=("13",))
