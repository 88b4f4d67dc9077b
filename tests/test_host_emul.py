"""`-m "not gpu"` suite: the host layer and the kernel LOGIC, run on the emulated build of the same sources
(tests/emul: device code interpreted on the CPU).  Inputs are tiny because every CUDA thread is a coroutine here; the
same bodies (tests/cases.py) run at realistic sizes on the H100 in test_gpu_parity.py."""
import numpy as np
import pytest

import cases
import zeekstd_b200 as zk
from util import make_ctx
from zeekstd_b200 import corpus


@pytest.fixture(scope="module")
def ctx(emul_lib):
    c = make_ctx(emul_lib)
    yield c
    c.close()


def test_seek_table(emul_lib):
    cases.check_seek_table(emul_lib)


def test_seek_table_parser_fuzz(emul_lib):
    cases.check_seek_table_fuzz(emul_lib)


@pytest.mark.parametrize("kind,level,fs,ck", [("text", 1, 20_000, False), ("text", 3, 9_000, True), ("structured", 3, 30_000, True),
                                               ("lowent", 5, 30_000, False), ("random", 1, 8_000, True), ("runs", 3, 30_000, True),
                                               ("text", 19, 30_000, True)])
def test_decode_matches_libzstd(ctx, kind, level, fs, ck):
    cases.check_decode_matches_libzstd(ctx, corpus.make_class(kind, 30_000, seed=level).numpy(), fs, level, ck)


def test_decode_tiny_frames_and_empty(ctx):
    x = corpus.make_class("text", 3_000, 1).numpy()
    cases.check_decode_matches_libzstd(ctx, x, 100, 3, False)     # 1-stream Huffman / raw literals / predefined tables
    cases.check_decode_matches_libzstd(ctx, x[:1], 100, 1, True)


@pytest.mark.parametrize("kind,level,fs,ck", [("text", 3, 40_000, True), ("text", 1, 11_000, False), ("structured", 3, 40_000, False),
                                               ("lowent", 3, 40_000, True), ("random", 3, 40_000, True), ("runs", 3, 40_000, True),
                                               ("text", 5, 40_000, True), ("lowent", 9, 40_000, False), ("structured", 19, 12_000, True)])
def test_compress_roundtrip(ctx, kind, level, fs, ck):
    cases.check_compress_roundtrip(ctx, corpus.make_class(kind, 40_000, seed=3).numpy(), fs, level, ck)


def test_compress_edge_sizes(ctx):
    x = corpus.make_class("text", 70_000, 9).numpy()
    for n, fs in ((0, 100), (1, 100), (31, 100), (100, 100), (101, 100), (32_768, 32_768), (32_769, 65_536), (65_537, 1 << 20)):
        cases.check_compress_roundtrip(ctx, x[:n], fs, 3, True)


def test_compress_high_entropy_literals(ctx):
    """Huffman streams longer than the encoder's shared-memory buffer (tiled packer); deep, length-limited trees"""
    rng = np.random.default_rng(5)
    for k, level in ((64, 1), (128, 3), (200, 1)):
        cases.check_compress_roundtrip(ctx, rng.integers(0, k, 70_000, dtype=np.uint8), 1 << 20, level, k % 3 == 0)
    p = 1.0 / np.arange(1, 257) ** 1.3; p /= p.sum()
    x = rng.choice(256, size=70_000, p=p).astype(np.uint8)
    cases.check_compress_roundtrip(ctx, x, 1 << 20, 1, True)
    cases.check_decode_matches_libzstd(ctx, x, 1 << 20, 3, True)


def test_golden_archives(ctx):
    cases.check_golden_archives(ctx)


def test_corruption_detected(ctx):
    cases.check_corruption_is_detected(ctx, trials=12)


def test_special_entries(ctx):
    cases.check_special_entries(ctx)


def test_patch_cycle(ctx):
    """lib.rs:289-300 patch_cycle (+ the two frame-size-policy variants of lib.rs:302-313)"""
    cases.check_patch_cycle(ctx)
    cases.check_patch_cycle(ctx, zk.FrameSizePolicy.Uncompressed(3000))
    cases.check_patch_cycle(ctx, zk.FrameSizePolicy.Compressed(700))


def test_prefix_batches(ctx):
    cases.check_prefix_batches(ctx)


def test_cycle_tiny_buffers(ctx):
    cases.check_cycle_tiny_buffers(ctx)
    cases.check_cycle_tiny_buffers(ctx, zk.FrameSizePolicy.Uncompressed(777))


def test_standalone_seek_table(ctx):
    cases.check_standalone_seek_table(ctx)


def test_encoder_decoder_io(ctx):
    assert cases.check_encoder_decoder_io(ctx) == 1
    assert cases.check_encoder_decoder_io(ctx, zk.FrameSizePolicy.Uncompressed(1000), chunk=333) == 13


@pytest.mark.parametrize("n", [1, 2, 17, 100, 1023])
def test_frame_size_policies_property(ctx, n):
    """lib.rs:315-357 proptests: frames as small as one byte, both policies"""
    cases.check_encoder_decoder_io(ctx, zk.FrameSizePolicy.Uncompressed(max(n, 40)), chunk=97)
    cases.check_encoder_decoder_io(ctx, zk.FrameSizePolicy.Compressed(n * 8), chunk=4096)


def test_one_byte_frames(ctx):
    data = cases.INPUT[:40]
    a = cases.new_seekable(ctx, zk.FrameSizePolicy.Uncompressed(1), data)
    dec = zk.Decoder(zk.DecodeOptions(a, ctx))
    assert dec.seek_table().num_frames() == 40 and dec.read_all() == data


def test_frame_counts_match_reference(ctx):
    cases.check_frame_counts_match_reference(ctx)


def test_raw_encoder_reset(ctx):
    cases.check_raw_encoder_reset(ctx)


def test_checksum_flag(ctx):
    cases.check_checksum_flag(ctx)


def test_encoder_bytes_are_pinned(ctx):
    cases.check_encoder_golden(ctx)


def test_high_level_tiers(ctx):
    """levels 7-9, 10-12 and >= 13 (8192-entry double table / 16384-entry table / 32768-entry table over a 256 KiB history, one warp per CTA):
    libzstd restores their frames, with and without a prefix, and each is denser than the tier below"""
    d = np.frombuffer(cases.golden_bytes("dickens_96k.txt"), dtype=np.uint8)
    sizes = [ctx.compress_frames(d, 1 << 20, lvl, False)[0].size for lvl in (4, 7, 10, 13)]
    assert sizes[0] > sizes[1] >= sizes[2] > sizes[3], sizes
    comp, cs, ds = ctx.compress_frames(d, 1 << 20, 13, True)
    assert comp[5] == 0x40 and cases.O.frame_stats(comp.tobytes())["zstd_frames"] == 1           # Window_Descriptor: 256 KiB
    _, ss = cases.O.oracle_decompress_ex(comp.tobytes(), d.size)
    assert ss["max_offset"] > 65_536                                                               # the wider window is used
    for lvl in (7, 10, 13, 19):
        for kind in ("text", "structured", "lowent", "random", "runs"):
            cases.check_compress_roundtrip(ctx, corpus.make_class(kind, 40_001 if lvl < 13 else 100_001, seed=lvl).numpy(), 33_000 if lvl < 13 else 100_001, lvl, lvl % 2 == 1)
    cases.check_prefix_batches(ctx, n=90_000, levels=(10, 13))


def test_window_limit(ctx):
    cases.check_window_limit(ctx)


def test_decoder_options(ctx):
    cases.check_decoder_options(ctx)


def test_decoder_state_machine(ctx):
    cases.check_decoder_state_machine(ctx)


def test_encoder_random_ops(ctx):
    assert cases.check_encoder_random_ops(ctx) > 20
    cases.check_encoder_random_ops(ctx, ops=30, seed=9, frame_size=333, prefix=True)


def test_decoder_random_ops(ctx):
    cases.check_decoder_random_ops(ctx)


def test_libzstd_archive_through_decoder(ctx):
    cases.check_libzstd_archive_through_decoder(ctx)



def test_range_reads_stop_early(ctx):
    cases.check_range_reads_stop_early(ctx, n=400_000, frame_size=200_000, reads=8)      # (the GPU suite runs the full-size version)


def test_cli_front_end(ctx, tmp_path):
    """cli/tests/integration/main.rs on emulator-sized inputs"""
    from zeekstd_b200 import corpus
    data = corpus.as_numpy(corpus.make_class("text", 6000, seed=5)).tobytes()
    with_p, without = cases.check_cli(ctx, tmp_path, data, ["123", "3K", "2M"])
    assert with_p < without * 0.7        # --patch-from: 3/4 of the new version is in the prefix


def test_zz_decoder_coverage_matrix(ctx):
    """runs last in this file: every cell of SURVEY.md 8a's matrix that fits emulator-sized inputs was decoded above"""
    cases.check_coverage_matrix([c for c in cases.MATRIX_CELLS if c not in ("frames_over_2MiB", "offsets_over_1MiB")])
