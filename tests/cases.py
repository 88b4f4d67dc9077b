"""Backend-independent test bodies.  Every function takes a zeekstd_b200.Context bound to the library under test
(the emulated CPU build for `-m "not gpu"`, the real sm_90a build for `-m gpu`) and checks it against the oracle
(libzstd through the reference's call sequence / the plain-C restatement).  The API tests are ports of the
reference's own tests (lib/src/lib.rs:69-357, encode.rs:802-871, decode.rs:581-940, seek_table.rs:1061-1278)."""
from __future__ import annotations

import io

import numpy as np

import zeekstd_b200 as zk
from oracle import oracle as O
from zeekstd_b200 import _native, corpus
from framegen import BackBits as _BackBits, lit_header as _lit_header, nseq_bytes as _nseq_bytes
from util import decode_frames, golden_bytes, golden_meta, offsets, split_frames

INPUT = golden_bytes("dickens_96k.txt")[:12_345]       # plays the role of lib.rs's INPUT (the reference uses its own source text)


# ------------------------------------------------------------------------------------------------ coverage bookkeeping
# Every archive a test feeds to the codec's DECODER is also walked by the restatement (oracle.frame_stats, and -- below
# COVER_SEQ_BYTES -- decoded by it for the sequence-level statistics); the totals are asserted cell by cell at the end of
# each suite (check_coverage_matrix): the decoder coverage matrix of SURVEY.md 8a is then proven to have been exercised
# on the build under test, not assumed.
COVERAGE: dict = {}
COVER_SEQ_BYTES = 48 << 20
MATRIX_CELLS = ("n_raw", "n_rle", "n_comp", "lit_raw", "lit_rle", "lit_huf", "lit_treeless", "lit_1stream", "lit_4stream", "huf_direct", "huf_fse",
                "mode_predef", "mode_rle", "mode_fse", "mode_repeat", "nseq0_blocks", "checksum_frames", "single_segment_frames",
                "skippable_frames", "multi_frame_entries", "rep1", "rep2", "rep3", "rep1_minus_1", "rep_ll0", "overlap", "dict_id_rejected",
                "frames_over_2MiB", "offsets_over_1MiB", "prefix_frames")


def cover(entries, d_total: int | None = None, prefix=None):
    """entries: list of the compressed bytes of seek-table entries that were decoded by the codec under test"""
    blob = b"".join(entries)
    for k, v in O.frame_stats(blob).items():
        COVERAGE[k] = COVERAGE.get(k, 0) + v
    for e in entries:
        fs = O.frame_stats(e)
        COVERAGE["multi_frame_entries"] = COVERAGE.get("multi_frame_entries", 0) + int(fs["zstd_frames"] > 1)
    if d_total is not None and d_total <= COVER_SEQ_BYTES:
        _, ss = O.oracle_decompress_ex(blob, d_total + 1, prefix=prefix)
        for k, v in ss.items():
            COVERAGE[k] = max(COVERAGE.get(k, 0), v) if k == "max_offset" else COVERAGE.get(k, 0) + v
        COVERAGE["offsets_over_1MiB"] = COVERAGE.get("offsets_over_1MiB", 0) + int(ss["max_offset"] > (1 << 20))


def check_coverage_matrix(cells=MATRIX_CELLS):
    missing = [c for c in cells if COVERAGE.get(c, 0) <= 0]
    assert not missing, f"decoder coverage matrix: cells never exercised in this run: {missing}; totals {COVERAGE}"
    return {c: COVERAGE[c] for c in cells}


# ------------------------------------------------------------------------------------------------ raw codec parity
def check_decode_matches_libzstd(ctx, data: np.ndarray, frame_size: int, level: int, checksum: bool):
    """libzstd-compressed frames must decode bit-exactly (== ZSTD_decompressStream output == the input)"""
    frames, cs, ds = O.ref_compress_frames(data, frame_size, level, checksum)
    out, st, rc = decode_frames(ctx, frames, ds, verify=True)
    assert rc == 0 and not st.any(), (rc, st[st != 0][:5])
    assert out == data.tobytes()
    cover(frames, data.size)
    if frame_size > (2 << 20) and data.size > (2 << 20):
        COVERAGE["frames_over_2MiB"] = COVERAGE.get("frames_over_2MiB", 0) + 1


def check_compress_roundtrip(ctx, data: np.ndarray, frame_size: int, level: int, checksum: bool):
    """our compressed frames must be spec-compliant: libzstd AND the restatement restore the input; so do we"""
    comp, cs, ds = ctx.compress_frames(data, frame_size, level, checksum)
    n_frames = max(1, -(-data.size // frame_size))
    assert len(cs) == n_frames and int(cs.sum()) == comp.size and int(ds.sum()) == data.size
    frames = split_frames(comp.tobytes(), cs)
    for i, fr in enumerate(frames):
        want = data[i * frame_size: i * frame_size + int(ds[i])].tobytes()
        assert O.ref_decompress_any(fr, len(want) + 1) == want            # real libzstd accepts it
        assert O.oracle_decompress(fr, len(want) + 1) == want
        assert ((fr[4] >> 2) & 1) == int(checksum)                          # Frame_Header_Descriptor checksum bit (encode.rs:861-869)
    out, st, rc = decode_frames(ctx, frames, ds, verify=True)
    assert rc == 0 and out == data.tobytes()
    return data.size / max(1, comp.size)


def check_golden_archives(ctx):
    meta = golden_meta()
    src = golden_bytes("dickens_96k.txt")
    for name, info in meta["archives"].items():
        a = golden_bytes(name + ".zst")
        dec = zk.Decoder(zk.DecodeOptions(a, ctx))
        assert dec.seek_table().num_frames() == info["num_frames"]
        assert dec.read_all() == src[: info["src_bytes"]], name
        st = O.OracleSeekTable.parse(a, "foot")
        cover([a[st.c[i]: st.c[i + 1]] for i in range(st.num_frames())], info["src_bytes"])


def check_corruption_is_detected(ctx, trials: int = 24):
    """flipping bits must never yield silently wrong data when the frame carries a checksum, and must never crash"""
    x = np.frombuffer(golden_bytes("dickens_96k.txt")[:40_000], dtype=np.uint8)
    frames, cs, ds = O.ref_compress_frames(x, 40_000, 3, True)
    good = frames[0]
    rng = np.random.default_rng(11)
    detected = 0
    for _ in range(trials):
        bad = bytearray(good)
        pos = int(rng.integers(0, len(bad)))
        bad[pos] ^= 1 << int(rng.integers(0, 8))
        out, st, rc = decode_frames(ctx, [bytes(bad)], ds, verify=True)
        if rc != 0:
            detected += 1
            assert zk.Error(rc, ctx.lib).is_zstd()
        else:
            assert out == x.tobytes()          # only harmless flips (e.g. in unused header bits) may pass
    assert detected >= trials * 0.8
    # truncated and garbage inputs
    for blob in (good[:-7], good[: len(good) // 2], b"\x00" * 64, good[:4]):
        out, st, rc = decode_frames(ctx, [blob], ds, verify=True)
        assert rc != 0
    check_crafted_frames_rejected(ctx)


def _frame(blocks) -> bytes:
    """magic, FHD 0 (no FCS, no checksum), window descriptor 0x50 (1 MiB), then (type, content[, regen]) blocks"""
    out = bytearray(b"\x28\xb5\x2f\xfd\x00\x50")
    for i, blk in enumerate(blocks):
        btype, content = blk[0], blk[1]
        size = blk[2] if btype == 1 else len(content)
        out += ((size << 3) | (btype << 1) | int(i == len(blocks) - 1)).to_bytes(3, "little") + content
    return bytes(out)


def crafted_overflow_frame() -> bytes:
    """ADVICE r1 (high): 40 000 sequences whose literal lengths sum to exactly 2^32 -- the wrapped totals look valid, every
    intermediate sum is far out of range.  Literals: Raw, 0 bytes; all three tables RLE (LL code 35 = 65536 + 16 bits,
    OF code 1 = repeat offsets, ML code 0 = 3)."""
    nseq = 40_000
    lls = [107_374] * (nseq - 1)
    lls.append((1 << 32) - sum(lls))
    assert 65_536 <= lls[-1] <= 131_071
    bw = _BackBits()
    for ll in reversed(lls):                      # the decoder reads OF, ML, LL extra bits of the FIRST sequence first
        bw.put(ll - 65_536, 16); bw.put(0, 1)
    body = bytes([0x00]) + bytes([0xFF, (nseq - 0x7F00) & 0xFF, (nseq - 0x7F00) >> 8]) + bytes([0x54, 35, 1, 0]) + bw.finish()
    assert len(body) <= 128 << 10
    return _frame([(2, body)])


def crafted_frames():
    """-> list of (name, frame bytes, decompressed-size claim) that libzstd rejects as corrupted"""
    treeless_first = _frame([(2, bytes([0x43, 0x40, 0x00, 0x01, 0x00]))])          # Treeless literals in the first block (ADVICE r1, high)
    # Repeat_Mode sequence tables in the first block with sequences: raw literals (4 bytes), nseq 1, modes LL=repeat
    repeat_first = _frame([(2, bytes([0x20]) + b"abcd" + bytes([0x01, 0xC0]) + bytes([0x01, 0x01]))])
    # a valid raw block, THEN a treeless block: the count pass must also see the missing tree in later blocks
    treeless_later = _frame([(0, b"hello world"), (2, bytes([0x43, 0x40, 0x00, 0x01, 0x00]))])
    # Window_Descriptor 0xAA = 2^31 * 1.25: a valid header field, but above what a default DCtx accepts when streaming
    # (ZSTD_WINDOWLOG_LIMIT_DEFAULT = 27): frameParameter_windowTooLarge (found by tests/emul/fuzz_decode.py)
    big_window = b"\x28\xb5\x2f\xfd\x00\xaa" + (len(b"hello") << 3 | 1).to_bytes(3, "little") + b"hello"
    return [("overflow", crafted_overflow_frame(), 120_000), ("treeless_first", treeless_first, 4), ("repeat_first", repeat_first, 8),
            ("treeless_later", treeless_later, 15), ("big_window", big_window, 5)]


# --- hand-built VALID frames for the cells of the matrix libzstd's encoder does not reach on demand ------------------
_LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
_ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]


def _rle_seq_block(lit_section: bytes, codes, seqs, repeat_tables: bool = False) -> bytes:
    """a Compressed block whose three sequence tables are RLE (one code each; the values vary through the extra bits only),
    or Repeat_Mode of the previous block's tables.  codes = (ll_code, of_code, ml_code); seqs = [(ll_x, of_x, ml_x)] extra bits"""
    llc, ofc, mlc = codes
    bw = _BackBits()
    for llx, ofx, mlx in reversed(seqs):          # the decoder reads OF, ML, LL of the first sequence first
        bw.put(llx, _LL_BITS[llc]); bw.put(mlx, _ML_BITS[mlc]); bw.put(ofx, ofc)
    tables = bytes([0xFC]) if repeat_tables else bytes([0x54, llc, ofc, mlc])
    return lit_section + _nseq_bytes(len(seqs)) + tables + bw.finish()


def crafted_valid_frame(seed: int = 1):
    """One zstd frame, five blocks: Raw history; RLE literals + RLE-mode tables (explicit offsets); Raw literals with
    litLen == 0 repeat codes (rep2/rep3 shifted and the rep1-1 case); the same tables again through Repeat_Mode; an RLE block.
    -> frame bytes (libzstd is the judge of what it decodes to)"""
    rng = np.random.default_rng(seed)
    hist = rng.integers(0, 256, 3000, dtype=np.uint8).tobytes()
    # B: 40 sequences, litLen 16/17 of 'Q' (RLE literals), offset code 9 (509..1020), matchLen 35/36
    seqs_b = [(int(rng.integers(2)), int(rng.integers(512)), int(rng.integers(2))) for _ in range(40)]
    n_lit_b = sum(16 + s[0] for s in seqs_b) + 5                      # five trailing literals
    blk_b = _rle_seq_block(_lit_header(1, n_lit_b) + b"Q", (16, 9, 32), seqs_b)
    # C: litLen 0 (code 0), offset code 1 -> Offset_Value 2/3 -> with litLen == 0: rep3 / rep1-1; matchLen 8 (code 5)
    seqs_c = [(0, int(rng.integers(2)), 0) for _ in range(30)]
    blk_c = _rle_seq_block(_lit_header(0, 3) + b"xyz", (0, 1, 5), seqs_c)
    # D: Repeat_Mode for all three tables (the RLE tables of C), offset values 2/3 again, raw literals
    seqs_d = [(0, int(rng.integers(2)), 0) for _ in range(20)]
    blk_d = _rle_seq_block(_lit_header(0, 0), (0, 1, 5), seqs_d, repeat_tables=True)
    return _frame([(0, hist), (2, blk_b), (2, blk_c), (2, blk_d), (1, b"\x7f", 777)])


def check_special_entries(ctx):
    """cells of SURVEY.md 8a's matrix that need particular producers: hand-built RLE literals / RLE + Repeat tables /
    rep1-1; ZSTD_compress() one-shot frames (Single_Segment, every Frame_Content_Size width); skippable frames before,
    between and after zstd frames of one seek-table entry; several zstd frames per entry; RLE blocks; direct Huffman
    weights; a non-zero Dictionary_ID (rejected with dictionary_wrong, like libzstd without a dictionary)"""
    rng = np.random.default_rng(5)
    text = np.frombuffer(golden_bytes("dickens_96k.txt"), dtype=np.uint8)
    entries, wants = [], []

    def add(entry: bytes):
        want = O.ref_decompress_any(entry, 4 << 20)                    # libzstd is the reference for what an entry decodes to
        assert O.oracle_decompress(entry, 4 << 20) == want
        entries.append(entry); wants.append(want)

    add(crafted_valid_frame(1)); add(crafted_valid_frame(2))
    for n in (0, 1, 255, 256, 300, 65_791, 65_792, 90_000):            # FCS field widths 1 / 2 (+256) / 4 bytes
        add(O.ref_compress_simple(text[:n], 3))
    one = O.ref_compress_simple(text[:5000], 1); two = O.ref_compress_frames(text[5000:40_000], 20_000, 3, True)[0]
    add(O.skippable_frame(b"meta", 3) + one + O.skippable_frame(b"") + two[0] + two[1] + O.skippable_frame(b"x" * 100, 15))
    add(O.skippable_frame(b"only skippable"))                          # an entry that decodes to nothing
    add(O.ref_compress_frames(np.zeros(400_000, dtype=np.uint8), 400_000, 3, True)[0][0])            # RLE blocks
    p = np.array([.4, .25, .15, .08, .05, .04, .02, .01])
    add(O.ref_compress_frames(rng.choice(8, size=150_000, p=p).astype(np.uint8), 150_000, 1, False)[0][0])   # direct weights + treeless
    ds = [len(w) for w in wants]
    out, st, rc = decode_frames(ctx, entries, ds, verify=True)
    assert rc == 0 and not st.any(), (rc, list(st))
    assert out == b"".join(wants)
    cover(entries, sum(ds))
    # Dictionary_ID: flag 1 (one byte), ID 7, spliced into a valid frame header -> dictionary_wrong (32) in both decoders
    good = O.ref_compress_frames(text[:3000], 3000, 3, False)[0][0]
    assert good[4] & 3 == 0
    bad = good[:4] + bytes([good[4] | 1, good[5], 7]) + good[6:]
    for fn in (O.ref_decompress_any, O.oracle_decompress):
        try:
            fn(bad, 1 << 20); raise AssertionError("a frame with a Dictionary_ID was accepted")
        except O.ZstdError as e:
            assert e.code == 32
    out, st, rc = decode_frames(ctx, [good, bad], [3000, 3000], verify=True)
    assert rc == -32 and list(st) == [0, -32] and out[:3000] == text[:3000].tobytes()
    bad0 = good[:4] + bytes([good[4] | 1, good[5], 0]) + good[6:]     # Dictionary_ID field present but zero: no dictionary needed
    assert O.ref_decompress_any(bad0, 1 << 20) == text[:3000].tobytes()
    out, st, rc = decode_frames(ctx, [bad0], [3000], verify=True)
    assert rc == 0 and out == text[:3000].tobytes()
    COVERAGE["dict_id_rejected"] = COVERAGE.get("dict_id_rejected", 0) + 1


def check_window_limit(ctx):
    """Window_Descriptor 0x88 (2^27, the streaming default limit) is accepted, 0x89 (2^27 * 1.125) is not -- as libzstd"""
    body = (len(b"hello") << 3 | 1).to_bytes(3, "little") + b"hello"
    for wd, code in ((0x88, 0), (0x89, 16), (0xF8, 16)):
        fr = b"\x28\xb5\x2f\xfd\x00" + bytes([wd]) + body
        out, sizes = O.ref_decompress_frames(np.frombuffer(fr, dtype=np.uint8), [0, len(fr)], [0, 5])
        assert sizes[0] == (5 if code == 0 else -code), (hex(wd), sizes)
        got, st, rc = decode_frames(ctx, [fr], [5], verify=True)
        assert rc == -code and (code or got[:5] == b"hello"), (hex(wd), rc)
    # Block_Maximum_Size = min(Window_Size, 128 KiB): a 1 KiB window (descriptor 0x00) takes a 1024-byte block, not a 1025-byte one,
    # whether the block is Raw, RLE (regenerated size) or Compressed (RLE literals, no sequences) -- corruption_detected as libzstd
    for nbytes, code in ((1024, 0), (1025, 20)):
        payload = bytes(range(256)) * 5
        for kind, blk in (("raw", ((nbytes << 3) | 1).to_bytes(3, "little") + payload[:nbytes]),
                          ("rle", ((nbytes << 3) | (1 << 1) | 1).to_bytes(3, "little") + b"z"),
                          ("lit", ((4 << 3) | (2 << 1) | 1).to_bytes(3, "little") + ((nbytes << 4) | (1 << 2) | 1).to_bytes(2, "little") + b"z\x00")):
            fr = b"\x28\xb5\x2f\xfd\x00\x00" + blk
            out, sizes = O.ref_decompress_frames(np.frombuffer(fr, dtype=np.uint8), [0, len(fr)], [0, nbytes])
            assert sizes[0] == (nbytes if code == 0 else -code), (kind, nbytes, sizes)
            try:
                assert len(O.oracle_decompress(fr, nbytes)) == nbytes and code == 0
            except O.ZstdError as e:
                assert e.code == code, (kind, nbytes, e.code)
            got, st, rc = decode_frames(ctx, [fr], [nbytes], verify=True)
            assert rc == -code, (kind, nbytes, rc)
            if code == 0:
                assert got[:nbytes] == (payload[:nbytes] if kind == "raw" else b"z" * nbytes)


def check_crafted_frames_rejected(ctx):
    """hand-built invalid frames: libzstd and the restatement say corruption; the codec must say so too, must not touch memory
    outside its buffers (tests/emul/asan_check.py runs this under ASan), and must still decode a good frame in the SAME batch"""
    x = np.frombuffer(golden_bytes("dickens_96k.txt")[:20_000], dtype=np.uint8)
    good, gcs, gds = O.ref_compress_frames(x, 20_000, 3, True)
    for name, fr, claim in crafted_frames():
        for fn in (O.ref_decompress_any, O.oracle_decompress):
            try:
                fn(fr, 1 << 20)
                raise AssertionError(f"{name}: the oracle accepted a crafted frame")
            except O.ZstdError as e:
                code = e.code
                assert code == (30 if name.startswith("treeless") else 16 if name == "big_window" else 20), (name, code)   # 30: dictionary_corrupted for a missing tree
        out, st, rc = decode_frames(ctx, [good[0], fr, good[0]], [gds[0], claim, gds[0]], verify=True)
        assert rc == -code and list(st) == [0, -code, 0], (name, rc, list(st))
        assert out[:20_000] == x.tobytes() and out[20_000 + claim:] == x.tobytes()


# ------------------------------------------------------------------------------------------------ API: encode side
def new_seekable(ctx, policy=None, data: bytes = INPUT, out_buf_len=None) -> bytes:
    """decode.rs:587-629: RawEncoder driven with a caller buffer, then the seek table appended"""
    enc = zk.EncodeOptions(ctx).frame_size_policy(policy or zk.FrameSizePolicy.default()).into_raw_encoder()
    buf = bytearray(out_buf_len or max(len(data), 64))
    seekable = bytearray()
    in_progress = out_progress = 0
    while in_progress < len(data):
        p = enc.compress(data[in_progress:], buf)
        seekable += buf[: p.out_progress]
        in_progress += p.in_progress
        out_progress += p.out_progress
    assert in_progress == len(data)
    while True:
        p = enc.end_frame(buf)
        seekable += buf[: p.out_progress]
        out_progress += p.out_progress
        if p.data_left == 0:
            break
    assert out_progress == len(seekable)
    ser = enc.into_seek_table().into_serializer()
    while True:
        n = ser.write_into(buf)
        if n == 0:
            break
        seekable += buf[:n]
    assert out_progress + ser.encoded_len() == len(seekable)
    return bytes(seekable)


def check_cycle_tiny_buffers(ctx, policy=None):
    """lib.rs:82-134 test_cycle: every stage in many small steps (buffer = len/500), then full decompression"""
    data = INPUT
    a = new_seekable(ctx, policy, data, out_buf_len=max(1, len(data) // 500))
    # libzstd decodes the frames of our archive
    st = O.OracleSeekTable.parse(a, "foot")
    assert O.ref_decompress_any(a[: st.c[-1]], len(data) + 1) == data
    dec = zk.Decoder(zk.DecodeOptions(a, ctx))
    out = bytearray()
    buf = bytearray(max(1, len(data) // 500))
    while True:
        n = dec.decompress(buf)
        if n == 0:
            break
        out += buf[:n]
    assert bytes(out) == data


def check_standalone_seek_table(ctx):
    """lib.rs:136-200: seek table kept apart from the frames, Head and Foot"""
    for fmt in (zk.Format.Head, zk.Format.Foot):
        enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Uncompressed(1000)).into_raw_encoder()
        frames = bytearray()
        buf = bytearray(4096)
        pos = 0
        while pos < len(INPUT):
            p = enc.compress(INPUT[pos:], buf)
            frames += buf[: p.out_progress]; pos += p.in_progress
        while True:
            p = enc.end_frame(buf)
            frames += buf[: p.out_progress]
            if p.data_left == 0:
                break
        table = enc.into_seek_table().into_format_serializer(fmt).to_bytes()
        st = zk.SeekTable.from_bytes(table, fmt, ctx.lib)
        assert st.size_comp() == len(frames) and st.size_decomp() == len(INPUT)
        dec = zk.DecodeOptions(bytes(frames), ctx).seek_table(st).into_decoder()
        assert dec.read_all() == INPUT


def check_encoder_decoder_io(ctx, policy=None, chunk: int = 1000):
    """lib.rs:266-287: std Encoder / Decoder through io copy; finish() returns the bytes written"""
    sink = io.BytesIO()
    opts = zk.EncodeOptions(ctx)
    if policy:
        opts.frame_size_policy(policy)
    enc = opts.into_encoder(sink)
    for i in range(0, len(INPUT), chunk):
        assert enc.compress(INPUT[i:i + chunk]) == len(INPUT[i:i + chunk])
    n = enc.finish()
    a = sink.getvalue()
    assert n == len(a)
    st = O.OracleSeekTable.parse(a, "foot")
    assert st.d[-1] == len(INPUT) and st.c[-1] + 17 + 8 * st.num_frames() == len(a)
    assert O.ref_decompress_any(a[: st.c[-1]], len(INPUT) + 1) == INPUT
    dec = zk.Decoder(zk.DecodeOptions(io.BytesIO(a), ctx))       # generic Read + Seek source
    out = io.BytesIO()
    while True:
        b = bytearray(777)
        k = dec.readinto(b)
        if not k:
            break
        out.write(b[:k])
    assert out.getvalue() == INPUT
    return st.num_frames()


def check_frame_counts_match_reference(ctx):
    """frame boundaries are a host-side contract: same (d_size) sequence as the reference for the same policy"""
    for fs in (1000, len(INPUT), len(INPUT) // 3, 4096):
        sink = io.BytesIO()
        enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Uncompressed(fs)).into_encoder(sink)
        enc.write(INPUT)
        enc.finish()
        ours = O.OracleSeekTable.parse(sink.getvalue(), "foot")
        _, ref = O.ref_seekable_archive(np.frombuffer(INPUT, dtype=np.uint8), fs, 1, False)
        assert ours.d == ref.d, fs
    # empty stream: one empty frame, like Encoder::finish() on no input
    sink = io.BytesIO()
    enc = zk.Encoder(sink, zk.EncodeOptions(ctx))
    enc.finish()
    ours = O.OracleSeekTable.parse(sink.getvalue(), "foot")
    _, ref = O.ref_seekable_archive(np.zeros(0, dtype=np.uint8), 0x200000, 1, False)
    assert ours.d == ref.d == [0, 0] and ours.num_frames() == 1
    assert O.ref_decompress_any(sink.getvalue()[: ours.c[-1]], 1) == b""


def check_raw_encoder_reset(ctx):
    """encode.rs:810-846: reset_frame + reset_seek_table reproduce an identical seek table"""
    enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Uncompressed(2000)).into_raw_encoder()
    buf = bytearray(len(INPUT) + 1024)

    def run():
        pos = 0
        while pos < len(INPUT):
            p = enc.compress(INPUT[pos:], buf); pos += p.in_progress
        while enc.end_frame(buf).data_left:
            pass
        return enc.seek_table().clone()

    enc.compress(INPUT[:500], buf)
    enc.reset_frame()
    a = run()
    enc.reset_seek_table()
    assert enc.seek_table().num_frames() == 0
    b = run()
    assert a == b and a.num_frames() == -(-len(INPUT) // 2000)


def check_checksum_flag(ctx):
    """encode.rs:848-870: with checksum_flag(true) every frame's descriptor has bit 2 set"""
    for flag in (True, False):
        sink = io.BytesIO()
        enc = zk.EncodeOptions(ctx).checksum_flag(flag).frame_size_policy(zk.FrameSizePolicy.Uncompressed(3000)).into_encoder(sink)
        enc.write(INPUT); enc.finish()
        a = sink.getvalue()
        st = zk.SeekTable.from_bytes(a, zk.Format.Foot, ctx.lib)
        for i in range(st.num_frames()):
            assert ((a[st.frame_start_comp(i) + 4] >> 2) & 1) == int(flag)


def check_patch_cycle(ctx, policy=None):
    """lib.rs:202-263 test_patch_cycle: a "binary patch" -- the new version compressed with the old one as raw-content prefix of
    every frame, every stage in many small steps, decoded with the same prefix.  Plus what the reference cannot check: libzstd
    (ZSTD_DCtx_refPrefix) restores our patch, and a patch written by libzstd (ZSTD_CCtx_refPrefix) decodes on our side."""
    old = INPUT
    new = INPUT + b"\nThe End"
    opts = zk.EncodeOptions(ctx)
    if policy:
        opts.frame_size_policy(policy)
    enc = opts.into_raw_encoder()
    buf = bytearray(max(1, len(INPUT) // 500))
    patch = bytearray()
    pos = 0
    while pos < len(new):
        p = enc.compress_with_prefix(new[pos:], buf, old)
        patch += buf[: p.out_progress]; pos += p.in_progress
    while True:
        p = enc.end_frame(buf)
        patch += buf[: p.out_progress]
        if p.data_left == 0:
            break
    ser = enc.into_seek_table().into_serializer()
    while True:
        n = ser.write_into(buf)
        if n == 0:
            break
        patch += buf[:n]
    patch = bytes(patch)
    st = O.OracleSeekTable.parse(patch, "foot")
    if policy is None:
        assert len(patch) < len(new) // 20, len(patch)          # the point of a patch: almost everything comes from the prefix
    # libzstd with the prefix restores it; without the prefix it cannot
    out, sizes = O.ref_decompress_frames(patch[: st.c[-1]], st.c, st.d, prefix=old)
    assert out.tobytes() == new
    if policy is None:
        _, sizes = O.ref_decompress_frames(patch[: st.c[-1]], st.c, st.d)
        assert any(s < 0 for s in sizes)
    dec = zk.Decoder(zk.DecodeOptions(patch, ctx))
    got = bytearray()
    while True:
        n = dec.decompress_with_prefix(buf, old)
        if n == 0:
            break
        got += buf[:n]
    assert bytes(got) == new
    # the other direction: the reference path writes the patch
    for fs in (len(new), 4000):
        frames, cs, ds = O.ref_compress_frames(np.frombuffer(new, dtype=np.uint8), fs, 3, True, prefix=old)
        out, stt, rc = ctx.decompress_frames(np.frombuffer(b"".join(frames) + b"\0" * 64, dtype=np.uint8), offsets(cs), offsets(ds), True, prefix=old)
        assert rc == 0 and out.tobytes() == new
        cover(frames, len(new), prefix=old)
        COVERAGE["prefix_frames"] = COVERAGE.get("prefix_frames", 0) + len(frames)


def check_prefix_batches(ctx, n: int = 300_000, frame_size: int = 50_000, levels=(3,)):
    """prefix mode of the batch codec on more than one frame and more than one block per frame: text whose vocabulary lives
    in the prefix; both implementations, both directions, several prefix lengths (shorter and longer than the encoder's window)"""
    text = np.frombuffer(golden_bytes("dickens_96k.txt"), dtype=np.uint8)
    data = np.concatenate([text[10_000:60_000]] * (n // 50_000 + 1))[:n].copy()
    data[::977] ^= 1                                                   # not an exact copy of the prefix
    for plen, level in [(p, l) for l in levels for p in (1, 1000, 40_000, 98_304)]:
        prefix = text[:plen]
        comp, cs, ds = ctx.compress_frames(data, frame_size, level, True, prefix=prefix)
        out, sizes = O.ref_decompress_frames(comp, offsets(cs), offsets(ds), prefix=prefix)          # libzstd restores ours
        assert sizes == [int(d) for d in ds] and out.tobytes() == data.tobytes(), plen
        back, st, rc = ctx.decompress_frames(np.concatenate([comp, np.zeros(64, np.uint8)]), offsets(cs), offsets(ds), True, prefix=prefix)
        assert rc == 0 and back.tobytes() == data.tobytes()
        if plen >= 40_000:
            plain = ctx.compress_frames(data, frame_size, level, True)[0]
            assert comp.size < plain.size, (plen, comp.size, plain.size)        # the prefix was found
        frames, rcs, rds = O.ref_compress_frames(data, frame_size, 3, True, prefix=prefix)             # ours restores libzstd's
        back, st, rc = ctx.decompress_frames(np.frombuffer(b"".join(frames) + b"\0" * 64, dtype=np.uint8), offsets(rcs), offsets(rds), True, prefix=prefix)
        assert rc == 0 and back.tobytes() == data.tobytes(), plen
        _, ss = O.oracle_decompress_ex(b"".join(frames), n + 1, prefix=prefix)
        if plen >= 1000:
            assert ss["prefix_matches"] > 0
        COVERAGE["prefix_frames"] = COVERAGE.get("prefix_frames", 0) + len(frames)
    # a wrong prefix must not decode silently (checksum on)
    back, st, rc = ctx.decompress_frames(np.frombuffer(b"".join(frames) + b"\0" * 64, dtype=np.uint8), offsets(rcs), offsets(rds), True, prefix=text[:plen - 5])
    assert rc != 0


# ------------------------------------------------------------------------------------------------ API: decode side
def check_decoder_options(ctx):
    """decode.rs:631-661"""
    a = new_seekable(ctx)
    st = zk.SeekTable.from_bytes(a, zk.Format.Foot, ctx.lib)
    oks = [zk.DecodeOptions(a, ctx), zk.DecodeOptions(a, ctx).lower_frame(st.num_frames() - 1), zk.DecodeOptions(a, ctx).upper_frame(st.num_frames() - 1),
           zk.DecodeOptions(a, ctx).offset(st.size_decomp()), zk.DecodeOptions(a, ctx).offset_limit(st.size_decomp()),
           zk.DecodeOptions(bytes([0, 128]), ctx).seek_table(st.clone())]
    errs = [zk.DecodeOptions(bytes([0, 128]), ctx), zk.DecodeOptions(a, ctx).lower_frame(st.num_frames()), zk.DecodeOptions(a, ctx).upper_frame(st.num_frames()),
            zk.DecodeOptions(a, ctx).offset(st.size_decomp() + 1), zk.DecodeOptions(a, ctx).offset_limit(st.size_decomp() + 1)]
    for o in oks:
        o.into_decoder()
    for o in errs:
        try:
            o.into_decoder()
            raise AssertionError("expected an error")
        except zk.Error:
            pass


def check_decoder_state_machine(ctx):
    """decode.rs:663-939, one body per reference test"""
    n_in = len(INPUT)
    out = bytearray(n_in)
    # decompress_and_reset (:663-682)
    a = new_seekable(ctx)
    dec = zk.Decoder(zk.DecodeOptions(a, ctx))
    assert dec.decompress(out) == n_in and bytes(out) == INPUT
    assert dec.decompress(out) == 0
    dec.reset()
    assert dec.decompress(out) == n_in and bytes(out) == INPUT
    # decompress_until_upper_frame (:684-699)
    fs = n_in // 7
    dec = zk.Decoder(zk.DecodeOptions(new_seekable(ctx, zk.FrameSizePolicy.Uncompressed(fs)), ctx))
    dec.set_lower_frame(0); dec.set_upper_frame(5)
    buf = bytearray(fs * 6)
    assert dec.decompress(buf) == fs * 6 and bytes(buf) == INPUT[: fs * 6]
    # decompress_last_frames (:701-716)
    fs = n_in // 9
    dec = zk.Decoder(zk.DecodeOptions(new_seekable(ctx, zk.FrameSizePolicy.Uncompressed(fs)), ctx))
    dec.set_lower_frame(5); dec.set_upper_frame(9)
    ln = n_in - fs * 5
    buf = bytearray(ln)
    assert dec.decompress(buf) == ln and bytes(buf) == INPUT[n_in - ln:]
    # upper_frame_greater_than_lower_frame (:718-730)
    fs = n_in // 13
    dec = zk.Decoder(zk.DecodeOptions(new_seekable(ctx, zk.FrameSizePolicy.Uncompressed(fs)), ctx))
    dec.set_lower_frame(9); dec.set_upper_frame(8)
    assert dec.decompress(out) == 0
    # reset_decompression (:732-745)
    dec = zk.Decoder(zk.DecodeOptions(a, ctx))
    dec.decompress(bytearray(128)); dec.reset()
    assert dec.decompress(out) == n_in and bytes(out) == INPUT
    # decompress_everything_after_partly_decompression (:747-771)
    fs = n_in // 32
    dec = zk.Decoder(zk.DecodeOptions(new_seekable(ctx, zk.FrameSizePolicy.Uncompressed(fs)), ctx))
    dec.set_lower_frame(23); dec.set_upper_frame(29)
    n = dec.decompress(out)
    assert n == fs * 30 - fs * 23 and bytes(out[:n]) == INPUT[fs * 23: fs * 30]
    dec.set_lower_frame(0); dec.set_upper_frame(dec.seek_table().num_frames() - 1)
    assert dec.decompress(out) == n_in and bytes(out) == INPUT
    # set_frame_boundaries (:773-795)
    dec = zk.Decoder(zk.DecodeOptions(a, ctx))
    nf = dec.seek_table().num_frames()
    dec.set_lower_frame(nf - 1); dec.set_upper_frame(nf - 1)
    for fn in (dec.set_lower_frame, dec.set_upper_frame):
        try:
            fn(nf); raise AssertionError
        except zk.Error as e:
            assert e.is_frame_index_too_large()
    # set_offset_boundaries (:797-819)
    dec = zk.Decoder(zk.DecodeOptions(a, ctx))
    size = dec.seek_table().size_decomp()
    dec.set_offset(size); dec.set_offset_limit(size)
    for fn in (dec.set_offset, dec.set_offset_limit):
        try:
            fn(size + 1); raise AssertionError
        except zk.Error as e:
            assert e.is_offset_out_of_range()
    # decompress_within_offset_boundaries (:821-851)
    fs = n_in // 34
    dec = zk.Decoder(zk.DecodeOptions(new_seekable(ctx, zk.FrameSizePolicy.Uncompressed(fs)), ctx))
    off = n_in // 3; lim = 2 * off
    dec.set_offset(off); dec.set_offset_limit(lim)
    n = dec.decompress(out)
    assert n == lim - off and bytes(out[:n]) == INPUT[off:lim]
    assert dec.offset() == lim
    dec.set_offset(off)                                   # limit persists across set_offset
    assert dec.decompress(out) == lim - off
    dec.reset()
    assert dec.offset() == 0 and dec.offset_limit() == size and dec.read_compressed() == 0
    assert dec.decompress(out) == n_in and bytes(out) == INPUT
    # seek (:853-908)
    fs = n_in // 19
    dec = zk.Decoder(zk.DecodeOptions(new_seekable(ctx, zk.FrameSizePolicy.Uncompressed(fs)), ctx))
    seek_pos = n_in // 4; end = n_in
    assert dec.seek(seek_pos, 0) == seek_pos and dec.offset() == seek_pos
    n = dec.decompress(out)
    assert dec.read_compressed() != 0 and n == end - seek_pos and bytes(out[:n]) == INPUT[seek_pos:end]
    assert dec.offset() == end
    back = -(2 * fs)
    start = n_in + back
    assert dec.read_compressed() != 0
    dec.seek(back, 2)
    assert dec.offset() == start and dec.read_compressed() == 0
    n = dec.decompress(out)
    assert n == end - start and bytes(out[:n]) == INPUT[start:end]
    dec.seek(-(n_in // 2), 1)                               # SeekFrom::Current
    assert dec.offset() == n_in - n_in // 2
    try:
        dec.seek(1, 2); raise AssertionError                # positive SeekFrom::End is an error (:561-563)
    except zk.Error as e:
        assert e.is_offset_out_of_range()
    # reset_dctx_on_frame_change (:910-939)
    dec = zk.Decoder(zk.DecodeOptions(new_seekable(ctx, zk.FrameSizePolicy.Uncompressed(100)), ctx))
    assert dec.read_compressed() == 0
    dec.set_offset(10)
    assert dec.readinto(bytearray(10)) == 10
    assert dec.read_compressed() != 0
    dec.set_offset(30)                                      # same frame, forward: no reset
    assert dec.offset() == 30 and dec.read_compressed() != 0
    n = dec.decompress(out)
    assert n == n_in - 30 and bytes(out[:n]) == INPUT[30:]
    dec.set_offset(101)                                     # other frame: reset
    assert dec.offset() == 101 and dec.read_compressed() == 0
    n = dec.decompress(out)
    assert n == n_in - 101 and bytes(out[:n]) == INPUT[101:]


def check_libzstd_archive_through_decoder(ctx):
    """cross-implementation parity the reference lacks (SURVEY.md section 4): archives written by the reference path
    (libzstd) are read back bit-exactly through our Decoder, whole and ranged"""
    data = np.frombuffer(golden_bytes("dickens_96k.txt"), dtype=np.uint8)
    a, st = O.ref_seekable_archive(data, 10_000, 3, True)
    dec = zk.Decoder(zk.DecodeOptions(a, ctx))
    assert dec.read_all() == data.tobytes()
    rng = np.random.default_rng(3)
    for _ in range(12):
        lo = int(rng.integers(0, data.size)); hi = int(rng.integers(lo, min(data.size, lo + 30_000) + 1))
        dec.set_offset(lo); dec.set_offset_limit(hi)
        assert dec.read_all() == data[lo:hi].tobytes()
        dec.set_offset_limit(data.size)


def check_range_reads_stop_early(ctx, n: int = 600_000, frame_size: int = 300_000, reads: int = 24):
    """SURVEY.md 8f.1: a range read decodes its last frame only as far as offset_limit (block granularity).  Multi-block
    frames (libzstd: 128 KiB blocks; ours: 32 KiB), checksum on: the prefix must be exact, growing the limit afterwards
    must still give the right bytes, and zk_decompress_frames_upto must leave at least the wanted prefix of every entry"""
    data = np.concatenate([corpus.make_class("text", n // 2, 11).numpy(), corpus.make_class("structured", n - n // 2, 12).numpy()])
    rng = np.random.default_rng(17)
    for archive in (O.ref_seekable_archive(data, frame_size, 1, True)[0], None):
        if archive is None:
            sink = io.BytesIO()
            enc = zk.EncodeOptions(ctx).checksum_flag(True).frame_size_policy(zk.FrameSizePolicy.Uncompressed(frame_size)).into_encoder(sink)
            enc.write(data.tobytes()); enc.finish(); archive = sink.getvalue()
        dec = zk.Decoder(zk.DecodeOptions(archive, ctx))
        for _ in range(reads):
            lo = int(rng.integers(0, data.size - 1)); hi = int(rng.integers(lo + 1, min(data.size, lo + 70_000) + 1))
            dec.set_offset(lo); dec.set_offset_limit(hi)
            assert dec.read_all() == data[lo:hi].tobytes()
            if rng.integers(2):                                  # continue past the old limit inside the same frame
                hi2 = min(data.size, hi + int(rng.integers(1, 200_000)))
                dec.set_offset_limit(hi2)
                assert dec.read_all() == data[hi:hi2].tobytes()
            dec.set_offset_limit(data.size)
    # the batch entry point directly
    frames, cs, ds = O.ref_compress_frames(data, frame_size, 1, True)
    comp = np.frombuffer(b"".join(frames) + b"\0" * 64, dtype=np.uint8)
    co = np.zeros(len(cs) + 1, dtype=np.uint64); co[1:] = np.cumsum(cs)
    do = np.zeros(len(ds) + 1, dtype=np.uint64); do[1:] = np.cumsum(ds)
    need = np.array([int(rng.integers(0, d + 1)) for d in ds], dtype=np.uint32)
    out = np.zeros(int(do[-1]) + 64, dtype=np.uint8); st = np.zeros(len(cs), dtype=np.int32)
    rc = ctx.lib.zk_decompress_frames_upto(ctx._h, comp.ctypes.data, co.ctypes.data_as(_native.u64p), do.ctypes.data_as(_native.u64p), len(cs),
                                           out.ctypes.data, need.ctypes.data_as(_native.u32p), 1, st.ctypes.data_as(_native.i32p))
    assert rc == 0 and not st.any()
    for i, d in enumerate(ds):
        a0 = int(do[i]); assert out[a0:a0 + int(need[i])].tobytes() == data[a0:a0 + int(need[i])].tobytes()


# ------------------------------------------------------------------------------------------------ seek table (host only)
def check_seek_table(lib):
    """seek_table.rs:1084-1277 + the known-answer vectors of SURVEY.md 8c, cross-checked against the oracle restatement"""
    from zeekstd_b200 import _native
    _native.set_default_lib(lib)
    st = zk.SeekTable(lib=lib)
    assert st.into_serializer().to_bytes().hex() == "5e2a4d1809000000" + "00000000" + "00" + "b1ea928f"
    st.log_frame(123, 456)
    assert st.into_format_serializer(zk.Format.Foot).to_bytes().hex() == "5e2a4d18110000007b000000c80100000100000000b1ea928f"
    assert st.into_format_serializer(zk.Format.Head).to_bytes().hex() == "5e2a4d18110000000100000000b1ea928f7b000000c8010000"
    st.log_frame(333, 444)
    assert st.into_serializer().to_bytes().hex() == "5e2a4d18190000007b000000c80100004d010000bc0100000200000000b1ea928f"
    # accessor arithmetic over 1234 frames (:1085-1115)
    NUM, CS, DS = 1234, 123, 456
    st = zk.SeekTable(lib=lib); orc = O.OracleSeekTable()
    for _ in range(NUM):
        st.log_frame(CS, DS); orc.log_frame(CS, DS)
    assert st.num_frames() == NUM and st.size_comp() == NUM * CS and st.size_decomp() == NUM * DS
    assert st.max_frame_size_comp() == CS and st.max_frame_size_decomp() == DS
    for i in (0, 1, 617, NUM - 1):
        assert st.frame_start_comp(i) == i * CS and st.frame_end_comp(i) == (i + 1) * CS and st.frame_size_comp(i) == CS
        assert st.frame_start_decomp(i) == i * DS and st.frame_end_decomp(i) == (i + 1) * DS and st.frame_size_decomp(i) == DS
        for probe in (i * DS, i * DS + 1, (i + 1) * DS - 1):
            assert st.frame_index_decomp(probe) == i == orc.frame_index_decomp(probe)
        assert st.frame_index_comp(i * CS + CS // 2) == i == orc.frame_index_comp(i * CS + CS // 2)
    assert st.frame_index_decomp(NUM * DS) == NUM - 1 and st.frame_index_decomp(NUM * DS + 99) == NUM - 1
    for fn in (st.frame_start_comp, st.frame_end_decomp, st.frame_size_comp):
        try:
            fn(NUM); raise AssertionError
        except zk.Error as e:
            assert e.is_frame_index_too_large()
    # resumable serialization with tiny buffers (:1117-1141, 1257-1260), both formats, vs the oracle bytes
    for fmt, name in ((zk.Format.Foot, "foot"), (zk.Format.Head, "head")):
        want = orc.serialize(name)
        for blen in (1, 2, 3, 7, 8, 9, 13, 63):
            ser = st.into_format_serializer(fmt)
            got = bytearray()
            while True:
                b = bytearray(blen)
                n = ser.write_into(b)
                if n == 0:
                    break
                got += b[:n]
            assert bytes(got) == want and ser.encoded_len() == len(want)
            ser.reset()
            assert ser.to_bytes() == want
        # serde cycle (:1143-1154)
        back = zk.SeekTable.from_bytes(want, fmt, lib)
        assert back == st
    for nframes in (0, 1, 2, 1023, 1024, 1025, 4095):
        t = zk.SeekTable(lib=lib)
        for i in range(nframes):
            t.log_frame(i * 7 + 1, i * 13 + 5)
        for fmt in (zk.Format.Head, zk.Format.Foot):
            assert zk.SeekTable.from_bytes(t.into_format_serializer(fmt).to_bytes(), fmt, lib) == t
    # entries with per-frame checksums (12 bytes, descriptor bit 7), as zstd's own C seekable code writes (:1187-1212)
    import struct
    body = b"".join(struct.pack("<III", 100 + i, 1000 + i, 0xDEADBEEF) for i in range(5))
    tbl = struct.pack("<II", 0x184D2A5E, len(body) + 9) + body + struct.pack("<IBI", 5, 0x80, 0x8F92EAB1)
    t = zk.SeekTable.from_bytes(b"x" * 33 + tbl, zk.Format.Foot, lib)
    assert t.num_frames() == 5 and t.frame_size_comp(4) == 104 and t.frame_size_decomp(4) == 1004
    # malformed tables
    good = st.into_serializer().to_bytes()
    for mutate, pred in ((lambda b: b[:-1] + b"\x00", "zstd10"), (lambda b: b[:-5] + b"\x04" + b[-4:], "zstd20"),
                         (lambda b: b"\x00" + b[1:], "zstd10"), (lambda b: b[:4] + b"\x01\x00\x00\x00" + b[8:], "zstd20"),
                         (lambda b: b[-8:], "range")):
        try:
            zk.SeekTable.from_bytes(mutate(good), zk.Format.Foot, lib)
            raise AssertionError("malformed table accepted")
        except zk.Error as e:
            if pred == "range":
                assert e.is_offset_out_of_range()
            else:
                assert e.is_zstd() and e.zstd_code() == int(pred[4:])


# ---------------------------------------------------------------------------------- CLI front end (cli/tests/integration/main.rs)
def _cli(ctx, argv, stdin: bytes = b""):
    """run zeekstd_b200.cli.main in-process with ctx as the default context; -> (rc, stdout bytes, stderr text)"""
    import contextlib
    import io
    import sys
    import zeekstd_b200 as zk
    from zeekstd_b200 import cli

    class _Std:
        def __init__(self, data=b""):
            self.buffer = io.BytesIO(data)
            self.text = io.StringIO()
        def isatty(self): return False
        def write(self, s): return self.text.write(s)
        def flush(self): pass
        def readline(self): return self.buffer.readline().decode()

    old_ctx = zk._default_ctx
    zk.set_default_context(ctx)
    so, se, si = _Std(), _Std(), _Std(stdin)
    old = sys.stdout, sys.stderr, sys.stdin
    sys.stdout, sys.stderr, sys.stdin = so, se, si
    try:
        try:
            rc = cli.main([str(a) for a in argv])
        except SystemExit as e:
            rc = int(e.code or 0)
    finally:
        sys.stdout, sys.stderr, sys.stdin = old
        zk.set_default_context(old_ctx)
    return rc, so.buffer.getvalue() + so.text.getvalue().encode(), se.text.getvalue()


def check_cli(ctx, tmp, data: bytes, frame_sizes, tag=""):
    """one body per test of cli/tests/integration/main.rs, on `data` instead of the whole corpus where sizes must stay small"""
    import os
    import zeekstd_b200 as zk
    from zeekstd_b200 import cli
    tmp = str(tmp)
    src = os.path.join(tmp, f"input{tag}.txt")
    with open(src, "wb") as f:
        f.write(data)

    # args.rs:331-435 value parsers
    assert cli.byte_value("10") == 10
    for s, v in (("10B", 10), ("10 B", 10), ("10K", 10240), ("10 kib", 10240), ("10   mib", 10 << 20), ("2G", 2 << 30), ("2 gib", 2 << 30)):
        assert cli.byte_value(s) == v, s
    for bad in ("10 X", " ", "abc B"):
        try:
            cli.byte_value(bad); raise AssertionError(bad)
        except Exception as e:
            assert not isinstance(e, AssertionError)
    for s in ("end", "End", "eND", "END"):
        assert cli.last_frame(s) == "end" and cli.offset_limit(s) is None
    assert cli.last_frame("7") == 7 and cli.offset_limit("3K") == 3072
    assert cli.human_bytes(1023) == "1023 B" and cli.human_bytes(10192446) == "9.72 MiB"

    for fs in frame_sizes:
        # cycle: file -> file -> file (:38-59)
        z = os.path.join(tmp, f"c{tag}_{fs}.zst")
        rc, _, err = _cli(ctx, ["compress", src, "--output-file", z, "--frame-size", fs], b"y")
        assert rc == 0, err
        back = os.path.join(tmp, f"back{tag}_{fs}")
        rc, _, err = _cli(ctx, ["decompress", z, "--output-file", back], b"y")
        assert rc == 0, err
        assert open(back, "rb").read() == data
        # what the CLI wrote is a seekable archive libzstd accepts
        arc = open(z, "rb").read()
        st = zk.SeekTable.from_bytes(arc)
        assert st.size_decomp() == len(data) and st.size_comp() + st.into_serializer().encoded_len() == len(arc)
        # stdin -> file (:61-76), file -> stdout (:78-97), stdin -> stdout (:99-117)
        z2 = os.path.join(tmp, f"s{tag}_{fs}.zst")
        rc, _, err = _cli(ctx, ["compress", "--output-file", z2, "--frame-size", fs], data)
        assert rc == 0 and open(z2, "rb").read() == arc, err
        rc, out, err = _cli(ctx, ["compress", src, "--stdout", "--frame-size", fs])
        assert rc == 0 and out == arc, err
        rc, out, err = _cli(ctx, ["--stdout", "--frame-size", fs], data)          # no sub-command = compress (main.rs:27-30)
        assert rc == 0 and out == arc, err
        rc, out, err = _cli(ctx, ["d", z, "-c"])
        assert rc == 0 and out == data, err
        # separate seek table (:119-153)
        z3, t3 = os.path.join(tmp, f"h{tag}_{fs}.zst"), os.path.join(tmp, f"h{tag}_{fs}.table")
        rc, _, err = _cli(ctx, ["compress", src, "--output-file", z3, "--frame-size", fs, "--seek-table-file", t3], b"y")
        assert rc == 0, err
        assert open(z3, "rb").read() == arc[:st.size_comp()]
        rc, out, err = _cli(ctx, ["decompress", z3, "--seek-table-file", t3, "-c"])
        assert rc == 0 and out == data, err
        rc, out, err = _cli(ctx, ["list", t3, "--seek-table-format", "head"])
        assert rc == 0 and out.count(b"\n") == 2, err

    # output name derivation (:189-290)
    one = os.path.join(tmp, f"name{tag}.bin")
    with open(one, "wb") as f:
        f.write(data[:1000])
    rc, _, err = _cli(ctx, ["compress", one], b"y")
    assert rc == 0 and os.path.exists(one + ".zst"), err
    os.remove(one)
    rc, _, err = _cli(ctx, ["decompress", one + ".zst"], b"y")
    assert rc == 0 and open(one, "rb").read() == data[:1000], err
    noext = os.path.join(tmp, f"noext{tag}")
    os.rename(one + ".zst", noext)
    rc, _, err = _cli(ctx, ["decompress", noext])
    assert rc != 0 and "unknown extension" in err
    other = noext + ".foo"
    os.rename(noext, other)
    rc, _, err = _cli(ctx, ["decompress", other])
    assert rc != 0 and "unknown extension" in err
    given = os.path.join(tmp, f"given{tag}.out")
    rc, _, err = _cli(ctx, ["decompress", other, "--output-file", given])
    assert rc == 0 and open(given, "rb").read() == data[:1000], err

    # overwrite rules (:292-361): prompt answered "n", stdin input never overwrites, --force does
    keep = open(given, "rb").read()
    rc, _, err = _cli(ctx, ["compress", src, "--output-file", given], b"n\n")
    assert rc != 0 and open(given, "rb").read() == keep
    rc, _, err = _cli(ctx, ["compress", "--output-file", given], data)
    assert rc != 0 and "not overwritten" in err and open(given, "rb").read() == keep
    rc, _, err = _cli(ctx, ["compress", src, "--output-file", given, "--quiet"])
    assert rc != 0 and open(given, "rb").read() == keep
    tab = os.path.join(tmp, f"exists{tag}.table")
    open(tab, "wb").write(b"x")
    fresh = os.path.join(tmp, f"fresh{tag}.zst")
    rc, _, err = _cli(ctx, ["compress", "--output-file", fresh, "--seek-table-file", tab], data)
    assert rc != 0 and open(tab, "rb").read() == b"x" and not os.path.exists(fresh), err
    rc, _, err = _cli(ctx, ["compress", src, "--output-file", given, "--force"])
    assert rc == 0 and open(given, "rb").read() != keep, err
    rc, _, err = _cli(ctx, ["compress", "--output-file", given, "--force"], data)
    assert rc == 0, err
    # a missing input creates nothing (:363-377)
    nothing = os.path.join(tmp, f"nothing{tag}.zst")
    rc, _, err = _cli(ctx, ["compress", os.path.join(tmp, "does-not-exist"), "--output-file", nothing])
    assert rc != 0 and not os.path.exists(nothing)

    # frame / offset selection (:379-520)
    n = len(data)
    fs6 = n // 6
    z6 = os.path.join(tmp, f"six{tag}.zst")
    assert _cli(ctx, ["compress", src, "-o", z6, "-s", fs6], b"y")[0] == 0
    rc, first, err = _cli(ctx, ["decompress", z6, "-c", "--from-frame", 0, "--to-frame", 0])
    assert rc == 0 and len(first) == fs6, err
    rc, rest, err = _cli(ctx, ["decompress", z6, "-c", "--from-frame", 1, "--to-frame", "end"])
    assert rc == 0 and first + rest == data, err
    t6 = os.path.join(tmp, f"six{tag}.table")
    assert _cli(ctx, ["compress", src, "-s", fs6, "-o", z6, "--seek-table-file", t6, "--force"])[0] == 0
    rc, first, err = _cli(ctx, ["decompress", z6, "--seek-table-file", t6, "-c", "--from-frame", 0, "--to-frame", 0])
    assert rc == 0 and first == data[:fs6], err
    zall = os.path.join(tmp, f"all{tag}.zst")
    assert _cli(ctx, ["compress", src, "-o", zall, "-s", n], b"y")[0] == 0
    assert _cli(ctx, ["decompress", zall, "-c", "--from-frame", 1])[0] != 0
    assert _cli(ctx, ["decompress", zall, "-c", "--from-frame", 0, "--to-frame", 1])[0] != 0
    fs9 = n // 9
    z9 = os.path.join(tmp, f"nine{tag}.zst")
    assert _cli(ctx, ["compress", src, "-o", z9, "-s", fs9], b"y")[0] == 0
    lo, hi = fs9 + fs9 // 2, 4 * fs9 + fs9 // 2
    rc, out, err = _cli(ctx, ["decompress", z9, "-c", "--from", lo, "--to", hi])
    assert rc == 0 and out == data[lo:hi], err

    # list (:522-590): summary = 2 lines, --detail = header + one line per frame
    fs14 = n // 14
    z14 = os.path.join(tmp, f"fourteen{tag}.zst")
    assert _cli(ctx, ["compress", src, "-o", z14, "-s", fs14], b"y")[0] == 0
    frames = -(-n // fs14)
    rc, out, err = _cli(ctx, ["list", z14])
    assert rc == 0 and out.count(b"\n") == 2 and out.split(b"\n")[1].split()[0] == str(frames).encode(), err
    rc, out, err = _cli(ctx, ["list", "--detail", z14])
    assert rc == 0 and out.count(b"\n") == frames + 1, err
    rc, out, err = _cli(ctx, ["-r", "list", z14, "--from-frame", 2, "--num-frames", 3])
    rows = out.decode().splitlines()
    assert rc == 0 and len(rows) == 4 and [r.split()[0] for r in rows[1:]] == ["2", "3", "4"] and rows[1].split()[2] == str(fs14), err
    assert _cli(ctx, ["list", z14, "--from-frame", 5, "--to-frame", 2])[0] != 0

    # patch mode (--patch-from / --patch-apply, command.rs:199-263 + compress.rs:32-38)
    m = min(n // 2, 48_000)              # new = old shifted by m/4: every match into the prefix is 3m/4 <= 36 000 bytes back, inside the
    old_v, new_v = data[:m], data[m // 4: m + m // 4]      # 64 KiB match window of these kernels (DESIGN.md 5)
    pf, nf = os.path.join(tmp, f"old{tag}"), os.path.join(tmp, f"new{tag}")
    open(pf, "wb").write(old_v); open(nf, "wb").write(new_v)
    zp, zn = os.path.join(tmp, f"patch{tag}.zst"), os.path.join(tmp, f"nopatch{tag}.zst")
    assert _cli(ctx, ["compress", nf, "-o", zp, "--patch-from", pf, "-s", len(new_v)])[0] == 0
    assert _cli(ctx, ["compress", nf, "-o", zn, "-s", len(new_v)])[0] == 0
    rc, out, err = _cli(ctx, ["decompress", zp, "-c", "--patch-apply", pf])
    assert rc == 0 and out == new_v, err
    rc, out, err = _cli(ctx, ["decompress", zp, "-c", "--patch-apply", pf, "--mmap-prefix"])
    assert rc == 0 and out == new_v, err
    return os.path.getsize(zp), os.path.getsize(zn)


def check_seek_table_fuzz(lib, iters: int = 3000, seed: int = 5):
    """mutated seek tables (both formats): the native parser and the restatement of seek_table.rs:144-225, 379-436 agree on
    accept / reject, on the zstd error code, and on every offset of an accepted table"""
    rng = np.random.default_rng(seed)
    parsed = rejected = 0
    for _ in range(iters):
        t = O.OracleSeekTable()
        for _ in range(int(rng.integers(0, 12))):
            t.log_frame(int(rng.integers(0, 1 << 20)), int(rng.integers(0, 1 << 22)))
        fmt = "head" if rng.integers(2) else "foot"
        b = bytearray(t.serialize(fmt))
        lead = bytes(rng.integers(0, 256, int(rng.integers(0, 20)), dtype=np.uint8)) if fmt == "foot" else b""
        for _ in range(int(rng.integers(0, 3))):
            k = int(rng.integers(4)); p = int(rng.integers(len(b)))
            if k == 0: b[p] ^= 1 << int(rng.integers(8))
            elif k == 1: b[p] = int(rng.integers(256))
            elif k == 2: del b[p:p + int(rng.integers(1, 5))]
            else: b[p:p] = bytes(rng.integers(0, 256, int(rng.integers(1, 5)), dtype=np.uint8))
        blob = lead + bytes(b)
        try:
            want, wexc = O.OracleSeekTable.parse(blob, fmt), None
        except Exception as e:
            want, wexc = None, e
        try:
            got, gexc = zk.SeekTable.from_bytes(blob, zk.Format.Head if fmt == "head" else zk.Format.Foot, lib), None
        except zk.Error as e:
            got, gexc = None, e
        assert (want is None) == (got is None), (fmt, blob.hex(), repr(wexc), repr(gexc))
        if want is not None:
            n = want.num_frames()
            assert got.num_frames() == n
            for i in range(n):
                assert got.frame_end_comp(i) == want.c[i + 1] and got.frame_end_decomp(i) == want.d[i + 1], (i, blob.hex())
            parsed += 1
        else:
            if isinstance(wexc, O.ZstdError):
                assert gexc.is_zstd() and gexc.zstd_code() == wexc.code, (repr(wexc), gexc.rc, blob.hex())
            rejected += 1
    assert parsed > iters // 4 and rejected > iters // 4


def check_decoder_random_ops(ctx, ops: int = 250, seed: int = 3, n: int = 24_000, frame_size: int = 1_700):
    """differential test of the Decoder's state machine against the contract of decode.rs:201-270, 344-445, 545-579 written as a
    model over the plain bytes: a call returns data[offset : min(offset + len(buf), limit)] and advances the offset; offsets and
    limits beyond size_decomp and frame indices beyond the table are errors that change nothing; reset restores (0, size_decomp).
    The archive is libzstd-written (ragged last frame), read through a file-like source."""
    import io
    rng = np.random.default_rng(seed)
    data = corpus.as_numpy(corpus.make_mix(n, seed=seed, mix=corpus.CLASS_MIX_MIXED, segment=4096)).tobytes()
    arc, _ = O.ref_seekable_archive(np.frombuffer(data, dtype=np.uint8), frame_size, 3, True)
    dec = zk.Decoder(zk.DecodeOptions(io.BytesIO(arc), ctx))
    total, nf = len(data), dec.seek_table().num_frames()
    assert dec.seek_table().size_decomp() == total and nf == -(-total // frame_size)
    off, lim = 0, total
    fresh = True                                   # read_compressed() == 0: nothing read since the last (implicit) reset, decode.rs:352-357, 402-414
    fstart = lambda i: min(i * frame_size, total)
    fidx = lambda o: min(o // frame_size, nf - 1)    # frame_index_decomp (seek_table.rs:916-934): offsets at or past the end map to the last frame

    def moved(o):                                    # set_offset resets the context exactly when the frame changes or the offset goes back
        return fidx(o) != fidx(off) or o < off

    def expect_err(fn, pred):
        try:
            fn()
        except zk.Error as e:
            assert pred(e), e.rc
            return
        raise AssertionError("no error")

    for _ in range(ops):
        k = int(rng.integers(10))
        if k <= 3:                                            # decompress
            ln = int(rng.choice([0, 1, 7, 100, frame_size - 1, frame_size, frame_size + 1, 3 * frame_size - 100, total]))
            buf = bytearray(ln)
            got = dec.decompress(buf)
            want = data[off: min(off + ln, lim)] if lim > off else b""
            assert got == len(want) and bytes(buf[:got]) == want, (off, lim, ln, got, len(want))
            if got:
                fresh = False
            off += got
        elif k == 4:
            o = int(rng.integers(0, total + 1)) if rng.integers(8) else total + int(rng.integers(1, 50))
            if o > total: expect_err(lambda: dec.set_offset(o), lambda e: e.is_offset_out_of_range())
            else: fresh = fresh or moved(o); dec.set_offset(o); off = o
        elif k == 5:
            l = int(rng.integers(0, total + 1)) if rng.integers(8) else total + int(rng.integers(1, 50))
            if l > total: expect_err(lambda: dec.set_offset_limit(l), lambda e: e.is_offset_out_of_range())
            else: dec.set_offset_limit(l); lim = l
        elif k == 6:
            i = int(rng.integers(0, nf + 2))
            if i >= nf: expect_err(lambda: dec.set_lower_frame(i), lambda e: e.is_frame_index_too_large())
            else: fresh = fresh or moved(fstart(i)); assert dec.set_lower_frame(i) == fstart(i); off = fstart(i)
        elif k == 7:
            i = int(rng.integers(0, nf + 2))
            if i >= nf: expect_err(lambda: dec.set_upper_frame(i), lambda e: e.is_frame_index_too_large())
            else: assert dec.set_upper_frame(i) == fstart(i + 1); lim = fstart(i + 1)
        elif k == 8:
            w = int(rng.integers(3))
            if w == 0: p = int(rng.integers(0, total + 20)); tgt = p
            elif w == 1: p = int(rng.integers(-off - 5, total - off + 20)); tgt = off + p
            else: p = int(rng.integers(-total - 5, 3)); tgt = total + p
            bad = tgt < 0 or tgt > total or (w == 2 and p > 0)
            if bad: expect_err(lambda: dec.seek(p, w), lambda e: e.is_offset_out_of_range())
            else: fresh = fresh or moved(tgt); assert dec.seek(p, w) == tgt; off = tgt
        else:
            dec.reset(); off, lim = 0, total; fresh = True
        assert dec.offset() == off and dec.offset_limit() == lim
        assert (dec.read_compressed() == 0) == fresh, (dec.read_compressed(), fresh, off, lim)


def check_encoder_random_ops(ctx, ops: int = 60, seed: int = 4, frame_size: int = 700, prefix: bool = False):
    """differential test of Encoder framing against the contract of encode.rs:311-354, 438-472, 528-544, 626-775 as a model: a frame
    holds at most frame_size input bytes; a frame that filled up is closed lazily by the next compress / end_frame / finish;
    end_frame and finish always close a frame, an empty one included.  The archive must be one libzstd restores."""
    import io
    rng = np.random.default_rng(seed)
    sink = io.BytesIO()
    pfx = corpus.as_numpy(corpus.make_class("text", 3000, seed=seed + 1)) if prefix else None
    enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.Uncompressed(frame_size)).checksum_flag(bool(seed & 1)).compression_level(3).into_encoder(sink)
    src = corpus.as_numpy(corpus.make_mix(ops * max(400, frame_size // 2), seed=seed, mix=corpus.CLASS_MIX_MIXED, segment=2048)).tobytes()
    if prefix:
        src = pfx.tobytes()[500:1500] + src[1000:]
    pos, cur, model = 0, 0, []
    for _ in range(ops):
        if rng.integers(6) == 0:
            enc.end_frame(); model.append(cur); cur = 0
            continue
        ln = int(rng.choice([0, 1, 13, frame_size - 1, frame_size, frame_size + 1, 3 * frame_size + 5, int(rng.integers(1, 2000))]))
        chunk = src[pos: pos + ln]
        done = 0
        while done < len(chunk):
            k = enc.compress_with_prefix(chunk[done:], pfx) if prefix else enc.compress(chunk[done:])
            assert k > 0
            done += k
        left = len(chunk)
        while left:
            if cur == frame_size:
                model.append(cur); cur = 0
            take = min(left, frame_size - cur); cur += take; left -= take
        pos += len(chunk)
    total_written = enc.finish()
    model.append(cur)
    arc = sink.getvalue()
    assert total_written == len(arc)
    st = zk.SeekTable.from_bytes(arc, lib=ctx.lib)
    got = [st.frame_size_decomp(i) for i in range(st.num_frames())]
    assert got == model, (got[:12], model[:12], len(got), len(model))
    cs = [st.frame_size_comp(i) for i in range(st.num_frames())]
    assert st.size_comp() + st.into_serializer().encoded_len() == len(arc)
    from util import offsets
    out, sizes = O.ref_decompress_frames(np.frombuffer(arc, dtype=np.uint8)[: st.size_comp()], offsets(cs), offsets(got), prefix=pfx)
    assert list(sizes) == got and out.tobytes() == src[:pos]
    return len(model)


def check_encoder_golden(ctx, skip=(), only=None):
    """The encoder's bytes are deterministic (DESIGN.md 3: ties between lanes are resolved as sequential insertion would) and the SAME on every
    build of the sources: tests/golden/encoder_golden.json was written from the CPU emulation build (any warp-scheduling seed gives these hashes);
    the nvcc build on a GPU must reproduce it byte for byte -- which is also what lets ratios measured on one build be quoted for the other."""
    import hashlib
    import json
    gold = json.loads(golden_bytes("encoder_golden.json"))
    d = np.frombuffer(golden_bytes("dickens_96k.txt"), dtype=np.uint8)
    for key, want in gold.items():
        if key in skip or (only is not None and key not in only):
            continue
        if key == "3+prefix":
            comp, cs, ds = ctx.compress_frames(d[20_000:], 40_000, 3, True, prefix=d[:30_000])
        else:
            comp, cs, ds = ctx.compress_frames(d, 40_000, int(key), True)
        assert int(comp.size) == want["size"] and hashlib.sha256(comp.tobytes()).hexdigest() == want["sha256"], (key, int(comp.size), want["size"])
