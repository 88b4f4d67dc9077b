"""K-D1s comes in two cell layouts: zk_seq2_kernel holds 768 cells per block (LL, OF and ML tables back to back, each as
large as its accuracy log), zk_seq2_full_kernel the format's 512 + 256 + 512.  A block whose parsed tables need more than
768 cells is passed from the first to the second.  These tests pin the rule (restated below from the table descriptions),
show that libzstd's high levels produce such blocks and this codec's encoder does not, and decode batches that mix the two
routes, Repeat tables that point at a full-route block, and descriptions above the format's logs.
Every case runs on the emulation build (`-m "not gpu"`) and on the H100 (`-m gpu`)."""
import numpy as np
import pytest

import framegen as G
import zeekstd_b200 as zk
from oracle import oracle as O
from test_crafted_sequences import FB, batch, expect, short_seqs
from util import golden_bytes, offsets, serial_status

COMPACT_CELLS = 768
PREDEF_CELLS = (64, 32, 64)          # LL, OF, ML
MAX_SYM = (35, 31, 52)


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def ctx(request):
    c = zk.Context(0, request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib"))
    yield c
    c.close()


# ------------------------------------------------------------------------------------------------ the rule, restated
def _ncount(b: bytes, pos: int, max_sym: int):
    """FSE table description at b[pos] (RFC 8878 4.1.1) -> (accuracy log, bytes it takes)"""
    bits, off = int.from_bytes(b[pos:pos + 128], "little"), 4
    al = (bits & 15) + 5
    remaining, threshold, nb, sym, prev0 = (1 << al) + 1, 1 << al, al + 1, 0, False
    while remaining > 1 and sym <= max_sym:
        if prev0:
            while True:
                r = (bits >> off) & 3
                off += 2; sym += r
                if r != 3:
                    break
        mx = 2 * threshold - 1 - remaining
        low = (bits >> off) & (threshold - 1)
        if low < mx:
            c = low; off += nb - 1
        else:
            c = (bits >> off) & (2 * threshold - 1)
            if c >= threshold:
                c -= mx
            off += nb
        c -= 1
        remaining -= -c if c < 0 else c
        sym += 1; prev0 = c == 0
        while remaining < threshold:
            nb -= 1; threshold >>= 1
    return al, (off + 7) // 8


def _lit_section(b: bytes) -> int:
    typ, sf = b[0] & 3, (b[0] >> 2) & 3
    if typ < 2:
        hdr, regen = ((1, b[0] >> 3) if sf in (0, 2) else (2, (b[0] >> 4) | (b[1] << 4)) if sf == 1 else
                      (3, (b[0] >> 4) | (b[1] << 4) | (b[2] << 12)))
        return hdr + (regen if typ == 0 else 1)
    v = int.from_bytes(b[:5], "little")
    hdr, comp = ((3, (v >> 14) & 0x3FF) if sf < 2 else (4, (v >> 18) & 0x3FFF) if sf == 2 else (5, (v >> 22) & 0x3FFFF))
    return hdr + comp


def seq_block_cells(entry: bytes) -> list:
    """cells each block with sequences needs (Repeat: the table it refers to), in order, over every zstd frame of an entry"""
    out, pos = [], 0
    while pos < len(entry):
        magic = int.from_bytes(entry[pos:pos + 4], "little")
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            pos += 8 + int.from_bytes(entry[pos + 4:pos + 8], "little")
            continue
        assert magic == 0xFD2FB528
        fhd = entry[pos + 4]
        fcs_flag, single, csum, did = fhd >> 6, (fhd >> 5) & 1, (fhd >> 2) & 1, fhd & 3
        pos += 5 + (0 if single else 1) + (4 if did == 3 else did) + ((single, 2, 4, 8)[fcs_flag])
        last_cells = [None, None, None]
        while True:
            bh = int.from_bytes(entry[pos:pos + 3], "little")
            last, typ, size = bh & 1, (bh >> 1) & 3, bh >> 3
            b = entry[pos + 3:pos + 3 + size]
            pos += 3 + (1 if typ == 1 else size)
            if typ == 2:
                q = _lit_section(b)
                n0 = b[q]
                nseq, q = (n0, q + 1) if n0 < 128 else ((((n0 - 128) << 8) + b[q + 1], q + 2) if n0 < 255 else (b[q + 1] + (b[q + 2] << 8) + 0x7F00, q + 3))
                if nseq:
                    modes, q = b[q], q + 1
                    for t in range(3):
                        m = (modes >> (6 - 2 * t)) & 3
                        if m == 0:
                            last_cells[t] = PREDEF_CELLS[t]
                        elif m == 1:
                            last_cells[t] = 1; q += 1
                        elif m == 2:
                            al, used = _ncount(b, q, MAX_SYM[t])
                            last_cells[t] = 1 << al; q += used
                    out.append(sum(last_cells))
            if last:
                break
        pos += 4 if csum else 0
    return out


def test_rule_reads_table_descriptions():
    """the restatement's description parser against the writer's descriptions at every accuracy log"""
    rng = np.random.default_rng(1)
    for al in range(5, 10):
        for k in range(20):
            syms = sorted({int(s) for s in rng.integers(0, 36, int(rng.integers(2, 30)))})
            t = G.Fse(G.norm_for(syms, al, neg=syms[1:1 + k % 3]), al)
            h = t.header()
            assert _ncount(h + b"\0" * 8, 0, 35) == (al, len(h))


def _text(n: int) -> np.ndarray:
    return np.frombuffer(golden_bytes("dickens.txt")[1_000_000:1_000_000 + n], dtype=np.uint8)


def _libzstd_l19(x: np.ndarray, frame: int):
    frames, cs, ds = O.ref_compress_frames(x, frame, 19, False)
    return list(frames), [int(d) for d in ds]


def test_libzstd_high_level_blocks_take_the_full_route():
    frames, _ = _libzstd_l19(_text(256 << 10), 128 << 10)
    cells = [c for f in frames for c in seq_block_cells(f)]
    assert cells and max(cells) > COMPACT_CELLS, cells


@pytest.mark.parametrize("level", [1, 3, 19])
def test_own_archives_stay_compact(ctx, level):
    x = _text(96 << 10)
    comp, cs, ds = ctx.compress_frames(x, 32 << 10, level, False)
    blob = comp.tobytes()
    co = offsets(cs)
    cells = [c for i in range(len(cs)) for c in seq_block_cells(blob[int(co[i]):int(co[i + 1])])]
    assert cells and max(cells) <= COMPACT_CELLS, cells


# ------------------------------------------------------------------------------------------------ decoding both routes
def _codes(s):
    f = lambda fn, xs: sorted({fn(v) for v in xs})   # noqa: E731
    return f(G.ll_code, [v[0] for v in s]), f(G.of_code, [v[1] + 3 for v in s]), f(G.ml_code, [v[2] for v in s])


def _fse(codes, al):
    return ("fse", G.norm_for(codes, al), al)


def crafted_cases(seed: int):
    """cases for batch(): frames on both sides of the 768-cell line, each checked against the cells the rule gives its blocks"""
    rng = np.random.default_rng(seed)
    s = short_seqs(rng, 300, reach=100)
    ll_c, of_c, ml_c = _codes(s)
    rep = (("repeat",),) * 3
    out = []

    def add(name, fb, cells):
        fr = fb.frame()
        assert seq_block_cells(G.frame_bytes(fr)) == cells, name
        out.append((name, [fr], 0, b""))
    add("compact_768", FB(rng).raw(128).seqs(s, tables=(_fse(ll_c, 8), _fse(of_c, 8), _fse(ml_c, 8))), [768])
    add("compact_ll9", FB(rng).raw(128).seqs(s, tables=(_fse(ll_c, 9), _fse(of_c, 5), ("predef",))), [512 + 32 + 64])
    add("full_800", FB(rng).raw(128).seqs(s, tables=(_fse(ll_c, 9), _fse(of_c, 8), _fse(ml_c, 5))), [512 + 256 + 32])
    add("full_1280", FB(rng).raw(128).seqs(s, tables=(_fse(ll_c, 9), _fse(of_c, 8), _fse(ml_c, 9))), [1280])
    # Repeat tables that point at a full-route block: all three (full again), and LL alone beside smaller ones (compact)
    add("repeat_of_full", FB(rng).raw(128).seqs(s[:150], tables=(_fse(ll_c, 9), _fse(of_c, 8), _fse(ml_c, 9)))
        .seqs(s[150:], tables=rep), [1280, 1280])
    add("repeat_ll_of_full_compact", FB(rng).raw(128).seqs(s[:150], tables=(_fse(ll_c, 9), _fse(of_c, 8), _fse(ml_c, 9)))
        .raw(40).seqs(s[150:], tables=(("repeat",), ("predef",), _fse(ml_c, 6))), [1280, 512 + 32 + 64])
    # a compact block, then a full one, then Repeat of the full one's tables, in one frame
    add("compact_full_repeat", FB(rng).raw(128).seqs(s[:100]).seqs(s[100:200], tables=(_fse(ll_c, 9), _fse(of_c, 8), _fse(ml_c, 9)))
        .seqs(s[200:], tables=rep), [160, 1280, 1280])
    return out


def test_mixed_routes_in_one_batch(ctx):
    """libzstd level-19 frames (full-route blocks), this codec's level-1 frames and crafted frames on both sides of the
    768-cell line, in one batch; everything must decode to what libzstd decodes"""
    x = _text(256 << 10)
    l19, l19_sizes = _libzstd_l19(x, 128 << 10)
    comp, cs, ds = ctx.compress_frames(x[:64 << 10], 32 << 10, 1, False)
    own = [comp.tobytes()[int(a):int(b)] for a, b in zip(offsets(cs)[:-1], offsets(cs)[1:])]
    cases = crafted_cases(2)
    entries, sizes, wants, names, _ = batch(cases)
    for f, d in zip(l19, l19_sizes):
        entries.append(f); sizes.append(d); names.append("libzstd_l19")
        wants.append(O.ref_decompress_any(f, d + 1))
    start = 0
    for f, d in zip(own, ds):
        entries.append(f); sizes.append(int(d)); names.append("own_l1")
        wants.append(x[start:start + int(d)].tobytes()); start += int(d)
    assert b"".join(wants[-len(own) - len(l19):-len(own)]) == x.tobytes()
    expect(ctx, (entries, sizes, wants, names, None))


def test_tables_above_the_format_logs(ctx):
    """LL / ML descriptions at log 10 and OF at log 9 (one above the format's maxima) fail with libzstd's code, beside good
    entries of both routes that decode intact"""
    rng = np.random.default_rng(3)
    s = short_seqs(rng, 60, reach=100)
    ll_c, of_c, ml_c = _codes(s)
    bad = {"ll_log10": (_fse(ll_c, 10), _fse(of_c, 5), ("predef",)),
           "of_log9": (("predef",), _fse(of_c, 9), ("predef",)),
           "ml_log10": (_fse(ll_c, 9), _fse(of_c, 8), _fse(ml_c, 10))}
    cases, code = [c for c in crafted_cases(4) if c[0] in ("compact_768", "full_1280", "repeat_ll_of_full_compact")], {}
    for name, t in bad.items():
        fr = FB(rng).raw(128).seqs(s, tables=t).frame()
        blob = G.frame_bytes(fr)
        for fn in (O.ref_decompress_any, O.oracle_decompress):
            with pytest.raises(O.ZstdError) as e:
                fn(blob, 1 << 20)
            code[name] = e.value.code
        cases.append((name, [fr], code[name], b""))
    b = batch(cases)
    want = {i: -code[n] for i, n in enumerate(b[3]) if n in code}
    assert len(want) == len(bad)
    assert {i: st for i, st in enumerate(serial_status(e, n) for e, n in zip(b[0], b[1])) if st} == want
    expect(ctx, b, want)
