"""Crafted frames on the decode kernels' own boundaries.  Every frame is written by tests/framegen.py, so each case sits
exactly where a kernel changes path: the single-warp executor's 4 KiB window (near / far split and reloads at 2 KiB), the
CTA executor's ring (R/2), the long-copy paths at 48 bytes, matches into the prefix (prefix mode), the plan kernel's segment
starts, the sequence-stream forms and the two-level Huffman table.  Every valid entry is checked three ways before the
codec sees it (executor == libzstd == the restatement) and must then decode to the executor's bytes under every context
listed for its family; invalid entries must get libzstd's status (and the serial walk's, util.serial_status) while good
entries in the same batch decode intact.
Every case runs on the emulation build (`-m "not gpu"`) and on the H100 (`-m gpu`)."""
import os

import numpy as np
import pytest

import zeekstd_b200 as zk
import framegen as G
from framegen import Block, Frame
from oracle import oracle as O
from util import offsets, serial_status


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    return request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib")


def _context(lib, env: dict):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return zk.Context(0, lib)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


# contexts by name; CTA ones pin W and R so that the emulator (4 SMs) and the H100 (132) run the same configuration:
# batches that use them hold >= 133 entries, so both see >= 4 entries per SM (host path: share 3) and W <= 5 runs _w5
CTX_ENV = {
    "default": {},
    "warp_all": {"ZK_EXEC_SHORT": str(1 << 30)},
    "cta": {"ZK_EXEC_SHORT": "0"},
    **{f"cta_r{r}_w{w}": {"ZK_EXEC_SHORT": "0", "ZK_RING_BYTES": str(r), "ZK_EXEC_WARPS": str(w)} for r in (1024, 4096) for w in (2, 5, 16)},
}
PIN_ENTRIES = 140
# prefix mode on both executors: single warps and CTAs as the defaults route them, all on single warps, all on CTAs, and
# CTAs pinned to a small ring
PREFIX_CTXS = ("default", "warp_all", "cta", "cta_r1024_w5")


@pytest.fixture(scope="module")
def ctxs(lib):
    made = {}

    def get(name):
        if name not in made:
            made[name] = _context(lib, CTX_ENV[name])
        return made[name]
    yield get
    for c in made.values():
        c.close()


# ------------------------------------------------------------------------------------------------ frame building
class FB:
    """builds one frame from sequences given as (ll, off, ml): off > 0 an explicit offset, off in (-1, -2, -3) the repeat
    code Offset_Value 1 / 2 / 3.  Literal and history bytes are random, so a byte read from a stale place shows."""

    def __init__(self, rng, checksum=False, fcs_width=None):
        self.rng, self.blocks, self.checksum, self.fcs_width = rng, [], checksum, fcs_width

    def _bytes(self, n):
        return self.rng.integers(0, 256, n, dtype=np.uint8).tobytes()

    def raw(self, n):
        self.blocks.append(Block("raw", self._bytes(n))); return self

    def rle(self, n):
        self.blocks.append(Block("rle", self._bytes(1), n=n)); return self

    def lits(self, n, **kw):
        self.blocks.append(Block("comp", self._bytes(n), **kw)); return self

    def seqs(self, seqs, trailing=0, **kw):
        s = [(ll, off + 3 if off > 0 else -off, ml) for ll, off, ml in seqs]
        self.blocks.append(Block("comp", self._bytes(sum(x[0] for x in s) + trailing), seqs=s, **kw)); return self

    def frame(self):
        return Frame(self.blocks, checksum=self.checksum, fcs_width=self.fcs_width)


def short_seqs(rng, n, reach=64, ll_max=6):
    """n sequences of a few literals and short matches within `reach` bytes (needs >= reach bytes of history)"""
    out = []
    for _ in range(n):
        ml = int(rng.integers(3, 12))
        out.append((int(rng.integers(0, ll_max)), int(rng.integers(1, reach)), ml))
    return out


def checked(frames, prefix=b""):
    """-> (entry bytes, expected bytes): the executor, libzstd and the restatement agree on them"""
    blob = G.entry_bytes(frames, prefix)
    want = G.execute(frames, prefix)
    if prefix:
        got, sizes = O.ref_decompress_frames(np.frombuffer(blob, np.uint8), [0, len(blob)], [0, len(want)], prefix=np.frombuffer(prefix, np.uint8))
        assert sizes == [len(want)] and got.tobytes() == want
        assert O.oracle_decompress_ex(blob, len(want) + 1, prefix=np.frombuffer(prefix, np.uint8))[0] == want
    else:
        assert O.ref_decompress_any(blob, len(want) + 1) == want
        assert O.oracle_decompress(blob, len(want) + 1) == want
    return blob, want


def _filler(n):
    return Frame([Block("raw", bytes([n & 255]) * n)])


def batch(cases, min_entries=0):
    """cases: list of (name, frames, expected status (0 = valid), prefix).  Between cases go one-raw-block filler entries
    sized so that the cases' output addresses take every value mod 16.  -> entries, sizes, wants, names, frames per entry"""
    entries, sizes, wants, names, fr = [], [], [], [], []
    pos = 0
    for i, (name, frames, status, prefix) in enumerate(cases):
        k = 16 + ((i - pos) % 16)
        f = _filler(k)
        entries.append(G.frame_bytes(f)); sizes.append(k); wants.append(bytes([k]) * k); names.append("filler"); fr.append([f])
        pos += k
        if status == 0:
            blob, want = checked(frames, prefix)
        else:
            blob, want = G.entry_bytes(frames, prefix), None
        entries.append(blob); sizes.append(len(want) if want is not None else sum(k.regen() for f in frames for k in f.blocks)); wants.append(want); names.append(name)
        fr.append(frames)
        pos += sizes[-1]
    while len(entries) < min_entries:
        f = _filler(17)
        entries.append(G.frame_bytes(f)); sizes.append(17); wants.append(bytes([17]) * 17); names.append("filler"); fr.append([f])
    return entries, sizes, wants, names, fr


def decode(ctx, entries, sizes, prefix=None):
    s0 = ctx.decode_segments
    comp = np.frombuffer(b"".join(entries) + b"\0" * 64, dtype=np.uint8)
    out, st, rc = ctx.decompress_frames(comp, offsets([len(e) for e in entries]), offsets(sizes), True,
                                        prefix=None if prefix is None else np.frombuffer(prefix, np.uint8))
    return out.tobytes(), [int(x) for x in st], ctx.decode_segments - s0


def expect(ctx, b, statuses=None, prefix=None):
    entries, sizes, wants, names, _ = b
    out, st, segs = decode(ctx, entries, sizes, prefix)
    do = offsets(sizes)
    for i, (w, name) in enumerate(zip(wants, names)):
        want_st = 0 if statuses is None else statuses.get(i, 0)
        assert st[i] == want_st, (name, i, st[i], want_st)
        if w is not None and want_st == 0:
            got = out[int(do[i]): int(do[i + 1])]
            if got != w:
                bad = next(j for j in range(len(w)) if got[j] != w[j])
                raise AssertionError(f"{name}: first wrong byte at {bad} of {len(w)}")
    return segs


# ------------------------------------------------------------------------------------------------ A / B: window and ring layouts
def window_cases(half: int, seed: int):
    """layouts against a window (or ring) of 2 * half bytes, named by what they hit"""
    rng = np.random.default_rng(seed)
    hist = 4 * half + 64
    D = (half - 1, half, half + 1, 2 * half - 1, 2 * half, 2 * half + 1)
    cases = []

    def add(name, fb):
        cases.append((name, [fb.frame()], 0, b""))

    def probe(d):   # a chunk whose first match reads d bytes before the chunk start, then ordinary short matches
        return [(0, d, 24)] + short_seqs(rng, 20)
    for d in D:
        add(f"raw_then_src{d}", FB(rng).raw(hist).seqs(probe(d)))
        add(f"rle_then_src{d}", FB(rng).raw(hist).rle(half + 300).seqs(probe(d)))
        add(f"litonly_then_src{d}", FB(rng).raw(hist).lits(half + 100).seqs(probe(d)))
        # a direct chunk (32 sequences, more than half a window of output), then a source d back
        big = [(half // 32 + 8, int(rng.integers(1, 64)), 4) for _ in range(32)]
        add(f"direct_chunk_then_src{d}", FB(rng).raw(hist).seqs(big + probe(d)))
        for t in (half, half + 1):
            add(f"trailing{t}_then_src{d}", FB(rng).raw(hist).seqs(short_seqs(rng, 8), trailing=t).seqs(probe(d)))
    # chunks of half - 1 / half / half + 1 bytes, then a source half / half + 1 back
    for n in (half - 1, half, half + 1):
        ll = (n - 31 * 4) - 4
        first = [(ll, int(rng.integers(1, 64)), 4)] + [(0, int(rng.integers(1, 64)), 4) for _ in range(31)]
        for d in (half, half + 1):
            add(f"chunk{n}_then_src{d}", FB(rng).raw(hist).seqs(first + probe(d)))
    # long / short overlapping copies: ml 47 / 48 (and longer) against every offset class
    offs = list(range(1, 8)) + [8, 9, 15, 16, 17, 24, 31, 32, 33, 40, 47, 48, 49, 64, 100]
    for ml in (47, 48, 49, 100):
        s = [(1, o, ml) for o in offs]
        add(f"overlap_ml{ml}", FB(rng).raw(256).seqs(s[:16]).seqs(s[16:] + s[:4]))
    # a source straddling the chunk start, and 32 matches each reading the previous one's destination
    add("straddle", FB(rng).raw(hist).seqs(short_seqs(rng, 32) + [(10, 20, 30), (0, 40, 50)] + short_seqs(rng, 8)))
    chain = [(1, 1 + 5, 5)] + [(1, 6, 5) for _ in range(31)]
    add("chain32", FB(rng).raw(64).seqs(chain + [(0, 5 + 1, 60)] * 2))
    # a long run of random short and far matches: copies cross the window wrap at every alignment
    mixed = [(int(rng.integers(0, 40)), int(rng.integers(1, 3 * half)), int(rng.integers(3, 70))) for _ in range(300)]
    add("wrap", FB(rng).raw(hist).seqs(mixed[:150]).seqs(mixed[150:]))
    return cases


def test_a_warp_window(ctxs):
    b = batch(window_cases(2048, 1))
    for name in ("default", "warp_all"):
        expect(ctxs(name), b)


@pytest.mark.parametrize("ring", [1024, 4096])
def test_b_cta_ring(ctxs, ring):
    cases = window_cases(ring // 2, 2)
    rng = np.random.default_rng(3)
    # more than ZK_D2_META = 64 chunks of short matches in one block
    cases.append(("chunks_over_64", [FB(rng).raw(128).seqs(short_seqs(rng, 70 * 32, reach=100, ll_max=2)).frame()], 0, b""))
    b = batch(cases, PIN_ENTRIES)
    for w in (2, 5, 16):
        expect(ctxs(f"cta_r{ring}_w{w}"), b)


# ------------------------------------------------------------------------------------------------ C: prefix mode
def test_c_prefix_and_in_order(ctxs):
    """matches into the raw-content prefix before every zstd frame, in both segment executors: whole, straddling the frame
    start, through repeat offsets, in every frame of an entry; a block reading into the prefix starts no segment unless it
    is the entry's first"""
    rng = np.random.default_rng(4)
    prefix = rng.integers(0, 256, 3000, dtype=np.uint8).tobytes()
    P = len(prefix)
    cases = [
        ("reach_prefix_start", [FB(rng).seqs([(5, 5 + P, 20)] + short_seqs(rng, 10, reach=5)).frame()]),
        ("straddle_prefix", [FB(rng).seqs([(3, 10, 40)] + short_seqs(rng, 5, reach=3)).frame()]),
        ("repeat_into_prefix", [FB(rng).seqs([(2, 100, 8), (3, 700, 8), (1, 2000, 8), (0, -1, 9), (4, -3, 7), (0, -3, 6), (1, -2, 5)]).frame()]),
        ("frames_each_with_prefix", [FB(rng, checksum=True).seqs([(4, 4 + P, 12), (0, 50, 6)]).frame(),
                                     FB(rng, fcs_width=4).seqs([(0, P, 30), (2, 8, 8)]).frame(),
                                     FB(rng).raw(500).seqs([(0, 500 + P, 16)]).frame()]),
    ]
    b = batch([(n, f, 0, prefix) for n, f in cases], PIN_ENTRIES)
    ref = sum(len(G.segment_starts(f)) for f in b[4])
    for name in PREFIX_CTXS:
        segs = expect(ctxs(name), b, prefix=prefix)
        assert segs == ref, (name, segs, ref)
    # one byte past the prefix start: corruption (-20), the good entries intact
    bad = [FB(rng).seqs([(5, 6 + P, 20)]).frame()]
    blob = G.entry_bytes(bad)
    with pytest.raises(O.ZstdError) as e:
        O.oracle_decompress_ex(blob, 1 << 16, prefix=np.frombuffer(prefix, np.uint8))
    assert e.value.code == 20
    _, sizes = O.ref_decompress_frames(np.frombuffer(blob, np.uint8), [0, len(blob)], [0, 25], prefix=np.frombuffer(prefix, np.uint8))
    assert sizes == [-20]
    b = batch([(n, f, 0, prefix) for n, f in cases] + [("past_prefix", bad, 20, prefix)], PIN_ENTRIES)
    i_bad = b[3].index("past_prefix")
    want = {i: st for i, st in enumerate(serial_status(e, n, True, np.frombuffer(prefix, np.uint8)) for e, n in zip(b[0], b[1])) if st}
    assert want == {i_bad: -20}
    for name in PREFIX_CTXS:
        expect(ctxs(name), b, want, prefix=prefix)


# ------------------------------------------------------------------------------------------------ D: segment starts
def segment_cases(seed: int):
    rng = np.random.default_rng(seed)
    three = lambda: [(2, 3, 5), (2, 6, 5), (2, 9, 5)]   # noqa: E731  (explicit offsets: concrete repeats; first in a block, reads 1 byte back)
    cases = []

    def add(name, frames):
        cases.append((name, frames, 0, b""))
    # back = 0 (the block reads only itself) vs back reaching exactly the previous block's last byte
    add("back0", [FB(rng).raw(300).seqs(three()).seqs([(8, 3, 5)] + three() + short_seqs(rng, 10, reach=8)).frame()])
    add("back_last_byte", [FB(rng).raw(300).seqs(three()).seqs([(0, 1, 9)] + three() + short_seqs(rng, 10, reach=8)).frame()])
    add("back_last_byte_late", [FB(rng).raw(300).seqs(three()).seqs([(6, 3, 5)] + three() + [(0, 6 + 5 + 3 * 7 + 1, 4)]).frame()])
    # repeat codes that resolve into an earlier block; blocks with fewer than three explicit offsets
    add("repeat_into_earlier", [FB(rng).raw(300).seqs(three()).seqs([(4, -1, 6), (0, -1, 5)] + three()).seqs(three()).frame()])
    add("two_explicit", [FB(rng).raw(300).seqs(three()).seqs([(3, 2, 5), (3, 3, 5)]).seqs(three()).frame()])
    # a late block with a symbolic offset suppresses every earlier split of the entry
    add("late_symbolic", [FB(rng).raw(300).seqs(three()).seqs(three()).raw(50).seqs(three()).seqs([(3, -1, 4)]).frame()])
    # frames starting mid-entry reset the repeat offsets to {1, 4, 8}
    add("frame_starts", [FB(rng).raw(100).seqs(three()).frame(), FB(rng).raw(40).seqs([(3, 5, 4), (0, 9, 4)]).frame(),
                         FB(rng).seqs([(20, 4, 6), (1, -1, 5)]).frame(), FB(rng).raw(20).seqs(three()).frame()])
    return cases


@pytest.mark.parametrize("name", ["default", "warp_all", "cta"])
def test_d_segments(ctxs, name):
    cases = segment_cases(5)
    b = batch(cases)
    segs = expect(ctxs(name), b)
    ref = sum(len(G.segment_starts(f)) for f in b[4])
    assert segs == ref, (segs, ref)


def test_d_reference_splits_where_expected():
    """the segment-rule reference itself on the named layouts (so a wrong reference cannot agree with a wrong kernel)"""
    cases = {n: f for n, f, _, _ in segment_cases(5)}
    assert G.segment_starts(cases["back0"]) == [0, 2]
    assert G.segment_starts(cases["back_last_byte"]) == [0]
    assert G.segment_starts(cases["back_last_byte_late"]) == [0]
    assert G.segment_starts(cases["late_symbolic"]) == [0]
    assert G.segment_starts(cases["frame_starts"]) == [0, 2, 4, 5]


# ------------------------------------------------------------------------------------------------ E: sequence stream
def test_e_sequence_stream(ctxs, lib):
    rng = np.random.default_rng(6)
    cases = []

    def add(name, fb):
        cases.append((name, [fb.frame()], 0, b""))
    for n in (1, 31, 32, 33, 127, 128, 129, 255, 256):
        add(f"nseq{n}", FB(rng).raw(128).seqs(short_seqs(rng, n, reach=100)))
    s = short_seqs(rng, 200, reach=100)
    codes = lambda f, xs: sorted({f(x) for x in xs})   # noqa: E731
    ll_c, ml_c = codes(G.ll_code, [x[0] for x in s]), codes(G.ml_code, [x[2] for x in s])
    of_c = codes(G.of_code, [x[1] + 3 for x in s])
    for al in (5, 6, 9):
        t = (("fse", G.norm_for(ll_c, al), al), ("fse", G.norm_for(of_c, min(al, 8)), min(al, 8)), ("fse", G.norm_for(ml_c, al), al))
        add(f"fse_al{al}", FB(rng).raw(128).seqs(s, tables=t).seqs(short_seqs(rng, 50, reach=100), tables=(("predef",),) * 3))
    # every LL code 0..31 at -1 with accuracy log 5, every OF code used at -1 where the table allows
    s32 = [(G.LL_BASE[c], int(rng.integers(1, 100)), 4) for c in range(32)]
    t = (("fse", [-1] * 32, 5), ("predef",), ("rle",))
    add("all_minus1", FB(rng).raw(128).seqs(s32, trailing=3, tables=t))
    # Repeat chains across blocks (through blocks without sequences, which keep the tables)
    t = (("fse", G.norm_for(ll_c, 7), 7), ("fse", G.norm_for(of_c, 6), 6), ("fse", G.norm_for(ml_c, 8), 8))
    fb = FB(rng).raw(128).seqs(s, tables=t).raw(30).seqs(s[:40], tables=(("repeat",),) * 3).lits(20).seqs(s[40:90], tables=(("repeat",),) * 3)
    add("repeat_chain", fb)
    # streams of every length in a range and every start alignment (the filler entries shift the compressed offsets)
    for n in range(40, 72):
        add(f"stream{n}", FB(rng).raw(128).seqs(short_seqs(rng, n, reach=100)))
    b = batch(cases)
    expect(ctxs("default"), b)


def test_e_large_nseq(ctxs):
    """nseq at the two-byte / three-byte header forms (32511 / 32512) and a 128 KiB block of 43 690 three-byte matches"""
    rng = np.random.default_rng(7)
    cases = []
    for n in (32511, 32512):
        cases.append((f"nseq{n}", [FB(rng).raw(16).seqs([(0, int(rng.integers(1, 16)), 3) for _ in range(n)]).frame()], 0, b""))
    cases.append(("nseq43690", [FB(rng).raw(2).seqs([(0, 1 + (i & 1), 3) for i in range(43_690)]).frame()], 0, b""))
    assert cases[-1][1][0].blocks[-1].regen() == (128 << 10) - 2
    b = batch(cases)
    expect(ctxs("default"), b)


# ------------------------------------------------------------------------------------------------ F: Huffman
def _huf_case(rng, weights, n, streams=4, wmode=None):
    syms = [s for s, w in enumerate(weights) if w]
    data = bytes(int(x) for x in rng.choice(syms, n))
    wm = wmode or ("direct" if len(weights) <= 129 else "fse")
    return [Frame([Block("comp", data, lit="huf", weights=weights, streams=streams, wmode=wm)])]


def huffman_cases(seed: int):
    rng = np.random.default_rng(seed)
    cases = []

    def add(name, frames):
        cases.append((name, frames, 0, b""))
    tree = lambda n1, n2, heavy, pad=0: [0] * pad + [1] * n1 + [2] * n2 + heavy   # noqa: E731
    for mb in range(1, 12):           # max_bits 1 .. 11: two weight-1 symbols and one of each weight 2 .. mb
        w = [1, 1] + list(range(2, mb + 1))
        add(f"max_bits{mb}", _huf_case(rng, w, 900))
    add("L504_mb11", _huf_case(rng, tree(2, 251, [4, 10, 11]), 3000))
    add("L504_mb10", _huf_case(rng, tree(2, 251, [10, 3, 3]), 3000))
    add("L508_mb9", _huf_case(rng, tree(2, 253, [3]), 3000))
    add("L256_mb11", _huf_case(rng, tree(2, 127, [9, 10, 11]), 3000))
    add("direct128", _huf_case(rng, [1] * 128 + [8], 2000, wmode="direct"))
    add("fse255", _huf_case(rng, tree(2, 251, [4, 10, 11]), 2000, wmode="fse"))
    add("4stream_regen6", _huf_case(rng, [1, 1, 2], 6))
    add("1stream_1023", _huf_case(rng, [1, 1, 2, 3, 4, 5], 1023, streams=1))
    add("4stream_uneven", _huf_case(rng, [1, 1, 2, 3, 4, 5], 1025))
    # Treeless literals after a tree in the same frame
    w = [1, 1, 2, 3, 4, 5]
    d1, d2 = bytes(int(x) for x in rng.integers(0, 6, 500)), bytes(int(x) for x in rng.integers(0, 6, 700))
    add("treeless_after_tree", [Frame([Block("comp", d1, lit="huf", weights=w, streams=4),
                                       Block("comp", d2, lit="treeless", weights=w, streams=4, seqs=[(5, 3 + 100, 8)])])])
    return cases


def test_f_huffman(ctxs):
    b = batch(huffman_cases(8))
    expect(ctxs("default"), b)


# ------------------------------------------------------------------------------------------------ G: errors at the same boundaries
def error_cases(seed: int):
    """-> (name, frames, libzstd code); each case is first confirmed invalid by libzstd and by the restatement"""
    rng = np.random.default_rng(seed)
    out = []

    def add(name, frames, code, libzstd_accepts=False):
        blob = G.entry_bytes(frames)
        for fn in (O.oracle_decompress,) if libzstd_accepts else (O.ref_decompress_any, O.oracle_decompress):
            with pytest.raises(O.ZstdError) as e:
                fn(blob, 1 << 20)
            assert e.value.code == code, (name, e.value.code)
        if libzstd_accepts:
            assert len(O.ref_decompress_any(blob, 1 << 20)) == sum(b.regen() for f in frames for b in f.blocks)
        out.append((name, frames, code, b""))
    add("offset_one_past", [FB(rng).raw(700).seqs([(4, 705, 6)]).frame()], 20)
    s = short_seqs(rng, 40, reach=64)
    md = 3000 + sum(ll + ml for ll, _, ml in s) + 2
    add("offset_one_past_late", [FB(rng).raw(3000).seqs(s).seqs([(2, md + 1, 4)]).frame()], 20)
    # Repeat_Offset1 - 1 == 0: the restatement and the codec report corruption; libzstd 1.5.5 silently uses offset 1
    # (DESIGN §5, the second known difference: stricter, never laxer)
    add("rep1_minus_1_zero", [FB(rng).raw(50).seqs([(3, 4, 4), (2, 1, 4), (0, -3, 5)]).frame()], 20, libzstd_accepts=True)
    add("huf_spare_bit", [Frame([Block("comp", bytes(int(x) for x in rng.integers(0, 6, 500)), lit="huf", weights=[1, 1, 2, 3, 4, 5],
                                       streams=1, lit_spare_bit=True)])], 20)
    fb = FB(rng).raw(100).seqs(short_seqs(rng, 40, reach=64))
    fb.blocks[-1].nseq_extra = 5
    add("nseq_past_stream", [fb.frame()], 20)
    # Treeless literals whose tree was defined in an earlier zstd frame of the same entry: every frame starts without one
    w = [1, 1, 2, 3, 4, 5]
    d = bytes(int(x) for x in rng.integers(0, 6, 400))
    add("treeless_after_earlier_frame", [Frame([Block("comp", d, lit="huf", weights=w, streams=4)]),
                                         Frame([Block("comp", d, lit="treeless", weights=w, streams=4)])], 30)
    return out


def _max_bits_frame(rng):
    """40 sequences of LL code 35, ML code 52, OF code 31 through FSE tables at the largest accuracy logs where those codes
    have -1 cells (every state update reads the full log): 89 bits a sequence"""
    seqs = [(65_536 + int(rng.integers(1 << 16)), (1 << 31) + int(rng.integers(1 << 31)), 65_539 + int(rng.integers(1 << 16))) for _ in range(40)]
    t = (("fse", G.norm_for([0, 35], 9, neg=[35]), 9), ("fse", G.norm_for([0, 31], 8, neg=[31]), 8), ("fse", G.norm_for([0, 52], 9, neg=[52]), 9))
    blk = Block("comp", b"", seqs=[(ll, ov, ml) for ll, ov, ml in seqs], tables=t)
    return Frame([Block("raw", b"x" * 10), blk])


def test_g_errors(ctxs):
    rng = np.random.default_rng(9)
    errs = error_cases(9)
    # the max-bit stream: literal lengths far past the (empty) literals -> corruption, never a timed-out tile wait (-1)
    mb = _max_bits_frame(rng)
    blob = G.frame_bytes(mb)
    for fn in (O.ref_decompress_any, O.oracle_decompress):
        with pytest.raises(O.ZstdError) as e:
            fn(blob, 1 << 20)
        assert e.value.code == 20
    errs.append(("max_bit_sequences", [mb], 20, b""))
    good = window_cases(2048, 10)[:6] + segment_cases(11)[:3]
    cases = []
    for i, g in enumerate(good):
        cases.append(g)
        if i < len(errs):
            cases.append(errs[i])
    cases += errs[len(good):]
    b = batch(cases)
    code = {e[0]: -e[2] for e in errs}
    want = {i: code[n] for i, n in enumerate(b[3]) if n in code}
    assert len(want) == len(errs)
    assert {i: st for i, st in enumerate(serial_status(e, n) for e, n in zip(b[0], b[1])) if st} == want
    for name in ("default", "warp_all", "cta"):
        expect(ctxs(name), b, want)


# ------------------------------------------------------------------------------------------------ the writer itself
def test_writer_agrees_with_libzstd_and_restatement():
    """random frames over every block type, literals form, table mode (Predefined, RLE, FSE with -1 counts at accuracy
    logs up to the maxima, Repeat) and repeat code: the executor's bytes are what libzstd and the restatement decode"""
    rng = np.random.default_rng(12)
    for i in range(300):
        fr = G.random_frame(rng)
        checked([fr])
    # single-segment frames take the one-byte Frame_Content_Size form
    fr = Frame([Block("raw", b"abc" * 50)], fcs_width=1)
    checked([fr])
