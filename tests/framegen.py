"""Test-only zstd frame writer and plain reference executor, written from RFC 8878.

The writer builds frames whose every choice is explicit: block types, the literals section (Raw, RLE, Huffman from given
per-symbol weights with direct or FSE-compressed weights, 1 or 4 streams, Treeless), and the sequences section as a list of
(literal length, Offset_Value, match length) -- repeat codes are chosen by the caller -- with each of the LL / OF / ML
tables Predefined, RLE, FSE from explicit normalized counts (any accuracy log, -1 allowed) or Repeat.  The executor turns
the same description into the bytes a decoder must produce, with plain Python ints; `segment_starts` restates the rule by
which the decoder splits an entry into independently executable runs of blocks (DESIGN §3.2)."""
from __future__ import annotations

from dataclasses import dataclass, field

# ------------------------------------------------------------------------------------------------ code tables (RFC 3.1.1.3.2.1)
LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
# default distributions (RFC 3.1.1.3.2.2)
PREDEF_LL = ([4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1], 6)
PREDEF_ML = ([1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7, 6)
PREDEF_OF = ([1, 1, 1, 1, 1, 1, 2, 2, 2] + [1] * 15 + [-1] * 5, 5)
MAX_AL = {"ll": 9, "of": 8, "ml": 9}
MAX_SYM = {"ll": 35, "of": 31, "ml": 52}
MAGIC = b"\x28\xb5\x2f\xfd"


def _code(base, v: int) -> int:
    c = 0
    while c + 1 < len(base) and base[c + 1] <= v:
        c += 1
    return c


def ll_code(v: int) -> int: return _code(LL_BASE, v)
def ml_code(v: int) -> int: return _code(ML_BASE, v)
def of_code(ov: int) -> int: return ov.bit_length() - 1


# ------------------------------------------------------------------------------------------------ bitstreams
class BackBits:
    """writer for zstd's backward bitstreams (RFC 8878 4.1): fields in the order they are WRITTEN, then the end mark"""

    def __init__(self):
        self.acc, self.n = 0, 0

    def put(self, value: int, bits: int):
        self.acc |= (value & ((1 << bits) - 1)) << self.n; self.n += bits

    def finish(self) -> bytes:
        self.put(1, 1)
        return self.acc.to_bytes((self.n + 7) // 8, "little")


class FwdBits:
    """little-endian forward bitstream (FSE table descriptions)"""

    def __init__(self):
        self.acc, self.n = 0, 0

    def put(self, value: int, bits: int):
        self.acc |= (value & ((1 << bits) - 1)) << self.n; self.n += bits

    def bytes(self) -> bytes:
        return self.acc.to_bytes((self.n + 7) // 8, "little")


def lit_header(kind: int, regen: int) -> bytes:
    """Literals_Section_Header for Raw (0) / RLE (1) literals"""
    if regen < 32:
        return bytes([(regen << 3) | kind])
    if regen < 4096:
        return ((regen << 4) | (1 << 2) | kind).to_bytes(2, "little")
    return ((regen << 4) | (3 << 2) | kind).to_bytes(3, "little")


def nseq_bytes(n: int) -> bytes:
    if n < 128:
        return bytes([n])
    if n < 0x7F00:
        return bytes([128 + (n >> 8), n & 0xFF])
    return bytes([0xFF, (n - 0x7F00) & 0xFF, (n - 0x7F00) >> 8])


# ------------------------------------------------------------------------------------------------ FSE (RFC 4.1.1)
class Fse:
    """decoding table of normalized counts `norm` at accuracy log `al` (-1 = "less than 1"), and the encoder that picks,
    for a symbol and the state the decoder must reach next, the one cell of the symbol whose range holds that state"""

    def __init__(self, norm, al: int):
        size = 1 << al
        assert sum(1 if p == -1 else p for p in norm) == size, (sum(norm), size)
        self.norm, self.al = list(norm), al
        sym = [None] * size
        high = size - 1
        for s, p in enumerate(norm):
            if p == -1:
                sym[high] = s; high -= 1
        step, pos = (size >> 1) + (size >> 3) + 3, 0
        for s, p in enumerate(norm):
            for _ in range(max(p, 0)):
                sym[pos] = s
                pos = (pos + step) & (size - 1)
                while pos > high:
                    pos = (pos + step) & (size - 1)
        assert pos == 0
        nxt = {s: (1 if p == -1 else p) for s, p in enumerate(norm) if p}
        self.sym, self.nb, self.base = sym, [0] * size, [0] * size
        for u in range(size):
            ns = nxt[sym[u]]; nxt[sym[u]] += 1
            self.nb[u] = al - (ns.bit_length() - 1)
            self.base[u] = (ns << self.nb[u]) - size
        self.cells = {}
        for u in range(size):
            self.cells.setdefault(sym[u], []).append(u)

    def cell_for(self, s: int, target: int) -> int:
        """the cell of symbol s from which the decoder's update reaches state `target`"""
        for u in self.cells[s]:
            if self.base[u] <= target < self.base[u] + (1 << self.nb[u]):
                return u
        raise AssertionError("no cell")

    def header(self) -> bytes:
        """Table description: accuracy log, then the counts with the variable-width code and 2-bit zero-run flags"""
        bw = FwdBits()
        bw.put(self.al - 5, 4)
        size = 1 << self.al
        remaining, threshold, nbits = size + 1, size, self.al + 1
        s, prev0 = 0, False
        norm = self.norm
        while remaining > 1:
            if prev0:
                start = s
                while not norm[s]:
                    s += 1
                while s >= start + 3:
                    bw.put(3, 2); start += 3
                bw.put(s - start, 2)
            count = norm[s]; s += 1
            mx = (2 * threshold - 1) - remaining
            remaining -= abs(count)
            v = count + 1
            if v >= threshold:
                v += mx
            bw.put(v, nbits if v >= mx else nbits - 1)
            prev0 = v == 1
            while remaining < threshold:
                nbits -= 1; threshold >>= 1
        assert remaining == 1
        return bw.bytes()


def norm_for(symbols, al: int, neg=(), heavy=None) -> list:
    """a normalized distribution over `symbols` at accuracy log `al`: every symbol at least one cell (`neg`: -1), the rest
    of the table on `heavy` (default: the first symbol not in neg)"""
    symbols = sorted(set(symbols))
    norm = [0] * (max(symbols) + 1)
    for s in symbols:
        norm[s] = -1 if s in neg else 1
    left = (1 << al) - len(symbols)
    assert left >= 0, "too many symbols for the accuracy log"
    big = [s for s in symbols if s not in neg]
    if left:
        assert big
        norm[heavy if heavy is not None else big[0]] += left
    return norm


def fse_encode_states(tab: Fse, codes):
    """cells c_0 .. c_{n-1} for the decoded codes and the update fields (value, bits) of the transitions c_i -> c_{i+1}"""
    n = len(codes)
    cells = [0] * n
    cells[-1] = tab.cells[codes[-1]][0]
    ups = [None] * n
    for i in range(n - 2, -1, -1):
        cells[i] = tab.cell_for(codes[i], cells[i + 1])
        ups[i] = (cells[i + 1] - tab.base[cells[i]], tab.nb[cells[i]])
    return cells, ups


# ------------------------------------------------------------------------------------------------ Huffman (RFC 4.2)
def huf_codes(weights):
    """weights: per-symbol weight for symbols 0..last (last nonzero; the stream stores all but the last).
    -> (max_bits, {symbol: (code, bits)})"""
    total = sum(1 << (w - 1) for w in weights if w)
    max_bits = total.bit_length() - 1
    assert total == 1 << max_bits and weights[-1], "weights must sum to a power of two, the last symbol weighted"
    codes, cell = {}, 0
    for w in range(1, max_bits + 1):
        for s, ws in enumerate(weights):
            if ws == w:
                nb = max_bits + 1 - w
                codes[s] = (cell >> (w - 1), nb)
                cell += 1 << (w - 1)
    assert cell == total
    return max_bits, codes


def huf_tree(weights, mode: str = "direct", al: int = 6) -> bytes:
    """Huffman_Tree_Description: direct 4-bit weights (at most 128) or FSE-compressed weights (two interleaved states)"""
    ws = list(weights[:-1])
    if mode == "direct":
        assert len(ws) <= 128
        padded = ws + [0] * (len(ws) & 1)
        return bytes([127 + len(ws)]) + bytes((padded[i] << 4) | padded[i + 1] for i in range(0, len(padded), 2))
    assert len(ws) >= 2
    tab = Fse(norm_for(ws, al, heavy=max(set(ws), key=ws.count)), al)
    m = len(ws)
    # decode order: state 1 gives ws[0], state 2 ws[1], state 1 ws[2], ...; the update after ws[m-2] runs out of bits
    cells = [0] * m
    cells[m - 1] = tab.cells[ws[m - 1]][0]
    cands = [u for u in tab.cells[ws[m - 2]] if tab.nb[u] > 0]
    assert cands, "the second-to-last weight needs a cell that reads bits"
    cells[m - 2] = cands[0]
    ups = [None] * m
    for k in range(m - 3, -1, -1):
        cells[k] = tab.cell_for(ws[k], cells[k + 2])
        ups[k] = (cells[k + 2] - tab.base[cells[k]], tab.nb[cells[k]])
    bw = BackBits()
    for k in range(m - 3, -1, -1):
        bw.put(*ups[k])
    bw.put(cells[1], al); bw.put(cells[0], al)
    body = tab.header() + bw.finish()
    assert len(body) < 128
    return bytes([len(body)]) + body


def huf_stream(data: bytes, codes, spare_bit: bool = False) -> bytes:
    bw = BackBits()
    if spare_bit:
        bw.put(0, 1)                              # read after the last symbol: the stream is not consumed exactly
    for b in reversed(data):
        bw.put(*codes[b])
    return bw.finish()


def huf_literals(data: bytes, weights, streams: int = 1, wmode: str = "direct", treeless: bool = False, spare_bit: bool = False,
                 split=None) -> bytes:
    """a Compressed (or Treeless) literals section.  split: the four stream sizes in bytes of output (default: RFC's equal split)"""
    _, codes = huf_codes(weights)
    tree = b"" if treeless else huf_tree(weights, wmode)
    if streams == 1:
        payload = tree + huf_stream(data, codes, spare_bit)
    else:
        seg = (len(data) + 3) // 4
        parts = [data[0:seg], data[seg:2 * seg], data[2 * seg:3 * seg], data[3 * seg:]]
        ss = [huf_stream(p, codes, spare_bit and i == 3) for i, p in enumerate(parts)]
        payload = tree + b"".join(len(s).to_bytes(2, "little") for s in ss[:3]) + b"".join(ss)
    regen, comp = len(data), len(payload)
    kind = 3 if treeless else 2
    if streams == 1:
        assert regen < 1024 and comp < 1024
        hdr = (kind | (0 << 2) | (regen << 4) | (comp << 14)).to_bytes(3, "little")
    elif regen < 1024 and comp < 1024:
        hdr = (kind | (1 << 2) | (regen << 4) | (comp << 14)).to_bytes(3, "little")
    elif regen < 16384 and comp < 16384:
        hdr = (kind | (2 << 2) | (regen << 4) | (comp << 18)).to_bytes(4, "little")
    else:
        hdr = (kind | (3 << 2) | (regen << 4) | (comp << 22)).to_bytes(5, "little")
    return hdr + payload


# ------------------------------------------------------------------------------------------------ frame description
@dataclass
class Block:
    """kind 'raw' / 'rle' (data = content; rle: one byte repeated n times) / 'comp' (data = literals, seqs = (ll, Offset_Value, ml)).
    lit: 'raw' | 'rle' | 'huf' | 'treeless'; tables: LL, OF, ML specs, each ('predef',) | ('rle',) | ('fse', norm, al) | ('repeat',)
    (('rle',) takes the one code the block uses).  'huf': weights (symbols 0..last), streams 1 / 4, wmode 'direct' / 'fse'."""
    kind: str
    data: bytes = b""
    n: int = 0
    seqs: list = field(default_factory=list)
    lit: str = "raw"
    weights: list | None = None
    streams: int = 1
    wmode: str = "direct"
    tables: tuple = (("predef",), ("predef",), ("predef",))
    lit_spare_bit: bool = False
    nseq_extra: int = 0                 # the header claims this many sequences more than the stream holds

    def regen(self) -> int:
        if self.kind == "raw":
            return len(self.data)
        if self.kind == "rle":
            return self.n
        return len(self.data) + sum(s[2] for s in self.seqs)


@dataclass
class Frame:
    blocks: list
    checksum: bool = False
    fcs_width: int | None = None      # None: no Frame_Content_Size; 1 (Single_Segment) / 2 / 4 / 8
    window_log: int = 22


def _seq_section(blk: Block, prev: dict) -> bytes:
    seqs = blk.seqs
    n = len(seqs)
    out = bytearray(nseq_bytes(n + blk.nseq_extra))
    if n == 0:
        return bytes(out)
    codes = {"ll": [ll_code(s[0]) for s in seqs], "of": [of_code(s[1]) for s in seqs], "ml": [ml_code(s[2]) for s in seqs]}
    modes, tabs, descs = 0, {}, b""
    for shift, key, spec in ((6, "ll", blk.tables[0]), (4, "of", blk.tables[1]), (2, "ml", blk.tables[2])):
        kind = spec[0]
        if kind == "predef":
            m, t = 0, Fse(*{"ll": PREDEF_LL, "of": PREDEF_OF, "ml": PREDEF_ML}[key])
        elif kind == "rle":
            assert len(set(codes[key])) == 1
            m, t = 1, ("rle", codes[key][0])
            descs += bytes([codes[key][0]])
        elif kind == "fse":
            m, t = 2, Fse(spec[1], spec[2])
            descs += t.header()
        else:
            m, t = 3, prev[key]
        modes |= m << shift
        tabs[key] = t
        prev[key] = t
    out += bytes([modes]) + descs
    states = {}
    for key in ("ll", "of", "ml"):
        t = tabs[key]
        if isinstance(t, Fse):
            states[key] = fse_encode_states(t, codes[key])
    bw = BackBits()
    for i in range(n - 1, -1, -1):
        ll, ov, ml = seqs[i]
        if i < n - 1:
            for key in ("of", "ml", "ll"):
                if key in states:
                    bw.put(*states[key][1][i])
        lc, mc, oc = codes["ll"][i], codes["ml"][i], codes["of"][i]
        bw.put(ll - LL_BASE[lc], LL_BITS[lc]); bw.put(ml - ML_BASE[mc], ML_BITS[mc]); bw.put(ov - (1 << oc), oc)
    for key in ("ml", "of", "ll"):
        if key in states:
            bw.put(states[key][0][0], tabs[key].al)
    return bytes(out) + bw.finish()


def _literals(blk: Block) -> bytes:
    d = blk.data
    if blk.lit == "raw":
        return lit_header(0, len(d)) + d
    if blk.lit == "rle":
        assert len(set(d)) <= 1
        return lit_header(1, len(d)) + (d[:1] or b"\0")
    return huf_literals(d, blk.weights, blk.streams, blk.wmode, blk.lit == "treeless", blk.lit_spare_bit)


def block_body(blk: Block, prev: dict) -> tuple[int, bytes, int]:
    """-> (block type, content, Block_Size field)"""
    if blk.kind == "raw":
        return 0, blk.data, len(blk.data)
    if blk.kind == "rle":
        return 1, blk.data[:1], blk.n
    body = _literals(blk) + _seq_section(blk, prev)
    return 2, body, len(body)


def frame_bytes(fr: Frame, prefix: bytes = b"") -> bytes:
    """the frame as bytes (Frame_Content_Size and the checksum from the executor's output of it)"""
    content = execute([fr], prefix) if (fr.checksum or fr.fcs_width is not None) else b""
    out = bytearray(MAGIC)
    single = fr.fcs_width == 1
    flag = {None: 0, 1: 0, 2: 1, 4: 2, 8: 3}[fr.fcs_width]
    out.append((flag << 6) | (int(single) << 5) | (int(fr.checksum) << 2))
    if not single:
        out.append((fr.window_log - 10) << 3)
    if fr.fcs_width is not None:
        v = len(content) - (256 if fr.fcs_width == 2 else 0)
        out += v.to_bytes(fr.fcs_width, "little")
    prev = {}
    for i, blk in enumerate(fr.blocks):
        btype, body, size = block_body(blk, prev)
        out += ((size << 3) | (btype << 1) | int(i == len(fr.blocks) - 1)).to_bytes(3, "little") + body
    if fr.checksum:
        from oracle import oracle as O
        out += (O.oracle_xxh64(content) & 0xFFFFFFFF).to_bytes(4, "little")
    return bytes(out)


def entry_bytes(frames, prefix: bytes = b"") -> bytes:
    """one seek-table entry: the frames back to back, each with its own header, Frame_Content_Size and checksum"""
    return b"".join(frame_bytes(f, prefix) for f in frames)


# ------------------------------------------------------------------------------------------------ reference executor
def resolve(reps: list, ll: int, ov: int) -> int:
    """Offset_Value -> offset, updating the repeat-offset history in place (RFC 3.1.1.5)"""
    if ov > 3:
        off = ov - 3
        reps[:] = [off, reps[0], reps[1]]
        return off
    idx = ov - 1 + (ll == 0)
    if idx == 0:
        return reps[0]
    off = reps[0] - 1 if idx == 3 else reps[idx]
    if idx == 1:
        reps[:] = [off, reps[0], reps[2]]
    else:
        reps[:] = [off, reps[0], reps[1]]
    return off


class ExecError(Exception):
    pass


def execute(frames, prefix: bytes = b"") -> bytes:
    """the bytes a decoder must produce for these frames (one entry), each frame seeing `prefix` before its first byte"""
    out = bytearray()
    for fr in frames:
        zs = len(out)
        reps = [1, 4, 8]
        for blk in fr.blocks:
            if blk.kind == "raw":
                out += blk.data; continue
            if blk.kind == "rle":
                out += blk.data[:1] * blk.n; continue
            lit, lp = blk.data, 0
            for ll, ov, ml in blk.seqs:
                out += lit[lp:lp + ll]; lp += ll
                if lp > len(lit):
                    raise ExecError("literals overrun")
                off = resolve(reps, ll, ov)
                avail = len(out) - zs + len(prefix)
                if off <= 0 or off > avail:
                    raise ExecError(f"offset {off} reaches before the frame (and prefix): {avail} bytes available")
                for _ in range(ml):
                    p = len(out) - off
                    out.append(out[p] if p >= zs else prefix[len(prefix) + (p - zs)])
            out += lit[lp:]
    return bytes(out)


# ------------------------------------------------------------------------------------------------ segment rule (DESIGN §3.2)
def block_facts(frames):
    """per block of the entry: (output position, starts a zstd frame, back or None (unknown), outgoing repeat offsets concrete).
    The repeat history entering every block is symbolic (slot k, delta d) -- blocks are entropy-decoded independently --
    and explicit offsets only shift it, as in the sequence kernel.  back is measured from the block's first byte, so a read
    into the prefix (prefix mode) counts as a read before the block."""
    facts, pos = [], 0
    for fr in frames:
        for bi, blk in enumerate(fr.blocks):
            if blk.kind != "comp" or not blk.seqs:
                facts.append((pos, bi == 0, 0, False)); pos += blk.regen(); continue
            reps = [("s", 0, 0), ("s", 1, 0), ("s", 2, 0)]
            back, op, sym = 0, 0, False
            for ll, ov, ml in blk.seqs:
                op += ll
                if ov > 3:
                    off = ("c", ov - 3)
                    reps = [off, reps[0], reps[1]]
                else:
                    idx = ov - 1 + (ll == 0)
                    if idx == 0:
                        off = reps[0]
                    else:
                        off = ((reps[0][0], reps[0][1], reps[0][2] + 1) if reps[0][0] == "s" else ("c", reps[0][1] - 1)) if idx == 3 else reps[idx]
                        reps = [off, reps[0], reps[2]] if idx == 1 else [off, reps[0], reps[1]]
                if off[0] == "s":
                    sym = True
                else:
                    back = max(back, off[1] - op)
                op += ml
            conc = all(r[0] == "c" for r in reps)
            facts.append((pos, bi == 0, None if sym else back, conc))
            pos += blk.regen()
    return facts


def segment_starts(frames) -> list:
    """indices of the blocks that start a segment: the entry's first block, or a block b such that every block from b on
    reads nothing before b's first byte, and b starts a zstd frame or leaves concrete repeat offsets"""
    facts = block_facts(frames)
    starts, low = [], None
    for b in range(len(facts) - 1, -1, -1):
        op, first, back, conc = facts[b]
        lo = float("-inf") if back is None else op - back
        low = lo if low is None else min(low, lo)
        if b == 0 or (low >= op and (first or conc)):
            starts.append(b)
    return sorted(starts)


# ------------------------------------------------------------------------------------------------ random frames (self-test)
def random_frame(rng) -> Frame:
    """a frame of 1-4 random blocks exercising every block type, literals form, table mode and repeat code, valid by construction"""
    blocks, out_len, reps, prev_codes = [], 0, [1, 4, 8], None
    huf_w = None
    for bi in range(int(rng.integers(1, 5))):
        kind = ["raw", "rle", "comp", "comp", "comp"][int(rng.integers(5))]
        if kind == "raw":
            n = int(rng.integers(0, 300)); blocks.append(Block("raw", rng.integers(0, 256, n, dtype="u1").tobytes())); out_len += n; continue
        if kind == "rle":
            n = int(rng.integers(1, 300)); blocks.append(Block("rle", bytes([int(rng.integers(256))]), n=n)); out_len += n; continue
        seqs, lits, pos = [], 0, out_len
        for _ in range(int(rng.integers(0, 3) and rng.integers(1, 150))):
            ll = int(rng.choice([0, 0, 1, 2, 5, 17, 40, 70]))
            pos += ll; lits += ll
            ml = int(rng.choice([3, 4, 7, 20, 35, 60, 140, 600]))
            ov = None
            if rng.random() < 0.4:
                ov = int(rng.integers(1, 4))
                trial = list(reps)
                off = resolve(trial, ll, ov)
                if not 0 < off <= pos:
                    ov = None
            if ov is None:
                if pos == 0:
                    pos -= ll; lits -= ll; continue
                ov = int(rng.integers(1, min(pos, 2000) + 1)) + 3
            resolve(reps, ll, ov)
            seqs.append((ll, ov, ml)); pos += ml
        trailing = int(rng.integers(0, 40))
        n_lit = lits + trailing
        lit_kind = ["raw", "rle", "huf", "huf"][int(rng.integers(4))] if n_lit else "raw"
        alphabet = [int(x) for x in rng.choice(256, 6, replace=False)]
        if lit_kind == "huf":
            if huf_w is not None and rng.random() < 0.5:
                lit_kind = "treeless"
            else:
                w = [0] * (max(alphabet) + 1)
                for s, wt in zip(sorted(alphabet), [1, 1, 2, 3, 4, 5]):
                    w[s] = wt
                huf_w = w
        if lit_kind == "rle":
            data = bytes([alphabet[0]]) * n_lit
        elif lit_kind in ("huf", "treeless"):
            syms = [s for s, x in enumerate(huf_w) if x]
            data = bytes(int(x) for x in rng.choice(syms, n_lit))
        else:
            data = rng.integers(0, 256, n_lit, dtype="u1").tobytes()
        streams = 1 if n_lit < 6 or (n_lit < 1000 and rng.random() < 0.5) else 4
        if lit_kind in ("huf", "treeless") and n_lit == 0:
            lit_kind = "raw"
        tables = []
        codes = ({ll_code(s[0]) for s in seqs}, {of_code(s[1]) for s in seqs}, {ml_code(s[2]) for s in seqs})
        for k, (key, cs) in enumerate(zip(("ll", "of", "ml"), codes)):
            m = int(rng.integers(4))
            if not seqs or m == 0:
                tables.append(("predef",) if max(cs | {0}) <= (35, 28, 52)[k] else ("fse", norm_for(cs, 8), 8))
            elif m == 1 and len(cs) == 1:
                tables.append(("rle",))
            elif m == 3 and prev_codes is not None and prev_codes[k][0] == "fse" and cs <= prev_codes[k][1]:
                tables.append(("repeat",))
            else:
                al = int(rng.integers(max(5, (len(cs) + 2).bit_length()), MAX_AL[key] + 1))
                neg = {c for c in cs if rng.random() < 0.3} - {min(cs)}
                tables.append(("fse", norm_for(cs, al, neg), al))
        if seqs:
            prev_codes = [(t[0] if t[0] != "repeat" else prev_codes[k][0], {c for c, p in enumerate(t[1]) if p} if t[0] == "fse" else
                           (prev_codes[k][1] if t[0] == "repeat" else set())) for k, t in enumerate(tables)]
        blocks.append(Block("comp", data, seqs=seqs, lit=lit_kind, weights=huf_w, streams=streams,
                            wmode="fse" if huf_w is None or len(huf_w) > 129 or rng.random() < 0.5 else "direct", tables=tuple(tables)))
        out_len += blocks[-1].regen()
    fcs = [None, None, 2, 4, 8][int(rng.integers(5))]
    return Frame(blocks, checksum=bool(rng.random() < 0.5), fcs_width=4 if fcs == 2 and out_len < 256 else fcs)
