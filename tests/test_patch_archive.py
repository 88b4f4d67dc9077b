"""Seekable patches against a seekable archive (zk_patch_ranges_archive, zk_compress_frames_patch_archive,
zk_decompress_frames_prefixes_archive, the Decoder's reference-archive read): the reference R is an archive and OLD its decoded content,
decoded on the GPU entry by entry.  Every call equals its raw-reference call on OLD, for every layout of R (this codec's uniform, sized,
content-defined and Compressed(n) archives, libzstd's, entries of several frames with a skippable frame, empty entries); a one-frame read
decodes exactly the entries of R under its slice; a corrupt entry of R fails only the patch entries that reach it; argument errors and
the CLI's refusals.  Emulation cases run on the emulation build (`-m "not gpu"`, small inputs); the headline case runs on the H100."""
import io

import numpy as np
import pytest

import cases
import zeekstd_b200 as zk
from oracle import oracle as O
from test_patch_ldm import _mix, edited_copy
from util import offsets
from zeekstd_b200 import _native

INVALID = -1006


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    return request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib")


@pytest.fixture(scope="module")
def ctx(lib):
    _native.set_default_lib(lib)
    c = zk.Context(0, lib)
    yield c
    c.close()


def _uniform(n: int, fs: int) -> list:
    return [min(fs, n - a) for a in range(0, n, fs)] or [0]


OLD = _mix(256 << 10, 1)
NEW = edited_copy(OLD, 2, 12)
SIZES = _uniform(NEW.size, 64 << 10)
MARGIN = 8 << 10


def _with_table(comp, cs, ds) -> bytes:
    """frames + their Foot seek table"""
    table = zk.SeekTable()
    for c, d in zip(np.asarray(cs).tolist(), np.asarray(ds).tolist()):
        table.log_frame(int(c), int(d))
    return bytes(np.asarray(comp, dtype=np.uint8).tobytes()) + table.into_serializer().to_bytes()


def _multi(old) -> zk.ReferenceArchive:
    """entries of three libzstd frames each, every one after a skippable frame, described by explicit offsets"""
    frames, cs, ds = O.ref_compress_frames(old, 8 << 10, 3, True)
    body, co, do = b"", [0], [0]
    for i in range(0, len(frames), 3):
        part = O.skippable_frame(b"entry %d" % i, i % 16) + b"".join(frames[i:i + 3])
        body += part
        co.append(len(body)); do.append(do[-1] + sum(ds[i:i + 3]))
    return zk.ReferenceArchive(np.frombuffer(body + b"\0" * 64, dtype=np.uint8), c_off=co, d_off=do)


def reference(ctx, kind: str, old=OLD) -> zk.ReferenceArchive:
    """R of `kind` whose decoded content is old"""
    if kind == "uniform":
        return zk.ReferenceArchive(_with_table(*ctx.compress_frames(old, 24 << 10, 3, True)))
    if kind == "sized":
        rng = np.random.default_rng(5)
        sizes, left = [], old.size
        while left:
            s = min(left, int(rng.integers(1, 48 << 10)))
            sizes.append(s); left -= s
        return zk.ReferenceArchive(_with_table(*ctx.compress_frames_sized(old, sizes, 1, False)))
    if kind == "empty":                                    # empty entries at the start, in the middle and at the end
        sizes = [0, 40 << 10, 0, 0, old.size - (120 << 10), 0, 80 << 10, 0]
        return zk.ReferenceArchive(_with_table(*ctx.compress_frames_sized(old, sizes, 3, True)))
    if kind == "content":
        comp, cs, ds, _ = ctx.compress_frames_cdc(old, 16 << 10, 3, True)
        return zk.ReferenceArchive(_with_table(comp, cs, ds))
    if kind == "csize":
        comp, cs, ds, _ = ctx.compress_frames_csize(old, 8 << 10, 3, False)
        return zk.ReferenceArchive(_with_table(comp, cs, ds))
    if kind == "libzstd":
        return zk.ReferenceArchive(O.ref_seekable_archive(old, 20 << 10, 3, True)[0])
    if kind == "multi":
        return _multi(old)
    raise KeyError(kind)


KINDS = ["uniform", "sized", "empty", "content", "csize", "libzstd", "multi"]


@pytest.fixture(scope="module")
def refs(ctx):
    return {k: reference(ctx, k) for k in KINDS}


@pytest.fixture(scope="module")
def raw(ctx):
    """the raw-reference results everything is compared with: ranges, the frames with and without checksums, the patch"""
    rg = ctx.patch_ranges(NEW, SIZES, OLD, MARGIN)
    frames = {ck: ctx.compress_frames_patch(NEW, SIZES, OLD, rg, 3, ck) for ck in (False, True)}
    return rg, frames, ctx.compress_patch_slices(NEW, SIZES, OLD, 3, True, MARGIN)


def test_reference_layouts(refs):
    """every layout decodes to OLD's length and has several entries; the ones meant to have them have empty entries"""
    for k, r in refs.items():
        assert r.old_len == OLD.size and r.n_entries >= 3, k
    assert (np.diff(refs["empty"].d_off) == 0).sum() == 5


@pytest.mark.parametrize("kind", KINDS)
def test_same_ranges(ctx, refs, raw, kind, monkeypatch):
    """contract 1: the ranges of the raw call, with the default run size and with 4 KiB runs (split inside entries and at their edges)"""
    assert ctx.patch_ranges(NEW, SIZES, refs[kind], MARGIN).tolist() == raw[0].tolist()
    monkeypatch.setenv("ZK_PATCH_PIECE_BYTES", "4096")
    assert ctx.patch_ranges(NEW, SIZES, refs[kind], MARGIN).tolist() == raw[0].tolist()


@pytest.mark.parametrize("kind", ["uniform", "empty", "libzstd", "multi"])
@pytest.mark.parametrize("ck", [False, True])
def test_same_archive(ctx, refs, raw, kind, ck, monkeypatch):
    """contract 2: the bytes and c_sizes of the raw call, with the default groups and with 64 KiB groups"""
    rg, frames, _ = raw
    want, wcs, _ = frames[ck]
    for group in (None, 64 << 10):
        if group:
            monkeypatch.setenv("ZK_PATCH_GROUP_BYTES", str(group))
        comp, cs, _ = ctx.compress_frames_patch(NEW, SIZES, refs[kind], rg, 3, ck)
        assert comp.tobytes() == want.tobytes() and cs.tolist() == wcs.tolist(), group


def test_same_patch(ctx, refs, raw):
    """compress_patch_slices against the archive writes the raw call's patch"""
    assert ctx.compress_patch_slices(NEW, SIZES, refs["content"], 3, True, MARGIN) == raw[2]


def _split(archive: bytes):
    table = zk.SeekTable.from_bytes(archive, zk.Format.Foot)
    co, do = table.offsets()
    old_len, rg, _ = zk.patch_slices_read(archive, table.num_frames())
    return co, do, old_len, rg


@pytest.mark.parametrize("kind", ["uniform", "sized", "csize", "multi"])
@pytest.mark.parametrize("verify", [False, True])
def test_same_restore(ctx, refs, raw, kind, verify, monkeypatch):
    """contract 3: output, statuses and return code of the raw-reference decode, in full and with need, with small groups too"""
    archive = raw[2]
    co, do, _, rg = _split(archive)
    pad = np.frombuffer(archive + b"\0" * 64, dtype=np.uint8)
    need = np.array([int(do[f + 1] - do[f]) // (f + 2) for f in range(len(SIZES))], dtype=np.uint32)
    for group in (None, 48 << 10):
        if group:
            monkeypatch.setenv("ZK_PATCH_GROUP_BYTES", str(group))
        for nd in (None, need):
            want, wst, wrc = ctx.decompress_frames(pad, co, do, verify, need=nd, prefix=OLD, prefix_ranges=rg)
            got, st, rc = ctx.decompress_frames(pad, co, do, verify, need=nd, prefix=refs[kind], prefix_ranges=rg)
            assert rc == wrc == 0 and st.tolist() == wst.tolist()
            if nd is None:
                assert got.tobytes() == want.tobytes() == NEW.tobytes()
            else:
                for f in range(len(SIZES)):
                    a = int(do[f])
                    assert got[a:a + int(nd[f])].tobytes() == NEW[a:a + int(nd[f])].tobytes(), f


def test_restore_crosses_over(ctx, refs, raw):
    """a patch made against v1.zst restores with raw v1, and one made against raw v1 restores with v1.zst (both are the same bytes)"""
    arch = ctx.compress_patch_slices(NEW, SIZES, refs["libzstd"], 3, True, MARGIN)
    assert arch == raw[2]
    co, do, _, rg = _split(arch)
    pad = np.frombuffer(arch + b"\0" * 64, dtype=np.uint8)
    for prefix in (OLD, refs["uniform"]):
        back, st, rc = ctx.decompress_frames(pad, co, do, True, prefix=prefix, prefix_ranges=rg)
        assert rc == 0 and back.tobytes() == NEW.tobytes()


def test_whole_reference_without_ranges(ctx, refs):
    """no ranges: every entry against all of OLD, as the raw call with the whole prefix"""
    tail = OLD[-(96 << 10):]
    comp, cs, ds = ctx.compress_frames(NEW[:64 << 10], 16 << 10, 3, True, prefix=tail)
    ref = zk.ReferenceArchive(_with_table(*ctx.compress_frames(tail, 40 << 10, 3, True)))
    pad = np.concatenate([comp, np.zeros(64, dtype=np.uint8)])
    got, st, rc = ctx.decompress_frames(pad, offsets(cs), offsets(ds), True, prefix=ref)
    assert rc == 0 and got.tobytes() == NEW[:64 << 10].tobytes()


def test_one_frame_decodes_its_entries(ctx, refs, raw):
    """contract 4: a one-frame read decodes exactly the entries of R whose output overlaps its slice, and uploads no prefix byte"""
    archive = raw[2]
    co, do, _, rg = _split(archive)
    for kind in ("uniform", "empty", "multi"):
        r = refs[kind]
        for f in (0, len(SIZES) // 2, len(SIZES) - 1):
            lo, hi = (int(v) for v in rg[f])
            want = sum(1 for g in range(r.n_entries) if r.d_off[g] < hi and r.d_off[g + 1] > lo and r.d_off[g + 1] > r.d_off[g])
            before, up = ctx.reference_entries_decoded, ctx.prefix_bytes_uploaded
            dec = zk.DecodeOptions(zk.BytesWrapper(archive), ctx).lower_frame(f).upper_frame(f).into_decoder()
            buf = bytearray(SIZES[f] + 1)
            k = dec.decompress_with_prefix(buf, r, rg)
            assert bytes(buf[:k]) == NEW[int(do[f]):int(do[f + 1])].tobytes()
            assert ctx.reference_entries_decoded - before == want and 0 < want < r.n_entries, (kind, f)
            assert ctx.prefix_bytes_uploaded == up


def _bytes(r: zk.ReferenceArchive) -> bytes:
    """the archive bytes R was built from"""
    return np.asarray(r._keep[0] if isinstance(r._keep, tuple) else r._keep).tobytes()


def _corrupt(r: zk.ReferenceArchive, g: int, how: str) -> zk.ReferenceArchive:
    """R with entry g damaged: a byte flipped in its first compressed block, or its checksum changed"""
    b = bytearray(_bytes(r))
    c0, c1 = int(r.c_off[g]), int(r.c_off[g + 1])
    if how == "block":
        b[c0 + 20] ^= 0x5A
    else:
        b[c1 - 1] ^= 0xFF
    return zk.ReferenceArchive(bytes(b), c_off=r.c_off, d_off=r.d_off)


@pytest.mark.parametrize("how", ["block", "checksum"])
def test_corrupt_reference_entry(ctx, refs, raw, how):
    """contract 5: the patch entries whose ranges overlap the damaged entry fail with its code, the others restore exactly; the compress
    and range calls return an error"""
    r = refs["uniform"]
    g = r.n_entries // 2
    bad = _corrupt(r, g, how)
    code = ctx.decompress_frames(np.frombuffer(_bytes(bad) + b"\0" * 64, dtype=np.uint8), bad.c_off, bad.d_off, True)[1][g]
    assert code < 0
    archive = raw[2]
    co, do, _, rg = _split(archive)
    pad = np.frombuffer(archive + b"\0" * 64, dtype=np.uint8)
    got, st, rc = ctx.decompress_frames(pad, co, do, True, prefix=bad, prefix_ranges=rg)
    e0, e1 = int(r.d_off[g]), int(r.d_off[g + 1])
    hit = [int(lo) < e1 and int(hi) > e0 for lo, hi in rg.tolist()]
    assert any(hit) and not all(hit)
    assert st.tolist() == [code if h else 0 for h in hit] and rc == code
    for f, h in enumerate(hit):
        if not h:
            assert got[int(do[f]):int(do[f + 1])].tobytes() == NEW[int(do[f]):int(do[f + 1])].tobytes(), f
    if how == "checksum":                                   # without verification a bad checksum is not seen
        got, st, rc = ctx.decompress_frames(pad, co, do, False, prefix=bad, prefix_ranges=rg)
        assert rc == 0 and got.tobytes() == NEW.tobytes()
    with pytest.raises(zk.Error) as e:
        ctx.patch_ranges(NEW, SIZES, bad, MARGIN)
    assert e.value.rc == code
    with pytest.raises(zk.Error) as e:
        ctx.compress_frames_patch(NEW, SIZES, bad, rg, 3, False)
    assert e.value.rc == code


def test_argument_errors(ctx, refs, raw):
    """contract 6: decreasing offsets, offsets past R's bytes, a range past OLD, a seekable patch as R"""
    lib = ctx.lib
    r = refs["uniform"]
    rg = raw[0]
    data = _bytes(r)
    co, do = r.c_off.copy(), r.d_off.copy()

    def calls(ref):
        yield lambda: ctx.patch_ranges(NEW, SIZES, ref, MARGIN)
        yield lambda: ctx.compress_frames_patch(NEW, SIZES, ref, rg, 3, False)

    dco = co.copy(); dco[2] = dco[1] - 1
    ddo = do.copy(); ddo[2] = ddo[1] - 1
    long_co = co.copy(); long_co[-1] = len(data) + 1
    for c_off, d_off in ((dco, do), (co, ddo), (long_co, do)):
        bad = zk.ReferenceArchive(data, c_off=c_off, d_off=d_off)
        for call in calls(bad):
            with pytest.raises(zk.Error) as e:
                call()
            assert e.value.rc == INVALID
    past = rg.copy(); past[1][1] = OLD.size + 1
    with pytest.raises(zk.Error) as e:
        ctx.compress_frames_patch(NEW, SIZES, r, past, 3, False)
    assert e.value.rc == INVALID
    archive = raw[2]
    cco, cdo, _, _ = _split(archive)
    pad = np.frombuffer(archive + b"\0" * 64, dtype=np.uint8)
    assert ctx.decompress_frames(pad, cco, cdo, True, prefix=r, prefix_ranges=past)[2] == INVALID
    # a seekable patch is refused by ReferenceArchive, and by the C calls when described by explicit offsets
    with pytest.raises(ValueError, match="is a seekable patch; restore it first"):
        zk.ReferenceArchive(archive)
    pco, pdo = zk.SeekTable.from_bytes(archive).offsets()
    a = np.frombuffer(archive, dtype=np.uint8)
    rc = lib.zk_patch_ranges_archive(ctx._h, NEW.ctypes.data, np.asarray(SIZES, dtype=np.uint32).ctypes.data_as(_native.u32p), len(SIZES),
                                     a.ctypes.data, a.size, pco.ctypes.data_as(_native.u64p), pdo.ctypes.data_as(_native.u64p), len(pco) - 1,
                                     MARGIN, np.zeros(2 * len(SIZES), dtype=np.uint64).ctypes.data_as(_native.u64p))
    assert rc == INVALID


def test_head_table_and_mapping(ctx, refs, tmp_path):
    """ReferenceArchive from a stand-alone Head seek table, and from a mapping of the file"""
    r = refs["uniform"]
    table = zk.SeekTable.from_bytes(_bytes(r))
    head = table.into_format_serializer(zk.Format.Head).to_bytes()
    hr = zk.ReferenceArchive(_bytes(r), seek_table=head, format=zk.Format.Head)
    assert hr.c_off.tolist() == r.c_off.tolist() and hr.d_off.tolist() == r.d_off.tolist()
    p = tmp_path / "v1.zst"; p.write_bytes(_bytes(r))
    mr = zk.ReferenceArchive(np.memmap(p, dtype=np.uint8, mode="r"))
    assert ctx.patch_ranges(NEW, SIZES, mr, MARGIN).tolist() == ctx.patch_ranges(NEW, SIZES, hr, MARGIN).tolist()


def test_decoder_random_ops(ctx, refs, raw):
    """the Decoder reading the patch against R, against the same Decoder with raw OLD: random offsets, limits, seeks and reads"""
    archive = raw[2]
    _, _, _, rg = _split(archive)
    r = refs["sized"]
    rng = np.random.default_rng(11)
    a = zk.DecodeOptions(zk.BytesWrapper(archive), ctx).into_decoder()
    b = zk.DecodeOptions(zk.BytesWrapper(archive), ctx).into_decoder()
    total = NEW.size
    for _ in range(40):
        k = int(rng.integers(6))
        if k <= 2:
            ln = int(rng.choice([1, 999, 24 << 10, 64 << 10, total]))
            ba, bb = bytearray(ln), bytearray(ln)
            na, nb = a.decompress_with_prefix(ba, r, rg), b.decompress_with_prefix(bb, OLD, rg)
            assert na == nb and ba[:na] == bb[:nb]
        elif k == 3:
            o = int(rng.integers(0, total + 1))
            a.set_offset(o); b.set_offset(o)
        elif k == 4:
            o = int(rng.integers(0, total + 1))
            a.set_offset_limit(o); b.set_offset_limit(o)
        else:
            o = int(rng.integers(-total, 1))
            assert a.seek(o, io.SEEK_END) == b.seek(o, io.SEEK_END)
        assert a.offset() == b.offset()


def test_cli(ctx, refs, tmp_path):
    v1, v2 = tmp_path / "v1", tmp_path / "v2"
    v1.write_bytes(OLD.tobytes()); v2.write_bytes(NEW.tobytes())
    z1 = tmp_path / "v1.zst"
    rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", "-s", "24K", "-o", z1, v1])
    assert rc == 0, err
    raw_p, arc_p, back = tmp_path / "raw.zst", tmp_path / "arc.zst", tmp_path / "back"
    base = ["compress", "-q", "-f", "-s", "64K", "--patch-slices", "--patch-margin", "8K"]
    rc, _, err = cases._cli(ctx, base + ["--patch-from", v1, "-o", raw_p, v2])
    assert rc == 0, err
    rc, _, err = cases._cli(ctx, base + ["--patch-from", z1, "--patch-archive", "-o", arc_p, v2])
    assert rc == 0, err
    assert arc_p.read_bytes() == raw_p.read_bytes()
    for ref, extra in ((z1, ["--patch-archive"]), (v1, [])):
        rc, _, err = cases._cli(ctx, ["decompress", "-q", "-f", "--patch-apply", ref, *extra, "-o", back, raw_p])
        assert rc == 0 and back.read_bytes() == NEW.tobytes(), err
    # a range read decodes only the entries of v1.zst under the slices it reads
    before = ctx.reference_entries_decoded
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "-f", "--from", "70000", "--to", "120000", "--patch-apply", z1, "--patch-archive",
                                  "-o", back, arc_p])
    assert rc == 0 and back.read_bytes() == NEW[70000:120000].tobytes(), err
    assert 0 < ctx.reference_entries_decoded - before < zk.SeekTable.from_bytes(z1.read_bytes()).num_frames()
    # refusals
    out = tmp_path / "r.zst"
    for argv, what in ((["compress", "--patch-from", z1, "--patch-archive", v2], "--patch-archive needs"),
                       (["compress", "--patch-from", z1, "--patch-archive", "--long", v2], "--patch-archive needs"),
                       (["compress", "--patch-from", arc_p, "--patch-slices", "--patch-archive", v2], "is a seekable patch; restore it first"),
                       (["decompress", "--patch-archive", arc_p], "--patch-archive needs")):
        rc, _, err = cases._cli(ctx, [argv[0], "-q", "-f", *argv[1:], "-o", out])
        assert rc != 0 and what in err and not out.exists(), (argv, err)
    # a reference of the wrong length names both lengths
    short = tmp_path / "short.zst"
    (tmp_path / "v1s").write_bytes(OLD[:-1].tobytes())
    rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", "-s", "24K", "-o", short, tmp_path / "v1s"])
    assert rc == 0, err
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "-f", "--patch-apply", short, "--patch-archive", "-o", back, arc_p])
    assert rc != 0 and str(OLD.size) in err and str(OLD.size - 1) in err


@pytest.mark.gpu
def test_headline(gpu_lib):
    """tens of MiB of OLD in 2 MiB frames, level 16 with checksums: the patches against v1 and v1.zst are the same bytes, every round trip
    is exact, and a one-frame read decodes at most 4 entries of v1.zst (its 6 MiB slice over 2 MiB entries)"""
    ctx = zk.Context(0, gpu_lib)
    old = _mix(48 << 20, 3)
    new = edited_copy(old, 11, 200)
    fs = 2 << 20
    sizes = _uniform(new.size, fs)
    r = zk.ReferenceArchive(_with_table(*ctx.compress_frames(old, fs, 3, True)))
    want = ctx.compress_patch_slices(new, sizes, old, 16, True)
    got = ctx.compress_patch_slices(new, sizes, r, 16, True)
    assert got == want
    co, do, _, rg = _split(got)
    pad = np.frombuffer(got + b"\0" * 64, dtype=np.uint8)
    for prefix in (old, r):
        back, st, rc = ctx.decompress_frames(pad, co, do, True, prefix=prefix, prefix_ranges=rg)
        assert rc == 0 and back.tobytes() == new.tobytes()
    f = len(sizes) // 2
    before, up = ctx.reference_entries_decoded, ctx.prefix_bytes_uploaded
    dec = zk.DecodeOptions(zk.BytesWrapper(got), ctx).lower_frame(f).upper_frame(f).into_decoder()
    buf = bytearray(fs + 1)
    k = dec.decompress_with_prefix(buf, r, rg)
    assert bytes(buf[:k]) == new[int(do[f]):int(do[f + 1])].tobytes()
    assert 0 < ctx.reference_entries_decoded - before <= 4 and ctx.prefix_bytes_uploaded == up
    ctx.close()
