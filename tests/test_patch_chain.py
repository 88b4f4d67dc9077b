"""Seekable patch chains (zk_patch_ranges_chain, zk_compress_frames_patch_chain, zk_decompress_frames_prefixes_chain, the Decoder's
chain read, ReferenceArchive(base=...), the CLI's --patch-base): the reference is v1.zst <- v2.patch <- v3.patch <- ..., and OLD the
head's decoded content, every level decoded on the GPU only where the level above reads it.  Every call equals its raw call on OLD at
depths 1 to 4; at depth 1 it equals the _archive call, entry counter included; the entries decoded are what a Python model of Need
gives; a corrupt entry at the root or in the middle fails exactly the patch entries that reach it; argument errors; libzstd restores every
level; the CLI.  Emulation cases run on the emulation build (`-m "not gpu"`, small versions); the headline case runs on the H100."""
import ctypes
import io
from bisect import bisect_right

import numpy as np
import pytest

import cases
import zeekstd_b200 as zk
from oracle import oracle as O
from test_patch_archive import OLD, _bytes, _uniform, _with_table, reference
from test_patch_ldm import _mix, edited_copy
from zeekstd_b200 import _native

INVALID = -1006
CHECKSUM_WRONG = -22
FS = 64 << 10
MARGIN = 8 << 10
GROUP = 1 << 30                                             # ZK_PATCH_GROUP_BYTES' default

# v1 .. v4: each an edit of the one before
VERSIONS = [OLD]
for _k in range(3):
    VERSIONS.append(edited_copy(VERSIONS[-1], 21 + _k, 10))


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    return request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib")


@pytest.fixture(scope="module")
def ctx(lib):
    _native.set_default_lib(lib)
    c = zk.Context(0, lib)
    yield c
    c.close()


def sizes_of(v) -> list:
    return _uniform(v.size, FS)


@pytest.fixture(scope="module")
def raw_patches(ctx):
    """v_{k+1}.patch made against raw v_k, k = 1 .. 3"""
    return [ctx.compress_patch_slices(VERSIONS[k + 1], sizes_of(VERSIONS[k + 1]), VERSIONS[k], 3, True, MARGIN) for k in range(3)]


def chain_of(root: zk.ReferenceArchive, patches, depth: int) -> zk.ReferenceArchive:
    """the ReferenceArchive of v_depth: root, then depth - 1 patches, each on the one below"""
    r = root
    for p in patches[:depth - 1]:
        r = zk.ReferenceArchive(p, base=r)
    return r


@pytest.fixture(scope="module")
def chains(ctx, raw_patches):
    """kind -> [None, chain of depth 1, 2, 3, 4] over the raw patches (test 1 shows that chain-made patches are the same bytes)"""
    out = {}
    for kind in ("uniform", "empty", "libzstd", "multi"):
        root = reference(ctx, kind, VERSIONS[0])
        out[kind] = [None] + [chain_of(root, raw_patches, d) for d in range(1, 5)]
    return out


def _split(archive: bytes):
    table = zk.SeekTable.from_bytes(archive, zk.Format.Foot)
    co, do = table.offsets()
    _, rg, _ = zk.patch_slices_read(archive, table.num_frames())
    return co, do, rg


@pytest.fixture(scope="module")
def v5(ctx):
    """a patch against v4 (the head of every depth-4 chain): NEW = an edit of v4, made against raw v4"""
    new = edited_copy(VERSIONS[3], 31, 10)
    return new, ctx.compress_patch_slices(new, sizes_of(new), VERSIONS[3], 3, True, MARGIN)


# ----------------------------------------------------------------------------------------------------------- a Python model of Need
def hull_groups(ranges, group=GROUP):
    """zk_hull_group over (lo, hi) pairs -> [(start, end, hlo, hhi)]"""
    out, f0, n = [], 0, len(ranges)
    while f0 < n:
        lo = hi = 0
        any_, f = False, f0
        while f < n:
            a, b = (int(x) for x in ranges[f])
            if a == b:
                f += 1
                continue
            nlo, nhi = (min(lo, a), max(hi, b)) if any_ else (a, b)
            if f > f0 and any_ and nhi - nlo > group:
                break
            lo, hi, any_ = nlo, nhi, True
            f += 1
        out.append((f0, f, lo, hi))
        f0 = f
    return out


class Level:
    """one level of a chain for the model: its entries' offsets, its slices (patch levels) and the entries damaged ({g: code})"""

    def __init__(self, r: zk.ReferenceArchive, bad=None):
        self.d = [int(x) for x in r.d_off]
        self.slices = None
        if r.base is not None:
            self.slices = zk.patch_slices_read(_bytes(r)[int(r.c_off[0]):], r.n_entries)[1].tolist()
        self.bad = bad or {}


def levels_of(r: zk.ReferenceArchive, bad=None) -> list:
    bad = bad or {}
    return [Level(x, bad.get(i)) for i, x in enumerate(r.chain)]


def need(levels, i, lo, hi, verify=True, group=GROUP):
    """Need(i, [lo, hi)) -> (entries decoded at every level, level i's list, their statuses)"""
    lv = levels[i]
    d = lv.d
    g = bisect_right(d, lo) - 1
    lst = []
    while g < len(d) - 1 and d[g] < hi:
        if d[g + 1] > d[g]:
            lst.append(g)
        g += 1
    st = [0] * len(lst)
    count = 0
    if lv.slices is not None:
        sl = [lv.slices[g] for g in lst]
        for k0, k1, hlo, hhi in hull_groups(sl, group):
            if hhi <= hlo:
                continue
            c, blst, bst = need(levels, i - 1, hlo, hhi, verify, group)
            count += c
            for k in range(k0, k1):
                a, b = sl[k]
                if a < b:
                    st[k] = failure(levels[i - 1], blst, bst, a, b)
    for k, g in enumerate(lst):
        if st[k]:
            continue                                        # its slice failed below: not decoded
        count += 1
        if g in lv.bad:
            code = lv.bad[g]
            full = not (k == len(lst) - 1 and d[g + 1] > hi)
            if code != CHECKSUM_WRONG or (verify and full):
                st[k] = code
    return count, lst, st


def failure(lv: Level, lst, st, lo, hi) -> int:
    for g, s in zip(lst, st):
        if s and lv.d[g + 1] > lo and lv.d[g] < hi:
            return s
    return 0


def apply_model(levels, ranges, verify=True, group=GROUP):
    """the decompress call over entries with these ranges -> (entries decoded, every entry's status)"""
    count, st = 0, [0] * len(ranges)
    for f0, f1, hlo, hhi in hull_groups(ranges, group):
        if hhi <= hlo:
            continue
        c, lst, lst_st = need(levels, len(levels) - 1, hlo, hhi, verify, group)
        count += c
        for f in range(f0, f1):
            a, b = (int(x) for x in ranges[f])
            if a < b:
                st[f] = failure(levels[-1], lst, lst_st, a, b)
    return count, st


# ----------------------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("kind", ["uniform", "empty", "libzstd", "multi"])
def test_chain_made_patches(ctx, raw_patches, kind):
    """test 1: every v_{k+1}.patch made against the chain under it is the raw call's patch against raw v_k"""
    r = reference(ctx, kind, VERSIONS[0])
    for k in range(3):
        new = VERSIONS[k + 1]
        got = ctx.compress_patch_slices(new, sizes_of(new), r, 3, True, MARGIN)
        assert got == raw_patches[k], (kind, k)
        r = zk.ReferenceArchive(got, base=r)
    assert r.depth == 4 and [x.old_len for x in r.chain] == [v.size for v in VERSIONS]


def _archive_args(r: zk.ReferenceArchive):
    return (r._addr, r._len, r.c_off.ctypes.data_as(_native.u64p), r.d_off.ctypes.data_as(_native.u64p), r.n_entries)


def test_depth_one_is_the_archive_call(ctx, chains):
    """at depth 1 the _chain calls return what the _archive calls return, and decode as many entries"""
    lib = ctx.lib
    r = chains["multi"][1]
    new = VERSIONS[1]
    ds = np.asarray(sizes_of(new), dtype=np.uint32)
    outs = []
    for chain in (False, True):
        rg = np.zeros((ds.size, 2), dtype=np.uint64)
        before = ctx.reference_entries_decoded
        args = r._chain() if chain else _archive_args(r)
        call = lib.zk_patch_ranges_chain if chain else lib.zk_patch_ranges_archive
        assert call(ctx._h, new.ctypes.data, ds.ctypes.data_as(_native.u32p), ds.size, *args, MARGIN, rg.ctypes.data_as(_native.u64p)) == 0
        cap = lib.zk_compress_bound_sized(ds.ctypes.data_as(_native.u32p), ds.size)
        dst = np.zeros(cap + 64, dtype=np.uint8)
        cs = np.zeros(ds.size, dtype=np.uint32)
        dl = ctypes.c_size_t()
        call = lib.zk_compress_frames_patch_chain if chain else lib.zk_compress_frames_patch_archive
        assert call(ctx._h, new.ctypes.data, ds.ctypes.data_as(_native.u32p), ds.size, 3, 1, *args, rg.ctypes.data_as(_native.u64p),
                    dst.ctypes.data, cap, cs.ctypes.data_as(_native.u32p), ctypes.byref(dl)) == 0
        co = np.concatenate([[0], np.cumsum(cs, dtype=np.uint64)]).astype(np.uint64)
        do = np.concatenate([[0], np.cumsum(ds, dtype=np.uint64)]).astype(np.uint64)
        pad = np.concatenate([dst[:dl.value], np.zeros(64, dtype=np.uint8)])
        out = np.zeros(new.size + 64, dtype=np.uint8)
        st = np.zeros(ds.size, dtype=np.int32)
        call = lib.zk_decompress_frames_prefixes_chain if chain else lib.zk_decompress_frames_prefixes_archive
        rc = call(ctx._h, pad.ctypes.data, co.ctypes.data_as(_native.u64p), do.ctypes.data_as(_native.u64p), ds.size, out.ctypes.data, None, 1,
                  st.ctypes.data_as(_native.i32p), *args, rg.ctypes.data_as(_native.u64p))
        outs.append((rg.tolist(), dst[:dl.value].tobytes(), cs.tolist(), out[:new.size].tobytes(), st.tolist(), rc,
                     ctx.reference_entries_decoded - before))
    assert outs[0] == outs[1] and outs[0][3] == new.tobytes()


def _patch_against(depth, raw_patches, v5):
    """(NEW, the patch of NEW against raw v_depth): v_{depth+1}.patch, or v5's for depth 4"""
    return (VERSIONS[depth], raw_patches[depth - 1]) if depth < 4 else v5


@pytest.mark.parametrize("depth", [1, 2, 3, 4])
def test_same_ranges_frames_restore(ctx, chains, raw_patches, depth, v5):
    """test 2: through a chain of depth d, the raw calls' ranges, frames (checksums on and off) and restores (verify on and off, full and
    with need, with and without ranges) on v_d.  Test 1 already makes the checksummed patches of depths 1-3 through chains"""
    old = VERSIONS[depth - 1]
    new, patch = _patch_against(depth, raw_patches, v5)
    sizes = sizes_of(new)
    r = chains["uniform"][depth]
    co, do, rg = _split(patch)
    assert ctx.patch_ranges(new, sizes, r, MARGIN).tolist() == rg.tolist()
    if depth == 4:
        assert ctx.compress_patch_slices(new, sizes, r, 3, True, MARGIN) == patch
        want = ctx.compress_frames_patch(new, sizes, old, rg, 3, False)
        got = ctx.compress_frames_patch(new, sizes, r, rg, 3, False)
        assert got[0].tobytes() == want[0].tobytes() and got[1].tolist() == want[1].tolist()
    pad = np.frombuffer(patch + b"\0" * 64, dtype=np.uint8)
    nd = np.array([int(do[f + 1] - do[f]) // (f + 2) for f in range(len(sizes))], dtype=np.uint32)
    for verify in (False, True):
        for need_ in (None, nd):
            g, st, rc = ctx.decompress_frames(pad, co, do, verify, need=need_, prefix=r, prefix_ranges=rg)
            assert rc == 0 and not st.any()
            if need_ is None:
                assert g.tobytes() == new.tobytes()
            else:
                for f in range(len(sizes)):
                    a = int(do[f])
                    assert g[a:a + int(nd[f])].tobytes() == new[a:a + int(nd[f])].tobytes(), f
    # without ranges: every entry against all of OLD
    wc, wcs, wds = ctx.compress_frames(new[:64 << 10], 16 << 10, 3, True, prefix=old)
    p2 = np.concatenate([wc, np.zeros(64, dtype=np.uint8)])
    c2, d2 = np.concatenate([[0], np.cumsum(wcs)]).astype(np.uint64), np.concatenate([[0], np.cumsum(wds)]).astype(np.uint64)
    w, _, wrc = ctx.decompress_frames(p2, c2, d2, True, prefix=old)
    g, _, rc = ctx.decompress_frames(p2, c2, d2, True, prefix=r)
    assert rc == wrc == 0 and g.tobytes() == w.tobytes() == new[:64 << 10].tobytes()


def test_small_groups_and_pieces(ctx, chains, v5, monkeypatch):
    """test 3: with 96 KiB groups and 32 KiB pieces (hulls split at inner levels, every head entry its own run) every output is the
    same, and the entries decoded are the model's under that group size"""
    new, patch = v5
    sizes = sizes_of(new)
    r = chains["empty"][4]
    old = VERSIONS[3]
    rg = ctx.patch_ranges(new, sizes, old, MARGIN)
    want = ctx.compress_frames_patch(new, sizes, old, rg, 3, True)
    monkeypatch.setenv("ZK_PATCH_GROUP_BYTES", str(96 << 10))
    monkeypatch.setenv("ZK_PATCH_PIECE_BYTES", str(32 << 10))
    assert ctx.patch_ranges(new, sizes, r, MARGIN).tolist() == rg.tolist()
    got = ctx.compress_frames_patch(new, sizes, r, rg, 3, True)
    assert got[0].tobytes() == want[0].tobytes() and got[1].tolist() == want[1].tolist()
    co, do, prg = _split(patch)
    pad = np.frombuffer(patch + b"\0" * 64, dtype=np.uint8)
    before = ctx.reference_entries_decoded
    g, st, rc = ctx.decompress_frames(pad, co, do, True, prefix=r, prefix_ranges=prg)
    assert rc == 0 and g.tobytes() == new.tobytes()
    assert ctx.reference_entries_decoded - before == apply_model(levels_of(r), prg.tolist(), group=96 << 10)[0]


def test_entries_decoded(ctx, chains, v5):
    """test 4: one-frame reads, a read across two frames and a full apply decode exactly the model's entries, and upload no prefix byte"""
    new, patch = v5
    co, do, rg = _split(patch)
    pad = np.frombuffer(patch + b"\0" * 64, dtype=np.uint8)
    n = len(rg)
    for kind in ("uniform", "multi"):
        r = chains[kind][4]
        lv = levels_of(r)
        for f0, f1 in ((0, 0), (n // 2, n // 2), (n - 1, n - 1), (1, 2)):
            want = apply_model(lv, rg[f0:f1 + 1].tolist())[0]
            before, up = ctx.reference_entries_decoded, ctx.prefix_bytes_uploaded
            dec = zk.DecodeOptions(zk.BytesWrapper(patch), ctx).lower_frame(f0).upper_frame(f1).into_decoder()
            buf = bytearray(int(do[f1 + 1] - do[f0]) + 1)
            k = dec.decompress_with_prefix(buf, r, rg)
            assert bytes(buf[:k]) == new[int(do[f0]):int(do[f1 + 1])].tobytes()
            assert ctx.reference_entries_decoded - before == want and want > 0, (kind, f0, f1)
            assert ctx.prefix_bytes_uploaded == up
        before, up = ctx.reference_entries_decoded, ctx.prefix_bytes_uploaded
        g, st, rc = ctx.decompress_frames(pad, co, do, True, prefix=r, prefix_ranges=rg)
        assert rc == 0 and g.tobytes() == new.tobytes()
        total = apply_model(lv, rg.tolist())[0]
        assert ctx.reference_entries_decoded - before == total and total >= sum(x.n_entries for x in r.chain) // 2
        assert ctx.prefix_bytes_uploaded == up


def _damaged(r: zk.ReferenceArchive, g: int, how: str) -> zk.ReferenceArchive:
    """r with entry g (one zstd frame) damaged, on the same base: its first block's type set to the reserved 3 (a decode error
    wherever the entry is decoded), or its checksum changed"""
    b = bytearray(_bytes(r))
    c0, c1 = int(r.c_off[g]), int(r.c_off[g + 1])
    if how == "block":
        fhd = b[c0 + 4]
        single, fcs = (fhd >> 5) & 1, fhd >> 6
        at = c0 + 5 + (1 - single) + (0, 1, 2, 4)[fhd & 3] + ((1 if single else 0), 2, 4, 8)[fcs]
        b[at] |= 0x06
    else:
        b[c1 - 1] ^= 0xFF
    return zk.ReferenceArchive(bytes(b), c_off=r.c_off, d_off=r.d_off, base=r.base)


def _code(ctx, level: int, bad: zk.ReferenceArchive, g: int) -> int:
    """the status of entry g of `bad` (level `level` of a chain) decoded whole with verification, against the raw version below it"""
    pad = np.frombuffer(_bytes(bad) + b"\0" * 64, dtype=np.uint8)
    if level == 0:
        return int(ctx.decompress_frames(pad, bad.c_off, bad.d_off, True)[1][g])
    rg = zk.patch_slices_read(_bytes(bad)[int(bad.c_off[0]):], bad.n_entries)[1]
    return int(ctx.decompress_frames(pad, bad.c_off, bad.d_off, True, prefix=VERSIONS[level - 1], prefix_ranges=rg)[1][g])


@pytest.mark.parametrize("where", ["root", "middle"])
@pytest.mark.parametrize("how", ["block", "checksum"])
def test_corrupt_entry(ctx, chains, raw_patches, v5, where, how):
    """test 5: one damaged entry at the root or at level 1, under a chain one level above it and under the depth-4 chain: the patch
    entries the model names fail with its code, the others restore exactly; the compress and range calls return the failure"""
    root = chains["uniform"][1]
    level = 0 if where == "root" else 1
    lower = chain_of(root, raw_patches, level + 1)              # the level damaged, with its own chain under it
    g = lower.n_entries - 1                                     # the last entry: failures above it stay away from the start
    bad_level = _damaged(lower, g, how)
    code = _code(ctx, level, bad_level, g)
    assert code < 0 and (code == CHECKSUM_WRONG) == (how == "checksum")
    # failures widen with every level (each entry above reads a slice around its own); one level up, some entries still restore
    for depth, new, patch in ((level + 2, VERSIONS[level + 2], raw_patches[level + 1]), (4, *v5)):
        r = chain_of(bad_level, raw_patches[level:], depth - level)
        assert r.depth == depth
        co, do, rg = _split(patch)
        pad = np.frombuffer(patch + b"\0" * 64, dtype=np.uint8)
        lv = levels_of(r, {level: {g: code}})
        for verify in (True, False) if how == "checksum" else (True,):   # a bad checksum alone leaves the content right
            got, st, rc = ctx.decompress_frames(pad, co, do, verify, prefix=r, prefix_ranges=rg)
            _, want = apply_model(lv, rg.tolist(), verify)
            assert st.tolist() == want and rc == next((s for s in want if s), 0), (depth, verify, want)
            assert any(want) == verify and (depth == 4 or not all(want)), (depth, verify, want)
            for f, s in enumerate(want):
                if not s:
                    assert got[int(do[f]):int(do[f + 1])].tobytes() == new[int(do[f]):int(do[f + 1])].tobytes(), f
    sizes = sizes_of(new)
    rg_raw = ctx.patch_ranges(new, sizes, VERSIONS[3], MARGIN)
    with pytest.raises(zk.Error) as e:
        ctx.patch_ranges(new, sizes, r, MARGIN)
    assert e.value.rc == code
    with pytest.raises(zk.Error) as e:
        ctx.compress_frames_patch(new, sizes, r, rg_raw, 3, False)
    assert e.value.rc == code


def test_argument_errors(ctx, chains, raw_patches):
    """test 6: every ZK_ERR_INVALID_ARG case of the _chain calls, and ReferenceArchive's base errors"""
    lib = ctx.lib
    r1 = chains["uniform"][1]
    p2 = raw_patches[0]
    t2 = zk.SeekTable.from_bytes(p2)
    c2, d2 = t2.offsets()
    new = VERSIONS[2]
    ds = np.asarray(sizes_of(new), dtype=np.uint32)

    def desc(data, c_off, d_off):
        a = np.frombuffer(data, dtype=np.uint8)
        co, do = np.ascontiguousarray(c_off, dtype=np.uint64), np.ascontiguousarray(d_off, dtype=np.uint64)
        d = _native.ReferenceArchiveDesc(a.ctypes.data, a.size, co.ctypes.data_as(_native.u64p), do.ctypes.data_as(_native.u64p), co.size - 1)
        return d, (a, co, do)

    def ranges_rc(descs, depth=None):
        arr = (_native.ReferenceArchiveDesc * max(len(descs), 1))(*descs)
        rg = np.zeros(2 * ds.size, dtype=np.uint64)
        return lib.zk_patch_ranges_chain(ctx._h, new.ctypes.data, ds.ctypes.data_as(_native.u32p), ds.size, arr,
                                         len(descs) if depth is None else depth, MARGIN, rg.ctypes.data_as(_native.u64p))

    root, k0 = desc(_bytes(r1), r1.c_off, r1.d_off)
    patch, k1 = desc(p2, c2, d2)
    assert ranges_rc([root, patch]) == 0
    assert ranges_rc([root], depth=0) == INVALID
    assert ranges_rc([root], depth=33) == INVALID
    assert ranges_rc([patch]) == INVALID                    # a root that is a patch
    assert ranges_rc([root, root]) == INVALID               # a level without a slice frame
    mco, mdo = np.delete(c2, 1), np.delete(d2, 1)           # entries 0 and 1 merged: a slice frame of another entry count
    merged, k2 = desc(p2, mco, mdo)
    assert ranges_rc([root, merged]) == INVALID
    short = zk.ReferenceArchive(_with_table(*ctx.compress_frames(VERSIONS[0][:-1000], 24 << 10, 3, True)))
    sroot, k3 = desc(_bytes(short), short.c_off, short.d_off)
    assert ranges_rc([sroot, patch]) == INVALID             # old_len is not the level below's length
    dco = c2.copy(); dco[2] = dco[1] - 1
    dec_, k4 = desc(p2, dco, d2)
    assert ranges_rc([root, dec_]) == INVALID               # offsets that decrease
    long_co = c2.copy(); long_co[-1] = len(p2) + 1
    lng, k5 = desc(p2, long_co, d2)
    assert ranges_rc([root, lng]) == INVALID                # past the level's bytes
    r2 = chains["uniform"][2]
    rg = ctx.patch_ranges(new, ds, r2, MARGIN)
    past = rg.copy(); past[1][1] = r2.old_len + 1
    with pytest.raises(zk.Error) as e:
        ctx.compress_frames_patch(new, ds, r2, past, 3, False)
    assert e.value.rc == INVALID
    comp, cs, _ = ctx.compress_frames_patch(new, ds, r2, rg, 3, False)
    co, do = np.concatenate([[0], np.cumsum(cs)]), np.concatenate([[0], np.cumsum(ds)])
    pad = np.concatenate([comp, np.zeros(64, dtype=np.uint8)])
    assert ctx.decompress_frames(pad, co, do, True, prefix=r2, prefix_ranges=past)[2] == INVALID
    # ReferenceArchive: a patch without a base, a base under a plain archive, a base of another length
    with pytest.raises(ValueError, match="is a seekable patch; restore it first"):
        zk.ReferenceArchive(p2)
    with pytest.raises(ValueError, match="plain"):
        zk.ReferenceArchive(_bytes(r1), base=r1)
    with pytest.raises(ValueError, match=f"{short.old_len}.*{VERSIONS[0].size}"):
        zk.ReferenceArchive(p2, base=short)


def test_libzstd_restores_every_level(raw_patches, v5):
    """test 7: libzstd restores every patch of the chain (test 1 shows they are the patches made through it) from the raw previous
    version, refPrefix on each frame's slice"""
    for k, (new, patch) in enumerate([(VERSIONS[k + 1], raw_patches[k]) for k in range(3)] + [v5]):
        old = VERSIONS[k]
        co, do, rg = _split(patch)
        flen = zk.patch_slices_size(len(rg))
        for f, (lo, hi) in enumerate(rg.tolist()):
            c0 = int(co[f]) + (flen if f == 0 else 0)
            fr = np.frombuffer(patch[c0:int(co[f + 1])] + b"\0" * 64, dtype=np.uint8)
            n = int(do[f + 1] - do[f])
            out, sizes = O.ref_decompress_frames(fr, [0, int(co[f + 1]) - c0], [0, n], prefix=old[lo:hi] if hi > lo else None)
            assert sizes == [n] and out.tobytes() == new[int(do[f]):int(do[f + 1])].tobytes(), (k, f)


def test_decoder_random_ops(ctx, chains, v5):
    """test 8: the Decoder reading v5.patch through a depth-4 chain, against the same Decoder with raw v4"""
    new, patch = v5
    _, _, rg = _split(patch)
    r = chains["empty"][4]
    rng = np.random.default_rng(13)
    a = zk.DecodeOptions(zk.BytesWrapper(patch), ctx).into_decoder()
    b = zk.DecodeOptions(zk.BytesWrapper(patch), ctx).into_decoder()
    total = new.size
    for _ in range(20):
        k = int(rng.integers(6))
        if k <= 2:
            ln = int(rng.choice([1, 999, 24 << 10, 64 << 10, total]))
            ba, bb = bytearray(ln), bytearray(ln)
            na, nb = a.decompress_with_prefix(ba, r, rg), b.decompress_with_prefix(bb, VERSIONS[3], rg)
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
    # a chain that differs at a lower level (the same head) is another prefix: the window is decoded again, against the new chain
    a.set_offset(0); a.set_offset_limit(total)
    buf = bytearray(total)
    assert a.decompress_with_prefix(buf, chains["uniform"][4], rg) == total and bytes(buf) == new.tobytes()


def test_cli(ctx, raw_patches, tmp_path):
    """test 9: compress and decompress with --patch-base, whole and with --from/--to and --from-frame/--to-frame, and each new error"""
    v = [tmp_path / f"v{k + 1}" for k in range(4)]
    for p, x in zip(v, VERSIONS):
        p.write_bytes(x.tobytes())
    z1 = tmp_path / "v1.zst"
    rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", "-s", "24K", "-o", z1, v[0]])
    assert rc == 0, err
    pat = [None, tmp_path / "v2.patch", tmp_path / "v3.patch", tmp_path / "v4.patch"]
    pat[1].write_bytes(raw_patches[0]); pat[2].write_bytes(raw_patches[1])
    chain = ["--patch-archive", "--patch-base", pat[1], "--patch-base", z1]
    rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", "-s", "64K", "--patch-slices", "--patch-margin", "8K", "--patch-from", pat[2], *chain,
                                  "-o", pat[3], v[3]])
    assert rc == 0 and pat[3].read_bytes() == raw_patches[2], err
    back = tmp_path / "back"
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "-f", "--patch-apply", pat[2], *chain, "-o", back, pat[3]])
    assert rc == 0 and back.read_bytes() == VERSIONS[3].tobytes(), err
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "-f", "--from", "70000", "--to", "150000", "--patch-apply", pat[2], *chain, "-o", back,
                                  pat[3]])
    assert rc == 0 and back.read_bytes() == VERSIONS[3][70000:150000].tobytes(), err
    do = zk.SeekTable.from_bytes(pat[3].read_bytes()).offsets()[1]
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "-f", "--from-frame", "1", "--to-frame", "2", "--patch-apply", pat[2], *chain, "-o", back,
                                  pat[3]])
    assert rc == 0 and back.read_bytes() == VERSIONS[3][int(do[1]):int(do[3])].tobytes(), err
    # errors
    out = tmp_path / "r.out"
    short = tmp_path / "short.zst"
    (tmp_path / "v1s").write_bytes(VERSIONS[0][:-1].tobytes())
    rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", "-s", "24K", "-o", short, tmp_path / "v1s"])
    assert rc == 0, err
    for argv, what in (
            (["decompress", "--patch-apply", pat[2], "--patch-base", pat[1], pat[3]], "--patch-base needs --patch-archive"),
            (["compress", "-s", "64K", "--patch-slices", "--patch-from", pat[2], "--patch-base", z1, v[3]], "--patch-base needs --patch-archive"),
            (["decompress", "--patch-apply", pat[2], "--patch-archive", "--patch-base", pat[1], pat[3]], "is a seekable patch; restore it first"),
            (["decompress", "--patch-apply", pat[1], "--patch-archive", "--patch-base", z1, "--patch-base", z1, pat[2]],
             "is not a seekable patch: --patch-base"),
            (["decompress", "--patch-apply", pat[1], "--patch-archive", "--patch-base", short, pat[2]],
             f"decodes to {VERSIONS[0].size - 1} bytes, the seekable patch {pat[1]} was made against {VERSIONS[0].size} bytes")):
        rc, _, err = cases._cli(ctx, [argv[0], "-q", "-f", *argv[1:], "-o", out])
        assert rc != 0 and what in err and not out.exists(), (argv, err)


@pytest.mark.gpu
def test_headline(gpu_lib):
    """test 10: a depth-4 chain of 64 MiB versions in 2 MiB frames at level 16 with checksums, default groups: every chain-made patch is
    the raw call's, a full apply and a one-frame read through the chain restore exactly and decode the model's entries"""
    ctx = zk.Context(0, gpu_lib)
    fs = 2 << 20
    vs = [_mix(64 << 20, 7)]
    for k in range(4):
        vs.append(edited_copy(vs[-1], 51 + k, 200))
    r = zk.ReferenceArchive(_with_table(*ctx.compress_frames(vs[0], fs, 3, True)))
    for k in range(4):
        new, sizes = vs[k + 1], _uniform(vs[k + 1].size, fs)
        want = ctx.compress_patch_slices(new, sizes, vs[k], 16, True)
        got = ctx.compress_patch_slices(new, sizes, r, 16, True)
        assert got == want, k
        if k == 3:
            break
        r = zk.ReferenceArchive(got, base=r)
    assert r.depth == 4
    new = vs[4]
    co, do, rg = _split(got)
    pad = np.frombuffer(got + b"\0" * 64, dtype=np.uint8)
    lv = levels_of(r)
    before, up = ctx.reference_entries_decoded, ctx.prefix_bytes_uploaded
    back, st, rc = ctx.decompress_frames(pad, co, do, True, prefix=r, prefix_ranges=rg)
    assert rc == 0 and back.tobytes() == new.tobytes()
    assert ctx.reference_entries_decoded - before == apply_model(lv, rg.tolist())[0] and ctx.prefix_bytes_uploaded == up
    f = len(rg) // 2
    before = ctx.reference_entries_decoded
    dec = zk.DecodeOptions(zk.BytesWrapper(got), ctx).lower_frame(f).upper_frame(f).into_decoder()
    buf = bytearray(fs + 1)
    k = dec.decompress_with_prefix(buf, r, rg)
    assert bytes(buf[:k]) == new[int(do[f]):int(do[f + 1])].tobytes()
    assert ctx.reference_entries_decoded - before == apply_model(lv, rg[f:f + 1].tolist())[0]
    ctx.close()
