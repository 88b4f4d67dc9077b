"""What a raw OLD costs the seekable-patch calls (zk_patch_ranges, zk_compress_frames_patch, zk_decompress_frames_prefixes with ranges).
Raw OLD is the root of a reference chain of one level, and every ranged call makes each group's hull of OLD resident before its entries
run.  So a ranged call uploads exactly the hulls of its groups of entries (the group rule, restated here), the anchor pass uploads no
prefix bytes, the ReferenceArchive calls upload none, and no raw call decodes a reference entry.  Emulation cases run on the emulation
build (`-m "not gpu"`); the same cases run on the H100 (`-m gpu`)."""
import numpy as np
import pytest

import zeekstd_b200 as zk
from test_patch_ldm import _mix, edited_copy
from util import offsets
from zeekstd_b200 import _native


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    return request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib")


@pytest.fixture(scope="module")
def ctx(lib):
    _native.set_default_lib(lib)
    c = zk.Context(0, lib)
    yield c
    c.close()


OLD = _mix(256 << 10, 1)
NEW = edited_copy(OLD, 2, 12)
SIZES = [min(32 << 10, NEW.size - a) for a in range(0, NEW.size, 32 << 10)]
MARGIN = 8 << 10
GROUPS = [None, 96 << 10, 48 << 10, 32 << 10]              # ZK_PATCH_GROUP_BYTES: the default (one group), then several groups
EMPTY = (0, 1, 5)                                           # the frames whose range the "gaps" ranges empty


def hulls(ranges, group) -> list:
    """the hull lengths of the groups with a non-empty hull: a group takes, from its first entry on, as many entries as keep the hull of
    their non-empty ranges within `group` bytes, and at least one non-empty range (empty ranges join any group)"""
    out, f, n = [], 0, len(ranges)
    while f < n:
        f0, lo, hi = f, None, None
        while f < n:
            a, b = (int(v) for v in ranges[f])
            if a != b:
                nlo, nhi = (a, b) if lo is None else (min(lo, a), max(hi, b))
                if f > f0 and lo is not None and nhi - nlo > group:
                    break
                lo, hi = nlo, nhi
            f += 1
        if lo is not None:
            out.append(hi - lo)
    return out


def _with_table(comp, cs, ds) -> bytes:
    table = zk.SeekTable()
    for c, d in zip(np.asarray(cs).tolist(), np.asarray(ds).tolist()):
        table.log_frame(int(c), int(d))
    return bytes(np.asarray(comp, dtype=np.uint8).tobytes()) + table.into_serializer().to_bytes()


@pytest.fixture(scope="module")
def anchored(ctx):
    return ctx.patch_ranges(NEW, SIZES, OLD, MARGIN)


@pytest.fixture(scope="module", params=["anchored", "gaps"])
def ranges(request, anchored):
    """the ranges patch_ranges finds; "gaps": the same with a few of them empty, leading ones included, so a group may have no hull"""
    if request.param == "anchored":
        return anchored
    rg = anchored.copy()
    rg[list(EMPTY)] = 0
    return rg


def _counters(ctx):
    return ctx.prefix_bytes_uploaded, ctx.reference_entries_decoded


def _group(monkeypatch, group):
    if group:
        monkeypatch.setenv("ZK_PATCH_GROUP_BYTES", str(group))
    return group or 1 << 30


def test_groups_of_the_fixture(anchored):
    """the ranges are non-empty and overlap, and the small groups split them several ways.  The "gaps" ranges start with empty ones
    followed by a range longer than the smallest group, and every group then holds exactly one non-empty range"""
    assert all(b > a for a, b in anchored.tolist())
    assert [len(hulls(anchored, g or 1 << 30)) for g in GROUPS] == [1, 4, len(SIZES), len(SIZES)]
    gaps = anchored.copy()
    gaps[list(EMPTY)] = 0
    assert int(gaps[2, 1] - gaps[2, 0]) > GROUPS[-1]
    assert hulls(gaps, GROUPS[-1]) == [int(b - a) for i, (a, b) in enumerate(anchored.tolist()) if i not in EMPTY]


def test_anchor_pass_uploads_no_prefix(ctx):
    """raw OLD's anchors stream through the staging buffer: no prefix bytes, no reference entries"""
    before = _counters(ctx)
    ctx.patch_ranges(NEW, SIZES, OLD, MARGIN)
    assert _counters(ctx) == before


@pytest.mark.parametrize("group", GROUPS)
def test_compress_uploads_group_hulls(ctx, ranges, group, monkeypatch):
    """compress_frames_patch uploads each non-empty group hull once, and decodes no reference entry"""
    g = _group(monkeypatch, group)
    up, dec = _counters(ctx)
    ctx.compress_frames_patch(NEW, SIZES, OLD, ranges, 3, True)
    assert ctx.prefix_bytes_uploaded - up == sum(hulls(ranges, g))
    assert ctx.reference_entries_decoded == dec


@pytest.mark.parametrize("group", GROUPS)
def test_ranged_decompress_uploads_group_hulls(ctx, ranges, group, monkeypatch):
    """the ranged decompress uploads each non-empty group hull once, decodes no reference entry, and restores NEW"""
    comp, cs, ds = ctx.compress_frames_patch(NEW, SIZES, OLD, ranges, 3, True)
    co, do = offsets(cs), offsets(ds)
    pad = np.concatenate([comp, np.zeros(64, dtype=np.uint8)])
    g = _group(monkeypatch, group)
    up, dec = _counters(ctx)
    out, st, rc = ctx.decompress_frames(pad, co, do, True, prefix=OLD, prefix_ranges=ranges)
    assert rc == 0 and not st.any() and out.tobytes() == NEW.tobytes()
    assert ctx.prefix_bytes_uploaded - up == sum(hulls(ranges, g))
    assert ctx.reference_entries_decoded == dec


def test_reference_archive_calls_upload_no_prefix(ctx, anchored, monkeypatch):
    """every call on a ReferenceArchive decodes entries into device memory and uploads no prefix bytes"""
    ref = zk.ReferenceArchive(_with_table(*ctx.compress_frames(OLD, 24 << 10, 3, True)))
    _group(monkeypatch, GROUPS[-1])
    up, dec = _counters(ctx)
    assert ctx.patch_ranges(NEW, SIZES, ref, MARGIN).tolist() == anchored.tolist()
    comp, cs, ds = ctx.compress_frames_patch(NEW, SIZES, ref, anchored, 3, True)
    pad = np.concatenate([comp, np.zeros(64, dtype=np.uint8)])
    out, st, rc = ctx.decompress_frames(pad, offsets(cs), offsets(ds), True, prefix=ref, prefix_ranges=anchored)
    assert rc == 0 and out.tobytes() == NEW.tobytes()
    assert ctx.prefix_bytes_uploaded == up and ctx.reference_entries_decoded > dec
