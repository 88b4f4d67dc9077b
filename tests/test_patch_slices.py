"""Seekable patches (zk_patch_ranges, zk_compress_frames_patch, the slice frame): every frame of NEW matched against the slice of OLD its
content anchors point at.  The ranges equal a plain-Python restatement of the rule and do not depend on how OLD and NEW are cut into pieces
or the frames into groups; every frame is the per-frame-prefix call of that frame alone; the archive restores through
decompress_frames_prefixes, the Decoder, the CLI and libzstd refPrefix; one frame restores from its slice alone; bad slice frames and CLI
misuse are refused.  Emulation cases run on the emulation build (`-m "not gpu"`, small inputs); the headline sizes run on the H100 (`-m gpu`)."""
import bisect

import numpy as np
import pytest

import cases
import zeekstd_b200 as zk
from oracle import oracle as O
from test_patch_ldm import _mix, edited_copy
from util import offsets
from zeekstd_b200 import _native

MASK = (1 << 64) - 1
THR = (1 << 64) - MASK // 65536
REACH = 1 << 27


def _gear(b: int) -> int:
    z = ((b + 1) * 0x9E3779B97F4A7C15) & MASK
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
    return z ^ (z >> 31)


GEAR = np.array([_gear(b) for b in range(256)], dtype=np.uint64)


def anchors(x) -> list:
    """(position, key) of every anchor of x: p >= 63 with h_p = sum_j gear(x[p - j]) * 2^j (j < 64) mod 2^64 >= THR, in position order"""
    x = np.asarray(x, dtype=np.uint8)
    n = x.size
    if n < 64:
        return []
    h = np.zeros(n - 63, dtype=np.uint64)
    with np.errstate(over="ignore"):
        for j in range(64):
            h += GEAR[x[63 - j:n - j]] << np.uint64(j)
    return [(int(i) + 63, int(h[i])) for i in np.nonzero(h >= np.uint64(THR))[0]]


def ref_ranges(old, new, sizes, margin: int) -> list:
    """the rule of zk_patch_ranges, restated"""
    table = {}
    for p, k in anchors(old):
        table.setdefault(k, []).append(p)
    na = anchors(new)
    out, a = [], 0
    for size in sizes:
        b = a + int(size)
        ln = b - a
        matches = []
        for c, k in na:
            if a <= c < b and k in table:
                ps = table[k]
                i = bisect.bisect_left(ps, c)
                cands = ([ps[i - 1]] if i > 0 else []) + ([ps[i]] if i < len(ps) else [])
                matches.append((c, min(cands, key=lambda o: (abs(o - c), o))))
        centre = None
        if matches:
            (c1, o1), (c2, o2) = matches[0], matches[-1]
            in_order = o2 >= o1 and abs((o2 - o1) - (c2 - c1)) <= ln
            lo = o1 - (c1 - a) - margin
            hi = (o2 + (b - c2) if in_order else o1 + (b - c1)) + margin
            centre = (o1 + (o2 if in_order else o1)) // 2
        else:
            lo, hi = a - margin, b + margin
        lo = min(max(lo, 0), len(old))
        hi = min(max(hi, lo), len(old))
        w = REACH - ln if ln < REACH else 0
        if hi - lo > w:
            centre = (lo + hi) // 2 if centre is None else centre
            s = max(lo, min(centre - w // 2, hi - w))
            lo, hi = s, s + w
        out.append((lo, hi))
        a = b
    return out


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


def _repeated(n: int, seed: int) -> np.ndarray:
    """OLD whose content repeats four times: every anchor key has four positions"""
    part = _mix(n // 4, seed)
    return np.concatenate([part] * 4)


def _cases():
    """name -> (OLD, NEW, frame sizes, margin): many anchors per frame with a moved region, duplicate keys, frames too short for an anchor,
    and content defined frames are covered by test_content_policy"""
    old = _mix(640 << 10, 1)
    new = edited_copy(old, 2, 12)
    rep = _repeated(512 << 10, 3)
    rnew = edited_copy(rep, 4, 6)
    moved = np.concatenate([old[96 << 10:], old[:96 << 10]])           # the first 96 KiB moved to the end
    return {
        "edited": (old, new, _uniform(new.size, 160 << 10), 16 << 10),
        "moved": (old, moved, _uniform(moved.size, 128 << 10), 8 << 10),
        "repeated": (rep, rnew, _uniform(rnew.size, 128 << 10), 0),
        "short_frames": (old[:96 << 10], new[:96 << 10], _uniform(96 << 10, 8 << 10), 4 << 10),
        "one_big_frame": (old, new, [new.size], 1 << 20),
    }


CASES = _cases()


@pytest.mark.parametrize("name", list(CASES))
def test_ranges_follow_the_rule(ctx, name):
    """emulation: the ranges are the restated rule's, and frames hold 0, 1 and many matched anchors"""
    old, new, sizes, m = CASES[name]
    got = ctx.patch_ranges(new, sizes, old, m)
    assert [tuple(int(v) for v in r) for r in got] == ref_ranges(old, new, sizes, m)


def test_anchor_counts_cover_the_cases():
    """the fixtures give frames without an anchor, with one matched anchor, and with several"""
    def matched(name):
        old, new, sizes, _ = CASES[name]
        keys = {k for _, k in anchors(old)}
        per, a = [], 0
        for s in sizes:
            per.append(sum(1 for c, k in anchors(new) if a <= c < a + s and k in keys))
            a += s
        return per
    assert 1 in matched("edited")
    assert matched("one_big_frame")[0] >= 3
    assert 0 in matched("short_frames")


def test_ranges_and_archive_do_not_depend_on_pieces_or_groups(ctx, monkeypatch):
    """emulation: OLD and NEW streamed in 4 KiB pieces and frames grouped by a 64 KiB hull give the same ranges and the same archive"""
    old, new, sizes, m = CASES["edited"]
    want_rg = ctx.patch_ranges(new, sizes, old, m)
    want = ctx.compress_patch_slices(new, sizes, old, 3, True, m)
    monkeypatch.setenv("ZK_PATCH_PIECE_BYTES", "4096")
    monkeypatch.setenv("ZK_PATCH_GROUP_BYTES", str(64 << 10))
    assert ctx.patch_ranges(new, sizes, old, m).tolist() == want_rg.tolist()
    assert ctx.compress_patch_slices(new, sizes, old, 3, True, m) == want


@pytest.mark.parametrize("ck", [False, True])
def test_frames_equal_the_per_frame_call(ctx, ck):
    """emulation: frame f is compress_frames_sized(prefix_ranges=[range], long_distance=True) of frame f alone"""
    old, new, sizes, m = CASES["moved"]
    rg = ctx.patch_ranges(new, sizes, old, m)
    comp, cs, ds = ctx.compress_frames_patch(new, sizes, old, rg, 3, ck)
    co, do = offsets(cs), offsets(ds)
    for f, (lo, hi) in enumerate(rg.tolist()):
        frame = new[int(do[f]):int(do[f + 1])]
        alone = ctx.compress_frames_sized(frame, [frame.size], 3, ck, prefix=old, long_distance=True, prefix_ranges=[(lo, hi)])[0]
        assert comp[int(co[f]):int(co[f + 1])].tobytes() == alone.tobytes(), f


def _split(archive: bytes):
    """archive -> (c_off, d_off, old_len, ranges, slice frame length)"""
    table = zk.SeekTable.from_bytes(archive, zk.Format.Foot)
    co, do = table.offsets()
    old_len, rg, flen = zk.patch_slices_read(archive, table.num_frames())
    return co, do, old_len, rg, flen


def _restores(ctx, archive: bytes, old, new):
    co, do, old_len, rg, flen = _split(archive)
    assert old_len == old.size
    pad = np.frombuffer(archive + b"\0" * 64, dtype=np.uint8)
    back, st, rc = ctx.decompress_frames(pad, co, do, True, prefix=old, prefix_ranges=rg)
    assert rc == 0 and not any(st) and back[: new.size].tobytes() == new.tobytes()
    dec = zk.DecodeOptions(zk.BytesWrapper(archive), ctx).into_decoder()
    out = bytearray()
    buf = bytearray(1 << 16)
    while True:
        k = dec.decompress_with_prefix(buf, old, rg)
        if k == 0:
            break
        out += buf[:k]
    assert bytes(out) == new.tobytes()
    # libzstd refPrefix restores every frame from OLD[lo, hi) alone, and no frame announces a window above 2^27
    for f, (lo, hi) in enumerate(rg.tolist()):
        c0 = int(co[f]) + (flen if f == 0 else 0)
        fr = np.frombuffer(archive[c0:int(co[f + 1])] + b"\0" * 64, dtype=np.uint8)
        n = int(do[f + 1] - do[f])
        out, sizes = O.ref_decompress_frames(fr, [0, int(co[f + 1]) - c0], [0, n], prefix=old[lo:hi] if hi > lo else None)
        assert sizes == [n] and out.tobytes() == new[int(do[f]):int(do[f + 1])].tobytes(), f
        wd = int(fr[5])
        assert (1 << (10 + (wd >> 3))) + ((1 << (10 + (wd >> 3))) >> 3) * (wd & 7) <= REACH, f


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("ck", [False, True])
def test_round_trip(ctx, name, ck):
    old, new, sizes, m = CASES[name]
    archive = ctx.compress_patch_slices(new, sizes, old, 3, ck, m)
    _restores(ctx, archive, old, new)


def test_content_policy(ctx):
    old, new, _, _ = CASES["edited"]
    sizes, _ = ctx.cut_frames_cdc(new, 64 << 10)
    assert len(sizes) > 3
    rg = ctx.patch_ranges(new, sizes, old, 64 << 10)
    assert [tuple(int(v) for v in r) for r in rg] == ref_ranges(old, new, sizes, 64 << 10)
    _restores(ctx, ctx.compress_patch_slices(new, sizes, old, 3, True, 64 << 10), old, new)


def test_one_frame_uploads_its_slice(ctx):
    """restoring one frame through the Decoder uploads its slice of OLD only"""
    old, new, sizes, m = CASES["edited"]
    archive = ctx.compress_patch_slices(new, sizes, old, 3, True, m)
    co, do, _, rg, _ = _split(archive)
    f = len(sizes) // 2
    lo, hi = (int(v) for v in rg[f])
    before = ctx.prefix_bytes_uploaded
    dec = zk.DecodeOptions(zk.BytesWrapper(archive), ctx).lower_frame(f).upper_frame(f).into_decoder()
    buf = bytearray(sizes[f] + 1)
    k = dec.decompress_with_prefix(buf, old, rg)
    assert bytes(buf[:k]) == new[int(do[f]):int(do[f + 1])].tobytes()
    assert 0 < ctx.prefix_bytes_uploaded - before <= hi - lo
    assert hi - lo < old.size


def test_slice_frame_errors(ctx):
    old, new, sizes, m = CASES["short_frames"]
    archive = ctx.compress_patch_slices(new, sizes, old, 3, False, m)
    co, do, old_len, rg, flen = _split(archive)
    n = len(sizes)
    head = bytearray(archive[:flen])
    assert zk.patch_slices_read(bytes(head), n)[0] == old_len

    def bad(b, frames=n):
        with pytest.raises(zk.Error) as e:
            zk.patch_slices_read(bytes(b), frames)
        assert e.value.rc == -1006

    bad(head[: flen - 1])                                    # truncated
    bad(head, n + 1)                                         # n differs from the seek table's
    for at, val in ((0, 0x5E), (4, 0x00), (8, ord("X")), (24, n + 1)):   # magic, payload size, tag, n
        b = bytearray(head); b[at] = val; bad(b)
    b = bytearray(head); b[28:36] = (10 ** 9).to_bytes(8, "little"); bad(b)              # lo > hi
    b = bytearray(head); b[36:44] = (old_len + 1).to_bytes(8, "little"); bad(b)          # hi > old_len
    with pytest.raises(zk.Error):
        zk.patch_slices_write(10, [(5, 4)])
    with pytest.raises(zk.Error):
        ctx.compress_frames_patch(new, sizes, old, [(0, old.size + 1)] * n)


def test_cli(ctx, tmp_path):
    old, new, _, _ = CASES["edited"]
    po = tmp_path / "old.bin"; po.write_bytes(old.tobytes())
    pn = tmp_path / "new.bin"; pn.write_bytes(new.tobytes())
    a, back = tmp_path / "a.zst", tmp_path / "back.bin"
    for policy in ("uncompressed", "content"):
        rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", "-s", "128K", "--frame-size-policy", policy, "--patch-from", po, "--patch-slices",
                                      "--patch-margin", "16K", "-o", a, pn])
        assert rc == 0, err
        sizes = ctx.cut_frames_cdc(new, 128 << 10)[0] if policy == "content" else _uniform(new.size, 128 << 10)
        assert a.read_bytes() == ctx.compress_patch_slices(new, sizes, old, 3, True, 16 << 10)
        rc, _, err = cases._cli(ctx, ["decompress", "-q", "-f", "--patch-apply", po, "-o", back, a])
        assert rc == 0 and back.read_bytes() == new.tobytes(), err
    # one frame from its slice
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "-f", "--from-frame", "2", "--to-frame", "2", "--patch-apply", po, "-o", back, a])
    sizes = ctx.cut_frames_cdc(new, 128 << 10)[0]
    s0 = int(sum(int(s) for s in sizes[:2]))
    assert rc == 0 and back.read_bytes() == new[s0:s0 + int(sizes[2])].tobytes(), err
    # errors: no --patch-apply, a reference of the wrong length
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "-f", "-o", back, a])
    assert rc != 0 and "this archive is a seekable patch; pass --patch-apply" in err
    short = tmp_path / "short.bin"; short.write_bytes(old[:-1].tobytes())
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "-f", "--patch-apply", short, "-o", back, a])
    assert rc != 0 and str(old.size) in err and str(old.size - 1) in err
    # refusals
    for extra, what in ((["--frame-size-policy", "compressed"], "--frame-size-policy"), (["--long-mode"], "--long-mode"),
                        (["--reuse-from", a], "--reuse-from")):
        out = tmp_path / "r.zst"
        rc, _, err = cases._cli(ctx, ["compress", "-q", "--patch-from", po, "--patch-slices", *extra, "-o", out, pn])
        assert rc != 0 and what in err and not out.exists(), (extra, err)
    rc, _, err = cases._cli(ctx, ["compress", "-q", "--patch-slices", "-o", tmp_path / "s.zst", pn])
    assert rc != 0 and "--patch-from" in err
    rc, _, err = cases._cli(ctx, ["compress", "-q", "--long", "--patch-from", po, "--frame-size-policy", "content", "-o", tmp_path / "t.zst", pn])
    assert rc != 0 and "--long needs --frame-size-policy uncompressed" in err


@pytest.mark.gpu
def test_headline(gpu_lib, monkeypatch):
    """OLD: 384 MiB of the bench's mix; NEW: OLD with 64 small edits and its first 8 MiB moved to the end; 2 MiB frames.  The slice patch is
    a fraction of NEW's plain archive and the whole-prefix --long patch, which cannot reach OLD's first 256 MiB, is several times larger.
    The bounds are the H100 run of DESIGN §6 with some room (the bytes are deterministic): 15.3 % of plain, 3.2x smaller than whole-prefix.
    The mix repeats dickens.txt slices, so many anchor keys recur in OLD and the nearest one is often another copy"""
    from zeekstd_b200 import corpus
    ctx = zk.Context(0, gpu_lib)
    n = 384 << 20
    old = corpus.make_mix(n, seed=1, segment=64 << 10).numpy()
    new = old.copy()
    rng = np.random.default_rng(9)
    for at in rng.integers(0, n - 64, 64):
        new[at:at + 32] = rng.integers(0, 256, 32, dtype=np.uint8)
    new = np.concatenate([new[8 << 20:], new[:8 << 20]])
    fs = 2 << 20
    sizes = _uniform(new.size, fs)
    plain = ctx.compress_frames_sized(new, sizes, 16, True)[0].size
    archive = ctx.compress_patch_slices(new, sizes, old, 16, True, fs)
    whole = ctx.compress_frames(new, fs, 16, True, prefix=old, long_distance=True)[0].size
    print(f"headline (H100): plain {plain}, slices {len(archive)}, whole-prefix --long {whole}")
    assert len(archive) <= 0.17 * plain
    assert whole >= 3 * len(archive)
    _restores(ctx, archive, old, new)
    # pieces and groups forced small: the same archive
    monkeypatch.setenv("ZK_PATCH_PIECE_BYTES", str(48 << 20))
    monkeypatch.setenv("ZK_PATCH_GROUP_BYTES", str(40 << 20))
    assert ctx.compress_patch_slices(new, sizes, old, 16, True, fs) == archive
    ctx.close()


@pytest.mark.gpu
def test_small_case_against_whole_prefix(gpu_lib):
    """test_patch_ldm's small case (OLD < 128 MiB, every frame reaches all of it): slices cost at most 1.5x the whole-prefix patch"""
    ctx = zk.Context(0, gpu_lib)
    old = _mix(8 << 20, 3)
    new = edited_copy(old, 11, 200)
    fs = 2 << 20
    sizes = _uniform(new.size, fs)
    archive = ctx.compress_patch_slices(new, sizes, old, 16, True)
    whole = ctx.compress_frames(new, fs, 16, True, prefix=old, long_distance=True)[0].size
    print(f"small case (H100): slices {len(archive)}, whole-prefix --long {whole}")
    assert len(archive) <= 1.5 * whole
    _restores(ctx, archive, old, new)
    ctx.close()
