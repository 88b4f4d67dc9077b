"""Compressing a new version against the archive of the previous one (zk_compress_frames_sized_reuse, Context.compress_frames_reuse,
`compress --reuse-from`) and the cut-only entry point (zk_cut_frames_cdc, Context.cut_frames_cdc).  The output is checked against
compress_frames_sized on the same frames byte for byte, `reused[]` against the rule restated in numpy (the lowest-index old entry of the
frame's size and key, copied iff its bytes are the frame's), foreign old archives against libzstd and the codec's decoder.  Every case runs
on the emulation build (`-m "not gpu"`, small inputs) and on the H100 (`-m gpu`, MiB-scale)."""
import ctypes

import numpy as np
import pytest

import cases
import zeekstd_b200 as zk
from golden.make_encoder_golden_ldm import edited_copy
from oracle import oracle as O
from util import offsets
from zeekstd_b200 import _native, corpus

KIB = 1 << 10
NONE = 0xFFFFFFFF


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    return request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib")


@pytest.fixture(scope="module")
def ctx(lib):
    _native.set_default_lib(lib)
    c = zk.Context(0, lib)
    yield c
    c.close()


def _emul(ctx) -> bool:
    return "emul" in ctx.lib._name


def _scale(ctx, emul: int, gpu: int) -> int:
    return emul if _emul(ctx) else gpu


def _mix(n: int, seed: int) -> np.ndarray:
    return corpus.as_numpy(corpus.make_mix(n, seed=seed, segment=16 * KIB))


def _uniform(n: int, s: int) -> np.ndarray:
    sizes = [s] * (n // s) + ([n % s] if n % s or n == 0 else [])
    return np.array(sizes, dtype=np.uint32)


def _seekable(comp, c_sizes, d_sizes) -> bytes:
    st = zk.SeekTable()
    for c, d in zip(np.asarray(c_sizes).tolist(), np.asarray(d_sizes).tolist()):
        st.log_frame(int(c), int(d))
    return bytes(np.asarray(comp, dtype=np.uint8).tobytes()) + st.into_serializer().to_bytes()


def _archive(ctx, x, sizes, level, checksum, long_mode=False) -> bytes:
    comp, cs, _ = ctx.compress_frames_sized(x, sizes, level, checksum, long_mode=long_mode)
    return _seekable(comp, cs, sizes)


def _frames(x, sizes):
    o = offsets(sizes)
    return [x[int(o[i]): int(o[i + 1])].tobytes() for i in range(len(sizes))]


def _predict(old_x, old_sizes, new_x, new_sizes, any_key: bool = False):
    """reused[] by the rule, every old entry decodable with a matching flag.  Full keys: the lowest-index old entry of equal bytes (a key
    collision between different bytes of one size is not expected).  any_key (ZK_REUSE_KEY_BITS=0): the lowest-index entry of equal size,
    copied only when its bytes are equal"""
    first_bytes, first_size = {}, {}
    for g, b in enumerate(_frames(old_x, old_sizes)):
        first_bytes.setdefault(b, g)
        first_size.setdefault(len(b), g)
    olds = _frames(old_x, old_sizes)
    out = []
    for b in _frames(new_x, new_sizes):
        if any_key:
            g = first_size.get(len(b))
            out.append(g if g is not None and olds[g] == b else NONE)
        else:
            out.append(first_bytes.get(b, NONE))
    return out


def _restores(ctx, x, comp, cs, ds):
    pad = np.concatenate([np.asarray(comp, dtype=np.uint8), np.zeros(64, np.uint8)])
    out, got = O.ref_decompress_frames(pad, offsets(cs), offsets(ds))
    assert out.tobytes() == x.tobytes() and got == [int(d) for d in ds]
    back, st, rc = ctx.decompress_frames(pad, offsets(cs), offsets(ds), True)
    assert rc == 0 and not any(st) and back[: x.size].tobytes() == x.tobytes()


def _copied_verbatim(old_arch: bytes, comp, cs, reused):
    """every reused frame of the output is the old entry's bytes"""
    co, _ = zk.SeekTable.from_bytes(old_arch).offsets()
    o = offsets(cs)
    comp = np.asarray(comp, dtype=np.uint8).tobytes()
    for f, g in enumerate(np.asarray(reused).tolist()):
        if g != NONE:
            assert comp[int(o[f]): int(o[f + 1])] == old_arch[int(co[g]): int(co[g + 1])]


def _pair(ctx, seed=7):
    old = _mix(_scale(ctx, 96 * KIB, 32 << 20), seed)
    new = edited_copy(old, seed + 1, _scale(ctx, 3, 24))
    s = _scale(ctx, 4096, 16 * KIB)
    return old, new, ctx.cut_frames_cdc(old, s)[0], ctx.cut_frames_cdc(new, s)[0]


# ---- 1. the same bytes as a fresh compress -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level,checksum,long_mode", [(-3, True, False), (1, False, False), (3, True, False), (3, False, False),
                                                      (13, True, False), (19, False, False), (19, True, False), (3, True, True)])
def test_same_bytes_as_a_fresh_compress(ctx, level, checksum, long_mode):
    old, new, osz, nsz = _pair(ctx)
    arch = _archive(ctx, old, osz, level, checksum, long_mode)
    full, fcs, _ = ctx.compress_frames_sized(new, nsz, level, checksum, long_mode=long_mode)
    comp, cs, reused = ctx.compress_frames_reuse(new, nsz, arch, level, checksum, long_mode)
    assert comp.tobytes() == full.tobytes() and cs.tolist() == fcs.tolist()
    want = _predict(old, osz, new, nsz)
    assert reused.tolist() == want
    share = sum(g != NONE for g in want) / len(want)
    assert share > (0.5 if _emul(ctx) else 0.9), share
    _copied_verbatim(arch, comp, cs, reused)


# ---- 2. uniform frames ---------------------------------------------------------------------------------------------------------------
def test_uniform_frames(ctx):
    s = _scale(ctx, 8 * KIB, 256 * KIB)
    old = _mix(_scale(ctx, 80 * KIB, 16 << 20), 3)
    new = edited_copy(old, 4, 2)
    osz, nsz = _uniform(old.size, s), _uniform(new.size, s)
    arch = _archive(ctx, old, osz, 3, True)
    full, fcs, _ = ctx.compress_frames_sized(new, nsz, 3, True)
    comp, cs, reused = ctx.compress_frames_reuse(new, nsz, arch, 3, True)
    assert comp.tobytes() == full.tobytes() and reused.tolist() == _predict(old, osz, new, nsz)
    first = int(np.flatnonzero(old[: min(old.size, new.size)] != new[: min(old.size, new.size)])[0])
    assert all(reused[f] == f for f in range(first // s))
    # an overwrite in place keeps every other frame
    ov = old.copy(); ov[s + 5: s + 9] ^= 0x5A
    comp, cs, reused = ctx.compress_frames_reuse(ov, osz, arch, 3, True)
    assert comp.tobytes() == ctx.compress_frames_sized(ov, osz, 3, True)[0].tobytes()
    assert reused.tolist() == [NONE if f == 1 else f for f in range(len(osz))]


# ---- 3. the verification path --------------------------------------------------------------------------------------------------------
def test_every_equal_size_entry_is_a_candidate_without_keys(ctx, monkeypatch):
    s = 4096
    old = _mix(_scale(ctx, 48 * KIB, 8 << 20), 5)
    osz = _uniform(old.size, s)
    fr = _frames(old, osz)
    # frames equal to old entry 0, to later old entries (the lowest candidate, entry 0, differs: not reused), and new bytes
    picks = [0, 3, 0, 2, len(osz) - 1, 0]
    new = np.frombuffer(b"".join(fr[p] if p < len(osz) - 1 else bytes(s) for p in picks) + bytes(100), dtype=np.uint8)
    nsz = _uniform(new.size, s)
    arch = _archive(ctx, old, osz, 3, True)
    full = ctx.compress_frames_sized(new, nsz, 3, True)[0].tobytes()
    monkeypatch.setenv("ZK_REUSE_KEY_BITS", "0")
    comp, cs, reused = ctx.compress_frames_reuse(new, nsz, arch, 3, True)
    assert comp.tobytes() == full
    want = _predict(old, osz, new, nsz, any_key=True)
    assert reused.tolist() == want and want[:4] == [0, NONE, 0, NONE]
    # the CDC pair: same bytes, and the rule's prediction
    old, new, osz, nsz = _pair(ctx, 9)
    arch = _archive(ctx, old, osz, 1, False)
    comp, cs, reused = ctx.compress_frames_reuse(new, nsz, arch, 1, False)
    assert comp.tobytes() == ctx.compress_frames_sized(new, nsz, 1, False)[0].tobytes()
    assert reused.tolist() == _predict(old, osz, new, nsz, any_key=True)


# ---- 4. foreign old entries ----------------------------------------------------------------------------------------------------------
def _changed_in_place(old, s, every=3):
    new = old.copy()
    for f in range(0, old.size // s, every):
        new[f * s + 7] ^= 0xA5
    return new


def test_foreign_old_entries(ctx):
    s = 8 * KIB
    old = _mix(_scale(ctx, 64 * KIB, 8 << 20), 11)
    new = _changed_in_place(old, s)
    osz = _uniform(old.size, s)
    want = _predict(old, osz, new, osz)
    assert any(g != NONE for g in want) and any(g == NONE for g in want)
    # another level, and libzstd: copied as they are
    frames, rcs, rds = O.ref_compress_frames(old, s, 3, True)
    for arch in (_archive(ctx, old, osz, 1, True), _seekable(np.frombuffer(b"".join(frames), np.uint8), rcs, rds)):
        comp, cs, reused = ctx.compress_frames_reuse(new, osz, arch, 3, True)
        assert reused.tolist() == want
        _copied_verbatim(arch, comp, cs, reused)
        _restores(ctx, new, comp, cs, osz)
    # the other checksum flag: nothing is reused
    arch = _archive(ctx, old, osz, 3, False)
    comp, cs, reused = ctx.compress_frames_reuse(new, osz, arch, 3, True)
    assert (reused == NONE).all() and comp.tobytes() == ctx.compress_frames_sized(new, osz, 3, True)[0].tobytes()


# ---- 5. edges ------------------------------------------------------------------------------------------------------------------------
def test_empty_inputs_and_frames(ctx):
    old = _mix(40 * KIB, 13)
    osz = np.array([4096, 0, 9000, 0, old.size - 13096], dtype=np.uint32)
    arch = _archive(ctx, old, osz, 3, True)
    comp, cs, reused = ctx.compress_frames_reuse(b"", [], arch, 3, True)
    assert comp.size == 0 and cs.size == 0 and reused.size == 0
    comp, cs, reused = ctx.compress_frames_reuse(b"", [0], arch, 3, True)
    assert reused.tolist() == [1] and comp.tobytes() == ctx.compress_frames_sized(b"", [0], 3, True)[0].tobytes()
    new = np.concatenate([old[4096:13096], old[:4096]])
    nsz = np.array([0, 9000, 0, 4096, 0], dtype=np.uint32)
    comp, cs, reused = ctx.compress_frames_reuse(new, nsz, arch, 3, True)
    assert reused.tolist() == [1, 2, 1, 0, 1] and comp.tobytes() == ctx.compress_frames_sized(new, nsz, 3, True)[0].tobytes()
    empty_arch = zk.SeekTable().into_serializer().to_bytes()
    comp, cs, reused = ctx.compress_frames_reuse(new, nsz, empty_arch, 3, True)
    assert (reused == NONE).all() and comp.tobytes() == ctx.compress_frames_sized(new, nsz, 3, True)[0].tobytes()


def test_corrupted_old_entry_is_not_reused(ctx):
    s = 8 * KIB
    old = _mix(_scale(ctx, 48 * KIB, 4 << 20), 17)
    osz = _uniform(old.size, s)
    comp0, cs0, _ = ctx.compress_frames_sized(old, osz, 3, True)
    o = offsets(cs0)
    # the last byte (the content checksum: the entry fails to decode) and the first (the magic: no zstd frame)
    for g, at in ((1, int(o[2]) - 1), (3, int(o[3]))):
        bad = comp0.copy()
        bad[at] ^= 0x40
        arch = _seekable(bad, cs0, osz)
        comp, cs, reused = ctx.compress_frames_reuse(old, osz, arch, 3, True)
        # the mix repeats itself, so a frame may copy an earlier entry of equal bytes: the lowest one other than g
        first = {}
        for h, b in enumerate(_frames(old, osz)):
            if h != g:
                first.setdefault(b, h)
        assert g not in reused.tolist() and reused.tolist() == [first.get(b, NONE) for b in _frames(old, osz)]
        assert comp.tobytes() == comp0.tobytes()


def test_own_archive_is_reused_whole(ctx):
    """every frame copies an old entry (the lowest of equal bytes: the mix repeats itself), and the output is the archive's bytes"""
    old, _, osz, _ = _pair(ctx, 21)
    comp0, cs0, _ = ctx.compress_frames_sized(old, osz, 19, True)
    comp, cs, reused = ctx.compress_frames_reuse(old, osz, _seekable(comp0, cs0, osz), 19, True)
    assert reused.tolist() == _predict(old, osz, old, osz) and comp.tobytes() == comp0.tobytes() and cs.tolist() == cs0.tolist()
    assert all(g <= f for f, g in enumerate(reused.tolist()))


def test_small_sub_batches_give_the_same_bytes(ctx, monkeypatch):
    old, new, osz, nsz = _pair(ctx, 23)
    arch = _archive(ctx, old, osz, 3, True)
    want = ctx.compress_frames_reuse(new, nsz, arch, 3, True)
    monkeypatch.setenv("ZK_HOST_SUB_BYTES_ENC", str(_scale(ctx, 10 * KIB, 1 << 20)))
    monkeypatch.setenv("ZK_HOST_SUB_BYTES", str(_scale(ctx, 7 * KIB, 512 * KIB)))
    got = ctx.compress_frames_reuse(new, nsz, arch, 3, True)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(want, got))


def _raw_call(ctx, new, nsz, old: bytes, co, do, dst_cap, old_len=None):
    lib = ctx.lib
    ds = np.ascontiguousarray(nsz, dtype=np.uint32)
    co = np.ascontiguousarray(co, dtype=np.uint64); do = np.ascontiguousarray(do, dtype=np.uint64)
    ob = np.frombuffer(old, np.uint8)
    dst = np.zeros(dst_cap + 64, np.uint8)
    cs = np.zeros(ds.size, np.uint32); ru = np.zeros(ds.size, np.uint32); dl = ctypes.c_size_t()
    rc = lib.zk_compress_frames_sized_reuse(ctx._h, new.ctypes.data, ds.ctypes.data_as(_native.u32p), ds.size, 3, 1, 0, ob.ctypes.data,
                                            ob.size if old_len is None else old_len, co.ctypes.data_as(_native.u64p),
                                            do.ctypes.data_as(_native.u64p), len(co) - 1, dst.ctypes.data, dst_cap,
                                            cs.ctypes.data_as(_native.u32p), ru.ctypes.data_as(_native.u32p), ctypes.byref(dl))
    return rc, dst[: dl.value]


def test_argument_errors_and_capacity(ctx):
    s = 8 * KIB
    old = _mix(40 * KIB, 29)
    new = _changed_in_place(old, s, 2)
    osz = _uniform(old.size, s)
    arch = _archive(ctx, old, osz, 3, True)
    co, do = zk.SeekTable.from_bytes(arch).offsets()
    bad_c = co.copy(); bad_c[2], bad_c[3] = bad_c[3], bad_c[2]
    bad_d = do.copy(); bad_d[1] = bad_d[2] + 1
    assert _raw_call(ctx, new, osz, arch, bad_c, do, 1 << 20)[0] == -1006
    assert _raw_call(ctx, new, osz, arch, co, bad_d, 1 << 20)[0] == -1006
    assert _raw_call(ctx, new, osz, arch, co, do, 1 << 20, old_len=int(co[-1]) - 1)[0] == -1006
    assert _raw_call(ctx, new, osz, arch, co, do, 1 << 20, old_len=int(co[-1]))[0] == 0
    bound = int(ctx.lib.zk_compress_bound_sized(np.ascontiguousarray(osz).ctypes.data_as(_native.u32p), osz.size)) + int(co[-1] - co[0])
    rc, out = _raw_call(ctx, new, osz, arch, co, do, bound)
    assert rc == 0 and out.tobytes() == ctx.compress_frames_sized(new, osz, 3, True)[0].tobytes()
    assert _raw_call(ctx, new, osz, arch, co, do, out.size - 1)[0] == -70
    assert _raw_call(ctx, new, osz, arch, co, do, out.size)[0] == 0


# ---- 6. the cut-only entry point -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [4096, 16 * KIB])
def test_cut_only_equals_the_compress_call(ctx, s):
    x = _mix(_scale(ctx, 150 * KIB, 24 << 20), 31)
    for n in (0, 1000, x.size // 2, x.size):
        for final in (True, False):
            _, _, ds, used = ctx.compress_frames_cdc(x[:n], s, 1, False, final=final)
            got, got_used = ctx.cut_frames_cdc(x[:n], s, final)
            assert got.tolist() == ds.tolist() and got_used == used


# ---- 7. the CLI ----------------------------------------------------------------------------------------------------------------------
def test_cli(ctx, tmp_path):
    old, new, _, _ = _pair(ctx, 37)
    po = tmp_path / "old.bin"; po.write_bytes(old.tobytes())
    pn = tmp_path / "new.bin"; pn.write_bytes(new.tobytes())
    oz = tmp_path / "old.zst"
    for args in (["--frame-size-policy", "content", "-s", "16K"], ["-s", "16K", "--no-checksum", "-l", "1"], ["-s", "64K", "--long-mode"]):
        rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", *args, "-o", oz, po])
        assert rc == 0, err
        plain, reuse, back = tmp_path / "plain.zst", tmp_path / "reuse.zst", tmp_path / "back.bin"
        rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", *args, "-o", plain, pn])
        assert rc == 0, err
        rc, _, err = cases._cli(ctx, ["compress", "-f", *args, "--reuse-from", oz, "-o", reuse, pn])
        assert rc == 0 and "reused " in err and reuse.read_bytes() == plain.read_bytes(), err
        rc, _, err = cases._cli(ctx, ["decompress", "-q", "-f", "-o", back, reuse])
        assert rc == 0 and back.read_bytes() == new.tobytes(), err
    # a separate seek table, as plain compress writes it
    for name, extra in (("plain", []), ("reuse", ["--reuse-from", oz])):
        rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", "-s", "16K", "--seek-table-file", tmp_path / f"{name}.st", *extra,
                                      "-o", tmp_path / f"{name}.zst", pn])
        assert rc == 0, err
    assert (tmp_path / "plain.zst").read_bytes() == (tmp_path / "reuse.zst").read_bytes()
    assert (tmp_path / "plain.st").read_bytes() == (tmp_path / "reuse.st").read_bytes()
    # refusals
    out = tmp_path / "x.zst"
    for args, msg in ((["--patch-from", po], "--reuse-from cannot be used with --patch-from"),
                      (["--patch-from", po, "--long"], "--reuse-from cannot be used with --patch-from"),
                      (["--long"], "--long needs --patch-from"),
                      (["--frame-size-policy", "compressed", "-s", "16K"], "--reuse-from needs --frame-size-policy uncompressed or content"),
                      (["--frame-size-policy", "content", "--long-mode"], "--long-mode needs --frame-size-policy uncompressed")):
        rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", *args, "--reuse-from", oz, "-o", out, pn])
        assert rc != 0 and msg in err and "Traceback" not in err, err
    # an old file without a Foot seek table
    rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", "--reuse-from", po, "-o", out, pn])
    assert rc == 1 and "not a seekable archive" in err, err


# ---- 8. large frames (GPU only) ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_large_frames(gpu_lib):
    _native.set_default_lib(gpu_lib)
    ctx = zk.Context(0, gpu_lib)
    try:
        # frames above 64 MiB: the key, the compare and the copies cross thousands of 32 KiB work items
        old = _mix(200 << 20, 41)
        osz = np.array([(80 << 20) + 13, 3, (70 << 20) - 5, old.size - (150 << 20) - 11], dtype=np.uint32)
        new = old.copy(); new[(130 << 20) + 23] ^= 1                 # 50 MiB into the third frame
        arch = _archive(ctx, old, osz, 3, True)
        comp, cs, reused = ctx.compress_frames_reuse(new, osz, arch, 3, True)
        assert reused.tolist() == [0, 1, NONE, 3]
        assert comp.tobytes() == ctx.compress_frames_sized(new, osz, 3, True)[0].tobytes()
        # one call of more than 1 GiB, content-defined frames
        old = _mix((1 << 30) + (5 << 20), 43)
        new = edited_copy(old, 44, 40)
        osz, nsz = ctx.cut_frames_cdc(old, 2 << 20)[0], ctx.cut_frames_cdc(new, 2 << 20)[0]
        arch = _archive(ctx, old, osz, 1, False)
        comp, cs, reused = ctx.compress_frames_reuse(new, nsz, arch, 1, False)
        assert comp.tobytes() == ctx.compress_frames_sized(new, nsz, 1, False)[0].tobytes()
        assert reused.tolist() == _predict(old, osz, new, nsz)
    finally:
        ctx.close()
