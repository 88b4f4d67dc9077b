"""Content-defined frames (FrameSizePolicy::ContentDefined(s), zk_compress_frames_cdc[_dev], Context.compress_frames_cdc): frame ends are
chosen by a 64-byte gear hash of the input, so an edit changes only the frames around it.  The frame sizes are checked against a numpy
restatement of the rule; the archive against compress_frames_sized with the same sizes (byte for byte), libzstd and the codec's decoder;
the cut against every way of splitting the work (sub-batches, a tiny candidate capacity, chunked calls, Encoder writes); the point of the
feature on edited copies; the CLI; pinned bytes.  Every case runs on the emulation build (`-m "not gpu"`, small inputs) and on the H100
(`-m gpu`, MiB-scale)."""
import ctypes
import hashlib
import io
import json
import os

import numpy as np
import pytest

import cases
import zeekstd_b200 as zk
from golden.make_encoder_golden_ldm import edited_copy
from oracle import oracle as O
from test_high_levels import _data
from test_sized_frames import LEVELS
from util import GOLDEN, offsets
from zeekstd_b200 import _native, corpus

M64 = (1 << 64) - 1
KIB = 1 << 10


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


# ---- the rule, restated ----------------------------------------------------------------------------------------------------------------
def _gear() -> np.ndarray:
    """splitmix64 of b + 1 for every byte value b (zkc_ldm_gear)"""
    z = (np.arange(256, dtype=np.uint64) + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


GEAR = _gear()


def _hashes(x: np.ndarray) -> np.ndarray:
    """h_p = sum over j = max(0, p - 63) .. p of gear(x_j) * 2^(p - j) mod 2^64, as 64 shifted adds"""
    g = GEAR[x]
    h = np.zeros(x.size, np.uint64)
    for k in range(min(64, x.size)):
        h[k:] += g[: x.size - k] << np.uint64(k)
    return h


def _rule(s: int):
    s = min(max(s, 4096), 1 << 30)
    mn, mx = s // 4, min(4 * s, 1 << 30)
    return mn, mx, (1 << 64) - M64 // (s - mn)


def _cut(x: np.ndarray, s: int, final: bool = True, h=None):
    """-> (frame sizes, consumed) by the rule; h: _hashes(x) if already known"""
    mn, mx, thr = _rule(s)
    n = x.size
    cand = np.flatnonzero((_hashes(x) if h is None else h) >= np.uint64(thr))
    sizes, b = [], 0
    while b < n:
        i = int(np.searchsorted(cand, b + mn - 1))
        if i < cand.size and cand[i] <= b + mx - 1:
            end = int(cand[i]) + 1
        elif b + mx <= n:
            end = b + mx
        else:
            if final:
                sizes.append(n - b); b = n
            break
        if end == n and not final:
            break
        sizes.append(end - b); b = end
    if n == 0 and final:
        sizes = [0]
    return sizes, b


def _bench_mix(n: int, seed: int) -> np.ndarray:
    return corpus.as_numpy(corpus.make_mix(n, seed=seed, segment=16 * KIB))


def _restores(ctx, x, comp, cs, ds):
    pad = np.concatenate([comp, np.zeros(64, np.uint8)])
    out, got = O.ref_decompress_frames(pad, offsets(cs), offsets(ds))
    assert out.tobytes() == x.tobytes() and got == [int(d) for d in ds]
    back, st, rc = ctx.decompress_frames(pad, offsets(cs), offsets(ds), True)
    assert rc == 0 and not any(st) and back[: x.size].tobytes() == x.tobytes()


def test_constant_runs_never_hold_a_candidate():
    """a run of byte b hashes to 2^64 - gear(b); the loosest threshold (s = 4096) is 2^64 - T with T < min gear"""
    run_hash = [(1 << 64) - int(g) for g in GEAR]
    loosest = _rule(4096)[2]
    assert max(run_hash) < loosest
    assert max(run_hash) == (1 << 64) - int(GEAR.min()) and 8.0e16 < int(GEAR.min()) < 8.2e16 and 5.9e15 < (1 << 64) - loosest < 6.1e15


@pytest.mark.parametrize("kind", ["dickens", "mix", "random"])
def test_sizes_follow_the_rule(ctx, kind):
    n = _scale(ctx, 200 * KIB, 16 << 20)
    x = {"dickens": lambda: _data("dickens", n), "mix": lambda: _bench_mix(n, 3), "random": lambda: _data("random", n, 4)}[kind]()
    h = _hashes(x)
    for s in ((1000, 4096, 5000, 12345) if _emul(ctx) else (1000, 64 * KIB, 100_000, 1 << 20)):
        for final in (True, False):
            comp, cs, ds, used = ctx.compress_frames_cdc(x, s, 1, False, final=final)
            want, wused = _cut(x, s, final, h)
            assert list(ds) == want and used == wused, (kind, s, final)
            assert int(np.sum(ds)) == used
        if s >= 4096:
            mn, mx, _ = _rule(s)
            assert all(mn <= d <= mx for d in want[:-1])


def test_constant_runs_are_cut_at_mx(ctx):
    s = 4096
    mn, mx, _ = _rule(s)
    n = _scale(ctx, 5 * mx + 777, 3 * (1 << 20) + 777)
    for v in (0, 0xFF, ord("a")):
        x = np.full(n, v, np.uint8)
        comp, cs, ds, _ = ctx.compress_frames_cdc(x, s, 3, True)
        assert list(ds) == [mx] * (n // mx) + [n % mx], v
        _restores(ctx, x, comp, cs, ds)
    # a run inside text: cut at mx from the last frame end before it
    x = np.concatenate([_data("dickens", 30_000), np.zeros(4 * mx + 10, np.uint8), _data("dickens", 20_000)])
    comp, cs, ds, _ = ctx.compress_frames_cdc(x, s, 3, False)
    assert list(ds) == _cut(x, s)[0] and mx in list(ds)


@pytest.mark.parametrize("s", [1000, 6000])
def test_input_lengths_at_the_limits(ctx, s):
    mn, mx, _ = _rule(s)
    x = _bench_mix(mx + 5000, 8)
    for n in (0, 1, mn - 1, mn, mx - 1, mx, mx + 1):
        for final in (True, False):
            comp, cs, ds, used = ctx.compress_frames_cdc(x[:n], s, 3, True, final=final)
            want, wused = _cut(x[:n], s, final)
            assert list(ds) == want and used == wused, (n, final)
            if final:
                _restores(ctx, x[:n], comp, cs, ds)
            else:
                assert comp.size == int(np.sum(cs))
    # a frame that ends exactly at the end of the input stays open without final
    ds = _cut(x, s)[0]
    end = int(np.sum(ds[:2]))
    assert ctx.compress_frames_cdc(x[:end], s, 3, False, final=False)[2].tolist() == ds[:1]
    assert ctx.compress_frames_cdc(x[:end], s, 3, False, final=True)[2].tolist() == ds[:2]


@pytest.mark.parametrize("level", LEVELS)
def test_same_bytes_as_the_sized_path(ctx, level):
    n = _scale(ctx, 60_000, 6 << 20)
    x = _data("text", n, level & 0xFF)
    prefix = _data("text", 50_000, 77)
    s = _scale(ctx, 5000, 256 * KIB)
    combos = [(False, None), (True, prefix)] if _emul(ctx) else [(False, None), (True, None), (False, prefix), (True, prefix)]
    for checksum, pf in combos:
        comp, cs, ds, used = ctx.compress_frames_cdc(x, s, level, checksum, pf)
        assert list(ds) == _cut(x, s)[0] and used == n
        ref, rcs, rds = ctx.compress_frames_sized(x, ds, level, checksum, pf)
        assert comp.tobytes() == ref.tobytes() and list(cs) == list(rcs), (level, checksum, pf is None)
        if pf is None:
            _restores(ctx, x, comp, cs, ds)


def test_seek_table_lists_the_frames(ctx):
    x = _bench_mix(_scale(ctx, 150 * KIB, 8 << 20), 5)
    s = _scale(ctx, 8192, 128 * KIB)
    comp, cs, ds, _ = ctx.compress_frames_cdc(x, s, 3, True)
    sink = io.BytesIO()
    enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.ContentDefined(s)).checksum_flag(True).compression_level(3).into_encoder(sink)
    enc.compress(x.tobytes()); enc.finish()
    arch = sink.getvalue()
    assert arch[: comp.size] == comp.tobytes()
    st = zk.SeekTable.from_bytes(arch)
    assert [st.frame_size_decomp(i) for i in range(st.num_frames())] == list(ds)
    assert [st.frame_size_comp(i) for i in range(st.num_frames())] == list(cs)
    dec = zk.DecodeOptions(arch, ctx).into_decoder()
    assert dec.read_all() == x.tobytes()


def test_sub_batches_and_capacity_do_not_change_the_output(ctx, monkeypatch):
    x = np.concatenate([_bench_mix(_scale(ctx, 120 * KIB, 12 << 20), 6), np.zeros(_scale(ctx, 70_000, 3 << 20), np.uint8),
                        _data("text", _scale(ctx, 40_000, 2 << 20), 6)])
    for s in (_scale(ctx, 4096, 64 * KIB), _scale(ctx, 20_000, 1 << 20)):
        ref = ctx.compress_frames_cdc(x, s, 1, True)
        assert list(ref[2]) == _cut(x, s)[0]
        for env, val in (("ZK_HOST_SUB_BYTES_ENC", 5000), ("ZK_HOST_SUB_BYTES_ENC", 100_000), ("ZK_CDC_CAP", 1), ("ZK_CDC_CAP", 3)):
            monkeypatch.setenv(env, str(val))
            got = ctx.compress_frames_cdc(x, s, 1, True)
            monkeypatch.delenv(env)
            assert got[0].tobytes() == ref[0].tobytes() and list(got[1]) == list(ref[1]) and list(got[2]) == list(ref[2]), (s, env, val)


def test_periodic_input_truncates_the_candidate_list(ctx, monkeypatch):
    """two bytes repeated, chosen so that one phase is a candidate: every other position is one (32 times the default capacity), and
    every frame has exactly mn bytes"""
    s = 4096
    mn, _, thr = _rule(s)
    pair = next((a, b) for a in range(256) for b in range(256) if a != b and _hashes(np.array([a, b] * 40, np.uint8))[-1] >= np.uint64(thr))
    n = _scale(ctx, 40 * mn + 5, 4096 * mn + 5)
    x = np.resize(np.array(pair, np.uint8), n)
    comp, cs, ds, _ = ctx.compress_frames_cdc(x, s, 3, False)
    want = _cut(x, s)[0]
    assert list(ds) == want and want[:-1] == [mn] * (len(want) - 1) and len(want) == n // 1024 + 1
    monkeypatch.setenv("ZK_CDC_CAP", "2")
    assert ctx.compress_frames_cdc(x, s, 3, False)[0].tobytes() == comp.tobytes()


def test_chunked_calls_give_the_same_frames(ctx):
    n = _scale(ctx, 160 * KIB, 12 << 20)
    x = _bench_mix(n, 9)
    s = _scale(ctx, 6000, 100_000)
    whole, cs0, ds0, _ = ctx.compress_frames_cdc(x, s, 3, True)
    rng = np.random.default_rng(7)
    parts, cs, ds = [], [], []
    rest, pos = x[:0], 0
    while pos < n:
        k = int(rng.integers(1, max(2, n // 5)))
        buf = np.concatenate([rest, x[pos:pos + k]]); pos += k
        comp, c, d, used = ctx.compress_frames_cdc(buf, s, 3, True, final=False)
        assert int(np.sum(d)) == used and used < max(buf.size, 1)
        parts.append(comp.tobytes()); cs += list(c); ds += list(d)
        rest = buf[used:]
    comp, c, d, used = ctx.compress_frames_cdc(rest, s, 3, True)
    assert used == rest.size
    parts.append(comp.tobytes()); cs += list(c); ds += list(d)
    assert b"".join(parts) == whole.tobytes() and cs == list(cs0) and ds == list(ds0)


def test_encoder_write_sizes_do_not_matter(ctx):
    x = _bench_mix(_scale(ctx, 100 * KIB, 6 << 20), 10)
    s = _scale(ctx, 5000, 64 * KIB)
    comp, cs, ds, _ = ctx.compress_frames_cdc(x, s, 3, False)
    rng = np.random.default_rng(3)
    data = x.tobytes()
    archives = set()
    for trial in range(3):
        sink = io.BytesIO()
        enc = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.ContentDefined(s)).compression_level(3).into_encoder(sink)
        p = 0
        while p < len(data):
            k = int(rng.integers(1, len(data) // (2 + 10 * trial) + 2))
            enc.compress(data[p:p + k]); p += k
        enc.finish()
        archives.add(sink.getvalue())
    assert len(archives) == 1
    assert archives.pop()[: comp.size] == comp.tobytes()


def test_refusals(ctx):
    opts = zk.EncodeOptions(ctx).frame_size_policy(zk.FrameSizePolicy.ContentDefined(64 * KIB))
    with pytest.raises(zk.Error) as e:
        opts.into_raw_encoder()
    assert e.value.rc == -1006
    with pytest.raises(zk.Error) as e:
        opts.long_distance_matching(True).into_encoder(io.BytesIO())
    assert e.value.rc == -1006
    lib = ctx.lib
    o = lib.zk_encode_options_new(ctx._h)
    lib.zk_encode_options_frame_size_policy(o, zk.FrameSizePolicy.CONTENT, 4096)
    h = ctypes.c_void_p()
    assert lib.zk_encode_options_into_raw_encoder(o, ctypes.byref(h)) == -1006
    lib.zk_encode_options_free(o)                                           # not consumed by the refusal


def test_documented_capacities_suffice_at_their_edge(ctx):
    lib = ctx.lib
    s = 4096
    rng_x = _data("random", _scale(ctx, 50_000, 3 << 20), 2)
    mn, _, thr = _rule(s)
    pair = next((a, b) for a in range(256) for b in range(256) if a != b and _hashes(np.array([a, b] * 40, np.uint8))[-1] >= np.uint64(thr))
    per_x = np.resize(np.array(pair, np.uint8), 30 * 1024 + 17)              # n // 1024 + 1 frames: the most any input can have

    def call(x, dst_cap, frames_cap):
        guard = 4096
        dst = np.full(dst_cap + guard, 0xA5, np.uint8)
        c = np.full(frames_cap + 16, 0xFFFFFFFF, np.uint32); d = c.copy()
        nf = ctypes.c_uint32(); dl = ctypes.c_size_t(); used = ctypes.c_size_t()
        rc = lib.zk_compress_frames_cdc(ctx._h, x.ctypes.data, x.size, s, 1, 1, None, 0, 1, dst.ctypes.data, dst_cap,
                                        c.ctypes.data_as(_native.u32p), d.ctypes.data_as(_native.u32p), frames_cap,
                                        ctypes.byref(nf), ctypes.byref(dl), ctypes.byref(used))
        assert (dst[dst_cap:] == 0xA5).all() and (c[frames_cap:] == 0xFFFFFFFF).all() and (d[frames_cap:] == 0xFFFFFFFF).all()
        return rc, nf.value, dl.value

    for x in (rng_x, per_x):
        rc, nf, dl = call(x, lib.zk_compress_bound(x.size, 1024), x.size // 1024 + 1)
        assert rc == 0 and nf == len(_cut(x, s)[0])
        assert call(x, dl, nf) == (0, nf, dl)
        assert call(x, dl - 1, nf)[0] == -70 and call(x, dl, nf - 1)[0] == -70
    assert call(per_x, 1 << 20, per_x.size // 1024 + 1)[1] == per_x.size // 1024 + 1


def _shared_after(ctx, old, new, policy, level, p0):
    """-> (frames of NEW's archive that end after byte p0 and appear byte for byte among OLD's frames, frames that end after p0)"""
    def frames(x):
        if policy == "content":
            comp, cs, ds, _ = ctx.compress_frames_cdc(x, 64 * KIB, level, True)
        else:
            comp, cs, ds = ctx.compress_frames(x, 64 * KIB, level, True)
        co, do = offsets(cs), offsets(ds)
        return [(int(do[i + 1]), comp[int(co[i]):int(co[i + 1])].tobytes()) for i in range(len(cs))]
    old_set = {f for _, f in frames(old)}
    after = [f for end, f in frames(new) if end > p0]
    return sum(f in old_set for f in after), len(after)


def test_edits_change_only_the_frames_around_them(ctx):
    """from the first edit on, Uncompressed(64 KiB) shares no frame with the old archive; ContentDefined(64 KiB) loses about two frames
    per edit (edited_copy also moves a region, which counts as two more edits)"""
    n = _scale(ctx, 2 << 20, 32 << 20)
    edits = _scale(ctx, 4, 24)
    level = _scale(ctx, -3, 3)
    for kind, seed in (("dickens", 1), ("mix", 2)):
        old = _data("dickens", n) if kind == "dickens" else _bench_mix(n, 21)
        new = edited_copy(old, seed, edits)
        m = min(old.size, new.size)
        p0 = int(np.argmax(old[:m] != new[:m]))                             # the first edited byte
        # the same count from the restatement, on the frames' input bytes
        want_old, want_new = _cut(old, 64 * KIB)[0], _cut(new, 64 * KIB)[0]
        old_frames = {old[a:a + d].tobytes() for a, d in zip(offsets(want_old)[:-1].tolist(), want_old)}
        after = [(a, d) for a, d in zip(offsets(want_new)[:-1].tolist(), want_new) if a + d > p0]
        same = sum(new[a:a + d].tobytes() in old_frames for a, d in after)
        assert len(after) - same <= 2 * (edits + 2), (kind, len(after), same)
        shared, total = _shared_after(ctx, old, new, "content", level, p0)
        assert (shared, total) == (same, len(after))
        ushared, utotal = _shared_after(ctx, old, new, "uncompressed", level, p0)
        assert ushared == 0 and utotal > 10, (kind, ushared, utotal)


def test_cli(ctx, tmp_path):
    x = _bench_mix(_scale(ctx, 300 * KIB, 8 << 20), 12)
    src = tmp_path / "in.bin"; src.write_bytes(x.tobytes())
    out = tmp_path / "in.bin.zst"; back = tmp_path / "back.bin"
    rc, _, err = cases._cli(ctx, ["compress", "-q", "-l", 3, "--frame-size-policy", "content", "-s", "64K", "-o", out, src])
    assert rc == 0, err
    comp, cs, ds, _ = ctx.compress_frames_cdc(x, 64 * KIB, 3, True)
    arch = out.read_bytes()
    assert arch[: comp.size] == comp.tobytes()
    rc, _, err = cases._cli(ctx, ["decompress", "-q", "-o", back, out])
    assert rc == 0 and back.read_bytes() == x.tobytes(), err
    rc, listing, err = cases._cli(ctx, ["list", "-d", out])
    rows = listing.decode().splitlines()[1:]
    assert rc == 0 and [int(r.split()[0]) for r in rows] == list(range(len(ds))), err
    prefix = tmp_path / "old.bin"; prefix.write_bytes(x[:1000].tobytes())
    rc, _, err = cases._cli(ctx, ["compress", "-q", "-f", "--frame-size-policy", "content", "--patch-from", prefix, "--long", "-o", out, src])
    assert rc != 0 and "--long needs --frame-size-policy uncompressed" in err


def test_pinned_bytes(ctx):
    from golden.make_cdc_golden import inputs
    want = json.load(open(os.path.join(GOLDEN, "cdc_golden.json")))
    for name, (x, s, level, ck) in inputs().items():
        comp, cs, ds, _ = ctx.compress_frames_cdc(x, s, level, ck)
        got = {"d_sizes": [int(v) for v in ds], "size": int(comp.size), "sha256": hashlib.sha256(comp.tobytes()).hexdigest()}
        assert got == want[name], name


@pytest.mark.gpu
def test_device_entry_point_matches_host(gpu_lib, monkeypatch):
    import torch
    from zeekstd_b200 import parallel
    ctx = zk.Context(0, gpu_lib)
    x = np.concatenate([_bench_mix(20 << 20, 13), np.zeros(1 << 20, np.uint8), _data("text", 3 << 20, 13)])
    xd = torch.from_numpy(x).cuda()
    dev = parallel.DeviceCodec(ctx)
    for level, s in ((1, 64 * KIB), (3, 2 << 20), (19, 256 * KIB), (-3, 4096)):
        for final in (True, False):
            comp, cs, ds, used = ctx.compress_frames_cdc(x, s, level, True, final=final)
            dcomp, dcs, dds, dused = dev.compress_cdc(xd, s, level, True, final=final)
            assert dcomp.cpu().numpy().tobytes() == comp.tobytes() and list(dcs) == list(cs) and list(dds) == list(ds) and dused == used
    ref = dev.compress_cdc(xd, 64 * KIB, 1, True)
    for env, val in (("ZK_DEV_SUB_BYTES", 1 << 20), ("ZK_CDC_CAP", 5)):
        monkeypatch.setenv(env, str(val))
        got = dev.compress_cdc(xd, 64 * KIB, 1, True)
        monkeypatch.delenv(env)
        assert got[0].cpu().numpy().tobytes() == ref[0].cpu().numpy().tobytes() and list(got[2]) == list(ref[2]), env
    ctx.close()
