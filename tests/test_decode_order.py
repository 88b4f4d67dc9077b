"""The decode stages hand out their work heaviest first (K-D0o / K-D1o, ZK_DEC_ORDER=1, the default) or in the order the
lists were filled (ZK_DEC_ORDER=0).  Only the order of execution changes: output bytes, per-entry statuses and segment counts
must be the same under both, for every level tier, with and without checksums, for libzstd's archives, range reads,
prefix mode, corrupt entries beside good ones and batches with fewer items than workers.  Every case runs on the emulation
build (`-m "not gpu"`) and on the H100 (`-m gpu`), where the mix is larger."""
import os

import numpy as np
import pytest

import zeekstd_b200 as zk
from util import decode_frames, golden_bytes, offsets, split_frames
from zeekstd_b200 import corpus


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    return request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib")


def _context(lib, order: int):
    old = os.environ.get("ZK_DEC_ORDER")
    os.environ["ZK_DEC_ORDER"] = str(order)
    try:
        return zk.Context(0, lib)
    finally:
        if old is None:
            del os.environ["ZK_DEC_ORDER"]
        else:
            os.environ["ZK_DEC_ORDER"] = old


@pytest.fixture(scope="module")
def ctxs(lib):
    c = (_context(lib, 0), _context(lib, 1))
    yield c
    for x in c:
        x.close()


def _scale(lib, n: int) -> int:
    """the emulation build interprets every thread on the CPU: its inputs are a sixteenth of the H100's"""
    return n if "emul" not in lib._name else n // 16


def _mix(n: int, seed: int) -> np.ndarray:
    return corpus.as_numpy(corpus.make_mix(n, seed=seed, segment=64 << 10))


def _same(ctxs, frames, sizes, verify=True, **kw):
    """decode with both orders -> the (shared) statuses; good entries' bytes and the segment counts must match"""
    res = []
    for c in ctxs:
        s0 = c.decode_segments
        if kw:
            comp = np.frombuffer(b"".join(frames) + b"\0" * 64, dtype=np.uint8)
            out, st, rc = c.decompress_frames(comp, offsets([len(f) for f in frames]), offsets(sizes), verify, **kw)
            out = out.tobytes()
        else:
            out, st, rc = decode_frames(c, frames, sizes, verify)
        res.append((out, list(st), rc, c.decode_segments - s0))
    (o0, st0, rc0, n0), (o1, st1, rc1, n1) = res
    assert st0 == st1 and rc0 == rc1 and n0 == n1, (st0, st1, rc0, rc1, n0, n1)
    d = offsets(sizes)
    need = kw.get("need")
    for e, s in enumerate(st0):
        if s == 0:
            end = int(d[e + 1]) if need is None else int(d[e]) + min(int(need[e]), int(sizes[e]))
            assert o0[int(d[e]):end] == o1[int(d[e]):end], e
    return st0, o1


LEVELS = [(1, False), (1, True), (3, False), (3, True), (-1, False), (-1, True), (19, False), (19, True)]


@pytest.mark.parametrize("level,checksum", LEVELS)
def test_mix_decodes_the_same_in_both_orders(lib, ctxs, level, checksum):
    n = _scale(lib, (16 << 20) if level != 19 else (4 << 20))
    x = _mix(n, 71 + level)
    comp, cs, ds = ctxs[1].compress_frames(x, max(n // 8, 64 << 10), level, checksum)
    st, out = _same(ctxs, split_frames(comp.tobytes(), cs), [int(d) for d in ds])
    assert not any(st) and out == x.tobytes()


@pytest.mark.parametrize("name", ["dickens_96k_l1_f32k", "dickens_96k_l19_f96k", "dickens_96k_l3_f96k_ck", "dickens_96k_l9_f20000_ck",
                                  "dickens_4k_l3_f100"])
def test_libzstd_archives_decode_the_same_in_both_orders(lib, ctxs, name):
    a = golden_bytes(name + ".zst")
    t = zk.SeekTable.from_bytes(a, zk.Format.Foot, lib)
    co, do = t.offsets()
    co = [int(v) for v in co]; do = [int(v) for v in do]
    frames = [a[co[i]:co[i + 1]] for i in range(len(co) - 1)]
    st, _ = _same(ctxs, frames, [do[i + 1] - do[i] for i in range(len(do) - 1)])
    assert not any(st)


def test_corrupt_entries_beside_good_ones(lib, ctxs):
    n = _scale(lib, 16 << 20)
    x = _mix(n, 5)
    comp, cs, ds = ctxs[1].compress_frames(x, max(n // 16, 32 << 10), 1, True)
    frames = split_frames(comp.tobytes(), cs)
    sizes = [int(d) for d in ds]
    rng = np.random.default_rng(3)
    for e in range(0, len(frames), 3):
        f = bytearray(frames[e])
        f[int(rng.integers(16, len(f) - 1))] ^= 1 << int(rng.integers(8))
        frames[e] = bytes(f)
    sizes[1] += 1                                          # a wrong entry size as well
    st, _ = _same(ctxs, frames, sizes)
    assert any(st) and not all(st)


def test_range_read(lib, ctxs):
    n = _scale(lib, 16 << 20)
    x = _mix(n, 9)
    comp, cs, ds = ctxs[1].compress_frames(x, max(n // 8, 64 << 10), 3, False)
    rng = np.random.default_rng(4)
    need = np.array([int(rng.integers(1, int(d) + 1)) for d in ds], dtype=np.uint32)
    st, _ = _same(ctxs, split_frames(comp.tobytes(), cs), [int(d) for d in ds], False, need=need)
    assert not any(st)


def test_prefix_mode(lib, ctxs):
    n = _scale(lib, 8 << 20)
    old = _mix(n, 12)
    new = old.copy()
    new[n // 3: n // 3 + 4096] ^= 0x5A
    comp, cs, ds = ctxs[1].compress_frames(new, max(n // 8, 64 << 10), 3, True, prefix=old)
    st, out = _same(ctxs, split_frames(comp.tobytes(), cs), [int(d) for d in ds], True, prefix=old)
    assert not any(st) and out[:n] == new.tobytes()


def test_fewer_items_than_workers(lib, ctxs):
    x = _mix(20000, 13)
    comp, cs, ds = ctxs[1].compress_frames(x, 20000, 1, True)
    st, out = _same(ctxs, split_frames(comp.tobytes(), cs), [int(d) for d in ds])
    assert not any(st) and out == x.tobytes()


def test_launches_grow_by_two_per_batch(lib, ctxs):
    x = _mix(20000, 14)
    comp, cs, ds = ctxs[1].compress_frames(x, 20000, 1, False)
    grew = []
    for c in ctxs:
        k0 = c.kernel_launches
        decode_frames(c, split_frames(comp.tobytes(), cs), [int(d) for d in ds], False)
        grew.append(c.kernel_launches - k0)
    assert grew[1] == grew[0] + 2, grew
