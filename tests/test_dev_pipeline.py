"""The device-pointer entry points run their sub-batches on ZK_DEV_SLOTS slot streams at once; compress chains only where each sub-batch's
frames start, on the device.  Cut into sub-batches of one frame, of three frames and of a size no frame count fills, over one, two and three
slots, a call must give what one sub-batch gives: the same archive and compressed sizes, the same output and statuses, the same error for
a destination that the output of a later sub-batch overflows.  Every case runs on the emulation build (`-m "not gpu"`, whose device memory
is host memory) and on the H100 (`-m gpu`); the caller's stream order is checked on the H100 only."""
import ctypes

import numpy as np
import pytest

import zeekstd_b200 as zk
from util import offsets
from zeekstd_b200 import _native as N
from zeekstd_b200 import corpus

FRAME = 8192
ONE = {"ZK_DEV_SUB_BYTES": str(1 << 30), "ZK_DEV_SLOTS": "1"}
CUTS = [1 * FRAME, 3 * FRAME, 2 * FRAME + FRAME // 2]          # one frame, three frames, a size no count of whole frames fills
PIPES = [{"ZK_DEV_SUB_BYTES": str(sub), "ZK_DEV_SLOTS": str(slots)} for sub in CUTS for slots in (1, 2, 3)]


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    return request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib")


@pytest.fixture(scope="module")
def ctx(lib):
    c = zk.Context(0, lib)
    yield c
    c.close()


class Mem:
    """device memory of the build under test: torch CUDA tensors on the H100, numpy arrays in the emulation build"""

    def __init__(self, lib):
        self.gpu = "emul" not in lib._name
        if self.gpu:
            import torch
            self.torch = torch

    def put(self, a: np.ndarray):
        a = np.concatenate([a, np.zeros(64, np.uint8)])
        return self.torch.from_numpy(a).cuda() if self.gpu else a

    def zeros(self, n: int):
        return self.torch.zeros(n + 64, dtype=self.torch.uint8, device="cuda") if self.gpu else np.zeros(n + 64, np.uint8)

    def ptr(self, t):
        return t.data_ptr() if self.gpu else t.ctypes.data

    def get(self, t, n: int) -> bytes:
        return (t[:n].cpu().numpy() if self.gpu else t[:n]).tobytes()


def _env(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _data(n: int, seed: int) -> np.ndarray:
    return corpus.make_mix(n, seed=seed, segment=4096).numpy()


def compress(lib, ctx, mem, x, level, checksum, sizes=None, cap=None, stream=None):
    """-> (rc, archive bytes, c_sizes, d_sizes) of zk_compress_frames[_sized]_dev"""
    src = x if stream is not None else mem.put(x)
    n = len(x) if stream is None else stream[1]
    nf = len(sizes) if sizes is not None else max(1, -(-n // FRAME))
    bound = lib.zk_compress_bound_sized(np.asarray(sizes, np.uint32).ctypes.data_as(N.u32p), nf) if sizes is not None else lib.zk_compress_bound(n, FRAME)
    cap = bound if cap is None else cap
    dst = mem.zeros(bound)
    cs = np.zeros(nf + 1, np.uint32); ds = np.zeros(nf + 1, np.uint32)
    k, dl = ctypes.c_uint32(), ctypes.c_size_t()
    st = stream[0] if stream is not None else None
    if sizes is not None:
        sz = np.asarray(sizes, np.uint32)
        rc = lib.zk_compress_frames_sized_dev(ctx._h, mem.ptr(src), sz.ctypes.data_as(N.u32p), nf, level, int(checksum), mem.ptr(dst), cap,
                                              cs.ctypes.data_as(N.u32p), ctypes.byref(dl), st)
        ds[:nf] = sz; k.value = nf
    else:
        rc = lib.zk_compress_frames_dev(ctx._h, mem.ptr(src), n, FRAME, level, int(checksum), mem.ptr(dst), cap, cs.ctypes.data_as(N.u32p),
                                        ds.ctypes.data_as(N.u32p), nf + 1, ctypes.byref(k), ctypes.byref(dl), st)
    if rc:
        return rc, b"", [], []
    return rc, mem.get(dst, dl.value), list(cs[: k.value]), list(ds[: k.value])


def decompress(lib, ctx, mem, arc: bytes, cs, ds, verify):
    """-> (rc, output bytes, statuses) of zk_decompress_frames_dev"""
    comp = mem.put(np.frombuffer(arc, np.uint8))
    n = int(sum(ds))
    out = mem.zeros(n)
    co, do = offsets(cs), offsets(ds)
    status = np.full(len(cs), 7, np.int32)
    rc = lib.zk_decompress_frames_dev(ctx._h, mem.ptr(comp), co.ctypes.data_as(N.u64p), do.ctypes.data_as(N.u64p), len(cs), mem.ptr(out),
                                      int(verify), status.ctypes.data_as(N.i32p), None)
    return rc, mem.get(out, n), list(status)


CASES = [(1, False, 7 * FRAME + 1000), (1, True, 7 * FRAME + 1000), (3, True, 7 * FRAME + 1000), (-3, False, 7 * FRAME + 1000),
         (19, True, 4 * FRAME + 300)]


@pytest.mark.parametrize("level,checksum,n", CASES)
def test_same_archive_and_output(lib, ctx, monkeypatch, level, checksum, n):
    mem = Mem(lib)
    x = _data(n, 40 + level)
    _env(monkeypatch, ONE)
    rc, arc, cs, ds = compress(lib, ctx, mem, x, level, checksum)
    assert rc == 0
    rc, out, st = decompress(lib, ctx, mem, arc, cs, ds, checksum)
    assert rc == 0 and out == x.tobytes() and st == [0] * len(cs)
    for env in PIPES:
        _env(monkeypatch, env)
        assert compress(lib, ctx, mem, x, level, checksum) == (0, arc, cs, ds), env
        assert decompress(lib, ctx, mem, arc, cs, ds, checksum) == (0, out, st), env


def test_sized_frames(lib, ctx, monkeypatch):
    mem = Mem(lib)
    sizes = [5000, 1, 12000, 0, 8192, 3 * FRAME, 700, 9000]
    x = _data(sum(sizes), 51)
    _env(monkeypatch, ONE)
    want = compress(lib, ctx, mem, x, 3, True, sizes)
    assert want[0] == 0
    back = decompress(lib, ctx, mem, want[1], want[2], want[3], True)
    assert back == (0, x.tobytes(), [0] * len(sizes))
    for env in PIPES:
        _env(monkeypatch, env)
        assert compress(lib, ctx, mem, x, 3, True, sizes) == want, env
        assert decompress(lib, ctx, mem, want[1], want[2], want[3], True) == back, env


def test_destination_too_small_in_a_later_sub_batch(lib, ctx, monkeypatch):
    mem = Mem(lib)
    x = _data(7 * FRAME + 1000, 61)
    _env(monkeypatch, ONE)
    rc, arc, cs, _ = compress(lib, ctx, mem, x, 1, False)
    assert rc == 0
    for cap in (int(sum(cs[:4])) + 5, len(arc) - 1):          # the overflow falls in sub-batch 5 of one frame, then in the last
        _env(monkeypatch, ONE)
        want = compress(lib, ctx, mem, x, 1, False, cap=cap)[0]
        assert want == -70                                     # ZK_ERR_ZSTD(ZSTD_error_dstSize_tooSmall)
        for env in PIPES:
            _env(monkeypatch, env)
            assert compress(lib, ctx, mem, x, 1, False, cap=cap)[0] == want, (env, cap)


def test_corrupt_frame_in_a_later_sub_batch(lib, ctx, monkeypatch):
    mem = Mem(lib)
    x = _data(7 * FRAME + 1000, 71)
    _env(monkeypatch, ONE)
    rc, arc, cs, ds = compress(lib, ctx, mem, x, 3, True)
    assert rc == 0
    co = offsets(cs)
    bad = bytearray(arc)
    for f in (4, 6):                                            # in the second sub-batch of three frames, and in the last
        mid = int(co[f]) + int(cs[f]) // 2
        bad[mid: mid + 8] = bytes(b ^ 0x5A for b in bad[mid: mid + 8])
    bad = bytes(bad)
    want = decompress(lib, ctx, mem, bad, cs, ds, True)
    assert want[0] != 0 and want[2][4] != 0 and want[2][6] != 0 and want[2][:4] == [0] * 4
    for env in PIPES:
        _env(monkeypatch, env)
        got = decompress(lib, ctx, mem, bad, cs, ds, True)
        assert (got[0], got[2]) == (want[0], want[2]), env


@pytest.mark.gpu
def test_caller_stream_order(gpu_lib, monkeypatch):
    """the input is written on the caller's stream just before the call and the output read on it just after, with no host synchronise"""
    import torch
    lib = gpu_lib
    ctx = zk.Context(0, lib)
    mem = Mem(lib)
    n = 64 * FRAME + 123
    x = torch.from_numpy(_data(n, 81)).cuda()
    _env(monkeypatch, {"ZK_DEV_SUB_BYTES": str(3 * FRAME), "ZK_DEV_SLOTS": "3"})
    s = torch.cuda.Stream()
    src = torch.zeros(n + 64, dtype=torch.uint8, device="cuda")
    big = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        big.fill_(3)                                            # keeps the stream busy before the input is written
        src[:n].copy_(x)
        rc, arc, cs, ds = compress(lib, ctx, mem, src, 1, True, stream=(s.cuda_stream, n))
    assert rc == 0
    comp = mem.put(np.frombuffer(arc, np.uint8))
    out = torch.zeros(n + 64, dtype=torch.uint8, device="cuda")
    co, do = offsets(cs), offsets(ds)
    with torch.cuda.stream(s):
        big.fill_(4)
        rc = lib.zk_decompress_frames_dev(ctx._h, comp.data_ptr(), co.ctypes.data_as(N.u64p), do.ctypes.data_as(N.u64p), len(cs),
                                          out.data_ptr(), 1, None, s.cuda_stream)
        got = out[:n].clone()
    assert rc == 0
    s.synchronize()
    assert torch.equal(got, x)
    _env(monkeypatch, ONE)
    assert compress(lib, ctx, mem, x.cpu().numpy(), 1, True)[1] == arc
    ctx.close()
