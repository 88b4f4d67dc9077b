"""The decoder's scratch retry: a batch whose blocks outnumber the first scratch estimate (total output / 32 KiB + 4 per entry + 64)
overflows, reports its exact needs and runs again.  The second attempt must get the same prefix and the same `need` array as the first.
Each case uses a fresh context, since a context keeps the needs an overflow reported and would not retry.  The host path retries in
zk_decompress_frames_prefix's pipeline, the device-pointer path inside zk_decode_batch.  The launch counts show that exactly one retry
ran.  Every case runs on the emulation build (`-m "not gpu"`) and on the H100 (`-m gpu`)."""
import numpy as np
import pytest

import framegen as G
import zeekstd_b200 as zk
from framegen import Block, Frame
from util import offsets
from zeekstd_b200 import _native

BLOCKS = 3000           # far above the first estimate for these few KiB of output
PREFIX = 2000


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    return request.getfixturevalue("emul_lib" if request.param == "emul" else "gpu_lib")


def _entry(rng, prefix: bytes, frames: int):
    """frames of BLOCKS // frames tiny blocks each: two literals and one match, whose offset reaches into the prefix when there is one"""
    out = []
    for _ in range(frames):
        blocks, pos = [], 0
        for _ in range(BLOCKS // frames):
            lits = rng.integers(0, 256, 2, dtype=np.uint8).tobytes()
            ml = int(rng.integers(3, 9))
            off = int(rng.integers(1, pos + 2 + len(prefix) + 1))
            blocks.append(Block("comp", lits, seqs=[(2, off + 3, ml)]))
            pos += 2 + ml
        out.append(Frame(blocks))
    return G.entry_bytes(out, prefix), G.execute(out, prefix)


def _launch_counts(lib, run):
    """(launches of the first run on a fresh context, of a second identical run); the second finds its scratch grown already"""
    ctx = zk.Context(0, lib)
    try:
        run(ctx)
        first = ctx.kernel_launches
        run(ctx)
        return first, ctx.kernel_launches - first
    finally:
        ctx.close()


@pytest.mark.parametrize("with_need", [False, True])
def test_host_retry_keeps_prefix_and_need(lib, with_need):
    rng = np.random.default_rng(7 + with_need)
    prefix = rng.integers(0, 256, PREFIX, dtype=np.uint8).tobytes()
    entries = [_entry(rng, prefix, frames) for frames in (1, 3)]
    comp = np.frombuffer(b"".join(e[0] for e in entries) + b"\0" * 64, np.uint8)
    sizes = [len(e[1]) for e in entries]
    need = np.array([s // 2 + 1 for s in sizes], np.uint32) if with_need else None
    do = offsets(sizes)

    def run(ctx):
        out, st, rc = ctx.decompress_frames(comp, offsets([len(e[0]) for e in entries]), do, False, need=need,
                                            prefix=np.frombuffer(prefix, np.uint8))
        assert rc == 0 and list(st) == [0, 0]
        for i, (_, want) in enumerate(entries):
            k = len(want) if need is None else int(need[i])
            assert out[int(do[i]): int(do[i]) + k].tobytes() == want[:k], i

    first, again = _launch_counts(lib, run)
    assert first == 2 * again


def test_device_retry(lib):
    rng = np.random.default_rng(11)
    blob, want = _entry(rng, b"", 2)
    comp = np.frombuffer(blob + b"\0" * 64, np.uint8)
    co, do = offsets([len(blob)]), offsets([len(want)])
    gpu = "emul" not in lib._name
    if gpu:
        import torch
        d_comp = torch.from_numpy(comp.copy()).cuda()
        d_out = torch.zeros(len(want) + 64, dtype=torch.uint8, device="cuda")
        comp_ptr, out_ptr = d_comp.data_ptr(), d_out.data_ptr()
    else:                                  # the emulation build's device memory is host memory
        out = np.zeros(len(want) + 64, np.uint8)
        comp_ptr, out_ptr = comp.ctypes.data, out.ctypes.data

    def run(ctx):
        st = np.ones(1, np.int32)
        rc = lib.zk_decompress_frames_dev(ctx._h, comp_ptr, co.ctypes.data_as(_native.u64p), do.ctypes.data_as(_native.u64p), 1, out_ptr,
                                          0, st.ctypes.data_as(_native.i32p), None)
        assert rc == 0 and st[0] == 0
        got = d_out.cpu().numpy() if gpu else out
        assert got[: len(want)].tobytes() == want

    first, again = _launch_counts(lib, run)
    assert first == 2 * again
