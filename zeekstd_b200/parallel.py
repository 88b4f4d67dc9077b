"""Frame sharding across GPUs (SURVEY.md 8e, BASELINE config 4): frames of the seekable format are independent
(seekable_format.md:23-29), so rank r of W owns a contiguous range of frames and no collective touches the codec itself.
The exchanges around it are torch.distributed point-to-point calls (NCCL over NVLink on the GPU box, gloo in the CPU
tests), CHUNKED and PIPELINED so that they overlap the codec:

  compress:   the root posts, up front, one grouped send per chunk round (chunk k of every other rank's shard); a rank
              posts all its receives up front and compresses chunk k as soon as it has landed, while chunk k+1.. are
              still in flight (NCCL runs them on its own stream).  Then one all-gather of the per-frame sizes (4+4 B per
              frame: this is what makes the global seek table -- the only host read-back of the step), and the ranks
              send their compressed bytes, which the root receives at the scanned offsets.
  decompress: the root posts every send (compressed chunk k of rank r, by seek-table offsets) AND every receive
              (decoded chunk k of rank r, straight into its final place) up front, on two communicators so both
              directions of the NVLink are used at once; a rank decodes chunk k when it lands and sends it back at once.

One process per GPU; `codec` is DeviceCodec (CUDA tensors, zk_*_frames_dev, zero-copy) or HostCodec (CPU tensors through
the host-pointer entry points; the gloo tests).  `stats` (optional dict) receives this rank's timings.
"""
from __future__ import annotations

import ctypes
import time

import numpy as np
import torch
import torch.distributed as dist

from . import _native

CHUNK_BYTES = 1 << 30            # uncompressed bytes per pipeline chunk (whole frames); >= 2 chunks per rank when possible.
                                 # The codec kernels are bound by per-frame latency, so a chunk costs about the same whatever its size
                                 # up to ~512 frames (tools/c4_probe.py: 256 MiB chunks run at half the GiB/s of 1 GiB chunks)


def frame_ranges(n_frames: int, world: int):
    """contiguous frame ranges, ceil(N/W) per rank (rank order == frame order)"""
    per = -(-n_frames // world) if n_frames else 0
    return [(min(r * per, n_frames), min((r + 1) * per, n_frames)) for r in range(world)]


def chunk_ranges(lo: int, hi: int, chunk_frames: int):
    """[lo, hi) cut into runs of <= chunk_frames frames"""
    return [(f, min(f + chunk_frames, hi)) for f in range(lo, hi, max(1, chunk_frames))]


def pick_chunk_frames(n_frames: int, world: int, frame_size: int, chunk_bytes: int = 0) -> int:
    per = -(-n_frames // world) if n_frames else 1
    cf = max(1, (chunk_bytes or CHUNK_BYTES) // max(1, frame_size))
    return max(1, min(cf, -(-per // 2)))           # at least two chunks per rank, so that something overlaps


def torch_stream_handle(device) -> ctypes.c_void_p:
    """cudaStream_t of torch's current stream; torch's default stream is the legacy NULL stream, which the C ABI
    spells cudaStreamLegacy (0x1) because NULL there means "the context's own stream"."""
    h = torch.cuda.current_stream(device).cuda_stream
    return ctypes.c_void_p(h if h else 1)


class DeviceCodec:
    """zero-copy codec over CUDA tensors (zk_*_frames_dev).  The kernels are enqueued on torch's CURRENT stream so they
    are ordered after the tensor ops / NCCL receives that produced their inputs.  Inputs are slices of larger buffers:
    the entry points want 16 readable bytes after the last one (callers allocate their buffers with PAD bytes of slack)."""
    PAD = 64

    def __init__(self, ctx):
        self.ctx, self.lib = ctx, ctx.lib
        self.device_ms = 0.0

    def empty(self, n: int, device):
        return torch.empty(n + self.PAD, dtype=torch.uint8, device=device)

    def compress_bound(self, n: int, frame_size: int) -> int:
        return int(self.lib.zk_compress_bound(n, frame_size))

    def compress_into(self, src: torch.Tensor, n: int, frame_size: int, level: int, checksum: bool, dst: torch.Tensor,
                      long_mode: bool = False):
        """src[:n] -> frames written from dst[0]; src and dst are views with PAD readable / writable bytes behind them.
        long_mode: every frame also matches its own bytes up to 2^27 back (zk_compress_frames_long_dev).
        -> (bytes written, c_sizes, d_sizes)"""
        if src.data_ptr() % 16:
            src = torch.cat([src[:n], torch.zeros(self.PAD, dtype=torch.uint8, device=src.device)])
        nfmax = n // frame_size + 2
        cs = np.zeros(nfmax, dtype=np.uint32); ds = np.zeros(nfmax, dtype=np.uint32)
        nf = ctypes.c_uint32(); dl = ctypes.c_size_t()
        cap = min(self.compress_bound(n, frame_size), dst.numel())
        name = "zk_compress_frames_long_dev" if long_mode else "zk_compress_frames_dev"
        rc = getattr(self.lib, name)(self.ctx._h, src.data_ptr(), n, frame_size, level, int(checksum), dst.data_ptr(), cap,
                cs.ctypes.data_as(_native.u32p), ds.ctypes.data_as(_native.u32p), nfmax, ctypes.byref(nf),
                ctypes.byref(dl), torch_stream_handle(src.device))
        if rc:
            raise RuntimeError(f"{name}: {rc}")
        self.device_ms += self.ctx.last_device_ms
        return int(dl.value), cs[: nf.value].astype(np.int64), ds[: nf.value].astype(np.int64)

    def decompress_into(self, comp: torch.Tensor, c_off, d_off, verify: bool, dst: torch.Tensor):
        """entries comp[c_off[i]:c_off[i+1]] -> dst[d_off[i]:d_off[i+1]] (offsets relative to the two views)"""
        co = np.ascontiguousarray(c_off, dtype=np.uint64); do = np.ascontiguousarray(d_off, dtype=np.uint64)
        n = len(co) - 1
        mis = comp.data_ptr() % 16                    # any byte offset inside the archive: hand over the aligned address
        tmp = None
        if dst.data_ptr() % 16:
            tmp = torch.empty(int(do[-1]) + self.PAD, dtype=torch.uint8, device=dst.device)
        target = tmp if tmp is not None else dst
        rc = self.lib.zk_decompress_frames_dev(self.ctx._h, comp.data_ptr() - mis, (co + np.uint64(mis)).ctypes.data_as(_native.u64p),
                                               do.ctypes.data_as(_native.u64p), n, target.data_ptr(), int(verify), None, torch_stream_handle(comp.device))
        if rc:
            raise RuntimeError(f"zk_decompress_frames_dev: {rc}")
        self.device_ms += self.ctx.last_device_ms
        if tmp is not None:
            dst[: int(do[-1])] = tmp[: int(do[-1])]

    # whole-buffer conveniences (tools, tests)
    def compress(self, x: torch.Tensor, frame_size: int, level: int, checksum: bool, long_mode: bool = False):
        n = x.numel()
        src = torch.cat([x, torch.zeros(self.PAD, dtype=torch.uint8, device=x.device)])
        dst = self.empty(self.compress_bound(n, frame_size), x.device)
        k, cs, ds = self.compress_into(src, n, frame_size, level, checksum, dst, long_mode)
        return dst[:k], cs, ds

    def compress_csize(self, x: torch.Tensor, target: int, level: int, checksum: bool, final: bool = True):
        """FrameSizePolicy::Compressed(target) (zk_compress_frames_csize_dev) -> (frames, c_sizes, d_sizes, consumed)"""
        n = x.numel()
        src = torch.cat([x, torch.zeros(self.PAD, dtype=torch.uint8, device=x.device)])
        cap = self.compress_bound(n, 32768)
        dst = self.empty(cap, x.device)
        nfmax = n // 32768 + 2
        cs = np.zeros(nfmax, dtype=np.uint32); ds = np.zeros(nfmax, dtype=np.uint32)
        nf = ctypes.c_uint32(); dl = ctypes.c_size_t(); used = ctypes.c_size_t()
        rc = self.lib.zk_compress_frames_csize_dev(self.ctx._h, src.data_ptr(), n, target, level, int(checksum), int(final), dst.data_ptr(), cap,
                                                   cs.ctypes.data_as(_native.u32p), ds.ctypes.data_as(_native.u32p), nfmax, ctypes.byref(nf),
                                                   ctypes.byref(dl), ctypes.byref(used), torch_stream_handle(x.device))
        if rc:
            raise RuntimeError(f"zk_compress_frames_csize_dev: {rc}")
        self.device_ms += self.ctx.last_device_ms
        return dst[: int(dl.value)], cs[: nf.value].astype(np.int64), ds[: nf.value].astype(np.int64), int(used.value)

    def compress_cdc(self, x: torch.Tensor, size: int, level: int, checksum: bool, final: bool = True):
        """FrameSizePolicy::ContentDefined(size) (zk_compress_frames_cdc_dev) -> (frames, c_sizes, d_sizes, consumed)"""
        n = x.numel()
        src = torch.cat([x, torch.zeros(self.PAD, dtype=torch.uint8, device=x.device)])
        cap = self.compress_bound(n, 1024)
        dst = self.empty(cap, x.device)
        nfmax = n // 1024 + 1
        cs = np.zeros(nfmax, dtype=np.uint32); ds = np.zeros(nfmax, dtype=np.uint32)
        nf = ctypes.c_uint32(); dl = ctypes.c_size_t(); used = ctypes.c_size_t()
        rc = self.lib.zk_compress_frames_cdc_dev(self.ctx._h, src.data_ptr(), n, size, level, int(checksum), int(final), dst.data_ptr(), cap,
                                                 cs.ctypes.data_as(_native.u32p), ds.ctypes.data_as(_native.u32p), nfmax, ctypes.byref(nf),
                                                 ctypes.byref(dl), ctypes.byref(used), torch_stream_handle(x.device))
        if rc:
            raise RuntimeError(f"zk_compress_frames_cdc_dev: {rc}")
        self.device_ms += self.ctx.last_device_ms
        return dst[: int(dl.value)], cs[: nf.value].astype(np.int64), ds[: nf.value].astype(np.int64), int(used.value)

    def decompress(self, comp: torch.Tensor, c_off, d_off, verify: bool):
        src = torch.cat([comp, torch.zeros(self.PAD, dtype=torch.uint8, device=comp.device)])
        out = self.empty(int(c_off[-1] * 0 + d_off[-1]), comp.device)
        self.decompress_into(src, c_off, d_off, verify, out)
        return out[: int(d_off[-1])]


class HostCodec:
    """same interface over CPU tensors through the host-pointer entry points (used by the gloo tests)"""
    PAD = 64

    def __init__(self, ctx):
        self.ctx = ctx
        self.device_ms = 0.0

    def empty(self, n: int, device="cpu"):
        return torch.empty(n + self.PAD, dtype=torch.uint8)

    def compress_bound(self, n: int, frame_size: int) -> int:
        return int(self.ctx.lib.zk_compress_bound(n, frame_size))

    def compress_into(self, src, n, frame_size, level, checksum, dst):
        comp, cs, ds = self.ctx.compress_frames(src[:n].numpy(), frame_size, level, checksum)
        dst[: comp.size] = torch.from_numpy(comp.copy())
        return int(comp.size), cs.astype(np.int64), ds.astype(np.int64)

    def decompress_into(self, comp, c_off, d_off, verify, dst):
        end = int(c_off[-1])
        out, st, rc = self.ctx.decompress_frames(np.concatenate([comp[:end].numpy(), np.zeros(64, dtype=np.uint8)]), c_off, d_off, verify)
        if rc:
            raise RuntimeError(f"zk_decompress_frames: {rc}")
        dst[: out.size] = torch.from_numpy(out.copy())

    def compress(self, x, frame_size, level, checksum):
        dst = self.empty(self.compress_bound(x.numel(), frame_size))
        k, cs, ds = self.compress_into(x, x.numel(), frame_size, level, checksum, dst)
        return dst[:k], cs, ds

    def decompress(self, comp, c_off, d_off, verify):
        out = self.empty(int(d_off[-1]))
        self.decompress_into(comp, c_off, d_off, verify, out)
        return out[: int(d_off[-1])]


# ------------------------------------------------------------------------------------------------ exchange helpers
class Groups:
    """two communicators: `down` carries root -> ranks traffic, `up` carries ranks -> root traffic, so that the two
    directions of a step never queue behind each other (one NCCL communicator executes its operations in order)"""

    def __init__(self, device=None):
        opts = None
        if dist.get_backend() == "nccl":
            # The exchange needs a small fraction of NVLink (16 GiB per ~0.3 s step); its kernels must not take SMs from the
            # codec, whose frames want to be resident all at once: a few CTAs per NCCL kernel are plenty.
            try:
                import os
                opts = dist.ProcessGroupNCCL.Options()
                opts.config.max_ctas = int(os.environ.get("ZK_NCCL_MAX_CTAS", "8"))
                opts.config.min_ctas = 1
            except Exception:
                opts = None
        self.down = dist.new_group(pg_options=opts) if opts is not None else dist.new_group()
        self.up = dist.new_group(pg_options=opts) if opts is not None else dist.new_group()
        self.bulk = dist.new_group()          # exchanges nothing overlaps with (the archive gather after compression): full width
        # NCCL creates a communicator at its FIRST use, collectively, with device-wide synchronisation inside.  If that first use
        # falls into a pass where receives posted ahead are already spinning on the GPU, the ranks deadlock (seen at N = 2: the
        # root sat in the creation of `up` waiting for a rank whose creation waited for a receive only the root could feed).
        # So every communicator does a collective and a point-to-point round trip in both directions NOW, while nothing is in flight.
        if device is not None and dist.get_backend() == "nccl":
            rank, world = dist.get_rank(), dist.get_world_size()
            for g in (self.down, self.up, self.bulk):
                t = torch.zeros(16, dtype=torch.uint8, device=device)
                dist.all_reduce(t, group=g)
                for root in range(world):
                    ops = []
                    if rank == root:
                        for r in range(world):
                            if r != root:
                                ops += [dist.P2POp(dist.isend, t, r, g), dist.P2POp(dist.irecv, torch.empty_like(t), r, g)]
                    else:
                        ops = [dist.P2POp(dist.irecv, torch.empty_like(t), root, g), dist.P2POp(dist.isend, t, root, g)]
                    if ops:
                        for q in dist.batch_isend_irecv(ops):
                            q.wait()
                torch.cuda.synchronize(device)
            dist.barrier()


_groups: Groups | None = None


def groups(device=None) -> Groups:
    global _groups
    if _groups is None:
        _groups = Groups(device)
    return _groups


def _post(ops):
    """post a round of point-to-point operations -> list of requests.  NCCL: one grouped launch (ncclGroupStart/End), so a
    round towards W-1 peers shares the links instead of queueing peer after peer."""
    if not ops:
        return []
    if dist.get_backend() == "nccl":
        return dist.batch_isend_irecv(ops)
    return [op.op(op.tensor, op.peer, group=op.group) for op in ops]


def _wait(reqs):
    for q in reqs:
        q.wait()


def _now(device):
    if isinstance(device, torch.device) and device.type == "cuda" or (isinstance(device, str) and device.startswith("cuda")):
        torch.cuda.synchronize(device)
    return time.perf_counter()


# ------------------------------------------------------------------------------------------------ the two sharded passes
def sharded_compress(codec, x_root, n_total: int, frame_size: int, level: int = 1, checksum: bool = False, root: int = 0, device="cpu",
                     chunk_bytes: int = 0, stats: dict | None = None):
    """x_root: the whole input on the root (a tensor with codec.PAD bytes of slack behind n_total), None elsewhere.
    -> on root: (frames tensor, c_sizes, d_sizes) for the WHOLE input; on other ranks: (None, c_sizes, d_sizes)"""
    rank, world = dist.get_rank(), dist.get_world_size()
    g = groups(device)
    t0 = _now(device) if stats is not None else 0.0
    n_frames = max(1, -(-n_total // frame_size))
    ranges = frame_ranges(n_frames, world)
    cf = pick_chunk_frames(n_frames, world, frame_size, chunk_bytes)
    chunks = [chunk_ranges(lo, hi, cf) for lo, hi in ranges]
    rounds = max(len(c) for c in chunks)
    byte = lambda f: min(f * frame_size, n_total)
    lo, hi = ranges[rank]
    b0, b1 = byte(lo), byte(hi)
    # 1. scatter: every receive / send of the pass is posted now; NCCL works through them while the codec runs
    recv_reqs = []
    if rank == root:
        mine = x_root[b0:] if x_root is not None else codec.empty(0, device)
        for k in range(rounds):
            ops = [dist.P2POp(dist.isend, x_root[byte(chunks[r][k][0]): byte(chunks[r][k][1])], r, g.down)
                   for r in range(world) if r != root and k < len(chunks[r]) and byte(chunks[r][k][1]) > byte(chunks[r][k][0])]
            recv_reqs.append(_post(ops))                      # the root's "receives" are its sends: waited on at the end
    else:
        mine = codec.empty(b1 - b0, device)
        for (f0, f1) in chunks[rank]:
            ops = [dist.P2POp(dist.irecv, mine[byte(f0) - b0: byte(f1) - b0], root, g.down)] if byte(f1) > byte(f0) else []
            recv_reqs.append(_post(ops))
    # 2. local compress, chunk by chunk, into one contiguous local archive
    own = hi > lo or (n_total == 0 and rank == 0)
    local = codec.empty(codec.compress_bound(b1 - b0, frame_size) if own else 0, device)
    pos = 0
    cs_l, ds_l = [], []
    codec.device_ms = 0.0
    if own:
        my_chunks = chunks[rank] if hi > lo else [(0, 1)]
        for k, (f0, f1) in enumerate(my_chunks):
            if rank != root and k < len(recv_reqs):
                _wait(recv_reqs[k])
            s0, s1 = byte(f0) - b0, byte(f1) - b0
            wrote, cs, ds = codec.compress_into(mine[s0:], s1 - s0, frame_size, level, checksum, local[pos:])
            pos += wrote; cs_l.append(cs); ds_l.append(ds)
    cs = np.concatenate(cs_l) if cs_l else np.zeros(0, dtype=np.int64)
    ds = np.concatenate(ds_l) if ds_l else np.zeros(0, dtype=np.int64)
    t1 = time.perf_counter()                                 # the codec calls are host-synchronous: no device sync needed here
    # 3. all-gather of the per-frame sizes (padded to the per-rank maximum) -> global seek table on every rank
    per = max(1, max(h - l for l, h in ranges))
    pad = torch.full((2, per), -1, dtype=torch.int64)
    pad[0, : len(cs)] = torch.from_numpy(cs); pad[1, : len(ds)] = torch.from_numpy(ds)
    pad = pad.to(device)
    if dist.get_backend() == "nccl":
        allp = torch.empty((world, 2, per), dtype=torch.int64, device=device)
        dist.all_gather_into_tensor(allp, pad)
    else:
        parts = [torch.empty_like(pad) for _ in range(world)]
        dist.all_gather(parts, pad)
        allp = torch.stack(parts)
    table = allp.cpu().numpy()                               # the one host read-back of the pass: the seek table
    counts = [int((table[r, 0] >= 0).sum()) for r in range(world)]
    c_all = np.concatenate([table[r, 0, : counts[r]] for r in range(world)]).astype(np.int64)
    d_all = np.concatenate([table[r, 1, : counts[r]] for r in range(world)]).astype(np.int64)
    # 4. variable-size gather of the compressed bytes to the root at the scanned offsets
    starts = np.concatenate([[0], np.cumsum(c_all)])
    first = np.concatenate([[0], np.cumsum(counts)])
    out = None
    if rank == root:
        out = codec.empty(int(starts[-1]), device)
        ops = []
        for r in range(world):
            o0, o1 = int(starts[first[r]]), int(starts[first[r + 1]])
            if o1 > o0 and r != root:
                ops.append(dist.P2POp(dist.irecv, out[o0:o1], r, g.bulk))
        reqs = _post(ops)
        o0, o1 = int(starts[first[root]]), int(starts[first[root + 1]])
        out[o0:o1] = local[:pos]
        _wait(reqs)
        for rr in recv_reqs:
            _wait(rr)
    elif pos:
        _wait(_post([dist.P2POp(dist.isend, local[:pos], root, g.bulk)]))
    if stats is not None:
        t2 = _now(device)
        stats.update(compress_total_ms=(t2 - t0) * 1e3, compress_until_codec_done_ms=(t1 - t0) * 1e3, compress_codec_ms=codec.device_ms,
                     compress_gather_ms=(t2 - t1) * 1e3, compress_chunks=len(chunks[rank]), chunk_frames=cf)
    if rank == root:
        return out[: int(starts[-1])], c_all, d_all
    return None, c_all, d_all


def sharded_decompress(codec, comp_root, c_sizes, d_sizes, verify: bool = True, root: int = 0, device="cpu", chunk_bytes: int = 0,
                       stats: dict | None = None, frame_size: int = 0):
    """c_sizes / d_sizes known on every rank (the seek table); comp_root: the archive on the root (PAD bytes of slack).
    -> on root: the decompressed tensor"""
    rank, world = dist.get_rank(), dist.get_world_size()
    g = groups(device)
    t0 = _now(device) if stats is not None else 0.0
    n_frames = len(c_sizes)
    c_off = np.concatenate([[0], np.cumsum(c_sizes)]).astype(np.int64); d_off = np.concatenate([[0], np.cumsum(d_sizes)]).astype(np.int64)
    ranges = frame_ranges(n_frames, world)
    fs = frame_size or int(max(1, np.max(d_sizes))) if n_frames else 1
    cf = pick_chunk_frames(n_frames, world, fs, chunk_bytes)
    chunks = [chunk_ranges(lo, hi, cf) for lo, hi in ranges]
    rounds = max([len(c) for c in chunks] + [0])
    lo, hi = ranges[rank]
    codec.device_ms = 0.0
    if rank == root:
        out = codec.empty(int(d_off[-1]), device)
        down, up = [], []
        for k in range(rounds):                              # everything is posted before the first frame is decoded
            sel = [r for r in range(world) if r != root and k < len(chunks[r])]
            down.append(_post([dist.P2POp(dist.isend, comp_root[int(c_off[chunks[r][k][0]]): int(c_off[chunks[r][k][1]])], r, g.down)
                               for r in sel if c_off[chunks[r][k][1]] > c_off[chunks[r][k][0]]]))
            up.append(_post([dist.P2POp(dist.irecv, out[int(d_off[chunks[r][k][0]]): int(d_off[chunks[r][k][1]])], r, g.up)
                             for r in sel if d_off[chunks[r][k][1]] > d_off[chunks[r][k][0]]]))
        for (f0, f1) in chunks[root]:                        # the root's own shard, decoded in place
            codec.decompress_into(comp_root[int(c_off[f0]):], c_off[f0: f1 + 1] - c_off[f0], d_off[f0: f1 + 1] - d_off[f0], verify, out[int(d_off[f0]):])
        t1 = time.perf_counter()
        for rr in down + up:
            _wait(rr)
        if stats is not None:
            t2 = _now(device)
            stats.update(decompress_total_ms=(t2 - t0) * 1e3, decompress_codec_ms=codec.device_ms, decompress_wait_ms=(t2 - t1) * 1e3,
                         decompress_chunks=len(chunks[rank]))
        return out[: int(d_off[-1])]
    cb0 = int(c_off[lo]); db0 = int(d_off[lo])
    mine = codec.empty(int(c_off[hi]) - cb0, device)
    out_local = codec.empty(int(d_off[hi]) - db0, device)
    recv = [_post([dist.P2POp(dist.irecv, mine[int(c_off[f0]) - cb0: int(c_off[f1]) - cb0], root, g.down)] if c_off[f1] > c_off[f0] else [])
            for (f0, f1) in chunks[rank]]
    sends = []
    for k, (f0, f1) in enumerate(chunks[rank]):
        _wait(recv[k])
        codec.decompress_into(mine[int(c_off[f0]) - cb0:], c_off[f0: f1 + 1] - c_off[f0], d_off[f0: f1 + 1] - d_off[f0], verify, out_local[int(d_off[f0]) - db0:])
        if d_off[f1] > d_off[f0]:
            sends.append(_post([dist.P2POp(dist.isend, out_local[int(d_off[f0]) - db0: int(d_off[f1]) - db0], root, g.up)]))
    t1 = time.perf_counter()
    for rr in sends:
        _wait(rr)
    if stats is not None:
        t2 = _now(device)
        stats.update(decompress_total_ms=(t2 - t0) * 1e3, decompress_codec_ms=codec.device_ms, decompress_wait_ms=(t2 - t1) * 1e3,
                     decompress_chunks=len(chunks[rank]))
    return None
