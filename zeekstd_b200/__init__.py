"""zeekstd_b200 -- H100-native seekable-Zstandard codec behind rorosen/zeekstd's API surface.

Python mirror of the reference's public items (lib/src/lib.rs:38-58) over the C ABI in
include/zeekstd_b200.h; every codec byte is produced by the CUDA kernels in csrc/.

    Encoder / RawEncoder / EncodeOptions / FrameSizePolicy     lib/src/encode.rs
    Decoder / DecodeOptions                                     lib/src/decode.rs
    SeekTable / Serializer / Format                             lib/src/seek_table.rs
    BytesWrapper / OffsetFrom / Seekable                        lib/src/seekable.rs
    Error                                                       lib/src/error.rs

There is no CPU fallback: constructing a Context without a usable CUDA device raises Error.
"""
from __future__ import annotations

import ctypes
import io
from ctypes import byref, c_size_t, c_uint32, c_uint64, c_void_p

import numpy as np

from . import _native
from ._native import CompressionProgress, EpilogueProgress

SEEKABLE_MAGIC_NUMBER = 0x8F92EAB1      # lib.rs:52
SEEKABLE_MAX_FRAMES = 0x08000000        # lib.rs:54
SEEK_TABLE_INTEGRITY_SIZE = 9           # lib.rs:56
SEEKABLE_MAX_FRAME_SIZE = 0x40000000    # lib.rs:58

_ERR_NUMBER_CONVERSION = -1001
_ERR_OFFSET_OUT_OF_RANGE = -1002
_ERR_FRAME_INDEX_TOO_LARGE = -1003
_ERR_IO = -1004
_ERR_NO_DEVICE = -1005
_ERR_CUDA = -1007


class Error(Exception):
    """lib/src/error.rs: opaque error with kind predicates; zstd codes keep libzstd's numbering."""

    def __init__(self, rc: int, lib=None):
        self.rc = int(rc)
        lib = lib or _native.default_lib()
        name = lib.zk_error_name(self.rc)
        detail = ""
        if self.rc == _ERR_CUDA:
            msg = lib.zk_last_cuda_error()
            detail = f" [{msg.decode()}]" if msg else ""
        super().__init__(f"{name.decode() if name else 'error'}{detail}; code {self.rc}")

    def is_number_conversion_failed(self) -> bool: return self.rc == _ERR_NUMBER_CONVERSION
    def is_offset_out_of_range(self) -> bool: return self.rc == _ERR_OFFSET_OUT_OF_RANGE
    def is_frame_index_too_large(self) -> bool: return self.rc == _ERR_FRAME_INDEX_TOO_LARGE
    def is_io(self) -> bool: return self.rc == _ERR_IO
    def is_cuda(self) -> bool: return self.rc == _ERR_CUDA
    def is_zstd(self) -> bool: return -1000 < self.rc < 0
    def zstd_code(self) -> int: return -self.rc if self.is_zstd() else 0


def _check(rc: int, lib=None):
    if rc != 0:
        raise Error(rc, lib)


def _buf(b):
    """-> (address, length, keepalive) for bytes-like / numpy input"""
    if isinstance(b, np.ndarray):
        a = np.ascontiguousarray(b).view(np.uint8).reshape(-1)
        return a.ctypes.data, a.size, a
    a = np.frombuffer(b, dtype=np.uint8) if len(b) else np.zeros(0, dtype=np.uint8)
    return a.ctypes.data, a.size, (a, b)


class Format:
    """seek_table::Format (seek_table.rs:228-241)"""
    Head = 0
    Foot = 1


class FrameSizePolicy:
    """encode.rs:21-39"""
    COMPRESSED = 0
    UNCOMPRESSED = 1
    CONTENT = 2

    def __init__(self, kind: int, size: int):
        self.kind, self.size = kind, size

    @classmethod
    def Compressed(cls, size: int): return cls(cls.COMPRESSED, size)

    @classmethod
    def Uncompressed(cls, size: int): return cls(cls.UNCOMPRESSED, size)

    @classmethod
    def ContentDefined(cls, size: int):
        """frames end where a rolling hash of the input says so, about `size` bytes apart on average (between size/4 and 4*size), so that
        an edit changes only the frames around it.  An extension of this codec: Encoder only (not RawEncoder, not with long-distance
        matching); Context.compress_frames_cdc is the batch form"""
        return cls(cls.CONTENT, size)

    @classmethod
    def default(cls): return cls.Uncompressed(0x200000)


class Context:
    """Owns the CUDA streams / HBM scratch (the role CCtx / DCtx play in the reference)."""

    def __init__(self, device: int = 0, lib=None):
        self.lib = lib or _native.default_lib()
        h = c_void_p()
        _check(self.lib.zk_ctx_create(device, 0, byref(h)), self.lib)
        self._h = h

    def close(self):
        if self._h:
            self.lib.zk_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def kernel_launches(self) -> int: return int(self.lib.zk_ctx_kernel_launches(self._h))

    @property
    def decode_segments(self) -> int:
        """execution segments the decoder has run so far: independent runs of blocks, several per entry where the data allows"""
        return int(self.lib.zk_ctx_decode_segments(self._h))

    @property
    def last_device_ms(self) -> float: return float(self.lib.zk_ctx_last_device_ms(self._h))

    # ---- batch codec (the hot path) ------------------------------------------------------------
    def compress_frames(self, data, frame_size: int = 0x200000, level: int = 0, checksum: bool = False, prefix=None, long_distance: bool = False,
                        long_mode: bool = False):
        """-> (compressed bytes (np.uint8), c_sizes, d_sizes).  Host buffers.  prefix: raw-content prefix of every frame.
        long_distance: match every frame against the whole prefix (its last 128 MiB), not only its last 32 KiB: patch mode.  Every level
        then writes what level 16 writes; without a prefix the flag changes nothing.
        long_mode: match every frame also against its own bytes up to 2^27 back (zstd --long), and against the whole prefix as
        long_distance does; every level writes what level 16 writes."""
        addr, n, keep = _buf(data)
        lib = self.lib
        cap = lib.zk_compress_bound(n, frame_size)
        dst = np.empty(cap + 64, dtype=np.uint8)
        nfmax = n // max(frame_size, 1) + 2
        cs = np.zeros(nfmax, dtype=np.uint32); ds = np.zeros(nfmax, dtype=np.uint32)
        nf = c_uint32(); dl = c_size_t()
        if prefix is not None or long_mode:
            paddr, pn, pkeep = _buf(prefix) if prefix is not None else (None, 0, None)
            fn = lib.zk_compress_frames_long if long_mode else lib.zk_compress_frames_ldm if long_distance else lib.zk_compress_frames_prefix
            _check(fn(self._h, addr, n, frame_size, level, int(checksum), paddr, pn, dst.ctypes.data, cap,
                                                 cs.ctypes.data_as(_native.u32p), ds.ctypes.data_as(_native.u32p), nfmax, byref(nf), byref(dl)), lib)
        else:
            _check(lib.zk_compress_frames(self._h, addr, n, frame_size, level, int(checksum), dst.ctypes.data, cap,
                                          cs.ctypes.data_as(_native.u32p), ds.ctypes.data_as(_native.u32p), nfmax, byref(nf),
                                          byref(dl)), lib)
        return dst[: dl.value], cs[: nf.value].copy(), ds[: nf.value].copy()

    def compress_frames_sized(self, data, frame_sizes, level: int = 0, checksum: bool = False, prefix=None, long_distance: bool = False,
                              long_mode: bool = False, prefix_ranges=None):
        """frames of caller-chosen sizes in one batch: frame f covers the next frame_sizes[f] bytes of data (their sum is its length)
        -> (compressed bytes (np.uint8), c_sizes, d_sizes).  Each frame is what compress_frames makes of its bytes alone
        (long_distance and long_mode as there).  prefix_ranges (n x 2 integers): frame f's prefix is only
        prefix[prefix_ranges[f][0]:prefix_ranges[f][1]] (zk_compress_frames_sized_prefixes), and the frame is what this call makes of it
        alone with that slice as the prefix."""
        addr, n, keep = _buf(data)
        ds = np.ascontiguousarray(frame_sizes, dtype=np.uint32).reshape(-1)
        if int(np.sum(ds, dtype=np.uint64)) != n:
            raise ValueError(f"frame sizes add up to {int(np.sum(ds, dtype=np.uint64))} bytes, the input has {n}")
        lib = self.lib
        dsp = ds.ctypes.data_as(_native.u32p)
        cap = lib.zk_compress_bound_sized(dsp, ds.size)
        dst = np.empty(cap + 64, dtype=np.uint8)
        cs = np.zeros(ds.size, dtype=np.uint32)
        dl = c_size_t()
        paddr, pn, pkeep = _buf(prefix) if prefix is not None else (None, 0, None)
        if prefix_ranges is not None:
            rg = _ranges(prefix_ranges, ds.size)
            _check(lib.zk_compress_frames_sized_prefixes(self._h, addr, dsp, ds.size, level, int(checksum), paddr, pn,
                                                         rg.ctypes.data_as(_native.u64p), int(long_distance), int(long_mode), dst.ctypes.data,
                                                         cap, cs.ctypes.data_as(_native.u32p), byref(dl)), lib)
            return dst[: dl.value], cs, ds.copy()
        fn = lib.zk_compress_frames_sized_long if long_mode else lib.zk_compress_frames_sized_ldm if long_distance else lib.zk_compress_frames_sized
        _check(fn(self._h, addr, dsp, ds.size, level, int(checksum), paddr, pn, dst.ctypes.data, cap,
                                            cs.ctypes.data_as(_native.u32p), byref(dl)), lib)
        return dst[: dl.value], cs, ds.copy()

    def compress_frames_csize(self, data, target: int, level: int = 0, checksum: bool = False, prefix=None, final: bool = True):
        """FrameSizePolicy::Compressed(target) on the batch path -> (compressed bytes (np.uint8), c_sizes, d_sizes, consumed).
        A frame closes after the first 32 KiB block at which its header + blocks reach `target` (or at 1 GiB of input).
        final=False: only closed frames are made and `consumed` input bytes are covered; pass the rest again with more input."""
        addr, n, keep = _buf(data)
        lib = self.lib
        cap = lib.zk_compress_bound(n, 32768)
        dst = np.empty(cap + 64, dtype=np.uint8)
        nfmax = n // 32768 + 2
        cs = np.zeros(nfmax, dtype=np.uint32); ds = np.zeros(nfmax, dtype=np.uint32)
        nf = c_uint32(); dl = c_size_t(); used = c_size_t()
        paddr, pn, pkeep = _buf(prefix) if prefix is not None else (None, 0, None)
        _check(lib.zk_compress_frames_csize(self._h, addr, n, target, level, int(checksum), paddr, pn, int(final), dst.ctypes.data, cap,
                                            cs.ctypes.data_as(_native.u32p), ds.ctypes.data_as(_native.u32p), nfmax, byref(nf), byref(dl),
                                            byref(used)), lib)
        return dst[: dl.value], cs[: nf.value].copy(), ds[: nf.value].copy(), int(used.value)

    def compress_frames_cdc(self, data, size: int, level: int = 0, checksum: bool = False, prefix=None, final: bool = True):
        """FrameSizePolicy::ContentDefined(size) on the batch path -> (compressed bytes (np.uint8), c_sizes, d_sizes, consumed).
        Frame boundaries depend on the input bytes and `size` only (the rule: include/zeekstd_b200.h, zk_compress_frames_cdc); frame f's
        bytes are what compress_frames_sized writes for the same sizes.  final=False: only closed frames are made and `consumed` input
        bytes are covered; pass the rest again with more input."""
        addr, n, keep = _buf(data)
        lib = self.lib
        cap = lib.zk_compress_bound(n, 1024)
        dst = np.empty(cap + 64, dtype=np.uint8)
        nfmax = n // 1024 + 1
        cs = np.zeros(nfmax, dtype=np.uint32); ds = np.zeros(nfmax, dtype=np.uint32)
        nf = c_uint32(); dl = c_size_t(); used = c_size_t()
        paddr, pn, pkeep = _buf(prefix) if prefix is not None else (None, 0, None)
        _check(lib.zk_compress_frames_cdc(self._h, addr, n, size, level, int(checksum), paddr, pn, int(final), dst.ctypes.data, cap,
                                          cs.ctypes.data_as(_native.u32p), ds.ctypes.data_as(_native.u32p), nfmax, byref(nf), byref(dl),
                                          byref(used)), lib)
        return dst[: dl.value], cs[: nf.value].copy(), ds[: nf.value].copy(), int(used.value)

    def cut_frames_cdc(self, data, size: int, final: bool = True):
        """the frame sizes of FrameSizePolicy::ContentDefined(size) without compressing -> (d_sizes (np.uint32), consumed): exactly what
        compress_frames_cdc returns for the same data, size and final (zk_cut_frames_cdc)."""
        addr, n, keep = _buf(data)
        nfmax = n // 1024 + 1
        ds = np.zeros(nfmax, dtype=np.uint32)
        nf = c_uint32(); used = c_size_t()
        _check(self.lib.zk_cut_frames_cdc(self._h, addr, n, size, int(final), ds.ctypes.data_as(_native.u32p), nfmax, byref(nf), byref(used)),
               self.lib)
        return ds[: nf.value].copy(), int(used.value)

    def compress_frames_reuse(self, data, frame_sizes, old, level: int = 0, checksum: bool = False, long_mode: bool = False):
        """compress_frames_sized(data, frame_sizes, level, checksum, long_mode=long_mode), copying every frame whose bytes an entry of the
        old seekable archive `old` (bytes ending in its Foot seek table) already holds -> (compressed bytes (np.uint8), c_sizes, reused):
        reused[f] is the old entry frame f copies, or 0xFFFFFFFF.  The rule (include/zeekstd_b200.h, zk_compress_frames_sized_reuse): the
        lowest-index old entry of frame f's size, checksum flag and key is copied verbatim iff its decoded bytes equal the frame's."""
        addr, n, keep = _buf(data)
        ds = np.ascontiguousarray(frame_sizes, dtype=np.uint32).reshape(-1)
        if int(np.sum(ds, dtype=np.uint64)) != n:
            raise ValueError(f"frame sizes add up to {int(np.sum(ds, dtype=np.uint64))} bytes, the input has {n}")
        oaddr, on, okeep = _buf(old)
        co, do = SeekTable.from_bytes(old, Format.Foot, self.lib).offsets()
        lib = self.lib
        dsp = ds.ctypes.data_as(_native.u32p)
        cap = lib.zk_compress_bound_sized(dsp, ds.size) + int(co[-1] - co[0])
        dst = np.empty(cap + 64, dtype=np.uint8)
        cs = np.zeros(ds.size, dtype=np.uint32); ru = np.zeros(ds.size, dtype=np.uint32)
        dl = c_size_t()
        _check(lib.zk_compress_frames_sized_reuse(self._h, addr, dsp, ds.size, level, int(checksum), int(long_mode), oaddr, on,
                                                  co.ctypes.data_as(_native.u64p), do.ctypes.data_as(_native.u64p), len(co) - 1,
                                                  dst.ctypes.data, cap, cs.ctypes.data_as(_native.u32p), ru.ctypes.data_as(_native.u32p),
                                                  byref(dl)), lib)
        return dst[: dl.value], cs, ru

    def decompress_frames(self, comp, c_off, d_off, verify_checksum: bool = True, out: np.ndarray | None = None, need=None, prefix=None,
                          prefix_ranges=None):
        """decode frames given N+1 cumulative offsets -> (np.uint8 output, per-frame status, rc).
        need (optional, one uint32 per frame): only that many leading bytes of each frame are wanted (range reads,
        zk_decompress_frames_upto): the rest of a frame's output range is then unspecified and its checksum is not verified.
        prefix_ranges (n x 2 integers): entry e is decoded against prefix[prefix_ranges[e][0]:prefix_ranges[e][1]] only
        (zk_decompress_frames_prefixes).  prefix may be a ReferenceArchive: its decoded content is the prefix, and only the entries
        under the ranges are decoded, on the GPU, at every level of its chain (zk_decompress_frames_prefixes_chain)."""
        addr, n, keep = _buf(comp)
        co = np.ascontiguousarray(c_off, dtype=np.uint64); do = np.ascontiguousarray(d_off, dtype=np.uint64)
        nf = len(co) - 1
        total = int(do[-1])
        if out is None:
            out = np.empty(total + 64, dtype=np.uint8)
        elif not (isinstance(out, np.ndarray) and out.dtype == np.uint8 and out.flags["C_CONTIGUOUS"] and out.size >= total):
            raise ValueError(f"out: need a C-contiguous np.uint8 array of at least {total} bytes")
        st = np.zeros(max(nf, 1), dtype=np.int32)
        nd = None if need is None else np.ascontiguousarray(need, dtype=np.uint32)
        if nd is not None and len(nd) != nf:
            raise ValueError("need: one entry per frame")
        if isinstance(prefix, ReferenceArchive):
            rg = None if prefix_ranges is None else _ranges(prefix_ranges, nf)
            rc = self.lib.zk_decompress_frames_prefixes_chain(self._h, addr, co.ctypes.data_as(_native.u64p), do.ctypes.data_as(_native.u64p),
                                                              nf, out.ctypes.data, None if nd is None else nd.ctypes.data_as(_native.u32p),
                                                              int(verify_checksum), st.ctypes.data_as(_native.i32p), *prefix._chain(),
                                                              None if rg is None else rg.ctypes.data_as(_native.u64p))
            return out[:total], st[:nf], rc
        paddr, pn, pkeep = _buf(prefix) if prefix is not None else (None, 0, None)
        if prefix_ranges is not None:
            rg = _ranges(prefix_ranges, nf)
            rc = self.lib.zk_decompress_frames_prefixes(self._h, addr, co.ctypes.data_as(_native.u64p), do.ctypes.data_as(_native.u64p), nf,
                                                        out.ctypes.data, None if nd is None else nd.ctypes.data_as(_native.u32p),
                                                        int(verify_checksum), st.ctypes.data_as(_native.i32p), paddr, pn,
                                                        rg.ctypes.data_as(_native.u64p))
            return out[:total], st[:nf], rc
        rc = self.lib.zk_decompress_frames_prefix(self._h, addr, co.ctypes.data_as(_native.u64p), do.ctypes.data_as(_native.u64p), nf,
                                                  out.ctypes.data, None if nd is None else nd.ctypes.data_as(_native.u32p),
                                                  int(verify_checksum), st.ctypes.data_as(_native.i32p), paddr, pn)
        return out[:total], st[:nf], rc


    # ---- seekable patches ------------------------------------------------------------------------
    @property
    def prefix_bytes_uploaded(self) -> int:
        """prefix bytes this context has copied to the device so far (zk_ctx_prefix_bytes_uploaded)"""
        return int(self.lib.zk_ctx_prefix_bytes_uploaded(self._h))

    @property
    def reference_entries_decoded(self) -> int:
        """entries of reference archives this context has decoded so far (zk_ctx_reference_entries_decoded)"""
        return int(self.lib.zk_ctx_reference_entries_decoded(self._h))

    def patch_ranges(self, new, frame_sizes, old, margin: int | None = None) -> np.ndarray:
        """the slice of `old` each frame of `new` is matched against in a seekable patch -> n x 2 np.uint64 (lo, hi), found on the GPU by
        content anchors (the rule: include/zeekstd_b200.h, zk_patch_ranges).  margin: bytes added on each side (default: the largest frame
        size, which is the frame size of uniform frames).  old may be a ReferenceArchive: the same ranges, with OLD decoded on the GPU
        (zk_patch_ranges_chain)"""
        addr, n, keep = _buf(new)
        ds = np.ascontiguousarray(frame_sizes, dtype=np.uint32).reshape(-1)
        if int(np.sum(ds, dtype=np.uint64)) != n:
            raise ValueError(f"frame sizes add up to {int(np.sum(ds, dtype=np.uint64))} bytes, the input has {n}")
        m = int(ds.max()) if margin is None and ds.size else int(margin or 0)
        rg = np.zeros((max(ds.size, 1), 2), dtype=np.uint64)
        if isinstance(old, ReferenceArchive):
            _check(self.lib.zk_patch_ranges_chain(self._h, addr, ds.ctypes.data_as(_native.u32p), ds.size, *old._chain(), m,
                                                  rg.ctypes.data_as(_native.u64p)), self.lib)
            return rg[: ds.size]
        oaddr, on, okeep = _buf(old)
        _check(self.lib.zk_patch_ranges(self._h, addr, ds.ctypes.data_as(_native.u32p), ds.size, oaddr, on, m,
                                        rg.ctypes.data_as(_native.u64p)), self.lib)
        return rg[: ds.size]

    def compress_frames_patch(self, new, frame_sizes, old, ranges, level: int = 0, checksum: bool = False):
        """frame f of `new` against old[ranges[f][0]:ranges[f][1]] with long-distance matching, for an `old` of any size
        (zk_compress_frames_patch) -> (compressed bytes (np.uint8), c_sizes, d_sizes).  Frame f is what compress_frames_sized(frame alone,
        prefix=old, long_distance=True, prefix_ranges=[ranges[f]]) writes.  old may be a ReferenceArchive: the same bytes, with each group's
        slices of OLD decoded on the GPU (zk_compress_frames_patch_chain)"""
        addr, n, keep = _buf(new)
        ds = np.ascontiguousarray(frame_sizes, dtype=np.uint32).reshape(-1)
        if int(np.sum(ds, dtype=np.uint64)) != n:
            raise ValueError(f"frame sizes add up to {int(np.sum(ds, dtype=np.uint64))} bytes, the input has {n}")
        rg = _ranges(ranges, ds.size)
        dsp = ds.ctypes.data_as(_native.u32p)
        cap = self.lib.zk_compress_bound_sized(dsp, ds.size)
        dst = np.empty(cap + 64, dtype=np.uint8)
        cs = np.zeros(max(ds.size, 1), dtype=np.uint32)
        dl = c_size_t()
        if isinstance(old, ReferenceArchive):
            _check(self.lib.zk_compress_frames_patch_chain(self._h, addr, dsp, ds.size, level, int(checksum), *old._chain(),
                                                           rg.ctypes.data_as(_native.u64p), dst.ctypes.data, cap, cs.ctypes.data_as(_native.u32p),
                                                           byref(dl)), self.lib)
            return dst[: dl.value], cs[: ds.size], ds.copy()
        oaddr, on, okeep = _buf(old)
        _check(self.lib.zk_compress_frames_patch(self._h, addr, dsp, ds.size, level, int(checksum), oaddr, on, rg.ctypes.data_as(_native.u64p),
                                                 dst.ctypes.data, cap, cs.ctypes.data_as(_native.u32p), byref(dl)), self.lib)
        return dst[: dl.value], cs[: ds.size], ds.copy()

    def compress_patch_slices(self, new, frame_sizes, old, level: int = 0, checksum: bool = False, margin: int | None = None) -> bytes:
        """a seekable patch of `new` against `old` -> the archive's bytes: the slice frame (the ranges of patch_ranges), then the frames
        of compress_frames_patch, then the Foot seek table.  Entry 0's compressed size includes the slice frame.  old may be a
        ReferenceArchive, chained or not: the same bytes."""
        ds = np.ascontiguousarray(frame_sizes, dtype=np.uint32).reshape(-1)
        if ds.size == 0:
            raise ValueError("a seekable patch has at least one frame")
        rg = self.patch_ranges(new, ds, old, margin)
        comp, cs, _ = self.compress_frames_patch(new, ds, old, rg, level, checksum)
        head = patch_slices_write(old.old_len if isinstance(old, ReferenceArchive) else _buf(old)[1], rg, self.lib)
        table = SeekTable(lib=self.lib)
        for f, (c, d) in enumerate(zip(cs.tolist(), ds.tolist())):
            table.log_frame(c + (len(head) if f == 0 else 0), d)
        return head + comp.tobytes() + table.into_serializer().to_bytes()


PATCH_SLICES_MAGIC = 0x184D2A5B


class ReferenceArchive:
    """a seekable archive as the reference (OLD) of a seekable patch: OLD is its decoded content, and the patch calls that take one decode
    on the GPU only the entries of it they need (DESIGN §3.4.2).  data: the archive's bytes or a mapping of it (kept, not copied).  Its
    entries come from the Foot seek table at its end (the default), from seek_table (a SeekTable, or the bytes of one in `format`, e.g.
    a stand-alone Head table), or from explicit c_off / d_off (n + 1 offsets each, as Context.decompress_frames takes them).
    A seekable patch (the slice frame at the start of its first entry) needs `base`: the ReferenceArchive of the version it was made
    against, which may itself be a patch with a base of its own.  OLD is then the patch applied to its base's decoded content, and the
    calls decode every level of the chain on the GPU, each only where the level above reads it (DESIGN §3.4.3).  Without `base` a patch is
    refused; a `base` under a plain archive, or one whose decoded length is not the slice frame's old_len, is a ValueError."""

    def __init__(self, data, seek_table=None, format: int = Format.Foot, c_off=None, d_off=None, lib=None, base=None):
        self.lib = lib or _native.default_lib()
        self._addr, self._len, self._keep = _buf(data)
        if c_off is not None or d_off is not None:
            if c_off is None or d_off is None:
                raise ValueError("c_off and d_off go together")
            co, do = np.ascontiguousarray(c_off, dtype=np.uint64), np.ascontiguousarray(d_off, dtype=np.uint64)
            if co.ndim != 1 or co.size == 0 or co.shape != do.shape:
                raise ValueError("c_off, d_off: n + 1 offsets each")
        else:
            if seek_table is None:
                seek_table = SeekTable.from_bytes(data, format, self.lib)
            elif not isinstance(seek_table, SeekTable):
                seek_table = SeekTable.from_bytes(seek_table, format, self.lib)
            co, do = seek_table.offsets()
        self.c_off, self.d_off = co, do
        c0 = int(co[0])
        view = self._keep if isinstance(self._keep, np.ndarray) else self._keep[0]
        patch = int(co[-1]) - c0 >= 4 and c0 + 4 <= self._len and int.from_bytes(view[c0:c0 + 4].tobytes(), "little") == PATCH_SLICES_MAGIC
        if base is None:
            if patch:
                raise ValueError("the reference archive is a seekable patch; restore it first")
        elif not isinstance(base, ReferenceArchive):
            raise ValueError("base: the ReferenceArchive of the version the patch was made against")
        elif not patch:
            raise ValueError("base is for a seekable patch; this reference archive is a plain one")
        else:
            old_len = patch_slices_read(view[c0:int(co[-1])], self.n_entries, self.lib)[0]
            if old_len != base.old_len:
                raise ValueError(f"the base decodes to {base.old_len} bytes, the seekable patch was made against {old_len} bytes")
            if base.depth >= _native.CHAIN_MAX_DEPTH:
                raise ValueError(f"a reference chain has at most {_native.CHAIN_MAX_DEPTH} levels")
        self.base = base

    @property
    def n_entries(self) -> int: return len(self.c_off) - 1

    @property
    def old_len(self) -> int:
        """bytes of OLD, the archive's decoded content"""
        return int(self.d_off[-1])

    @property
    def depth(self) -> int:
        """levels of the chain this reference heads: 1 for a plain archive"""
        return 1 if self.base is None else self.base.depth + 1

    @property
    def chain(self) -> list:
        """the ReferenceArchive of every level, root first (the last is this one)"""
        return [self] if self.base is None else self.base.chain + [self]

    def _chain(self):
        """the (chain, depth) arguments of the _chain calls (the array keeps no level alive: hold self while it is used)"""
        levels = self.chain
        arr = (_native.ReferenceArchiveDesc * len(levels))()
        for d, r in zip(arr, levels):
            d.comp, d.len, d.n = r._addr, r._len, r.n_entries
            d.c_off, d.d_off = r.c_off.ctypes.data_as(_native.u64p), r.d_off.ctypes.data_as(_native.u64p)
        return arr, len(levels)


def patch_slices_size(n_frames: int) -> int:
    """bytes of the slice frame of a seekable patch of n_frames frames"""
    return 28 + 16 * n_frames


def patch_slices_read(buf, n_frames: int, lib=None):
    """the slice frame at the start of a seekable patch's first entry -> (old_len, ranges (n_frames x 2 np.uint64), frame length).  Raises
    Error (ZK_ERR_INVALID_ARG) for anything that is not a valid slice frame of n_frames slices (zk_patch_slices_read)"""
    lib = lib or _native.default_lib()
    addr, n, keep = _buf(buf)
    rg = np.zeros((max(n_frames, 1), 2), dtype=np.uint64)
    ol = c_uint64(); fl = c_size_t()
    _check(lib.zk_patch_slices_read(addr, n, n_frames, byref(ol), rg.ctypes.data_as(_native.u64p), byref(fl)), lib)
    return int(ol.value), rg[:n_frames], int(fl.value)


def patch_slices_write(old_len: int, ranges, lib=None) -> bytes:
    """the slice frame of a seekable patch whose frames have these (lo, hi) ranges of an OLD of old_len bytes (zk_patch_slices_write)"""
    lib = lib or _native.default_lib()
    rg = np.ascontiguousarray(np.asarray(ranges, dtype=np.uint64).reshape(-1, 2))
    out = np.zeros(lib.zk_patch_slices_size(len(rg)), dtype=np.uint8)
    w = c_size_t()
    _check(lib.zk_patch_slices_write(old_len, rg.ctypes.data_as(_native.u64p) if rg.size else None, len(rg), out.ctypes.data, out.size,
                                     byref(w)), lib)
    return out[: w.value].tobytes()


def _ranges(prefix_ranges, n: int) -> np.ndarray:
    """n (lo, hi) prefix ranges -> a C-contiguous n x 2 np.uint64 array"""
    rg = np.asarray(prefix_ranges)
    if rg.size and (rg.dtype.kind not in "iu" or int(rg.min()) < 0):
        raise ValueError("prefix_ranges: non-negative integers")
    rg = np.ascontiguousarray(rg, dtype=np.uint64).reshape(-1, 2) if rg.size else np.zeros((0, 2), dtype=np.uint64)
    if len(rg) != n:
        raise ValueError(f"prefix_ranges: one (lo, hi) pair per frame, {n} expected, {len(rg)} given")
    return rg if n else np.zeros((1, 2), dtype=np.uint64)


_default_ctx: Context | None = None


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(0)
    return _default_ctx


def set_default_context(ctx: Context | None) -> None:
    global _default_ctx
    _default_ctx = ctx


# ---------------------------------------------------------------------------------------------- SeekTable
class SeekTable:
    """lib/src/seek_table.rs:267-935"""

    def __init__(self, _h=None, _owned=True, lib=None, _keep=None):
        self.lib = lib or _native.default_lib()
        self._h = _h if _h is not None else c_void_p(self.lib.zk_seek_table_new())
        self._owned = _owned
        self._keep = _keep

    def __del__(self):
        try:
            if self._owned and self._h:
                self.lib.zk_seek_table_free(self._h)
        except Exception:
            pass

    @classmethod
    def from_bytes(cls, buf, format: int = Format.Foot, lib=None):
        """SeekTable::from_seekable_format(&mut BytesWrapper::new(buf), format), :379-436"""
        lib = lib or _native.default_lib()
        addr, n, keep = _buf(buf)
        h = c_void_p()
        _check(lib.zk_seek_table_from_bytes(addr, n, format, byref(h)), lib)
        return cls(h, True, lib)

    from_seekable = from_bytes

    @classmethod
    def from_reader(cls, reader, lib=None):
        """stand-alone Head-format seek table, :461-493"""
        return cls.from_bytes(reader.read(), Format.Head, lib)

    def clone(self): return SeekTable(c_void_p(self.lib.zk_seek_table_clone(self._h)), True, self.lib)
    def log_frame(self, c_size: int, d_size: int): _check(self.lib.zk_seek_table_log_frame(self._h, c_size, d_size), self.lib)
    def num_frames(self) -> int: return int(self.lib.zk_seek_table_num_frames(self._h))
    def frame_index_comp(self, off: int) -> int: return int(self.lib.zk_seek_table_frame_index_comp(self._h, off))
    def frame_index_decomp(self, off: int) -> int: return int(self.lib.zk_seek_table_frame_index_decomp(self._h, off))

    def _get(self, fn, index):
        v = c_uint64()
        _check(fn(self._h, index, byref(v)), self.lib)
        return int(v.value)

    def frame_start_comp(self, i): return self._get(self.lib.zk_seek_table_frame_start_comp, i)
    def frame_start_decomp(self, i): return self._get(self.lib.zk_seek_table_frame_start_decomp, i)
    def frame_end_comp(self, i): return self._get(self.lib.zk_seek_table_frame_end_comp, i)
    def frame_end_decomp(self, i): return self._get(self.lib.zk_seek_table_frame_end_decomp, i)
    def frame_size_comp(self, i): return self._get(self.lib.zk_seek_table_frame_size_comp, i)
    def frame_size_decomp(self, i): return self._get(self.lib.zk_seek_table_frame_size_decomp, i)
    def max_frame_size_comp(self): return int(self.lib.zk_seek_table_max_frame_size_comp(self._h))
    def max_frame_size_decomp(self): return int(self.lib.zk_seek_table_max_frame_size_decomp(self._h))
    def size_comp(self): return int(self.lib.zk_seek_table_size_comp(self._h))
    def size_decomp(self): return int(self.lib.zk_seek_table_size_decomp(self._h))

    def offsets(self):
        n = self.num_frames() + 1
        c = np.zeros(n, dtype=np.uint64); d = np.zeros(n, dtype=np.uint64)
        self.lib.zk_seek_table_offsets(self._h, c.ctypes.data_as(_native.u64p), d.ctypes.data_as(_native.u64p), n)
        return c, d

    def into_serializer(self): return self.into_format_serializer(Format.Foot)
    def into_format_serializer(self, format: int): return Serializer(c_void_p(self.lib.zk_seek_table_into_serializer(self._h, format)), self.lib)

    def __eq__(self, other):
        a, b = self.offsets(), other.offsets()
        return a[0].tolist() == b[0].tolist() and a[1].tolist() == b[1].tolist()


class Serializer(io.RawIOBase):
    """seek_table.rs:955-1059 (resumable; also readable like `impl Read`)"""

    def __init__(self, h, lib):
        super().__init__()
        self._h, self.lib = h, lib

    def __del__(self):
        try:
            if self._h:
                self.lib.zk_serializer_free(self._h)
        except Exception:
            pass

    def write_into(self, buf) -> int:
        mv = memoryview(buf)
        if len(mv) == 0:
            return 0
        arr = (ctypes.c_uint8 * len(mv)).from_buffer(mv)
        return int(self.lib.zk_serializer_write_into(self._h, arr, len(mv)))

    def reset(self): self.lib.zk_serializer_reset(self._h)
    def encoded_len(self) -> int: return int(self.lib.zk_serializer_encoded_len(self._h))
    def readable(self): return True
    def readinto(self, b): return self.write_into(b)

    def to_bytes(self) -> bytes:
        out = bytearray(self.encoded_len())
        n = self.write_into(out)
        return bytes(out[:n])


# ---------------------------------------------------------------------------------------------- encode
class EncodeOptions:
    """encode.rs:110-207 (builder)"""

    def __init__(self, ctx: Context | None = None):
        self.ctx = ctx or default_context()
        self._policy = FrameSizePolicy.default()
        self._checksum = False
        self._level = 0
        self._ldm = False
        self._long = False

    def frame_size_policy(self, policy: FrameSizePolicy): self._policy = policy; return self
    def checksum_flag(self, flag: bool): self._checksum = bool(flag); return self
    def compression_level(self, level: int): self._level = int(level); return self

    def long_distance_matching(self, flag: bool):
        """match the frames of compress_with_prefix against the whole prefix (what the reference CLI sets on the CCtx it passes to
        with_cctx for patch files).  Every level then runs as level 16; into_encoder refuses it with FrameSizePolicy.Compressed and
        FrameSizePolicy.ContentDefined"""
        self._ldm = bool(flag); return self

    def long_mode(self, flag: bool):
        """match every frame also against its own bytes up to 2^27 back (zstd --long), and the frames of compress_with_prefix against
        the whole prefix as long_distance_matching does.  Every level then runs as level 16; into_encoder refuses it with
        FrameSizePolicy.Compressed and FrameSizePolicy.ContentDefined"""
        self._long = bool(flag); return self

    def _native_opts(self):
        lib = self.ctx.lib
        o = c_void_p(lib.zk_encode_options_new(self.ctx._h))
        lib.zk_encode_options_frame_size_policy(o, self._policy.kind, self._policy.size)
        lib.zk_encode_options_checksum_flag(o, int(self._checksum))
        lib.zk_encode_options_compression_level(o, self._level)
        lib.zk_encode_options_long_distance_matching(o, int(self._ldm))
        lib.zk_encode_options_long_mode(o, int(self._long))
        return o

    def into_raw_encoder(self): return RawEncoder(self)
    def into_encoder(self, writer): return Encoder(writer, self)


class RawEncoder:
    """encode.rs:266-545"""

    def __init__(self, opts: EncodeOptions | None = None):
        opts = opts or EncodeOptions()
        self.ctx, self.lib = opts.ctx, opts.ctx.lib
        h = c_void_p()
        self._h = None
        o = opts._native_opts()
        rc = self.lib.zk_encode_options_into_raw_encoder(o, byref(h))
        if rc:                                              # refused options (FrameSizePolicy.ContentDefined) are not consumed
            self.lib.zk_encode_options_free(o)
        _check(rc, self.lib)
        self._h = h

    def __del__(self):
        try:
            if self._h:
                self.lib.zk_raw_encoder_free(self._h)
        except Exception:
            pass

    def compress(self, input, output) -> CompressionProgress:
        """-> progress with .in_progress / .out_progress (encode.rs:398)"""
        addr, n, keep = _buf(input)
        mv = memoryview(output)
        oarr = (ctypes.c_uint8 * len(mv)).from_buffer(mv) if len(mv) else None
        p = CompressionProgress()
        _check(self.lib.zk_raw_encoder_compress(self._h, addr, n, oarr, len(mv), byref(p)), self.lib)
        return p

    def compress_with_prefix(self, input, output, prefix=None) -> CompressionProgress:
        """encode.rs:311-354: `prefix` (bytes-like, or None) becomes the raw-content prefix of a frame when passed on the
        frame's first call; the caller keeps it alive until the frame is closed"""
        if prefix is None:
            return self.compress(input, output)
        addr, n, keep = _buf(input)
        paddr, pn, pkeep = _buf(prefix)
        self._prefix_keep = pkeep
        mv = memoryview(output)
        oarr = (ctypes.c_uint8 * len(mv)).from_buffer(mv) if len(mv) else None
        p = CompressionProgress()
        _check(self.lib.zk_raw_encoder_compress_with_prefix(self._h, addr, n, oarr, len(mv), paddr, pn, byref(p)), self.lib)
        return p

    def end_frame(self, output) -> EpilogueProgress:
        mv = memoryview(output)
        oarr = (ctypes.c_uint8 * len(mv)).from_buffer(mv) if len(mv) else None
        p = EpilogueProgress()
        _check(self.lib.zk_raw_encoder_end_frame(self._h, oarr, len(mv), byref(p)), self.lib)
        return p

    def seek_table(self) -> SeekTable:
        return SeekTable(c_void_p(self.lib.zk_raw_encoder_seek_table(self._h)), False, self.lib, _keep=self)

    def into_seek_table(self) -> SeekTable:
        h = c_void_p(self.lib.zk_raw_encoder_into_seek_table(self._h))
        self._h = None
        return SeekTable(h, True, self.lib)

    def reset_frame(self): self.lib.zk_raw_encoder_reset_frame(self._h)
    def reset_seek_table(self): self.lib.zk_raw_encoder_reset_seek_table(self._h)


class Encoder(io.RawIOBase):
    """encode.rs:568-800: compresses into any object with .write(bytes) (W: std::io::Write)"""

    def __init__(self, writer, opts: EncodeOptions | None = None):
        super().__init__()
        opts = opts or EncodeOptions()
        self.ctx, self.lib = opts.ctx, opts.ctx.lib
        self._writer = writer

        def _write(user, data, n):
            try:
                writer.write(ctypes.string_at(data, n))
                return 0
            except Exception:
                return -1

        def _flush(user):
            try:
                if hasattr(writer, "flush"):
                    writer.flush()
                return 0
            except Exception:
                return -1

        self._wcb = _native.WRITE_FN(_write)
        self._fcb = _native.FLUSH_FN(_flush)
        h = c_void_p()
        self._h = None
        o = opts._native_opts()
        rc = self.lib.zk_encode_options_into_encoder(o, self._wcb, self._fcb, None, byref(h))
        if rc:                                              # refused options are not consumed
            self.lib.zk_encode_options_free(o)
        _check(rc, self.lib)
        self._h = h

    def __del__(self):
        try:
            if self._h:
                self.lib.zk_encoder_free(self._h)
        except Exception:
            pass

    def compress(self, buf) -> int:
        addr, n, keep = _buf(buf)
        c = c_size_t()
        _check(self.lib.zk_encoder_compress(self._h, addr, n, byref(c)), self.lib)
        return int(c.value)

    def compress_with_prefix(self, buf, prefix=None) -> int:
        """encode.rs:641-665"""
        if prefix is None:
            return self.compress(buf)
        addr, n, keep = _buf(buf)
        paddr, pn, pkeep = _buf(prefix)
        self._prefix_keep = pkeep
        c = c_size_t()
        _check(self.lib.zk_encoder_compress_with_prefix(self._h, addr, n, paddr, pn, byref(c)), self.lib)
        return int(c.value)

    def writable(self): return True
    def write(self, b): return self.compress(b)

    def end_frame(self) -> int:
        w = c_size_t()
        _check(self.lib.zk_encoder_end_frame(self._h, byref(w)), self.lib)
        return int(w.value)

    def flush(self):
        if getattr(self, "_h", None):
            _check(self.lib.zk_encoder_flush(self._h), self.lib)

    def finish(self) -> int: return self.finish_format(Format.Foot)

    def finish_format(self, format: int) -> int:
        t = c_uint64()
        h, self._h = self._h, None
        _check(self.lib.zk_encoder_finish_format(h, format, byref(t)), self.lib)
        return int(t.value)

    def written_compressed(self) -> int: return int(self.lib.zk_encoder_written_compressed(self._h))
    def seek_table(self) -> SeekTable: return SeekTable(c_void_p(self.lib.zk_encoder_seek_table(self._h)), False, self.lib, _keep=self)


# ---------------------------------------------------------------------------------------------- decode
class OffsetFrom:
    """seekable.rs:8-13"""
    START = 0
    END = 1


class BytesWrapper:
    """seekable.rs:43-97: a seekable view over bytes"""

    def __init__(self, src):
        self.src = src


class DecodeOptions:
    """decode.rs:13-114 (builder).  src: BytesWrapper / bytes-like, or a file-like object with read+seek."""

    def __init__(self, src, ctx: Context | None = None):
        self.ctx = ctx or default_context()
        self.src = src
        self._seek_table = None
        self._lower = self._upper = self._offset = self._limit = None

    def seek_table(self, st: SeekTable): self._seek_table = st; return self
    def lower_frame(self, i: int): self._lower = i; return self
    def upper_frame(self, i: int): self._upper = i; return self
    def offset(self, v: int): self._offset = v; return self
    def offset_limit(self, v: int): self._limit = v; return self
    def into_decoder(self): return Decoder(self)


class Decoder(io.RawIOBase):
    """decode.rs:121-579 (incl. impl Read / impl Seek)"""

    def __init__(self, src_or_opts):
        super().__init__()
        opts = src_or_opts if isinstance(src_or_opts, DecodeOptions) else DecodeOptions(src_or_opts)
        self.ctx, self.lib = opts.ctx, opts.ctx.lib
        lib = self.lib
        src = opts.src
        self._keep = None
        if isinstance(src, BytesWrapper):
            src = src.src
        if isinstance(src, (bytes, bytearray, memoryview, np.ndarray)):
            addr, n, keep = _buf(src)
            self._keep = keep
            o = c_void_p(lib.zk_decode_options_new_bytes(self.ctx._h, addr, n))
        else:
            f = src

            def _set_offset(user, whence, off):
                try:
                    return f.seek(off, 0 if whence == 0 else 2)
                except Exception:
                    return -1

            def _read(user, buf, n):
                try:
                    data = f.read(n)
                    ctypes.memmove(buf, data, len(data))
                    return len(data)
                except Exception:
                    return -1

            self._cbs = (_native.SET_OFFSET_FN(_set_offset), _native.READ_FN(_read))
            sk = _native.Seekable(None, self._cbs[0], self._cbs[1])
            o = c_void_p(lib.zk_decode_options_new_seekable(self.ctx._h, sk))
            self._keep = f
        if opts._seek_table is not None: lib.zk_decode_options_seek_table(o, opts._seek_table._h)
        if opts._lower is not None: lib.zk_decode_options_lower_frame(o, opts._lower)
        if opts._upper is not None: lib.zk_decode_options_upper_frame(o, opts._upper)
        if opts._offset is not None: lib.zk_decode_options_offset(o, opts._offset)
        if opts._limit is not None: lib.zk_decode_options_offset_limit(o, opts._limit)
        h = c_void_p()
        _check(lib.zk_decode_options_into_decoder(o, byref(h)), lib)
        self._h = h

    def __del__(self):
        try:
            if self._h:
                self.lib.zk_decoder_free(self._h)
        except Exception:
            pass

    def decompress(self, buf) -> int:
        mv = memoryview(buf)
        if len(mv) == 0:
            return 0
        arr = (ctypes.c_uint8 * len(mv)).from_buffer(mv)
        p = c_size_t()
        _check(self.lib.zk_decoder_decompress(self._h, arr, len(mv), byref(p)), self.lib)
        return int(p.value)

    def decompress_with_prefix(self, buf, prefix=None, ranges=None) -> int:
        """decode.rs:201-270: every frame is decoded against the raw-content prefix.  ranges (one (lo, hi) pair per seek-table entry): entry
        e is decoded against prefix[lo:hi] only, and only the slices of the frames read go to the device (a seekable patch,
        zk_decoder_decompress_with_prefix_ranges).  prefix may be a ReferenceArchive: each window of frames then decodes only the entries
        of it under its ranges, on the GPU (zk_decoder_decompress_with_reference_chain)"""
        if prefix is None:
            return self.decompress(buf)
        mv = memoryview(buf)
        if len(mv) == 0:
            return 0
        arr = (ctypes.c_uint8 * len(mv)).from_buffer(mv)
        p = c_size_t()
        if isinstance(prefix, ReferenceArchive):
            self._prefix_keep = prefix
            rp = None
            if ranges is not None:
                if getattr(self, "_ranges_src", None) is not ranges:    # the same array on every call keeps the decoded window valid
                    self._ranges_src, self._ranges = ranges, _ranges(ranges, self.seek_table().num_frames())
                rp = self._ranges.ctypes.data_as(_native.u64p)
            _check(self.lib.zk_decoder_decompress_with_reference_chain(self._h, arr, len(mv), *prefix._chain(), rp, byref(p)), self.lib)
            return int(p.value)
        paddr, pn, pkeep = _buf(prefix)
        self._prefix_keep = pkeep
        if ranges is None:
            _check(self.lib.zk_decoder_decompress_with_prefix(self._h, arr, len(mv), paddr, pn, byref(p)), self.lib)
        else:
            if getattr(self, "_ranges_src", None) is not ranges:    # the same array on every call keeps the decoded window valid
                self._ranges_src, self._ranges = ranges, _ranges(ranges, self.seek_table().num_frames())
            _check(self.lib.zk_decoder_decompress_with_prefix_ranges(self._h, arr, len(mv), paddr, pn, self._ranges.ctypes.data_as(_native.u64p),
                                                                     byref(p)), self.lib)
        return int(p.value)

    def readable(self): return True
    def seekable(self): return True
    def readinto(self, b): return self.decompress(b)

    def read_all(self) -> bytes:
        out = bytearray(self.offset_limit() - self.offset())
        n = 0
        while n < len(out):
            k = self.decompress(memoryview(out)[n:])
            if k == 0:
                break
            n += k
        return bytes(out[:n])

    def reset(self): self.lib.zk_decoder_reset(self._h)

    def set_lower_frame(self, i: int) -> int:
        v = c_uint64(); _check(self.lib.zk_decoder_set_lower_frame(self._h, i, byref(v)), self.lib); return int(v.value)

    def set_upper_frame(self, i: int) -> int:
        v = c_uint64(); _check(self.lib.zk_decoder_set_upper_frame(self._h, i, byref(v)), self.lib); return int(v.value)

    def set_offset(self, off: int): _check(self.lib.zk_decoder_set_offset(self._h, off), self.lib)
    def set_offset_limit(self, lim: int): _check(self.lib.zk_decoder_set_offset_limit(self._h, lim), self.lib)
    def read_compressed(self) -> int: return int(self.lib.zk_decoder_read_compressed(self._h))
    def offset(self) -> int: return int(self.lib.zk_decoder_offset(self._h))
    def offset_limit(self) -> int: return int(self.lib.zk_decoder_offset_limit(self._h))
    def seek_table(self) -> SeekTable: return SeekTable(c_void_p(self.lib.zk_decoder_seek_table(self._h)), False, self.lib, _keep=self)

    def seek(self, pos: int, whence: int = 0) -> int:
        """impl Seek (decode.rs:545-579): whence 0 Start, 1 Current, 2 End (Python convention)"""
        v = c_uint64()
        native_whence = {0: 0, 1: 2, 2: 1}[whence]
        _check(self.lib.zk_decoder_seek(self._h, native_whence, pos, byref(v)), self.lib)
        return int(v.value)


__all__ = ["Context", "default_context", "set_default_context", "Error", "Format", "FrameSizePolicy", "SeekTable", "Serializer",
           "EncodeOptions", "RawEncoder", "Encoder", "CompressionProgress", "EpilogueProgress", "DecodeOptions", "Decoder",
           "BytesWrapper", "OffsetFrom", "SEEKABLE_MAGIC_NUMBER", "SEEKABLE_MAX_FRAMES", "SEEK_TABLE_INTEGRITY_SIZE",
           "SEEKABLE_MAX_FRAME_SIZE"]
