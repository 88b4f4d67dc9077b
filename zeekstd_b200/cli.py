"""Command-line front end with the reference CLI's arguments and behaviour (SURVEY.md 8f.4), over the GPU codec.

    python -m zeekstd_b200 [compress] [-l N] [-s 2M] [--frame-size-policy ..]
                           [--patch-from F [--long | --patch-slices [--patch-archive [--patch-base B]...]]] [--long-mode]
                           [--reuse-from OLD.zst] [INPUT] [-o OUT]
    python -m zeekstd_b200 decompress [--from N | --from-frame I] [--to N|end | --to-frame I|end]
                           [--patch-apply F [--patch-archive [--patch-base B]...]] INPUT [-o OUT]
    python -m zeekstd_b200 list [--from-frame I] [--to-frame I|end | --num-frames N] [-d] [--seek-table-format head|foot] INPUT

What each piece follows in the reference: argument set and value parsers cli/src/args.rs:10-329; sub-commands, output
path derivation, overwrite checks and the list tables cli/src/command.rs:33-473; the compress loop (Encoder fed from a
reader, optional stand-alone Head-format seek table) cli/src/compress.rs:55-106; the decompress loop
cli/src/decompress.rs:21-117.  The codec underneath is this package's Encoder / Decoder, i.e. the CUDA path: there is no
CPU route.  Compression levels are 1..19 as in the reference CLI (16..19 run the high-level tier: a 2 MiB window and a
price-based parse), plus zstd's negative fast levels (`-l -5` or `--compression-level=-5`; acceleration = -level, clamped
at -131072).  `--patch-from F` alone matches every frame against the last 32 KiB of F.  With `--long` (zstd's name for it) the
window-log / long-distance-matching parameters the reference sets for patch files take effect: every frame is matched against
the whole of F (its last 128 MiB when it is larger), which is what makes the archive a patch.  Long-distance matching is part
of the high-level tier, so with `--long` every compression level writes what level 16 writes, and the frame size policy must be
`uncompressed`.  `--long-mode` is a different switch, with or without `--patch-from`: every frame is also matched against its own
bytes up to 128 MiB back (what `zstd --long` does), so large frames (`-s 64M`) find repeats that lie beyond level 16's 2 MiB
window; with `--patch-from` it also matches the whole of F as `--long` does.  It too runs every level as level 16 and needs
`--frame-size-policy uncompressed`.  `--mmap-prefix` / `--no-mmap-prefix` choose between np.memmap and a read.  `--frame-size-policy content` (an
extension of this codec) ends frames where a rolling hash of the data says so, about `-s` bytes apart on average, so that an edit
of the input changes only the frames around it and rsync, dedup stores and range-fetching clients can reuse the rest.
`--reuse-from OLD.zst` (an extension of this codec) compresses a new version against the archive of the previous one: every frame
whose bytes a frame of OLD.zst holds is copied from it, only the others are compressed; with `uncompressed` or `content` frames.
`--patch-from F --patch-slices` (an extension of this codec) writes a seekable patch against an F of any size: every frame is matched
against its own slice of F, found by content anchors and recorded in a skippable frame at the start of the archive, and `decompress
--patch-apply F` reads only the slices of the frames it restores.  With `--patch-archive` (also an extension) F is a seekable archive
whose decoded content is the reference: it is decoded on the GPU, and only the entries under the slices a command needs are.  The flag
is explicit because a raw reference file may itself be a .zst file.  When F is itself a seekable patch, `--patch-base B` names the
archive it was made against, and is repeated for B's own reference, nearest first, down to a plain seekable archive: every level of
that chain is decoded on the GPU, each only where the level above reads it, and no version is restored on the host.
"""
from __future__ import annotations

import argparse
import os
import stat
import sys
import time

import numpy as np

IN_CHUNK = 1 << 17            # CCtx::in_size() of the reference's read loop (compress.rs:60)
OUT_CHUNK = 8 << 20           # the reference uses DCtx::out_size(); larger here so one call spans whole frames
MMAP_THRESHOLD = 0x0010_0000  # args.rs:10 (the reference's comment says 128 MiB; the constant is 1 MiB)


class CliError(Exception):
    pass


# ------------------------------------------------------------------------------------------- value parsers (args.rs:12-112)
def byte_value(s: str) -> int:
    digits = ""
    for ch in s:
        if ch.isascii() and ch.isdigit():
            digits += ch
        else:
            break
    unit = "".join(ch for ch in s[len(digits):] if not ch.isspace())
    if not digits:
        raise argparse.ArgumentTypeError(f"invalid byte value: {s!r}")
    v = int(digits)
    mul = {"B": 1, "": 1, "K": 1 << 10, "kib": 1 << 10, "M": 1 << 20, "mib": 1 << 20, "G": 1 << 30, "gib": 1 << 30}.get(unit)
    if mul is None:
        raise argparse.ArgumentTypeError(f"Unknown unit: {unit!r}")
    v *= mul
    if v >= 1 << 64:
        raise argparse.ArgumentTypeError("Byte value too large")
    return v


def offset_limit(s: str):
    return None if s.lower() == "end" else byte_value(s)


def last_frame(s: str):
    if s.lower() == "end":
        return "end"
    try:
        v = int(s)
    except ValueError:
        raise argparse.ArgumentTypeError(f"invalid frame index: {s!r}")
    if not 0 <= v < 1 << 32:
        raise argparse.ArgumentTypeError(f"invalid frame index: {s!r}")
    return v


def num_frames(s: str) -> int:
    try:
        v = int(s)
    except ValueError:
        raise argparse.ArgumentTypeError(f"invalid frame number: {s!r}")
    if v <= 0:
        raise argparse.ArgumentTypeError("frame number must be greater than 0")
    return v


def u32(s: str) -> int:
    v = int(s)
    if not 0 <= v < 1 << 32:
        raise argparse.ArgumentTypeError(f"out of range: {s!r}")
    return v


def human_bytes(n: int) -> str:
    """indicatif::HumanBytes: binary prefixes, two decimals, plain integer below 1 KiB"""
    if n < 1024:
        return f"{n} B"
    v = float(n)
    for p in ("Ki", "Mi", "Gi", "Ti", "Pi", "Ei"):
        v /= 1024.0
        if v < 1024.0 or p == "Ei":
            return f"{v:.2f} {p}B"
    return f"{n} B"


def raw_bytes(n: int) -> str:
    return str(n)


# ------------------------------------------------------------------------------------------------------------ parser
def _add_flags(p, top: bool):
    d = {} if top else {"default": argparse.SUPPRESS}
    p.add_argument("-q", "--quiet", action="store_true", help="Suppress output. Ignored in list mode.", **d)
    p.add_argument("-r", "--raw-bytes", action="store_true", help="Disable human-readable formatting for all byte numbers.", **d)


def _add_common(p):
    p.add_argument("-f", "--force", action="store_true", help="Disable input and output checks.")
    p.add_argument("-c", "--stdout", action="store_true", help="Write to STDOUT.")
    p.add_argument("--no-progress", action="store_true", help="Do not show the progress counter.")
    p.add_argument("--mmap-prefix", action="store_true", help="Force memory-mapping prefix (patch) files.")
    p.add_argument("--no-mmap-prefix", action="store_true", help="Force disable memory-mapping prefix (patch) files.")
    p.add_argument("--seek-table-file", default=None, help='Path to the seek table file. If specified, implies the "Head" seek table format.')


def _level(s: str) -> int:
    """1..19, or a negative level: zstd's fast mode (the codec clamps levels below -131072 to it, as libzstd does)"""
    v = int(s)
    if not (1 <= v <= 19 or -(1 << 31) <= v < 0):
        raise argparse.ArgumentTypeError("compression level must be between 1 and 19, or negative for fast mode")
    return v


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="zeekstd_b200", description="Compress and decompress data using the Zstandard Seekable Format (H100 codec).")
    _add_flags(ap, True)
    sub = ap.add_subparsers(dest="command")

    c = sub.add_parser("compress", aliases=["c"], help="Compress INPUT_FILE (default); reads from STDIN if INPUT_FILE is `-` or not provided")
    _add_flags(c, False); _add_common(c)
    c.add_argument("-l", "--compression-level", type=_level, default=3,
                   help="Compression level: 1-19 (16-19: 2 MiB window, price-based parse, the smallest archives), or negative (-1 down to "
                        "-131072) for fast mode: faster, lower ratio, literals stored without Huffman coding. Default 3.")
    c.add_argument("--no-checksum", action="store_true", help="Don't include frame checksums.")
    c.add_argument("-s", "--frame-size", type=byte_value, default=byte_value("2M"))
    c.add_argument("--frame-size-policy", choices=["compressed", "uncompressed", "content"], default="uncompressed",
                   help="content: content-defined frames of about --frame-size bytes on average (between a quarter and four times it), "
                        "so that an edit changes only the frames around it.")
    c.add_argument("--patch-from", default=None, help="Provide a reference point for Zstandard's diff engine.")
    c.add_argument("--long", action="store_true",
                   help="With --patch-from: long-distance matching against the whole reference file (its last 128 MiB), so that the archive "
                        "is a patch. Every compression level then runs as level 16; needs --frame-size-policy uncompressed.")
    c.add_argument("--long-mode", action="store_true",
                   help="Match every frame also against its own bytes up to 128 MiB back (zstd --long), and with --patch-from against the "
                        "whole reference file as --long does: large frames find far repeats. Every compression level then runs as level 16; "
                        "needs --frame-size-policy uncompressed.")
    c.add_argument("--patch-slices", action="store_true",
                   help="With --patch-from: a seekable patch. Every frame is matched against its own slice of the reference file, found by "
                        "content anchors, so the file may be of any size and one frame restores from its slice alone. Implies long-distance "
                        "matching (level 16's tier); needs --frame-size-policy uncompressed or content.")
    c.add_argument("--patch-margin", type=byte_value, default=None,
                   help="With --patch-slices: bytes added on each side of a frame's slice (default: the frame size).")
    c.add_argument("--patch-archive", action="store_true",
                   help="With --patch-slices: the --patch-from file is a seekable archive, and the reference is its decoded content, "
                        "decoded on the GPU entry by entry. The patch is the one made against the decoded file.")
    c.add_argument("--patch-base", action="append", default=None, metavar="FILE",
                   help="With --patch-archive, when the --patch-from archive is itself a seekable patch: the archive it was made against. "
                        "Repeat it for that file's own reference, nearest first, ending at a plain seekable archive.")
    c.add_argument("--reuse-from", default=None, metavar="OLD.zst",
                   help="The archive of a previous version of the input (ending in its seek table): every frame whose bytes one of its "
                        "frames already holds is copied from it, only the others are compressed. The output is what compress writes "
                        "when OLD.zst was written with the same settings. Needs --frame-size-policy uncompressed or content.")
    c.add_argument("input_file", nargs="?", default="-")
    c.add_argument("-o", "--output-file", default=None)

    d = sub.add_parser("decompress", aliases=["d"], help="Decompress INPUT_FILE")
    _add_flags(d, False); _add_common(d)
    g0 = d.add_mutually_exclusive_group()
    g0.add_argument("--from", dest="from_", type=int, default=None, help="The offset (of the uncompressed data) where decompression starts.")
    g0.add_argument("--from-frame", type=u32, default=None)
    g1 = d.add_mutually_exclusive_group()
    g1.add_argument("--to", type=offset_limit, default="end", help="Accepts the special value 'end'.")
    g1.add_argument("--to-frame", type=last_frame, default=None)
    d.add_argument("--patch-apply", default=None)
    d.add_argument("--patch-archive", action="store_true",
                   help="With --patch-apply: the reference is a seekable archive; only its entries under the slices of the frames restored "
                        "are decoded, on the GPU.")
    d.add_argument("--patch-base", action="append", default=None, metavar="FILE",
                   help="With --patch-archive, when the --patch-apply archive is itself a seekable patch: the archive it was made against. "
                        "Repeat it for that file's own reference, nearest first, ending at a plain seekable archive.")
    d.add_argument("input_file")
    d.add_argument("-o", "--output-file", default=None)

    li = sub.add_parser("list", aliases=["l"], help="Print information about seekable Zstandard-compressed files")
    _add_flags(li, False)
    li.add_argument("--from-frame", type=u32, default=None)
    g2 = li.add_mutually_exclusive_group()
    g2.add_argument("--to-frame", type=last_frame, default=None)
    g2.add_argument("--num-frames", type=num_frames, default=None)
    li.add_argument("-d", "--detail", action="store_true")
    li.add_argument("--seek-table-format", choices=["head", "foot"], default="foot")
    li.add_argument("input_file")
    return ap


_COMMANDS = {"compress": "compress", "c": "compress", "decompress": "decompress", "d": "decompress", "list": "list", "l": "list"}
_TOP_FLAGS = {"-q", "--quiet", "-r", "--raw-bytes", "-h", "--help"}


def parse_args(argv):
    """main.rs:12-31: without a sub-command the arguments are those of `compress`"""
    argv = list(argv)
    i = 0
    while i < len(argv) and argv[i] in _TOP_FLAGS:
        i += 1
    if i == len(argv) or argv[i] not in _COMMANDS:
        if i == len(argv) and not argv:
            build_parser().print_help(sys.stderr)
            raise SystemExit(2)
        argv.insert(i, "compress")
    ns = build_parser().parse_args(argv)
    ns.command = _COMMANDS[ns.command]
    return ns


# ------------------------------------------------------------------------------------------------------ file checks
def _checked_out_file(path: str, in_path, quiet: bool, force: bool):
    """command.rs:45-78"""
    exists = os.path.exists(path)
    is_chr = exists and stat.S_ISCHR(os.stat(path).st_mode)
    if not force and exists and not is_chr:
        if quiet or in_path is None:
            raise CliError(f"{path} already exists; not overwritten")
        sys.stderr.write(f"{path} already exists; overwrite (y/n) ? ")
        sys.stderr.flush()
        if sys.stdin.readline().rstrip("\r\n") != "y":
            raise CliError(f"{path} already exists")
    try:
        return open(path, "wb")
    except OSError as e:
        raise CliError(f"Failed to open output file: {e}")


def _out_path(ns, in_path):
    """command.rs:93-126"""
    if ns.command == "list" or ns.stdout:
        return None
    if ns.output_file is not None:
        return ns.output_file
    if in_path is None:
        return None
    if ns.command == "compress":
        return in_path + ".zst"
    root, ext = os.path.splitext(in_path)
    if ext != ".zst":
        raise CliError(f"{in_path}: unknown extension (.zst expected); cannot derive the output file name")
    return root


def _new_writer(out_path, in_path, quiet: bool, force: bool):
    if out_path is not None:
        return _checked_out_file(out_path, in_path, quiet, force)
    if not force and sys.stdout.isatty():
        raise CliError("stdout is a terminal, aborting")
    return sys.stdout.buffer


def _load_reference(zk, path, bases=None):
    """a reference archive (--patch-archive): the file mapped, its Foot seek table parsed.  bases (--patch-base, nearest first): when it
    is a seekable patch, the chain of archives under it, ending at a plain one"""
    paths = [path] + list(bases or [])
    ref = None
    for i in range(len(paths) - 1, -1, -1):                # root first
        p = paths[i]
        try:
            data = np.memmap(p, dtype=np.uint8, mode="r") if os.path.getsize(p) > 0 else np.zeros(0, dtype=np.uint8)
        except OSError as e:
            raise CliError(f"Failed to load reference archive: {e}")
        try:
            table = zk.SeekTable.from_bytes(data, zk.Format.Foot)
        except zk.Error as e:
            raise CliError(f"Failed to parse the seek table of {p}: {e}")
        co, _ = table.offsets()
        c0, c1 = int(co[0]), int(co[-1])
        patch = c1 - c0 >= 4 and c0 + 4 <= data.size and int.from_bytes(data[c0:c0 + 4].tobytes(), "little") == zk.PATCH_SLICES_MAGIC
        if ref is None and patch:
            raise CliError(f"{p} is a seekable patch; restore it first")
        if ref is not None:
            if not patch:
                raise CliError(f"{p} is not a seekable patch: --patch-base {paths[i + 1]} goes only after a seekable patch")
            try:
                old_len = zk.patch_slices_read(data[c0:c1], table.num_frames())[0]
            except zk.Error as e:
                raise CliError(f"Failed to read the slices of the seekable patch {p}: {e}")
            if old_len != ref.old_len:
                raise CliError(f"{paths[i + 1]} decodes to {ref.old_len} bytes, the seekable patch {p} was made against {old_len} bytes")
        try:
            ref = zk.ReferenceArchive(data, seek_table=table, base=ref)
        except ValueError as e:
            raise CliError(str(e))
    return ref


def _load_prefix(path, use_mmap: bool):
    """command.rs:349-384"""
    if path is None:
        return None
    try:
        if use_mmap and os.path.getsize(path) > 0:
            return np.memmap(path, dtype=np.uint8, mode="r")
        return np.fromfile(path, dtype=np.uint8)
    except OSError as e:
        raise CliError(f"Failed to load prefix (patch) file: {e}")


def _use_mmap(ns, prefix_len) -> bool:
    """args.rs:162-172"""
    if ns.mmap_prefix:
        return True
    if ns.no_mmap_prefix:
        return False
    return prefix_len is not None and prefix_len >= MMAP_THRESHOLD


class _Progress:
    """the reference's indicatif counter ("{pos} of {len}" on stderr, 5 Hz), shown on a terminal only"""

    def __init__(self, total, fmt, enabled: bool, pos: int = 0):
        self.total, self.fmt, self.pos, self.last = total, fmt, pos, 0.0
        self.on = enabled and sys.stderr.isatty()

    def inc(self, n: int):
        self.pos += n
        if self.on and time.monotonic() - self.last >= 0.2:
            self.last = time.monotonic()
            tot = self.fmt(self.total) if self.total is not None else "?"
            sys.stderr.write(f"\r{self.fmt(self.pos)} of {tot}")
            sys.stderr.flush()

    def finish(self):
        if self.on:
            sys.stderr.write("\r" + " " * 48 + "\r")
            sys.stderr.flush()


# --------------------------------------------------------------------------------------------------------- commands
def _read_seek_table(zk, path: str, fmt: int):
    """SeekTable::from_seekable_format over a file without reading the archive: only the table's bytes are fetched
    (Foot: the integrity field gives the frame count, seek_table.rs:379-436; Head: the skippable header gives the size)"""
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        if fmt == zk.Format.Head:
            head = f.read(8)
            n = int.from_bytes(head[4:8], "little") + 8 if len(head) == 8 else 8
            f.seek(0)
            return zk.SeekTable.from_bytes(f.read(min(n, size)), zk.Format.Head)
        tail_n = min(size, zk.SEEK_TABLE_INTEGRITY_SIZE)
        f.seek(size - tail_n)
        tail = f.read(tail_n)
        want = size
        if tail_n == zk.SEEK_TABLE_INTEGRITY_SIZE:
            frames = int.from_bytes(tail[0:4], "little")
            per = 12 if tail[4] & 0x80 else 8
            want = min(size, 8 + frames * per + zk.SEEK_TABLE_INTEGRITY_SIZE)
        f.seek(size - want)
        return zk.SeekTable.from_bytes(f.read(want), zk.Format.Foot)


def _run_compress(zk, ns, fmt_bytes) -> int:
    in_path = None if ns.input_file == "-" else ns.input_file
    out_path = _out_path(ns, in_path)
    if in_path is not None:
        try:
            reader = open(in_path, "rb")
        except OSError as e:
            raise CliError(f"Failed to open input file: {e}")
    else:
        if not ns.force and sys.stdin.isatty():
            raise CliError("stdin is a terminal, aborting")
        reader = sys.stdin.buffer
    if ns.frame_size >= 1 << 32:
        raise CliError("Frame size too big")
    if ns.long and not ns.patch_from:
        raise CliError("--long needs --patch-from: long-distance matching runs against the reference file")
    if ns.long and ns.frame_size_policy in ("compressed", "content"):
        raise CliError("--long needs --frame-size-policy uncompressed")
    if ns.long_mode and ns.frame_size_policy in ("compressed", "content"):
        raise CliError("--long-mode needs --frame-size-policy uncompressed")
    if ns.patch_slices:
        if not ns.patch_from:
            raise CliError("--patch-slices needs --patch-from: the slices are taken from the reference file")
        if ns.frame_size_policy == "compressed":
            raise CliError("--patch-slices needs --frame-size-policy uncompressed or content")
        if ns.long_mode:
            raise CliError("--patch-slices cannot be used with --long-mode: a frame is matched against its slice of the reference file only")
        if ns.reuse_from is not None:
            raise CliError("--patch-slices cannot be used with --reuse-from: a copied frame must depend on its own bytes alone")
        if ns.frame_size == 0:
            raise CliError("--patch-slices needs a frame size above 0")
    elif ns.patch_margin is not None:
        raise CliError("--patch-margin needs --patch-slices")
    if ns.patch_base and not ns.patch_archive:
        raise CliError("--patch-base needs --patch-archive: it names the reference archive's own reference")
    if ns.patch_archive and (not ns.patch_slices or ns.long):
        raise CliError("--patch-archive needs --patch-from and --patch-slices: whole-prefix patches against an archive are not supported")
    if ns.reuse_from is not None:
        if ns.patch_from:
            raise CliError("--reuse-from cannot be used with --patch-from: a copied frame must depend on its own bytes alone")
        if ns.frame_size_policy == "compressed":
            raise CliError("--reuse-from needs --frame-size-policy uncompressed or content")
        if ns.frame_size == 0:
            raise CliError("--reuse-from needs a frame size above 0")
    prefix_len = os.path.getsize(ns.patch_from) if ns.patch_from and os.path.exists(ns.patch_from) else None
    ns.reference = _load_reference(zk, ns.patch_from, ns.patch_base) if ns.patch_archive else None
    st_file = None
    if ns.seek_table_file is not None:
        try:
            st_file = _checked_out_file(ns.seek_table_file, in_path, ns.quiet, ns.force)
        except CliError as e:
            raise CliError(f"Failed to create seek table file: {e}")
    in_len = os.path.getsize(in_path) if in_path is not None and os.path.isfile(in_path) else None
    bar = _Progress(in_len, fmt_bytes, not ns.quiet and not ns.no_progress)
    writer = _new_writer(out_path, in_path, ns.quiet, ns.force)

    if ns.reuse_from is not None:
        return _run_compress_reuse(zk, ns, fmt_bytes, reader, writer, in_path, out_path, st_file)
    if ns.patch_slices:
        return _run_compress_slices(zk, ns, fmt_bytes, reader, writer, in_path, out_path, st_file)
    policy = {"compressed": zk.FrameSizePolicy.Compressed, "uncompressed": zk.FrameSizePolicy.Uncompressed,
              "content": zk.FrameSizePolicy.ContentDefined}[ns.frame_size_policy](ns.frame_size)
    enc = (zk.EncodeOptions().frame_size_policy(policy).checksum_flag(not ns.no_checksum)
           .compression_level(ns.compression_level).long_distance_matching(ns.long).long_mode(ns.long_mode)
           .into_encoder(writer))
    prefix = _load_prefix(ns.patch_from, _use_mmap(ns, prefix_len))

    read = 0
    while True:
        buf = reader.read(IN_CHUNK)
        if not buf:
            break
        read += len(buf)
        bar.inc(len(buf))
        mv, pos = memoryview(buf), 0
        while pos < len(mv):
            pos += enc.compress_with_prefix(mv[pos:], prefix)
    if st_file is not None:
        enc.end_frame()
        enc.flush()
        written = enc.written_compressed()
        ser = enc.seek_table().clone().into_format_serializer(zk.Format.Head)
        blob = ser.to_bytes()
        st_file.write(blob)
        st_file.close()
        written += len(blob)
    else:
        written = enc.finish()
    bar.finish()
    if writer is not sys.stdout.buffer:
        writer.close()
    else:
        writer.flush()
    if not ns.quiet:
        ratio = 100.0 / read * written if read else float("nan")
        sys.stderr.write(f"{in_path or 'STDIN'} : {ratio:.2f}% ( {fmt_bytes(read)} => {fmt_bytes(written)}, {out_path or 'STDOUT'})\n")
    return 0


def _load_whole(path, what: str):
    """a file's bytes, memory-mapped from MMAP_THRESHOLD bytes on"""
    try:
        if os.path.getsize(path) >= MMAP_THRESHOLD:
            return np.memmap(path, dtype=np.uint8, mode="r")
        return np.fromfile(path, dtype=np.uint8)
    except OSError as e:
        raise CliError(f"Failed to read {what}: {e}")


def _policy_sizes(zk, ctx, ns, data):
    """the frame sizes the encoder's policy gives the whole input (uncompressed or content)"""
    n = int(data.size)
    if ns.frame_size_policy == "content":
        return ctx.cut_frames_cdc(data, ns.frame_size)[0]
    fs = min(ns.frame_size, zk.SEEKABLE_MAX_FRAME_SIZE)
    sizes = np.full(n // fs, fs, dtype=np.uint32)
    if n % fs or n == 0:
        sizes = np.append(sizes, np.uint32(n % fs))
    return sizes


def _write_archive(zk, ns, writer, st_file, parts, table) -> int:
    """the frames' bytes, then the seek table (Foot, or Head into its own file) -> bytes written"""
    written = 0
    for part in parts:
        writer.write(part)
        written += len(part)
    if st_file is not None:
        blob = table.into_format_serializer(zk.Format.Head).to_bytes()
        st_file.write(blob)
        st_file.close()
    else:
        blob = table.into_serializer().to_bytes()
        writer.write(blob)
    written += len(blob)
    if writer is not sys.stdout.buffer:
        writer.close()
    else:
        writer.flush()
    return written


def _run_compress_slices(zk, ns, fmt_bytes, reader, writer, in_path, out_path, st_file) -> int:
    """compress with --patch-slices: the whole input in one seekable patch (Context.patch_ranges, Context.compress_frames_patch); entry 0
    starts with the slice frame"""
    if in_path is not None and os.path.isfile(in_path):
        reader.close()
        data = _load_whole(in_path, "input file")
    else:
        data = np.frombuffer(reader.read(), dtype=np.uint8)
    old = ns.reference if ns.reference is not None else _load_whole(ns.patch_from, "prefix (patch) file")
    ctx = zk.default_context()
    sizes = _policy_sizes(zk, ctx, ns, data)
    margin = ns.frame_size if ns.patch_margin is None else ns.patch_margin
    ranges = ctx.patch_ranges(data, sizes, old, margin)
    comp, cs, _ = ctx.compress_frames_patch(data, sizes, old, ranges, ns.compression_level, not ns.no_checksum)
    head = zk.patch_slices_write(old.old_len if ns.reference is not None else int(old.size), ranges)
    table = zk.SeekTable()
    for f, (c, d) in enumerate(zip(cs.tolist(), sizes.tolist())):
        table.log_frame(c + (len(head) if f == 0 else 0), d)
    written = _write_archive(zk, ns, writer, st_file, [head, comp.tobytes()], table)
    if not ns.quiet:
        n = int(data.size)
        ratio = 100.0 / n * written if n else float("nan")
        sys.stderr.write(f"{in_path or 'STDIN'} : {ratio:.2f}% ( {fmt_bytes(n)} => {fmt_bytes(written)}, {out_path or 'STDOUT'})\n")
    return 0


def _run_compress_reuse(zk, ns, fmt_bytes, reader, writer, in_path, out_path, st_file) -> int:
    """compress with --reuse-from: the whole input in one batch call (Context.compress_frames_reuse) with the frame sizes the encoder's
    policy gives, then the archive and seek table exactly as the encoder writes them"""
    if in_path is not None and os.path.isfile(in_path):
        reader.close()
        data = _load_whole(in_path, "input file")
    else:
        data = np.frombuffer(reader.read(), dtype=np.uint8)
    old = _load_whole(ns.reuse_from, "--reuse-from archive")
    ctx = zk.default_context()
    n = int(data.size)
    if ns.frame_size_policy == "content":
        sizes, _ = ctx.cut_frames_cdc(data, ns.frame_size)
    else:
        fs = min(ns.frame_size, zk.SEEKABLE_MAX_FRAME_SIZE)
        sizes = np.full(n // fs, fs, dtype=np.uint32)
        if n % fs or n == 0:
            sizes = np.append(sizes, np.uint32(n % fs))
    try:
        zk.SeekTable.from_bytes(old, zk.Format.Foot)
    except zk.Error as e:
        raise CliError(f"{ns.reuse_from}: not a seekable archive ending in its seek table: {e}")
    comp, cs, reused = ctx.compress_frames_reuse(data, sizes, old, ns.compression_level, not ns.no_checksum, ns.long_mode)
    table = zk.SeekTable()
    for c, d in zip(cs.tolist(), sizes.tolist()):
        table.log_frame(c, d)
    writer.write(comp.tobytes())
    written = int(comp.size)
    if st_file is not None:
        blob = table.into_format_serializer(zk.Format.Head).to_bytes()
        st_file.write(blob)
        st_file.close()
    else:
        blob = table.into_serializer().to_bytes()
        writer.write(blob)
    written += len(blob)
    if writer is not sys.stdout.buffer:
        writer.close()
    else:
        writer.flush()
    if not ns.quiet:
        n_reused = int(np.count_nonzero(reused != 0xFFFFFFFF))
        sys.stderr.write(f"reused {n_reused} of {len(sizes)} frames\n")
        ratio = 100.0 / n * written if n else float("nan")
        sys.stderr.write(f"{in_path or 'STDIN'} : {ratio:.2f}% ( {fmt_bytes(n)} => {fmt_bytes(written)}, {out_path or 'STDOUT'})\n")
    return 0


def _run_decompress(zk, ns, fmt_bytes) -> int:
    in_path = ns.input_file
    out_path = _out_path(ns, in_path)
    if ns.patch_base and not ns.patch_archive:
        raise CliError("--patch-base needs --patch-archive: it names the reference archive's own reference")
    if ns.patch_archive and not ns.patch_apply:
        raise CliError("--patch-archive needs --patch-apply: it says that the reference file is a seekable archive")
    reference = _load_reference(zk, ns.patch_apply, ns.patch_base) if ns.patch_archive else None
    prefix_len = os.path.getsize(ns.patch_apply) if ns.patch_apply and os.path.exists(ns.patch_apply) else None
    if reference is not None:
        prefix_len = reference.old_len
    writer = _new_writer(out_path, in_path, ns.quiet, ns.force)
    try:
        src = open(in_path, "rb")
    except OSError as e:
        raise CliError(f"Failed to open input file: {e}")
    try:
        if ns.seek_table_file is not None:
            try:
                with open(ns.seek_table_file, "rb") as f:
                    table = zk.SeekTable.from_reader(f)
            except OSError as e:
                raise CliError(f"Failed to open seek table file: {e}")
        else:
            table = _read_seek_table(zk, in_path, zk.Format.Foot)
    except zk.Error as e:
        raise CliError(f"Failed to parse seek table: {e}")
    try:
        offset = table.frame_start_decomp(ns.from_frame) if ns.from_frame is not None else (ns.from_ or 0)
    except zk.Error as e:
        raise CliError(f"Failed to get decompression offset: {e}")
    try:
        if ns.to_frame is not None:
            limit = table.size_decomp() if ns.to_frame == "end" else table.frame_end_decomp(ns.to_frame)
        else:
            limit = table.size_decomp() if ns.to is None else ns.to
    except zk.Error as e:
        raise CliError(f"Failed to get decompression offset limit: {e}")
    # a seekable patch: entry 0 starts with the slice frame, which holds every frame's slice of the reference file
    ranges = None
    n_frames = table.num_frames()
    if n_frames:
        head = src.read(zk.patch_slices_size(n_frames))
        src.seek(0)
        if len(head) >= 4 and int.from_bytes(head[:4], "little") == zk.PATCH_SLICES_MAGIC:
            if not ns.patch_apply:
                raise CliError("this archive is a seekable patch; pass --patch-apply")
            try:
                old_len, ranges, _ = zk.patch_slices_read(head, n_frames)
            except zk.Error as e:
                raise CliError(f"Failed to read the slices of the seekable patch: {e}")
            if prefix_len != old_len:
                has = "decodes to" if reference is not None else "has"
                raise CliError(f"{ns.patch_apply} {has} {prefix_len} bytes, the seekable patch was made against {old_len} bytes")
    if reference is not None and ranges is None:
        raise CliError("--patch-archive needs a seekable patch (compress --patch-slices): whole-prefix patches against an archive are not supported")
    bar = _Progress(limit, fmt_bytes, not ns.quiet and not ns.no_progress, pos=offset)
    try:
        dec = zk.DecodeOptions(src).seek_table(table).offset(offset).offset_limit(limit).into_decoder()
    except zk.Error as e:
        raise CliError(f"Failed to create decoder: {e}")
    # the slices of a patch are read from a mapping: only those of the frames decoded are paged in (of a reference archive, only the
    # entries under them are decoded)
    prefix = reference if reference is not None else _load_prefix(ns.patch_apply, ranges is not None or _use_mmap(ns, prefix_len))

    buf = bytearray(OUT_CHUNK)
    view = memoryview(buf)
    written = 0
    while True:
        try:
            n = dec.decompress_with_prefix(view, prefix, ranges)
        except zk.Error as e:
            raise CliError(f"Failed to decompress data: {e}")
        if n == 0:
            break
        bar.inc(n)
        writer.write(view[:n])
        written += n
    bar.finish()
    if writer is not sys.stdout.buffer:
        writer.close()
    else:
        writer.flush()
    src.close()
    if not ns.quiet:
        sys.stderr.write(f"{in_path} : {fmt_bytes(written)}\n")
    return 0


def _run_list(zk, ns, fmt_bytes) -> int:
    if not os.path.exists(ns.input_file):
        raise CliError("Failed to open input file")
    try:
        st = _read_seek_table(zk, ns.input_file, zk.Format.Head if ns.seek_table_format == "head" else zk.Format.Foot)
    except zk.Error as e:
        raise CliError(f"Failed to read seek table: {e}")
    if ns.num_frames is not None:
        end = (ns.from_frame or 0) + ns.num_frames - 1
    elif ns.to_frame is not None:
        end = st.num_frames() - 1 if ns.to_frame == "end" else ns.to_frame
    else:
        end = None
    out = sys.stdout
    if ns.from_frame is None and end is None and not ns.detail:
        n = st.num_frames()
        comp, unc = st.frame_end_comp(n - 1), st.frame_end_decomp(n - 1)
        ratio = unc / comp if comp else float("nan")
        out.write(f"{'Frames': <15} {'Compressed': <15} {'Uncompressed': <15} {'Max Frame Size': <15} {'Ratio': <10} {'Filename': <15}\n")
        out.write(f"{n: <15} {fmt_bytes(comp): <15} {fmt_bytes(unc): <15} {fmt_bytes(st.max_frame_size_decomp()): <15} {ratio: <10.3f} {ns.input_file: <15}\n")
        return 0
    start = ns.from_frame or 0
    if end is None:
        end = st.num_frames() - 1
    if start > end:
        raise CliError(f"Start frame ({start}) cannot be greater than end frame ({end})")
    out.write(f"{'Frame Index': <15} {'Compressed': <15} {'Uncompressed': <15} {'Compressed Offset': <20} {'Uncompressed Offset': <20}\n")
    lines = []
    for i in range(start, end + 1):
        try:
            row = (fmt_bytes(st.frame_size_comp(i)), fmt_bytes(st.frame_size_decomp(i)), fmt_bytes(st.frame_start_comp(i)), fmt_bytes(st.frame_start_decomp(i)))
        except zk.Error as e:
            out.write("".join(lines))
            raise CliError(str(e))
        lines.append(f"{i: <15} {row[0]: <15} {row[1]: <15} {row[2]: <20} {row[3]: <20}\n")
        if len(lines) == 100:
            out.write("".join(lines)); lines = []
    out.write("".join(lines))
    return 0


def main(argv=None) -> int:
    ns = parse_args(sys.argv[1:] if argv is None else argv)
    import zeekstd_b200 as zk
    fmt_bytes = raw_bytes if ns.raw_bytes else human_bytes
    try:
        if ns.command == "compress":
            return _run_compress(zk, ns, fmt_bytes)
        if ns.command == "decompress":
            return _run_decompress(zk, ns, fmt_bytes)
        return _run_list(zk, ns, fmt_bytes)
    except CliError as e:
        sys.stderr.write(f"Error: {e}\n")
        return 1
    except zk.Error as e:
        sys.stderr.write(f"Error: {e}\n")
        return 1


if __name__ == "__main__":
    sys.exit(main())
