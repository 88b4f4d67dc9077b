/*
 * zeekstd_b200.h -- C ABI of the H100-native seekable-zstd codec.
 *
 * Drop-in boundary for the hot path of rorosen/zeekstd.  The reference crosses into native code
 * (libzstd via zstd-safe) at exactly these call sites, which this ABI replaces:
 *
 *   lib/src/encode.rs:341-345   cctx.compress_stream2(out, in, ZSTD_e_continue)   -> zk_compress_frames*
 *   lib/src/encode.rs:444-448   cctx.compress_stream2(out, empty, ZSTD_e_end)     -> zk_compress_frames*
 *   lib/src/encode.rs:281-284   cctx.set_parameter(CompressionLevel/ChecksumFlag)  -> level / checksum args
 *   lib/src/encode.rs:504-506   cctx.reset(SessionOnly)                            -> (frames are independent)
 *   lib/src/decode.rs:243-245   dctx.decompress_stream(out, in)                    -> zk_decompress_frames*
 *   lib/src/decode.rs:354-356   dctx.reset(SessionOnly)                            -> (stateless per call)
 *   lib/src/error.rs:68,125     zstd_safe::get_error_name                          -> zk_error_name
 *
 * The libzstd interface is a one-context, 128 KiB-at-a-time stream; it cannot express a batch.  Each
 * independent frame of the seekable format (seekable_format.md:23-29) is one unit of data parallelism,
 * so the batch entry points take whole frames.  On top of them the "mirror" layer (zk_raw_encoder_*,
 * zk_encoder_*, zk_decoder_*, zk_seek_table_*) re-exposes the reference's Rust API surface one C
 * function per method so that a Rust (or any FFI) wrapper is mechanical -- see INTEGRATION.md.
 *
 * Conventions
 *   - plain C, opaque handles, no exceptions cross the boundary, caller owns all byte buffers;
 *   - return value int32_t: 0 = ok, < 0 = error (ZK_ERR_* or -(libzstd ZSTD_ErrorCode), e.g. -20
 *     corruption_detected, -22 checksum_wrong, -70 dstSize_tooSmall) -- the numeric zstd codes are kept
 *     so that Error::is_zstd()/get_error_name() (error.rs:40-45,101-113) stay meaningful;
 *   - a zk_ctx is NOT thread-safe (one per host thread / GPU), like CCtx/DCtx; calls are synchronous;
 *   - there is NO CPU fallback: zk_ctx_create fails with ZK_ERR_NO_DEVICE when no CUDA device exists.
 */
#ifndef ZEEKSTD_B200_H
#define ZEEKSTD_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ constants (lib/src/lib.rs:49-62) */
#define ZK_SEEKABLE_MAGIC_NUMBER 0x8F92EAB1u
#define ZK_SEEKABLE_MAX_FRAMES 0x08000000u
#define ZK_SEEK_TABLE_INTEGRITY_SIZE 9u
#define ZK_SEEKABLE_MAX_FRAME_SIZE 0x40000000u
#define ZK_SKIPPABLE_HEADER_SIZE 8u
#define ZK_DEFAULT_FRAME_SIZE 0x200000u /* FrameSizePolicy::default(), encode.rs:33-39 */
#define ZK_PATCH_SLICES_MAGIC 0x184D2A5Bu /* the skippable frame of a seekable patch's slices (zk_patch_slices_write) */
#define ZK_CHAIN_MAX_DEPTH 32u /* the most archives in a reference chain (the _chain calls of the patch block) */

/* Compression levels (the `level` argument of every compress entry point and of zk_encode_options_compression_level), as in libzstd:
 *   0                 the default, level 3;
 *   1 .. 22           the ratio tiers of DESIGN.md 3 (13 .. 15: a 256 KiB window; from 16 on: hash chains over a 2 MiB window of
 *                     the frame and a price-based parse; higher levels run that tier too);
 *   -1 .. -131072     fast mode with acceleration -level: sparser match probing, literals stored without Huffman coding.
 *                     Lower levels clamp to ZK_MIN_COMPRESSION_LEVEL, as in libzstd (ZSTD_minCLevel()). */
#define ZK_MIN_COMPRESSION_LEVEL (-131072)

/* ------------------------------------------------------------------ errors (lib/src/error.rs:101-113) */
#define ZK_OK 0
#define ZK_ERR_NUMBER_CONVERSION (-1001) /* Kind::NumberConversionFailed */
#define ZK_ERR_OFFSET_OUT_OF_RANGE (-1002) /* Kind::OffsetOutOfRange       */
#define ZK_ERR_FRAME_INDEX_TOO_LARGE (-1003) /* Kind::FrameIndexTooLarge     */
#define ZK_ERR_IO (-1004) /* Kind::IO                     */
#define ZK_ERR_NO_DEVICE (-1005) /* no CUDA device / CUDA failure: the product never falls back to the CPU */
#define ZK_ERR_INVALID_ARG (-1006)
#define ZK_ERR_CUDA (-1007) /* a CUDA runtime call or a kernel failed after the context was created; zk_last_cuda_error() has the text */
/* Kind::Zstd(code): returned as -(ZSTD_ErrorCode), i.e. in [-120, -1] */
#define ZK_ERR_ZSTD(code) (-(int32_t)(code))
#define ZK_IS_ZSTD_ERR(rc) ((rc) < 0 && (rc) > -1000)

const char* zk_error_name(int32_t rc);
/* cudaGetErrorString of the most recent CUDA failure seen by this thread ("" if none) */
const char* zk_last_cuda_error(void);

/* ------------------------------------------------------------------ context (CCtx/DCtx, encode.rs:130, decode.rs:31) */
typedef struct zk_ctx zk_ctx;
int32_t zk_ctx_create(int32_t device_ordinal, uint32_t flags, zk_ctx** out);
void zk_ctx_destroy(zk_ctx* ctx);
/* number of CUDA kernels this context has launched so far (bench.py reports it as gpu_launches) */
uint64_t zk_ctx_kernel_launches(const zk_ctx* ctx);
/* number of execution segments (independent runs of blocks of a seek-table entry) the decoder has run so far */
uint64_t zk_ctx_decode_segments(const zk_ctx* ctx);
/* prefix bytes this context has copied to the device so far, by every call that takes a prefix */
uint64_t zk_ctx_prefix_bytes_uploaded(const zk_ctx* ctx);
/* entries of reference archives this context has decoded so far, by the calls that take one (the _archive calls of the patch block) */
uint64_t zk_ctx_reference_entries_decoded(const zk_ctx* ctx);
/* kernel-only device time (ms, CUDA events on the context's stream) of the most recent batch call */
float zk_ctx_last_device_ms(const zk_ctx* ctx);
const char* zk_version(void);
/* per-kernel device time (CUDA events on the launching stream), accumulated while enabled.
 * slots: 0 scan, 1 seq, 2 huf, 3 exec, 4 xxh64, 5 match, 6 entropy-enc, 7 frame assembly; arrays of 8 */
void zk_ctx_profile(zk_ctx* ctx, int32_t enable);
void zk_ctx_profile_read(const zk_ctx* ctx, float* ms, uint32_t* launches);

/* ------------------------------------------------------------------ batch codec: the hot path */
/* Upper bound of the compressed size of n input bytes cut into frames of frame_size (excl. seek table). */
size_t zk_compress_bound(size_t n, uint32_t frame_size);

/*
 * Compress src[0..n) into ceil(n / frame_size) independent zstd frames written back to back into dst
 * (FrameSizePolicy::Uncompressed, encode.rs:528-544).  c_sizes / d_sizes (capacity frames_cap) receive
 * what RawEncoder would pass to SeekTable::log_frame (encode.rs:466).  n == 0 produces one empty frame,
 * like Encoder::finish() on an empty stream (encode.rs:755-756).  HOST pointers (pinned memory is faster).
 */
int32_t zk_compress_frames(zk_ctx* ctx, const uint8_t* src, size_t n, uint32_t frame_size, int32_t level,
                           int32_t checksum, uint8_t* dst, size_t dst_cap, uint32_t* c_sizes, uint32_t* d_sizes,
                           uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len);

/*
 * Decompress n_frames seek-table entries.  Entry f occupies comp[c_off[f] .. c_off[f+1]) and decodes to
 * dst[d_off[f] .. d_off[f+1]) (the N+1 cumulative offsets of SeekTable, seek_table.rs:97-101, rebased by
 * the caller to the two pointers).  status[f] (optional) = 0 or -(zstd code).  With verify_checksum != 0
 * frames that carry a content checksum are verified (-22 on mismatch).  HOST pointers.
 * Returns 0 or the first failing frame's status.
 */
int32_t zk_decompress_frames(zk_ctx* ctx, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off,
                             uint32_t n_frames, uint8_t* dst, int32_t verify_checksum, int32_t* status);

/* Range reads (SURVEY.md 8f.1; decode.rs:228-266 decodes a frame only as far as offset_limit): like
 * zk_decompress_frames, but entry i is only guaranteed to hold its first d_need[i] bytes afterwards (the decoder stops at
 * the first block boundary at or after that point; the rest of the entry's output range is unspecified).  A prefix is
 * not checksum-verified, as in the reference (decode.rs:425-427).  d_need == NULL or d_need[i] >= the entry's size: everything. */
int32_t zk_decompress_frames_upto(zk_ctx* ctx, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off,
                                  uint32_t n_frames, uint8_t* dst, const uint32_t* d_need, int32_t verify_checksum, int32_t* status);

/*
 * Prefix / patch mode: the same calls with a raw-content prefix that precedes EVERY frame (the reference re-applies it per
 * frame: cctx.ref_prefix at each frame start, encode.rs:332-338; dctx.ref_prefix before the first frame and after every frame
 * end, decode.rs:211-214, 246-255).  Matches may reach back into the prefix; frames made this way only decode with the same
 * prefix (libzstd: ZSTD_CCtx_refPrefix / ZSTD_DCtx_refPrefix).  prefix == NULL or prefix_len == 0: the plain calls.  HOST pointers.
 */
int32_t zk_compress_frames_prefix(zk_ctx* ctx, const uint8_t* src, size_t n, uint32_t frame_size, int32_t level,
                                  int32_t checksum, const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap,
                                  uint32_t* c_sizes, uint32_t* d_sizes, uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len);
int32_t zk_decompress_frames_prefix(zk_ctx* ctx, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off,
                                    uint32_t n_frames, uint8_t* dst, const uint32_t* d_need, int32_t verify_checksum,
                                    int32_t* status, const uint8_t* prefix, size_t prefix_len);

/*
 * Device-resident variants (zero-copy; used for roofline measurements and multi-GPU pipelines).
 * d_* are CUDA device pointers, 16-byte aligned, with >= 16 readable bytes after the last byte;
 * offset / size arrays stay on the HOST.  cuda_stream is a cudaStream_t (NULL = the context's own
 * non-blocking stream; pass cudaStreamLegacy (0x1) to order the work on the legacy default stream, e.g.
 * after PyTorch ops).  The call returns after the work has completed on that stream.
 */
int32_t zk_compress_frames_dev(zk_ctx* ctx, const void* d_src, size_t n, uint32_t frame_size, int32_t level,
                               int32_t checksum, void* d_dst, size_t dst_cap, uint32_t* c_sizes, uint32_t* d_sizes,
                               uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len, void* cuda_stream);
int32_t zk_decompress_frames_dev(zk_ctx* ctx, const void* d_comp, const uint64_t* c_off, const uint64_t* d_off,
                                 uint32_t n_frames, void* d_dst, int32_t verify_checksum, int32_t* status,
                                 void* cuda_stream);

/*
 * FrameSizePolicy::Compressed(target) over a whole buffer: frames close after the first 32 KiB block at which header + blocks >= target
 * (or at 1 GiB of input).  "header + blocks" is the 10-byte frame header plus every block with its 3-byte block header; the 4-byte
 * checksum does not count (encode.rs:537-544).  The cut depends only on the input, target, level, checksum flag and prefix.
 * final == 0: only closed frames are written; *consumed = input bytes they cover, the rest must be passed again with more input (a
 * frame that would end exactly at the end of the input stays open).  final != 0: the rest becomes the last frame; n == 0 gives one
 * empty frame.  target == 0 behaves like 1.  dst_cap >= zk_compress_bound(n, 32768) and frames_cap >= n / 32768 + 2 always suffice;
 * less returns -70 (dstSize_tooSmall).  HOST pointers.
 */
int32_t zk_compress_frames_csize(zk_ctx* ctx, const uint8_t* src, size_t n, uint32_t target, int32_t level, int32_t checksum,
                                 const uint8_t* prefix, size_t prefix_len, int32_t final, uint8_t* dst, size_t dst_cap,
                                 uint32_t* c_sizes, uint32_t* d_sizes, uint32_t frames_cap, uint32_t* n_frames,
                                 size_t* dst_len, size_t* consumed);
/* the same on device pointers (conventions of zk_compress_frames_dev; no prefix, like the other _dev entry points) */
int32_t zk_compress_frames_csize_dev(zk_ctx* ctx, const void* d_src, size_t n, uint32_t target, int32_t level, int32_t checksum,
                                     int32_t final, void* d_dst, size_t dst_cap, uint32_t* c_sizes, uint32_t* d_sizes,
                                     uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len, size_t* consumed, void* cuda_stream);

/*
 * FrameSizePolicy::ContentDefined(size) over a whole buffer: frame boundaries chosen by the content, so that an edit changes only the frames
 * around it and later frames keep their bytes.  size (the target mean frame size) is clamped to [4096, 2^30]; mn = size / 4,
 * mx = min(4 size, 2^30), T = floor((2^64 - 1) / (size - mn)).  Position p is a candidate when h_p >= 2^64 - T, where
 * h_p = sum over j = max(0, p - 63) .. p of gear(src[j]) * 2^(p - j) mod 2^64 and gear(b) is splitmix64 of b + 1 (the sampling hash of
 * zk_compress_frames_ldm).  A frame that starts at byte b ends at the first candidate e with b + mn - 1 <= e <= b + mx - 1 (e - b + 1
 * bytes), else after mx bytes.  The cut depends on the input bytes and size only: not on level, checksum, prefix, or how the input is
 * split into calls.  A run of one byte value never holds a candidate, so it is cut every mx bytes.  Frame f's bytes are what
 * zk_compress_frames_sized writes for the same sizes, at every level.
 * final == 0: only closed frames are written; *consumed = input bytes they cover, the rest must be passed again with more input (a frame
 * that would end exactly at the end of the input stays open).  final != 0: the rest becomes the last frame; n == 0 gives one empty frame.
 * Every frame but the last has at least 1024 bytes, so dst_cap >= zk_compress_bound(n, 1024) and frames_cap >= n / 1024 + 1 always
 * suffice; less than a call needs returns -70 (dstSize_tooSmall).  HOST pointers.
 */
int32_t zk_compress_frames_cdc(zk_ctx* ctx, const uint8_t* src, size_t n, uint32_t size, int32_t level, int32_t checksum,
                               const uint8_t* prefix, size_t prefix_len, int32_t final, uint8_t* dst, size_t dst_cap,
                               uint32_t* c_sizes, uint32_t* d_sizes, uint32_t frames_cap, uint32_t* n_frames,
                               size_t* dst_len, size_t* consumed);
/* the same on device pointers (conventions of zk_compress_frames_dev; no prefix, like the other _dev entry points) */
int32_t zk_compress_frames_cdc_dev(zk_ctx* ctx, const void* d_src, size_t n, uint32_t size, int32_t level, int32_t checksum,
                                   int32_t final, void* d_dst, size_t dst_cap, uint32_t* c_sizes, uint32_t* d_sizes,
                                   uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len, size_t* consumed, void* cuda_stream);

/*
 * Frames of caller-chosen sizes in one batch (a frame boundary at any byte, as Encoder::end_frame, encode.rs:438-472): frame f covers the
 * next frame_sizes[f] bytes of src, whose length is the sum of the sizes.  Frame f's bytes are exactly what zk_compress_frames_prefix
 * writes for those bytes alone with frame_size = max(frame_sizes[f], 1): a size of 0 gives the empty frame of n == 0, and every level,
 * the checksum and the prefix behave as there.  The frames are written back to back into dst; c_sizes (n_frames entries) receives their
 * compressed sizes (the d_sizes are frame_sizes).  n_frames == 0 writes nothing.  A size above 1 GiB returns -42 (parameter_outOfBound),
 * more than ZK_SEEKABLE_MAX_FRAMES frames ZK_ERR_FRAME_INDEX_TOO_LARGE, and a dst_cap below what the frames need -70 (dstSize_tooSmall);
 * dst_cap >= zk_compress_bound_sized(frame_sizes, n_frames) always suffices.  HOST pointers.
 */
int32_t zk_compress_frames_sized(zk_ctx* ctx, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                 int32_t checksum, const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap,
                                 uint32_t* c_sizes, size_t* dst_len);
/* the same on device src / dst (frame_sizes and c_sizes stay on the host; no prefix, like the other _dev entry points) */
int32_t zk_compress_frames_sized_dev(zk_ctx* ctx, const void* d_src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                     int32_t checksum, void* d_dst, size_t dst_cap, uint32_t* c_sizes, size_t* dst_len,
                                     void* cuda_stream);
/* Upper bound of the compressed size of frames of these sizes (excl. seek table). */
size_t zk_compress_bound_sized(const uint32_t* frame_sizes, uint32_t n_frames);

/*
 * Long-distance matching (patch mode): zk_compress_frames_prefix / zk_compress_frames_sized with every frame matched against the WHOLE
 * prefix, not only its last 32 KiB -- what the reference CLI asks of libzstd for `--patch-from` (WindowLog and
 * EnableLongDistanceMatching on the CCtx it hands to EncodeOptions::with_cctx, cli/src/compress.rs:31-37).  A frame that repeats the
 * prefix with a few edits shrinks to the edits.  A non-empty frame announces a Window_Size of min(frame content + prefix_len, 2^27) (at
 * least what the prefix calls announce), which a default libzstd DCtx and zk_decompress_frames_prefix accept; no offset exceeds it, so with a
 * prefix above 128 MiB only its last 128 MiB are matched, and the far end of the prefix is out of reach late in a large frame.
 * Long-distance matching is part of the high-level tier: every `level`, negative ones included, writes what level 16 writes here.
 * prefix == NULL or prefix_len == 0: exactly the plain call at `level`.  The index of the prefix is rebuilt on every call (and for
 * every 96 MiB of input within one).  zk_compress_frames_csize has no such variant: its exact cut needs a bounded history per block.
 * HOST pointers.
 */
int32_t zk_compress_frames_ldm(zk_ctx* ctx, const uint8_t* src, size_t n, uint32_t frame_size, int32_t level,
                               int32_t checksum, const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap,
                               uint32_t* c_sizes, uint32_t* d_sizes, uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len);
int32_t zk_compress_frames_sized_ldm(zk_ctx* ctx, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                     int32_t checksum, const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap,
                                     uint32_t* c_sizes, size_t* dst_len);

/*
 * Long mode (what `zstd --long` does within a frame): zk_compress_frames_prefix / zk_compress_frames_sized with every frame also matched
 * against ITS OWN earlier bytes up to the window back, not only the last 2 MiB that level 16 searches.  A frame of many MiB that repeats
 * itself far apart (a disk image, a tar of similar trees, a log rotated twice) shrinks to what differs.  Frames stay independent: a
 * frame's bytes depend only on its own bytes, the checksum flag and the prefix, never on its neighbours in the batch, the sub-batch size,
 * host vs device memory or where the encoder's internal passes cut the batch, so the sized call equals one call per frame.  A non-empty
 * frame announces a Window_Size of min(max(frame content + prefix_len, 128 KiB), 2^27), as with zk_compress_frames_ldm, and no offset
 * exceeds it.  With a prefix, every frame
 * is also matched against the whole prefix exactly as by zk_compress_frames_ldm, so long mode is a superset of that switch; without one it
 * needs none.  Long matches are at least 64 bytes.  Part of the high-level tier: every `level` writes what level 16 writes here.  The
 * index of the input costs about 1 byte of device scratch per input byte and is rebuilt on every call.  zk_compress_frames_csize and
 * zk_compress_frames_cdc have no such variant.  HOST pointers; the _dev pair takes device src / dst (sizes on the host) and no prefix, like
 * every _dev entry point.
 */
int32_t zk_compress_frames_long(zk_ctx* ctx, const uint8_t* src, size_t n, uint32_t frame_size, int32_t level,
                                int32_t checksum, const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap,
                                uint32_t* c_sizes, uint32_t* d_sizes, uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len);
int32_t zk_compress_frames_sized_long(zk_ctx* ctx, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                      int32_t checksum, const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap,
                                      uint32_t* c_sizes, size_t* dst_len);
int32_t zk_compress_frames_long_dev(zk_ctx* ctx, const void* d_src, size_t n, uint32_t frame_size, int32_t level, int32_t checksum,
                                    void* d_dst, size_t dst_cap, uint32_t* c_sizes, uint32_t* d_sizes, uint32_t frames_cap,
                                    uint32_t* n_frames, size_t* dst_len, void* cuda_stream);
int32_t zk_compress_frames_sized_long_dev(zk_ctx* ctx, const void* d_src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                          int32_t checksum, void* d_dst, size_t dst_cap, uint32_t* c_sizes, size_t* dst_len,
                                          void* cuda_stream);

/*
 * Per-frame prefixes (batched deltas, seekable patches): frames of caller-chosen sizes, frame f matched against its own range
 * prefix[ranges[2f] .. ranges[2f+1]) of one prefix buffer -- each object against its own previous version, or each frame of a new image
 * against the slice of the old image around it -- in one batch instead of one call per frame.
 *   - Frame bytes: frame f is exactly what zk_compress_frames_sized (ldm and long_mode 0), zk_compress_frames_sized_ldm (ldm != 0) or
 *     zk_compress_frames_sized_long (long_mode != 0) writes for frame f alone with its range as the prefix, at every level, with either
 *     checksum setting, Window_Descriptor included.  Exceptions: under ldm, a frame whose range is empty is what zk_compress_frames_sized
 *     writes for it at level 16 with no prefix, and an empty frame (size 0) is level 16's empty frame.
 *   - Tiers: with ldm or long_mode set and a non-empty prefix buffer, every frame runs the high-level tier (level 16's bytes), whatever
 *     its range, so one call never mixes tiers; without either flag a frame with an empty range is the plain frame at `level`.
 *   - ranges == NULL gives every frame the whole buffer: the call then equals zk_compress_frames_sized / _sized_ldm / _sized_long on the
 *     same arguments.  A range with lo > hi or hi > prefix_len, or a prefix_len above 2^31 - 1, returns ZK_ERR_INVALID_ARG.  Empty frames,
 *     more than ZK_SEEKABLE_MAX_FRAMES frames and a short dst_cap behave as in zk_compress_frames_sized; n_frames == 0 writes nothing.
 *   - The prefix buffer is uploaded once per call.  With ldm or long_mode, every distinct range is indexed once (its last min(length,
 *     2^27 - 1) bytes, about 1 byte of device scratch per indexed byte); the call cuts its batch so that this stays bounded, and a frame
 *     whose range is 2^31 - 1 bytes long always runs.
 * zk_decompress_frames_prefixes decodes entry e (every zstd frame in it) against prefix[ranges[2e] .. ranges[2e+1]): exactly as
 * zk_decompress_frames_prefix decodes that entry alone with its range as the prefix, d_need, checksum verification and every error code
 * included (an offset that reaches before the start of the entry's range is -20, corruption_detected).  ranges == NULL: every entry
 * against the whole buffer, which is zk_decompress_frames_prefix.  With ranges, only the hull of the non-empty ranges of the entries it
 * decodes goes to the device, in groups of consecutive entries whose hull is at most 1 GiB, so the buffer may be of any size (host
 * memory, mmapped files included) and only a single range is limited to 2^31 - 1 bytes; a range with lo > hi or hi > prefix_len returns
 * ZK_ERR_INVALID_ARG.  HOST pointers.
 */
int32_t zk_compress_frames_sized_prefixes(zk_ctx* ctx, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                          int32_t checksum, const uint8_t* prefix, size_t prefix_len, const uint64_t* ranges,
                                          int32_t ldm, int32_t long_mode, uint8_t* dst, size_t dst_cap, uint32_t* c_sizes, size_t* dst_len);
int32_t zk_decompress_frames_prefixes(zk_ctx* ctx, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off, uint32_t n_frames,
                                      uint8_t* dst, const uint32_t* d_need, int32_t verify_checksum, int32_t* status,
                                      const uint8_t* prefix, size_t prefix_len, const uint64_t* ranges);

/*
 * Seekable patches (DESIGN §3.4): every frame of NEW matched against the slice of OLD that holds its content, so OLD may be of any size, a
 * frame's offsets never exceed 2^27 (a default libzstd DCtx restores it with ZSTD_DCtx_refPrefix(OLD[lo, hi))), and one frame restores
 * from its slice alone.
 *   zk_patch_ranges: frame f covers the next frame_sizes[f] bytes of new_src -> its slice [ranges[2f], ranges[2f+1]) of old.  The slices are
 *     a pure function of old, new, the frame sizes and margin (not of how the work is split): an anchor is a position p >= 63 whose gear hash
 *     of the 64 bytes ending at p (the hash of zk_compress_frames_cdc) is >= 2^64 - floor((2^64 - 1) / 65536); each anchor c of frame
 *     f = [a, b) takes OLD's anchor of the same hash nearest to c (the lower on a tie); with (c1, o1) the first match and (c2, o2) the last,
 *     the slice is [o1 - (c1 - a) - margin, o2 + (b - c2) + margin) when o2 >= o1 and |(o2 - o1) - (c2 - c1)| <= b - a, else
 *     [o1 - (c1 - a) - margin, o1 + (b - c1) + margin); with no match [a - margin, b + margin); clamped to [0, old_len) and then cut to at
 *     most 2^27 - (b - a) bytes around (o1 + o2) / 2 (o1 for a move; without a match, the clamped slice's centre).  old_len and margin
 *     below 2^62.  Both buffers in HOST memory (old may be mmapped); they stream through the device in pieces of at most 1 GiB.
 *   zk_compress_frames_patch: frame f is exactly what zk_compress_frames_sized_prefixes(ldm = 1) writes for frame f alone with old as the
 *     buffer and its range (level 16's tier; an empty range: level 16's frame without a prefix).  Consecutive frames whose ranges' hull is
 *     at most 1 GiB run as one such call on that hull of old, so old may be of any size.  Argument errors as in the sized call; a range
 *     with lo > hi or hi > old_len returns ZK_ERR_INVALID_ARG.
 *   The archive records the slices in one skippable frame at the start of entry 0 (its compressed size includes it):
 *     u32 ZK_PATCH_SLICES_MAGIC, u32 payload size, "ZKSLICE1", u64 old_len, u32 n, n x (u64 lo, u64 hi), little-endian.
 *   zk_patch_slices_write writes it (zk_patch_slices_size(n) bytes; a short dst_cap is -70); zk_patch_slices_read parses it from the start
 *     of src and validates every field: the magic, the payload size, the tag, n == n_frames (the seek table's frame count), lo <= hi <=
 *     old_len; anything else is ZK_ERR_INVALID_ARG.  ranges (2 n_frames) may be NULL; *frame_len: the frame's bytes.
 */
int32_t zk_patch_ranges(zk_ctx* ctx, const uint8_t* new_src, const uint32_t* frame_sizes, uint32_t n_frames, const uint8_t* old,
                        uint64_t old_len, uint64_t margin, uint64_t* ranges);
int32_t zk_compress_frames_patch(zk_ctx* ctx, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                 int32_t checksum, const uint8_t* old, uint64_t old_len, const uint64_t* ranges, uint8_t* dst, size_t dst_cap,
                                 uint32_t* c_sizes, size_t* dst_len);
size_t zk_patch_slices_size(uint32_t n_frames);
int32_t zk_patch_slices_write(uint64_t old_len, const uint64_t* ranges, uint32_t n_frames, uint8_t* dst, size_t dst_cap, size_t* written);
int32_t zk_patch_slices_read(const uint8_t* src, size_t len, uint32_t n_frames, uint64_t* old_len, uint64_t* ranges, size_t* frame_len);

/*
 * Seekable patches against a seekable archive (DESIGN §3.4.2): the reference R is a seekable archive, ref_n entries of ref_comp (ref_len
 * bytes) at ref_c_off / ref_d_off (ref_n + 1 offsets each, as zk_decompress_frames takes them), and OLD is its decoded content, old_len =
 * ref_d_off[ref_n].  R may be mmapped; only the compressed entries that a call needs cross to the device, and they are decoded there, on
 * slot 0, into the context's prefix buffer: no byte of OLD is uploaded (zk_ctx_prefix_bytes_uploaded does not grow) or copied to the host.
 *   zk_patch_ranges_archive returns exactly zk_patch_ranges(new_src, frame_sizes, OLD, old_len, margin), whatever R's entry layout.
 *   zk_compress_frames_patch_archive writes exactly the bytes and c_sizes of zk_compress_frames_patch(..., OLD, old_len, ranges, ...).
 *   zk_decompress_frames_prefixes_archive gives the output, statuses and return code of zk_decompress_frames_prefixes(..., OLD, old_len,
 *     ranges), d_need and checksum verification included; ranges == NULL: every entry against all of OLD.
 *   zk_decoder_decompress_with_reference_archive (the Decoder block) reads a seekable patch that way.
 * For each group of entries (zk_decompress_frames_prefixes' groups, hull [hlo, hhi) <= 1 GiB) only the entries of R whose output overlaps
 * the hull are decoded, the last one only as far as hhi (no checksum on that partial entry, as with d_need); empty entries never are.
 * zk_ctx_reference_entries_decoded counts them.  Full entries of R are checked against their checksums on the compress and range calls
 * always, on the decompress call when verify_checksum is set.
 * An entry of R that fails to decode: every entry being decompressed whose range overlaps its output gets its status (the return code is
 * the first non-zero status, as in the raw-reference call; the others decode normally); the compress and range calls return it.
 * ZK_ERR_INVALID_ARG: R's offsets decrease, ref_d_off[0] != 0, ref_c_off[ref_n] > ref_len, a range with lo > hi or hi > old_len, or R is
 * itself a seekable patch (ZK_PATCH_SLICES_MAGIC at ref_c_off[0]: such a reference goes to the _chain calls below, with its own reference
 * under it).  Other argument errors as in the raw calls.  Each _archive call is its _chain call with depth 1.
 */
int32_t zk_patch_ranges_archive(zk_ctx* ctx, const uint8_t* new_src, const uint32_t* frame_sizes, uint32_t n_frames, const uint8_t* ref_comp,
                                size_t ref_len, const uint64_t* ref_c_off, const uint64_t* ref_d_off, uint32_t ref_n, uint64_t margin,
                                uint64_t* ranges);
int32_t zk_compress_frames_patch_archive(zk_ctx* ctx, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                         int32_t checksum, const uint8_t* ref_comp, size_t ref_len, const uint64_t* ref_c_off,
                                         const uint64_t* ref_d_off, uint32_t ref_n, const uint64_t* ranges, uint8_t* dst, size_t dst_cap,
                                         uint32_t* c_sizes, size_t* dst_len);
int32_t zk_decompress_frames_prefixes_archive(zk_ctx* ctx, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off, uint32_t n,
                                              uint8_t* dst, const uint32_t* d_need, int32_t verify_checksum, int32_t* status,
                                              const uint8_t* ref_comp, size_t ref_len, const uint64_t* ref_c_off, const uint64_t* ref_d_off,
                                              uint32_t ref_n, const uint64_t* ranges);

/*
 * Seekable patch chains (DESIGN §3.4.3): the reference is a chain R_0 ... R_{depth-1} of archives (root first, 1 <= depth <=
 * ZK_CHAIN_MAX_DEPTH), each described as the _archive calls take one (host memory; comp may be mmapped).  R_0 is a plain seekable archive;
 * every R_i with i >= 1 is a seekable patch whose slice frame (zk_patch_slices_read, n slices) has old_len = R_{i-1}'s decoded length and is
 * applied against R_{i-1}'s decoded content.  OLD is the decoded content of the head R_{depth-1}.  The library reads each patch level's
 * slice frame itself.
 *   Every _chain call returns exactly what its raw call returns on OLD (the same ranges, archive bytes, c_sizes, output, statuses and
 *   return code); with depth 1 it is its _archive call, which runs this same code.  No byte of any level's content goes to the host.
 *   What is decoded: Need(i, [lo, hi)) decodes the non-empty entries of R_i whose output overlaps [lo, hi) into level i's device arena, the
 *   last one only as far as hi.  For i >= 1 their slices are grouped in list order as zk_decompress_frames_prefixes groups ranges (hull at
 *   most 1 GiB, empty slices skipped); for each group with a non-empty hull Need(i - 1, hull) runs first, then the group's entries are
 *   decoded against it.  The top of the chain runs Need(depth - 1, ...) where the _archive calls decode R.  zk_ctx_reference_entries_decoded
 *   counts every entry decoded at every level, each time it is decoded.
 *   Failures propagate upward: an entry of R_{i-1} that fails (corrupt, or a bad checksum on a full entry with verification on) gives its
 *   status to every entry of R_i in the same group whose slice overlaps its output (the first failing entry's in list order); those are not
 *   decoded and count as failed for level i + 1.  At the top, statuses are as in the _archive calls.  The decompress call verifies full
 *   entries at every level when verify_checksum is set; the compress and range calls always do, and return the first failure.
 * ZK_ERR_INVALID_ARG: depth == 0 or > ZK_CHAIN_MAX_DEPTH, a root that is a seekable patch, an R_i (i >= 1) without a valid slice frame of
 * its entry count, an old_len that differs from R_{i-1}'s decoded length, any level failing the _archive calls' offset rules, a range
 * past OLD's length.  Device memory: per level below the head, about its hull plus one entry plus one 128 KiB block.
 */
typedef struct { const uint8_t* comp; size_t len; const uint64_t* c_off; const uint64_t* d_off; uint32_t n; } zk_reference_archive;
int32_t zk_patch_ranges_chain(zk_ctx* ctx, const uint8_t* new_src, const uint32_t* frame_sizes, uint32_t n_frames,
                              const zk_reference_archive* chain, uint32_t depth, uint64_t margin, uint64_t* ranges);
int32_t zk_compress_frames_patch_chain(zk_ctx* ctx, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                       int32_t checksum, const zk_reference_archive* chain, uint32_t depth, const uint64_t* ranges, uint8_t* dst,
                                       size_t dst_cap, uint32_t* c_sizes, size_t* dst_len);
int32_t zk_decompress_frames_prefixes_chain(zk_ctx* ctx, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off, uint32_t n,
                                            uint8_t* dst, const uint32_t* d_need, int32_t verify_checksum, int32_t* status,
                                            const zk_reference_archive* chain, uint32_t depth, const uint64_t* ranges);

/*
 * The content-defined cut alone (FrameSizePolicy::ContentDefined(size), the rule of zk_compress_frames_cdc): frame_sizes, *n_frames and
 * *consumed are exactly the d_sizes, frame count and consumed of zk_compress_frames_cdc on the same src, n, size and final, at any level;
 * nothing is compressed.  frames_cap >= n / 1024 + 1 always suffices; less than a call needs returns -70 (dstSize_tooSmall).  HOST pointers.
 */
int32_t zk_cut_frames_cdc(zk_ctx* ctx, const uint8_t* src, size_t n, uint32_t size, int32_t final, uint32_t* frame_sizes,
                          uint32_t frames_cap, uint32_t* n_frames, size_t* consumed);

/*
 * Compress a new version against the archive of the previous one: every frame whose bytes an old entry already holds is copied from the
 * old archive, only the others are compressed.  src and frame_sizes as in zk_compress_frames_sized; long_mode != 0 compresses as
 * zk_compress_frames_sized_long (frames are independent there too).  The old archive: old_comp (old_len bytes) with old_n entries, entry g at
 * old_comp[old_c_off[g] .. old_c_off[g+1]) decoding to old_d_off[g+1] - old_d_off[g] bytes (the offsets of zk_decompress_frames, HOST
 * arrays of old_n + 1 entries).  Writes the frames back to back into dst, c_sizes[f], and reused[f]: the old entry frame f copies, or
 * 0xFFFFFFFF.  The rule for frame f:
 *   1. Old entry g is a candidate when its decompressed size equals frame_sizes[f], it decodes without error (checksum verified), the
 *      Content_Checksum_flag of its first zstd frame equals checksum != 0, and key(g) == key(f).  key(x) is XXH64 (seed 0) of the
 *      little-endian 8-byte XXH64s of x's consecutive 32 KiB chunks (the last one may be shorter; no bytes: the XXH64 of nothing).
 *   2. Frame f copies the lowest-index candidate verbatim iff its decoded bytes equal frame f's bytes, compared byte by byte: equality is
 *      proven, never assumed from the key.  With no candidate, or when the bytes differ, frame f is what zk_compress_frames_sized (or
 *      _sized_long) writes for it; no further candidate is tried.
 * So the result always restores src, and it equals zk_compress_frames_sized[_long] on the same arguments byte for byte whenever the
 * entries it copies were written by this codec at the same level, checksum flag and mode.  Entries written otherwise (another level,
 * libzstd) still decode to the frame's bytes and are copied as they are.  An old entry that fails to decode is not a candidate, never an
 * error of the call.  There is no prefix, no long-distance switch and no Compressed(n) variant: a copied frame's bytes must depend on its
 * own bytes alone.  ZK_REUSE_KEY_BITS (environment, tests; default 64) keeps only that many low bits of every key.
 * Old offsets that decrease, or an old_c_off[old_n] above old_len, return ZK_ERR_INVALID_ARG; other argument errors are those of
 * zk_compress_frames_sized.  dst_cap >= zk_compress_bound_sized(frame_sizes, n_frames) + old_c_off[old_n] - old_c_off[0] suffices when
 * every old entry is at most zk_compress_bound_sized of its own decompressed size (as this codec's entries are) or is copied at most once;
 * a dst_cap below what the frames need returns -70 (dstSize_tooSmall).  c_sizes and reused may be NULL.  Runs unpipelined; the old
 * entries of a matching size are decoded twice (once to index them, once to compare them), so device memory stays bounded by the
 * sub-batch, never by the old archive.  HOST pointers.
 */
int32_t zk_compress_frames_sized_reuse(zk_ctx* ctx, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                       int32_t checksum, int32_t long_mode, const uint8_t* old_comp, size_t old_len,
                                       const uint64_t* old_c_off, const uint64_t* old_d_off, uint32_t old_n, uint8_t* dst, size_t dst_cap,
                                       uint32_t* c_sizes, uint32_t* reused, size_t* dst_len);

/* ------------------------------------------------------------------ SeekTable (lib/src/seek_table.rs) */
typedef struct zk_seek_table zk_seek_table;
typedef enum { ZK_FORMAT_HEAD = 0, ZK_FORMAT_FOOT = 1 } zk_format; /* seek_table.rs:228-241 */

zk_seek_table* zk_seek_table_new(void);                                             /* SeekTable::new  :314 */
void zk_seek_table_free(zk_seek_table* st);
zk_seek_table* zk_seek_table_clone(const zk_seek_table* st);
/* SeekTable::from_seekable_format over a memory span (BytesWrapper), seek_table.rs:379-436 */
int32_t zk_seek_table_from_bytes(const uint8_t* buf, size_t len, zk_format format, zk_seek_table** out);
int32_t zk_seek_table_log_frame(zk_seek_table* st, uint32_t c_size, uint32_t d_size); /* :513-525 */
uint32_t zk_seek_table_num_frames(const zk_seek_table* st);                           /* :540 */
uint32_t zk_seek_table_frame_index_comp(const zk_seek_table* st, uint64_t offset);    /* :560 */
uint32_t zk_seek_table_frame_index_decomp(const zk_seek_table* st, uint64_t offset);  /* :580 */
int32_t zk_seek_table_frame_start_comp(const zk_seek_table* st, uint32_t index, uint64_t* out);
int32_t zk_seek_table_frame_start_decomp(const zk_seek_table* st, uint32_t index, uint64_t* out);
int32_t zk_seek_table_frame_end_comp(const zk_seek_table* st, uint32_t index, uint64_t* out);
int32_t zk_seek_table_frame_end_decomp(const zk_seek_table* st, uint32_t index, uint64_t* out);
int32_t zk_seek_table_frame_size_comp(const zk_seek_table* st, uint32_t index, uint64_t* out);
int32_t zk_seek_table_frame_size_decomp(const zk_seek_table* st, uint32_t index, uint64_t* out);
uint64_t zk_seek_table_max_frame_size_comp(const zk_seek_table* st);
uint64_t zk_seek_table_max_frame_size_decomp(const zk_seek_table* st);
uint64_t zk_seek_table_size_comp(const zk_seek_table* st);
uint64_t zk_seek_table_size_decomp(const zk_seek_table* st);
/* copies the N+1 cumulative offsets (c then d may be NULL); returns N+1 */
uint32_t zk_seek_table_offsets(const zk_seek_table* st, uint64_t* c_off, uint64_t* d_off, uint32_t cap);

/* Serializer (seek_table.rs:955-1051): resumable at byte granularity */
typedef struct zk_serializer zk_serializer;
zk_serializer* zk_seek_table_into_serializer(const zk_seek_table* st, zk_format format); /* :885-905 */
void zk_serializer_free(zk_serializer* s);
size_t zk_serializer_write_into(zk_serializer* s, uint8_t* buf, size_t len);          /* :967-1005 */
void zk_serializer_reset(zk_serializer* s);                                            /* :1021 */
size_t zk_serializer_encoded_len(const zk_serializer* s);                             /* :1038 */

/* ------------------------------------------------------------------ EncodeOptions / RawEncoder / Encoder (lib/src/encode.rs) */
typedef struct zk_encode_options zk_encode_options;
typedef struct zk_raw_encoder zk_raw_encoder;
typedef struct zk_encoder zk_encoder;
/* encode.rs:21-31; ZK_POLICY_CONTENT: content-defined frames (zk_compress_frames_cdc), an extension of this codec */
typedef enum { ZK_POLICY_COMPRESSED = 0, ZK_POLICY_UNCOMPRESSED = 1, ZK_POLICY_CONTENT = 2 } zk_frame_size_policy;
typedef struct { size_t in_progress, out_progress; } zk_compression_progress;           /* encode.rs:43-65 */
typedef struct { size_t out_progress, data_left; } zk_epilogue_progress;                /* encode.rs:69-92 */
/* Write sink (W: std::io::Write, encode.rs:570): must consume all len bytes; return 0 on success */
typedef int32_t (*zk_write_fn)(void* user, const uint8_t* data, size_t len);
typedef int32_t (*zk_flush_fn)(void* user);

zk_encode_options* zk_encode_options_new(zk_ctx* ctx);                                  /* encode.rs:124 */
void zk_encode_options_free(zk_encode_options* o);
void zk_encode_options_frame_size_policy(zk_encode_options* o, zk_frame_size_policy kind, uint32_t size); /* :158 */
void zk_encode_options_checksum_flag(zk_encode_options* o, int32_t flag);               /* :166 */
void zk_encode_options_compression_level(zk_encode_options* o, int32_t level);          /* :176 */
/* flag != 0: frames given a prefix (the *_compress_with_prefix calls) are matched against the whole of it, as by zk_compress_frames_ldm
 * (the counterpart of the CCtx the reference CLI prepares for with_cctx); every level then runs as level 16.  RawEncoder honours it
 * under both policies (its trial compressions included), Encoder under Uncompressed(n): with Compressed(n) or ContentDefined(n)
 * zk_encode_options_into_encoder returns ZK_ERR_INVALID_ARG and does not consume the options */
void zk_encode_options_long_distance_matching(zk_encode_options* o, int32_t flag);
/* flag != 0: long mode (zk_compress_frames_long): every frame is also matched against its own bytes up to 2^27 back, and frames given a
 * prefix against the whole of it; every level then runs as level 16.  Independent of the long-distance switch above, and a superset of
 * it.  RawEncoder honours it under both policies, Encoder under Uncompressed(n): with Compressed(n) or ContentDefined(n)
 * zk_encode_options_into_encoder returns ZK_ERR_INVALID_ARG and does not consume the options */
void zk_encode_options_long_mode(zk_encode_options* o, int32_t flag);
/* consume the options (like `self`).  ZK_POLICY_CONTENT: Encoder only (it buffers and cuts like Compressed(n), through
 * zk_compress_frames_cdc); zk_encode_options_into_raw_encoder returns ZK_ERR_INVALID_ARG for it, since a RawEncoder reports each call's
 * progress before the frame's end is known, and does not consume the options */
int32_t zk_encode_options_into_raw_encoder(zk_encode_options* o, zk_raw_encoder** out); /* :188 */
int32_t zk_encode_options_into_encoder(zk_encode_options* o, zk_write_fn write, zk_flush_fn flush, void* user,
                                       zk_encoder** out);                               /* :204 */

void zk_raw_encoder_free(zk_raw_encoder* e);
int32_t zk_raw_encoder_compress(zk_raw_encoder* e, const uint8_t* input, size_t in_len, uint8_t* output,
                                size_t out_len, zk_compression_progress* progress);     /* :398 / 311-354 */
/* RawEncoder::compress_with_prefix: the prefix given at a frame's FIRST call is that frame's raw-content prefix (it must stay
 * valid until the frame is closed -- 'b: 'a in the reference); NULL = none */
int32_t zk_raw_encoder_compress_with_prefix(zk_raw_encoder* e, const uint8_t* input, size_t in_len, uint8_t* output,
                                            size_t out_len, const uint8_t* prefix, size_t prefix_len,
                                            zk_compression_progress* progress);            /* :311-354 */
int32_t zk_raw_encoder_end_frame(zk_raw_encoder* e, uint8_t* output, size_t out_len,
                                 zk_epilogue_progress* progress);                       /* :438-472 */
const zk_seek_table* zk_raw_encoder_seek_table(const zk_raw_encoder* e);               /* :479 */
zk_seek_table* zk_raw_encoder_into_seek_table(zk_raw_encoder* e);                      /* :492 (consumes e) */
void zk_raw_encoder_reset_frame(zk_raw_encoder* e);                                     /* :501-507 */
void zk_raw_encoder_reset_seek_table(zk_raw_encoder* e);                                /* :524 */

void zk_encoder_free(zk_encoder* e);
int32_t zk_encoder_compress(zk_encoder* e, const uint8_t* buf, size_t len, size_t* consumed); /* :692 / 641-665 */
int32_t zk_encoder_compress_with_prefix(zk_encoder* e, const uint8_t* buf, size_t len, const uint8_t* prefix,
                                        size_t prefix_len, size_t* consumed);               /* :641-665 */
int32_t zk_encoder_end_frame(zk_encoder* e, size_t* written);                          /* :704-717 */
int32_t zk_encoder_flush(zk_encoder* e);                                                /* impl Write::flush :796 */
/* finish()/finish_format() consume the encoder; *total = bytes written to the sink incl. seek table */
int32_t zk_encoder_finish(zk_encoder* e, uint64_t* total);                              /* :743 */
int32_t zk_encoder_finish_format(zk_encoder* e, zk_format format, uint64_t* total);     /* :755-775 */
uint64_t zk_encoder_written_compressed(const zk_encoder* e);                            /* :615 */
const zk_seek_table* zk_encoder_seek_table(const zk_encoder* e);                        /* :609 */

/* ------------------------------------------------------------------ Seekable source + Decoder (lib/src/seekable.rs, decode.rs) */
/* trait Seekable (seekable.rs:16-39) as callbacks.  whence: 0 = OffsetFrom::Start(u64), 1 = OffsetFrom::End(i64) */
typedef struct {
    void* user;
    int64_t (*set_offset)(void* user, int32_t whence, int64_t offset); /* -> new absolute position or < 0 */
    int64_t (*read)(void* user, uint8_t* buf, size_t len);             /* -> bytes read (0 = EOF) or < 0 */
} zk_seekable;

typedef struct zk_decode_options zk_decode_options;
typedef struct zk_decoder zk_decoder;

/* DecodeOptions::new(src) with src = BytesWrapper over memory (seekable.rs:43-97); bytes must outlive the decoder */
zk_decode_options* zk_decode_options_new_bytes(zk_ctx* ctx, const uint8_t* src, size_t len);
/* DecodeOptions::new(src) with a generic Seekable */
zk_decode_options* zk_decode_options_new_seekable(zk_ctx* ctx, zk_seekable src);
void zk_decode_options_free(zk_decode_options* o);
void zk_decode_options_seek_table(zk_decode_options* o, const zk_seek_table* st);     /* decode.rs:69 (copied) */
void zk_decode_options_lower_frame(zk_decode_options* o, uint32_t index);              /* :77 */
void zk_decode_options_upper_frame(zk_decode_options* o, uint32_t index);              /* :85 */
void zk_decode_options_offset(zk_decode_options* o, uint64_t offset);                  /* :95 */
void zk_decode_options_offset_limit(zk_decode_options* o, uint64_t limit);             /* :105 */
int32_t zk_decode_options_into_decoder(zk_decode_options* o, zk_decoder** out);        /* :111 / 152-187 (consumes o) */

void zk_decoder_free(zk_decoder* d);
int32_t zk_decoder_decompress(zk_decoder* d, uint8_t* buf, size_t len, size_t* produced); /* :314 / 201-270 */
/* Decoder::decompress_with_prefix: every frame is decoded against the raw-content prefix (decode.rs:211-214, 246-255) */
int32_t zk_decoder_decompress_with_prefix(zk_decoder* d, uint8_t* buf, size_t len, const uint8_t* prefix,
                                          size_t prefix_len, size_t* produced);            /* :201-270 */
/* the same with entry e decoded against prefix[ranges[2e] .. ranges[2e+1]) (ranges: two per seek-table entry, as zk_decompress_frames_prefixes
 * takes them): a seekable patch read with its slices; each window of frames uploads only the hull of its own entries' ranges */
int32_t zk_decoder_decompress_with_prefix_ranges(zk_decoder* d, uint8_t* buf, size_t len, const uint8_t* prefix, size_t prefix_len,
                                                 const uint64_t* ranges, size_t* produced);
/* the same with the prefix being the decoded content of the reference archive R (zk_decompress_frames_prefixes_archive's arguments): each
 * window of frames decodes only the entries of R under its own entries' ranges */
int32_t zk_decoder_decompress_with_reference_archive(zk_decoder* d, uint8_t* buf, size_t len, const uint8_t* ref_comp, size_t ref_len,
                                                     const uint64_t* ref_c_off, const uint64_t* ref_d_off, uint32_t ref_n,
                                                     const uint64_t* ranges, size_t* produced);
/* the same with the prefix being OLD of a reference chain (zk_decompress_frames_prefixes_chain's arguments).  The decoder keeps a copy of
 * the depth descriptors: a call whose chain differs from the previous call's at any level decodes its window again */
int32_t zk_decoder_decompress_with_reference_chain(zk_decoder* d, uint8_t* buf, size_t len, const zk_reference_archive* chain, uint32_t depth,
                                                   const uint64_t* ranges, size_t* produced);
void zk_decoder_reset(zk_decoder* d);                                                    /* :346-350 */
int32_t zk_decoder_set_lower_frame(zk_decoder* d, uint32_t index, uint64_t* offset);    /* :367 */
int32_t zk_decoder_set_upper_frame(zk_decoder* d, uint32_t index, uint64_t* offset);    /* :383 */
int32_t zk_decoder_set_offset(zk_decoder* d, uint64_t offset);                           /* :402-414 */
int32_t zk_decoder_set_offset_limit(zk_decoder* d, uint64_t limit);                      /* :432-437 */
uint64_t zk_decoder_read_compressed(const zk_decoder* d);                                /* :448 */
uint64_t zk_decoder_offset(const zk_decoder* d);                                         /* :458 */
uint64_t zk_decoder_offset_limit(const zk_decoder* d);                                   /* :463 */
const zk_seek_table* zk_decoder_seek_table(const zk_decoder* d);                        /* :453 */
/* impl Seek for Decoder (decode.rs:545-579): whence 0 = Start, 1 = End, 2 = Current */
int32_t zk_decoder_seek(zk_decoder* d, int32_t whence, int64_t offset, uint64_t* new_offset);

#ifdef __cplusplus
}
#endif
#endif /* ZEEKSTD_B200_H */
