// zk_encode.h -- host-visible interface of the batched compress path (zk_encode.cu).
#pragma once
#include "zk_common.cuh"
#include <vector>

struct ZkEncodeWs {                    // HBM scratch owned by a zk_ctx slot, grown on demand
    void* buf = nullptr; size_t cap = 0;
    void* cut = nullptr; size_t cut_cap = 0;              // content-defined cut (zk_encode_cdc): kept apart from buf, which the frames of a cut then use
    void* reuse = nullptr; size_t reuse_cap = 0;          // span tables and results of zk_reuse_run
    void* patch = nullptr; size_t patch_cap = 0;          // anchors and anchor tables of zk_patch_anchors / zk_patch_join
    uint32_t* h_sizes = nullptr; size_t cap_frames = 0;   // pinned: per-frame compressed sizes
    int sm_count = 0;
    unsigned long long launches = 0;
    uint32_t pending_frames = 0;
    bool attr_set = false, attr_set_wide = false, attr_set_walk = false, attr_set_hc = false, attr_set_cdc = false;
    int prio = 0;                     // CUDA stream priority of the side stream (matches the slot's stream)
    cudaStream_t side = nullptr; cudaEvent_t ev_a = nullptr, ev_b = nullptr, ev_c = nullptr;   // K-C2s runs beside K-C2l
    cudaEvent_t ev_chain = nullptr;   // recorded after the last batch's frame scan when it had a chain (ZkEncodeParams::chain)
    ZkProf prof;
};

// What a call asks of every batch it enqueues
struct ZkEncodeParams {
    int level = 0, checksum = 0;
    const uint8_t* prefix = nullptr; uint32_t prefix_len = 0;   // device memory: the prefix buffer the frames' prefixes lie in (nullptr: none)
    const uint32_t* ranges = nullptr; // host, two per frame of the batch: frame f's prefix is prefix[ranges[2f], ranges[2f + 1]); nullptr: the
                                      // whole buffer for every frame
    bool ldm = false;                 // long-distance matching against the whole of each frame's prefix (nothing without one)
    bool long_mode = false;           // long mode: every frame also matches its own bytes up to 2^27 back (and the prefix as ldm does)
    // batches that write one output one after another, each enqueued before the one before it completed: chain[0] (device) holds the
    // bytes before the batch's frames, which it writes from d_dst + chain[0] on, and its frame scan writes chain[1] after waiting for
    // chain_wait (that of the batch before: its ZkEncodeWs::ev_chain; nullptr: none).  dst_cap bounds the whole output
    unsigned long long* chain = nullptr;
    cudaEvent_t chain_wait = nullptr;
};

// The frames of a batch: the caller's sizes (each <= 1 GiB; 0: an empty frame), or the uniform layout of n bytes (frame_size bytes each, the
// last frame shorter, one empty frame of no input).  n is the bytes they cover.
struct ZkFrames {
    const uint32_t* sizes;            // nullptr: uniform
    size_t n; uint32_t frame_size, count;
    uint32_t size(uint32_t f) const {
        if (sizes) return sizes[f];
        const size_t lo = (size_t)f * frame_size;
        return (uint32_t)(n - lo < frame_size ? n - lo : frame_size);
    }
    // the sub-batch from frame f0: as many frames as fit max_bytes of input, at least one -> its end frame; *bytes: its input
    uint32_t next_sub(uint32_t f0, size_t max_bytes, size_t* bytes) const {
        size_t b = size(f0); uint32_t e = f0 + 1;
        if (!sizes) {                 // frames before the last are full: the same rule in closed form
            const uint32_t per = frame_size <= max_bytes ? (uint32_t)(max_bytes / frame_size) : 1u;
            e = count - f0 < per ? count : f0 + per;
            b = (e == count ? n : (size_t)e * frame_size) - (size_t)f0 * frame_size;
            if (e < count && b + size(e) <= max_bytes) { b += size(e); e++; }   // a short last frame that still fits
        } else while (e < count && b + sizes[e] <= max_bytes) b += sizes[e++];
        *bytes = b;
        return e;
    }
    // frames [f0, f0 + cnt), which cover `bytes`
    ZkFrames sub(uint32_t f0, uint32_t cnt, size_t bytes) const { return {sizes ? sizes + f0 : nullptr, bytes, frame_size, cnt}; }
    size_t bound() const;             // the most bytes they compress to
};

// Enqueue the compression of `fr`, read back to back from d_src, into frames written back to back at d_dst.  zk_encode_collect then waits
// for it: c_sizes (host, one entry per frame) receives each frame's compressed size, *dst_len the bytes written.
int zk_encode_enqueue(ZkEncodeWs* ws, cudaStream_t stream, const uint8_t* d_src, const ZkFrames& fr, const ZkEncodeParams& p, uint8_t* d_dst,
                      size_t dst_cap);
int zk_encode_collect(ZkEncodeWs* ws, cudaStream_t stream, uint32_t* c_sizes, size_t* dst_len);
void zk_encode_ws_free(ZkEncodeWs* ws);
size_t zk_encode_bound(size_t n, uint32_t frame_size);
size_t zk_encode_bound_sized(const uint32_t* frame_sizes, uint32_t n_frames);

// FrameSizePolicy::Compressed(target) over one pass of n <= 1 GiB bytes at d_src: frames close after the first 32 KiB block at which
// header + blocks >= target, or at 1 GiB of input.  at_end: the pass ends the caller's input; final_: and no more input follows, so
// the rest becomes the last frame (otherwise a frame that would end at the end of the input stays open).  Frames are written back to
// back at d_dst.  The arrays in *out live in the workspace's pinned buffer until the next call.  Synchronous on `stream`.
struct ZkCsizeOut {
    uint32_t n_frames = 0;
    size_t consumed = 0, total = 0;      // input bytes the frames cover; bytes written
    const uint32_t* c_sizes = nullptr;   // n_frames compressed sizes
    const uint32_t* d_sizes = nullptr;   // n_frames input sizes
};
int zk_encode_csize(ZkEncodeWs* ws, cudaStream_t stream, const uint8_t* d_src, size_t n, uint32_t target, const ZkEncodeParams& p, int final_,
                    int at_end, uint8_t* d_dst, size_t dst_cap, ZkCsizeOut* out);

// FrameSizePolicy::ContentDefined(size): size clamped to [4096, 2^30]; frames of mn .. mx bytes end at the first position whose 64-byte gear
// hash is >= thr (zk_cdc.inc states the rule)
struct ZkCdcRule { uint32_t mn, mx; unsigned long long thr; };
ZkCdcRule zk_cdc_rule(uint32_t size);
// The cut only, over one pass of n <= 1 GiB bytes at d_src that starts a frame (at_end / final_ as for zk_encode_csize).  cap: candidate
// positions kept (0: n / 64 + 1); fewer only shortens what one pass covers.  *out->sizes lives in the workspace's pinned buffer until the
// next call.  Synchronous on `stream`.
struct ZkCdcOut {
    uint32_t n_frames = 0;
    size_t consumed = 0;                 // input bytes the frames cover
    const uint32_t* sizes = nullptr;     // n_frames frame sizes
};
int zk_encode_cdc(ZkEncodeWs* ws, cudaStream_t stream, const uint8_t* d_src, size_t n, uint32_t size, int final_, int at_end, uint32_t cap,
                  ZkCdcOut* out);

// zk_compress_frames_sized_reuse (zk_reuse.inc): one launch over n spans, each split into 32 KiB work items.  Span s covers
// a_buf[a, a + len) and b_buf[b, b + len) (device buffers with 16 readable bytes after their last span; spans start at any byte).
//   ZK_REUSE_KEYS     out (host, n words): the key of the a side, XXH64 of the little-endian XXH64s of its consecutive 32 KiB chunks
//   ZK_REUSE_COMPARE  out (host, n u32): non-zero iff the a side equals the b side
//   ZK_REUSE_COPY     the a side to the b side (the two must not overlap); out unused
// Synchronous on `stream`.
enum ZkReuseOp { ZK_REUSE_KEYS, ZK_REUSE_COMPARE, ZK_REUSE_COPY };
struct ZkReuseSpan { unsigned long long a, b; uint32_t len; };
int zk_reuse_run(ZkEncodeWs* ws, cudaStream_t stream, ZkReuseOp op, const uint8_t* a_buf, uint8_t* b_buf, const ZkReuseSpan* spans, uint32_t n,
                 void* out);

// Seekable patches (zk_patch.inc states the rule).  An anchor is a position p >= 63 whose 64-byte gear hash h_p is >= ZK_PATCH_THR, about one
// per 64 KiB; its key is h_p.
#define ZK_PATCH_THR (0ull - ~0ull / 65536ull)
// The anchors of one piece of n <= 1 GiB bytes at d_src (16 readable bytes after it), at positions 63 .. n - 1 of the piece, appended in
// position order to *keys / *pos (positions plus base).  Synchronous on `stream`.
int zk_patch_anchors(ZkEncodeWs* ws, cudaStream_t stream, const uint8_t* d_src, size_t n, unsigned long long base,
                     std::vector<unsigned long long>* keys, std::vector<unsigned long long>* pos);
// The anchors of OLD and NEW (each in position order) and NEW's frames: frame f covers NEW [fa[f], fa[f + 1]) and holds NEW's anchors
// [fanc[f], fanc[f + 1])
struct ZkPatchTables {
    std::vector<unsigned long long> okeys, opos, nkeys, npos, fa;
    std::vector<uint32_t> fanc;
};
// OLD's anchors sorted by (key, position) on the device, then frame f's range of OLD -> ranges[2f], ranges[2f + 1] (host).  Synchronous.
int zk_patch_join(ZkEncodeWs* ws, cudaStream_t stream, const ZkPatchTables& t, uint32_t n_frames, unsigned long long old_len,
                  unsigned long long margin, unsigned long long* ranges);
