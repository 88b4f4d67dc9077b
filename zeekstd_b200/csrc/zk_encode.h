// zk_encode.h -- host-visible interface of the batched compress path (zk_encode.cu).
#pragma once
#include "zk_common.cuh"

struct ZkEncodeWs {                    // HBM scratch owned by a zk_ctx slot, grown on demand
    void* buf = nullptr; size_t cap = 0;
    void* cut = nullptr; size_t cut_cap = 0;              // content-defined cut (zk_encode_cdc): kept apart from buf, which the frames of a cut then use
    uint32_t* h_sizes = nullptr; size_t cap_frames = 0;   // pinned: per-frame compressed sizes
    int sm_count = 0;
    unsigned long long launches = 0;
    uint32_t pending_frames = 0;
    bool attr_set = false, attr_set_wide = false, attr_set_walk = false, attr_set_hc = false, attr_set_cdc = false;
    const uint8_t* prefix = nullptr; uint32_t prefix_len = 0;   // device pointer: raw-content prefix for the NEXT enqueue (one-shot)
    bool ldm = false;                 // long-distance matching against that prefix for the NEXT enqueue (one-shot; nothing without a prefix)
    int prio = 0;                     // CUDA stream priority of the side stream (matches the slot's stream)
    bool no_side = false;             // host pipelines: concurrency comes from the other sub-batches; every extra stream costs a hardware queue
    cudaStream_t side = nullptr; cudaEvent_t ev_a = nullptr, ev_b = nullptr, ev_c = nullptr;   // K-C2s runs beside K-C2l
    ZkProf prof;
};

// Compress n bytes at d_src into ceil(n/frame_size) frames written back to back at d_dst.
// c_sizes (host, n_frames entries) receives each frame's compressed size.  Synchronous on `stream`.
int zk_encode_batch(ZkEncodeWs* ws, cudaStream_t stream, const uint8_t* d_src, size_t n, uint32_t frame_size, int level,
                    int checksum, uint8_t* d_dst, size_t dst_cap, uint32_t* c_sizes, uint32_t n_frames, size_t* dst_len);
int zk_encode_enqueue(ZkEncodeWs* ws, cudaStream_t stream, const uint8_t* d_src, size_t n, uint32_t frame_size, int level,
                      int checksum, uint8_t* d_dst, size_t dst_cap, uint32_t n_frames);
// The same with caller-chosen frame sizes: frame f covers frame_sizes[f] bytes (each <= 1 GiB; 0: an empty frame) of d_src, back to back
int zk_encode_enqueue_sized(ZkEncodeWs* ws, cudaStream_t stream, const uint8_t* d_src, const uint32_t* frame_sizes, uint32_t n_frames,
                            int level, int checksum, uint8_t* d_dst, size_t dst_cap);
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
    const uint32_t* starts = nullptr;    // n_frames + 1 first blocks (32 KiB units from d_src); the last one is the end of the last frame
};
int zk_encode_csize(ZkEncodeWs* ws, cudaStream_t stream, const uint8_t* d_src, size_t n, uint32_t target, int level, int checksum,
                    int final_, int at_end, const uint8_t* d_prefix, uint32_t prefix_len, uint8_t* d_dst, size_t dst_cap, ZkCsizeOut* out);

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
