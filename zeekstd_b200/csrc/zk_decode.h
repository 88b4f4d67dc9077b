// zk_decode.h -- host-visible interface of the batched decode path (zk_decode.cu).
#pragma once
#include "zk_common.cuh"
#include <string.h>

struct ZkDecodeArgs {                 // kernel parameter block (by value)
    const uint8_t* comp;              // compressed bytes; entry e occupies [c_off[e], c_off[e+1])
    const unsigned long long* c_off;  // device, n_entries + 1
    const unsigned long long* d_off;  // device, n_entries + 1; entry e decodes to dst + d_off[e]
    uint8_t* dst;
    uint32_t n_entries;
    ZkBlock* blocks; ZkEntry* entries; ZkCounters* counters; uint32_t* work_counter;
    uint8_t* lit; uint32_t* seq_lit_end; uint32_t* seq_out_end; uint32_t* seq_off;
    uint32_t* huf_list; uint32_t* seq_list;   // compacted indices of blocks with Huffman literals / with sequences; seq_list has
                                              // 2 x cap_blocks entries: the second half lists the blocks zk_seq2_kernel passes to
                                              // zk_seq2_full_kernel
    uint32_t* seg_list;                       // compacted indices of the first blocks of execution segments (long ones from the
                                              // front, short ones from the back: together never more than cap_blocks)
    uint32_t exec_short;                      // segments of at most this many output bytes run on one warp each; 0 = none
    unsigned long long cap_blocks, cap_lit, cap_seq;
    const uint8_t* prefix;            // the buffer of the raw-content prefixes of the zstd frames (Decoder::decompress_with_prefix, decode.rs:211-214, 246-255); device pointer or nullptr
    const uint32_t* pranges;          // device, two per entry: every zstd frame of entry e has the prefix prefix[pranges[2e], pranges[2e + 1])
    const uint32_t* d_need;           // per entry: only this many leading bytes are wanted (range reads); nullptr = everything
    uint32_t* seg_key;                // beside seg_list, same positions: the segment's cost, ZK_ORD_ALPHA x sequences + output bytes
};

struct ZkDecodeWs {                   // HBM scratch owned by a zk_ctx, grown on demand, reused across batches
    ZkBlock* blocks = nullptr; size_t cap_blocks = 0;
    ZkEntry* entries = nullptr; size_t cap_entries = 0;
    ZkCounters* counters = nullptr;
    uint8_t* lit = nullptr; size_t cap_lit = 0;
    uint32_t* seq_lit_end = nullptr; uint32_t* seq_out_end = nullptr; uint32_t* seq_off = nullptr; size_t cap_seq = 0;
    uint64_t* c_off = nullptr; uint64_t* d_off = nullptr;
    uint32_t* d_need = nullptr; uint32_t* h_need = nullptr;
    uint32_t* d_pr = nullptr; uint32_t* h_pr = nullptr;     // prefix mode: the entries' prefix ranges (ZkDecodeArgs::pranges)
    uint32_t* huf_list = nullptr; uint32_t* seq_list = nullptr; uint32_t* seg_list = nullptr;
    uint32_t* ord_list = nullptr;     // the three work lists ordered by cost (seq 2 x cap_blocks, huf, seg), read by their consumers
    uint32_t* seg_key = nullptr;
    uint32_t order = 1;               // ZK_DEC_ORDER: 1 = run every work list heaviest first (zk_order_kernel), 0 = in the order it was filled
    bool attr_set = false; uint32_t ring_override = 0;
    uint32_t exec_warps = 0;          // ZK_EXEC_WARPS: warps per K-D2 CTA (at most 16); 0 = chosen from the entries per SM
    uint32_t seq2_ctas = 0;           // ZK_SEQ2_CTAS: persistent K-D1s CTAs per SM; 0 = seq2_fit
    uint32_t seq2_fit = 0;            // K-D1s CTAs in three quarters of an SM's shared memory (queried at the first launch; DESIGN §6)
    uint32_t exec_short = 128 << 10;  // ZK_EXEC_SHORT: output bytes up to which a segment runs on one warp (zk_exec_warp_kernel); 0 = CTAs only
    uint32_t huf_pad = 0;             // extra dynamic smem per Huffman CTA: fewer resident CTAs -> more L1 for the streams (tuning)
    int prio = 0;                     // CUDA stream priority of the side stream (matches the slot's stream)
    uint32_t huf_ctas = 0;            // persistent K-D1h CTAs per SM (tuning: ZK_HUF_CTAS); 0: half of huf_fit
    uint32_t huf_fit = 0;             // K-D1h CTAs that fit on an SM (occupancy query at the first launch; 0 = not asked yet)
    cudaEvent_t ev_up = nullptr, ev_done = nullptr, ev_down = nullptr;
    cudaStream_t side = nullptr; cudaEvent_t ev_scan = nullptr, ev_huf = nullptr;   // Huffman kernel runs beside the FSE kernel
    ZkEntry* h_entries = nullptr; ZkCounters* h_counters = nullptr; uint64_t* h_off = nullptr;   // pinned
    size_t want_blocks = 0, want_lit = 0, want_seq = 0;   // exact needs reported by a batch that overflowed
    uint32_t pending_n = 0;
    int sm_count = 0;
    unsigned long long launches = 0;  // kernels launched so far (bench.py's gpu_launches)
    unsigned long long segments = 0;  // execution segments run so far (zk_ctx_decode_segments)
    ZkProf prof;
};

// What a call asks of every batch it enqueues
struct ZkDecodeParams {
    const uint8_t* prefix = nullptr; uint32_t prefix_len = 0;   // device memory: the prefix buffer of the zstd frames (nullptr: none)
    const uint32_t* ranges = nullptr; // host, two per entry: the prefix of entry e's frames is prefix[ranges[2e], ranges[2e + 1]); nullptr: all of it
    const uint32_t* need = nullptr;   // host, one per entry: leading bytes wanted (ZkDecodeArgs::d_need); nullptr = everything
    int share = 1;                    // how many batches share the GPU concurrently (host pipeline depth)
    bool side = true;                 // K-D1h on the side stream; host pipelines get their concurrency from the other sub-batches instead,
                                      // and every extra stream costs a hardware queue
    cudaStream_t up = nullptr, down = nullptr;      // host pipelines: dedicated upload / download streams (not owned); nullptr = everything on `stream`
};

// Decode n seek-table entries.  d_comp / d_dst are device pointers (16-byte aligned, 16 readable bytes of
// padding after the last byte); c_off / d_off are HOST arrays of n+1 cumulative offsets relative to those
// pointers (seek_table.rs:97-101).  status_out[n] (host, optional) receives 0 or -(zstd code) per entry.
// Returns 0, or the first non-zero entry status, or -(code) for a launch/allocation failure.
// Synchronous with respect to `stream` on return.
int zk_decode_batch(ZkDecodeWs* ws, cudaStream_t stream, const uint8_t* d_comp, const uint64_t* c_off, const uint64_t* d_off,
                    uint32_t n, uint8_t* d_dst, int verify_checksum, const ZkDecodeParams& p, int32_t* status_out);
int zk_decode_enqueue(ZkDecodeWs* ws, cudaStream_t stream, const uint8_t* d_comp, const uint64_t* c_off, const uint64_t* d_off,
                      uint32_t n, uint8_t* d_dst, int verify_checksum, const ZkDecodeParams& p);
int zk_decode_collect(ZkDecodeWs* ws, cudaStream_t stream, const ZkDecodeParams& p, int32_t* status_out);
void zk_decode_ws_free(ZkDecodeWs* ws);
