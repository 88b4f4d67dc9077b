// zk_ctx.h -- the context behind the C ABI's opaque zk_ctx (include/zeekstd_b200.h).
// Owns the CUDA streams, events, pinned/HBM staging and the per-slot codec workspaces.
#pragma once
#include "zk_decode.h"
#include "zk_encode.h"
#include "../../include/zeekstd_b200.h"

#define ZK_SLOTS 8                        // pipeline depth of the host<->device paths (H2D | kernels | D2H overlap)

struct ZkSlot {
    cudaStream_t stream = nullptr;
    ZkDecodeWs dws;
    ZkEncodeWs ews;
    uint8_t* d_in = nullptr; size_t cap_in = 0;      // device staging for the host-pointer entry points
    uint8_t* d_out = nullptr; size_t cap_out = 0;
};

struct zk_ctx {
    int device = 0;
    int sm_count = 132;
    ZkSlot slot[ZK_SLOTS];
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join[ZK_SLOTS] = {};    // device-pointer calls: the slot streams start after, and the caller's stream
                                                          // continues after, the work of the caller's stream
    void* d_chain = nullptr; size_t cap_chain = 0;        // device-pointer compress: the output offset of every sub-batch (ZkEncodeParams::chain)
    cudaStream_t up = nullptr, down = nullptr;            // dedicated copy streams of the host-pointer decompress pipeline
    float last_ms = 0.f;
    void* d_prefix = nullptr; size_t cap_prefix = 0;      // device copy of the raw-content prefix of the calls that take one
    unsigned long long prefix_uploaded = 0;               // prefix bytes copied to the device so far (zk_ctx_prefix_bytes_uploaded)
    unsigned long long ref_decoded = 0;                   // reference-archive entries decoded so far (zk_ctx_reference_entries_decoded)
    void* d_level[ZK_CHAIN_MAX_DEPTH - 1] = {};           // a reference chain's arenas below its head (level i's decoded content; the
    size_t cap_level[ZK_CHAIN_MAX_DEPTH - 1] = {};        // head's is d_prefix)
    void* d_reuse[4] = {}; size_t cap_reuse[4] = {};      // zk_compress_frames_sized_reuse: old entries, their decoded bytes, the changed
                                                          // frames, the assembled output
    unsigned long long launches() const {
        unsigned long long n = 0;
        for (int i = 0; i < ZK_SLOTS; i++) n += slot[i].dws.launches + slot[i].ews.launches;
        return n;
    }
};

int zk_slot_ensure(ZkSlot* s, size_t need_in, size_t need_out);
