// zk_api.cu -- the batch half of the C ABI (include/zeekstd_b200.h): context + zk_{de,}compress_frames[_dev].
// The API-mirror half (SeekTable / RawEncoder / Encoder / Decoder) lives in zk_host.cpp and is built on
// top of these entry points only.
#include "zk_ctx.h"
#include "../../include/zeekstd_b200.h"
#include <stdio.h>
#include <time.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

static thread_local char zk_tls_cuda_msg[256] = "";
void zk_note_cuda_error(const char* what, int code) {
    snprintf(zk_tls_cuda_msg, sizeof zk_tls_cuda_msg, "%s: %s", what, cudaGetErrorString((cudaError_t)code));
}
extern "C" const char* zk_last_cuda_error(void) { return zk_tls_cuda_msg; }

static int zk_host_slots(bool enc);
static size_t zk_env_size(const char* name, size_t dflt) {
    const char* s = getenv(name);
    if (!s || !*s) return dflt;
    return (size_t)strtoull(s, nullptr, 10);
}

// sub-batches in flight of the host-pointer pipelines (tuning knobs, swept by tools/e2e_sweep4.sh): decompress wants many
// (its exec stage is latency-bound per frame), compress few (its kernels fill the machine from one 128 MiB sub-batch)
static int zk_host_slots(bool enc) {
    size_t v = zk_env_size(enc ? "ZK_HOST_SLOTS_ENC" : "ZK_HOST_SLOTS", enc ? 4 : 8);
    return (int)(v < 1 ? 1 : (v > ZK_SLOTS ? ZK_SLOTS : v));
}

extern "C" const char* zk_version(void) {
#ifdef ZK_EMUL
    return "zeekstd_b200 0.1 (ZK_EMUL test build: device code interpreted on the CPU; not a product build)";
#else
    return "zeekstd_b200 0.1 (sm_90a)";
#endif
}

extern "C" const char* zk_error_name(int32_t rc) {
    switch (rc) {
    case 0: return "No error detected";
    case ZK_ERR_NUMBER_CONVERSION: return "number conversion failed";
    case ZK_ERR_OFFSET_OUT_OF_RANGE: return "offset out of range";
    case ZK_ERR_FRAME_INDEX_TOO_LARGE: return "frame index too large";
    case ZK_ERR_IO: return "io error";
    case ZK_ERR_NO_DEVICE: return "no usable CUDA device (zeekstd_b200 has no CPU fallback)";
    case ZK_ERR_INVALID_ARG: return "invalid argument";
    case ZK_ERR_CUDA: return "CUDA runtime or kernel failure (see zk_last_cuda_error)";
    // strings of ZSTD_getErrorName for the codes this codec can raise
    case -1: return "Error (generic)";
    case -10: return "Unknown frame descriptor";
    case -12: return "Version not supported";
    case -14: return "Unsupported frame parameter";
    case -16: return "Frame requires too much memory for decoding";
    case -20: return "Data corruption detected";
    case -22: return "Restored data doesn't match checksum";
    case -30: return "Dictionary is corrupted";
    case -32: return "Dictionary mismatch";
    case -42: return "Parameter is out of bound";
    case -64: return "Allocation error : not enough memory";
    case -70: return "Destination buffer is too small";
    case -72: return "Src size is incorrect";
    default: return "Unspecified error code";
    }
}

int zk_slot_ensure(ZkSlot* s, size_t need_in, size_t need_out) {
    const int rc = zk_grow((void**)&s->d_in, &s->cap_in, need_in, 1);
    return rc ? rc : zk_grow((void**)&s->d_out, &s->cap_out, need_out, 1);
}

extern "C" int32_t zk_ctx_create(int32_t device_ordinal, uint32_t flags, zk_ctx** out) {
    (void)flags;
    if (!out) return ZK_ERR_INVALID_ARG;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { (void)cudaGetLastError(); return ZK_ERR_NO_DEVICE; }
    if (device_ordinal < 0 || device_ordinal >= ndev) return ZK_ERR_INVALID_ARG;
    ZK_CUDA_OK(cudaSetDevice(device_ordinal));
    cudaDeviceProp prop;
    ZK_CUDA_OK(cudaGetDeviceProperties(&prop, device_ordinal));
    zk_ctx* c = new zk_ctx();
    c->device = device_ordinal;
    c->sm_count = prop.multiProcessorCount > 0 ? prop.multiProcessorCount : 132;
    // ZK_HOST_PRIO (default 1): slot i runs at stream priority (greatest + i): concurrent sub-batches of the host pipelines then
    // complete staggered (oldest slot first) instead of all at once, which keeps the D2H engine busy from early on
    int least = 0, greatest = 0;
    const bool use_prio = zk_env_size("ZK_HOST_PRIO", 1) != 0;
    if (use_prio) cudaDeviceGetStreamPriorityRange(&least, &greatest);
    for (int i = 0; i < ZK_SLOTS; i++) {
        const int prio = use_prio ? (greatest + i < least ? greatest + i : least) : 0;
        if (cudaStreamCreateWithPriority(&c->slot[i].stream, cudaStreamNonBlocking, prio) != cudaSuccess) { delete c; return ZK_ERR_NO_DEVICE; }
        c->slot[i].dws.prio = c->slot[i].ews.prio = prio;
        c->slot[i].dws.sm_count = c->sm_count;
        c->slot[i].dws.ring_override = (uint32_t)zk_env_size("ZK_RING_BYTES", 0);   // tuning / tests: power of two >= 1024
        c->slot[i].dws.exec_warps = (uint32_t)zk_env_size("ZK_EXEC_WARPS", 0);
        c->slot[i].dws.huf_pad = (uint32_t)zk_env_size("ZK_HUF_PAD", 0);
        c->slot[i].dws.exec_short = (uint32_t)zk_env_size("ZK_EXEC_SHORT", 128 << 10);
        c->slot[i].dws.seq2_ctas = (uint32_t)zk_env_size("ZK_SEQ2_CTAS", 0);
        c->slot[i].dws.huf_ctas = (uint32_t)zk_env_size("ZK_HUF_CTAS", 0);
        c->slot[i].ews.sm_count = c->sm_count;
    }
    cudaEventCreate(&c->ev0); cudaEventCreate(&c->ev1);
    if (zk_env_size("ZK_HOST_COPY_STREAMS", 1) != 0) {
        cudaStreamCreateWithFlags(&c->up, cudaStreamNonBlocking); cudaStreamCreateWithFlags(&c->down, cudaStreamNonBlocking);
    }
    *out = c;
    return 0;
}

extern "C" void zk_ctx_destroy(zk_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    for (int i = 0; i < ZK_SLOTS; i++) {
        ZkSlot& s = c->slot[i];
        if (s.stream) cudaStreamSynchronize(s.stream);
        zk_decode_ws_free(&s.dws);
        zk_encode_ws_free(&s.ews);
        if (s.d_in) cudaFree(s.d_in);
        if (s.d_out) cudaFree(s.d_out);
        if (s.stream) cudaStreamDestroy(s.stream);
    }
    if (c->up) cudaStreamDestroy(c->up);
    if (c->down) cudaStreamDestroy(c->down);
    if (c->d_prefix) cudaFree(c->d_prefix);
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    delete c;
}

extern "C" uint64_t zk_ctx_kernel_launches(const zk_ctx* c) { return c ? c->launches() : 0; }
extern "C" uint64_t zk_ctx_decode_segments(const zk_ctx* c) {
    unsigned long long n = 0;
    for (int i = 0; c && i < ZK_SLOTS; i++) n += c->slot[i].dws.segments;
    return n;
}
extern "C" float zk_ctx_last_device_ms(const zk_ctx* c) { return c ? c->last_ms : 0.f; }
extern "C" size_t zk_compress_bound(size_t n, uint32_t frame_size) { return zk_encode_bound(n, frame_size); }

extern "C" void zk_ctx_profile(zk_ctx* c, int32_t enable) {
    if (!c) return;
    for (int i = 0; i < ZK_SLOTS; i++) {
        c->slot[i].dws.prof.enabled = enable != 0; c->slot[i].ews.prof.enabled = enable != 0;
        for (int k = 0; k < ZK_PROF_SLOTS; k++) { c->slot[i].dws.prof.ms[k] = c->slot[i].ews.prof.ms[k] = 0.f; c->slot[i].dws.prof.count[k] = c->slot[i].ews.prof.count[k] = 0; }
    }
}
extern "C" void zk_ctx_profile_read(const zk_ctx* c, float* ms, uint32_t* launches) {
    for (int k = 0; k < ZK_PROF_SLOTS; k++) {
        float t = 0.f; uint32_t n = 0;
        for (int i = 0; c && i < ZK_SLOTS; i++) { t += c->slot[i].dws.prof.ms[k] + c->slot[i].ews.prof.ms[k]; n += c->slot[i].dws.prof.count[k] + c->slot[i].ews.prof.count[k]; }
        if (ms) ms[k] = t;
        if (launches) launches[k] = n;
    }
}


// ---------------------------------------------------------------------------------------------
// prefix / patch mode (SURVEY.md 8f.3): every frame is coded against the same raw-content prefix
//   RawEncoder::compress_with_prefix   encode.rs:311-338  (cctx.ref_prefix at the start of every frame)
//   Decoder::decompress_with_prefix    decode.rs:201-214, 246-255  (dctx.ref_prefix before the first frame and after every frame end)
// The prefix is uploaded once per call and stays resident; K-C1 searches its tail from the first block of every frame, K-D2
// resolves offsets that reach before a frame's first byte into it.
// ---------------------------------------------------------------------------------------------
// the prefix of one call (host memory; nullptr or len 0: none) -> its device copy *d_prefix, *d_len (nullptr, 0: none)
static int32_t zk_upload_prefix(zk_ctx* c, const uint8_t* prefix, size_t len, const uint8_t** d_prefix, uint32_t* d_len) {
    *d_prefix = nullptr; *d_len = 0;
    if (!prefix || len == 0) return 0;
    if (len > 0x7FFFFFFFull) return ZK_ERR_INVALID_ARG;
    ZK_CUDA_OK(cudaSetDevice(c->device));
    const int32_t rc = zk_grow(&c->d_prefix, &c->cap_prefix, len + 64, 1);
    if (rc) return rc;
    for (int i = 0; i < ZK_SLOTS; i++) if (c->slot[i].stream) cudaStreamSynchronize(c->slot[i].stream);    // nobody reads the old prefix any more
    ZK_CUDA_OK(cudaMemcpy(c->d_prefix, prefix, len, cudaMemcpyHostToDevice));
    *d_prefix = (const uint8_t*)c->d_prefix; *d_len = (uint32_t)len;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// decompress
// ---------------------------------------------------------------------------------------------
// split [0,n) into sub-batches bounded by output bytes so scratch stays proportional to the sub-batch
static uint32_t zk_next_sub(const uint64_t* d_off, uint32_t first, uint32_t n, size_t max_bytes, uint32_t max_entries) {
    uint32_t e = first + 1;
    while (e < n && e - first < max_entries && d_off[e + 1] - d_off[first] <= max_bytes) e++;
    return e;
}

extern "C" int32_t zk_decompress_frames_dev(zk_ctx* c, const void* d_comp, const uint64_t* c_off, const uint64_t* d_off,
                                            uint32_t n, void* d_dst, int32_t verify, int32_t* status, void* cuda_stream) {
    if (!c || (n && (!d_comp || !c_off || !d_off || !d_dst))) return ZK_ERR_INVALID_ARG;
    if (n == 0) return 0;
    ZK_CUDA_OK(cudaSetDevice(c->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : c->slot[0].stream;
    const size_t sub_bytes = zk_env_size("ZK_DEV_SUB_BYTES", (size_t)1 << 30);
    ZkDecodeParams p;                                       // device-resident data: nothing to copy but offsets and statuses
    p.side = zk_env_size("ZK_DEV_SIDE", 1) != 0;
    cudaEventRecord(c->ev0, st);
    int32_t worst = 0;
    for (uint32_t first = 0; first < n;) {
        uint32_t end = zk_next_sub(d_off, first, n, sub_bytes, 1u << 20);
        int rc = zk_decode_batch(&c->slot[0].dws, st, (const uint8_t*)d_comp, c_off + first, d_off + first, end - first, (uint8_t*)d_dst,
                                 verify, p, status ? status + first : nullptr);
        if (rc && !worst) worst = rc;
        if (rc == ZK_INT_CUDA || rc == -(int)ZKZ_MEMORY_ALLOCATION) return rc;
        first = end;
    }
    cudaEventRecord(c->ev1, st);
    cudaEventSynchronize(c->ev1);
    cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1);
    return worst;
}

// ZK_E2E_TRACE=1: per-sub-batch timeline of the host-pointer paths (CUDA events on the slot streams), printed to stderr.
struct ZkTrace {
    bool on = false; cudaEvent_t t0 = nullptr; std::vector<cudaEvent_t> ev; std::vector<int> tag; std::vector<double> host; double h0 = 0;
    static double now() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; }
    void begin(cudaStream_t st) {
        on = getenv("ZK_E2E_TRACE") != nullptr; if (!on) return;
        cudaEventCreate(&t0); cudaEventRecord(t0, st); h0 = now();
    }
    void mark(cudaStream_t st, int sub, int what) {
        if (!on) return;
        cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, st); ev.push_back(e); tag.push_back(sub * 8 + what); host.push_back(now() - h0);
    }
    void end(const char* name) {
        if (!on) return;
        cudaDeviceSynchronize();
        static const char* W[] = {"h2d0", "h2d1", "kern1", "d2h0", "d2h1"};
        for (size_t i = 0; i < ev.size(); i++) {
            float ms = 0; cudaEventElapsedTime(&ms, t0, ev[i]);
            fprintf(stderr, "%s sub %d %s gpu %.3f host %.3f\n", name, tag[i] >> 3, W[tag[i] & 7], ms, host[i]);
            cudaEventDestroy(ev[i]);
        }
        cudaEventDestroy(t0);
    }
};

// one host-pointer decompress call
struct ZkDecCall {
    const uint8_t* comp; const uint64_t* c_off; const uint64_t* d_off; uint8_t* dst; int verify; int32_t* status;
    ZkDecodeParams p;                                       // p.need: the whole call's
};
struct ZkSubDec { uint32_t first = 0, count = 0; std::vector<uint64_t> c_rel, d_rel; bool busy = false; };

static int zk_dec_sub_enqueue(zk_ctx* c, int si, ZkSubDec& sb, const ZkDecCall& q, ZkTrace* tr = nullptr, int k = 0) {
    ZkSlot& s = c->slot[si];
    uint32_t f = sb.first, cnt = sb.count;
    const uint64_t* c_off = q.c_off; const uint64_t* d_off = q.d_off;
    size_t cbytes = (size_t)(c_off[f + cnt] - c_off[f]), obytes = (size_t)(d_off[f + cnt] - d_off[f]);
    int rc = zk_slot_ensure(&s, cbytes + 32, obytes + 32);
    if (rc) return rc;
    sb.c_rel.resize(cnt + 1); sb.d_rel.resize(cnt + 1);
    for (uint32_t j = 0; j <= cnt; j++) { sb.c_rel[j] = c_off[f + j] - c_off[f]; sb.d_rel[j] = d_off[f + j] - d_off[f]; }
    cudaStream_t us = q.p.up ? q.p.up : s.stream, ds = q.p.down ? q.p.down : s.stream;
    if (tr) tr->mark(us, k, 0);
    ZK_CUDA_OK(cudaMemcpyAsync(s.d_in, q.comp + c_off[f], cbytes, cudaMemcpyHostToDevice, us));
    if (tr) tr->mark(us, k, 1);
    ZkDecodeParams p = q.p;
    if (p.need) p.need += f;
    rc = zk_decode_enqueue(&s.dws, s.stream, s.d_in, sb.c_rel.data(), sb.d_rel.data(), cnt, s.d_out, q.verify, p);
    if (rc) return rc;
    if (tr) tr->mark(s.stream, k, 2);
    if (obytes) ZK_CUDA_OK(cudaMemcpyAsync(q.dst + d_off[f], s.d_out, obytes, cudaMemcpyDeviceToHost, ds));
    if (ds != s.stream) ZK_CUDA_OK(cudaEventRecord(s.dws.ev_down, ds));        // what zk_decode_collect waits for
    if (tr) tr->mark(ds, k, 4);
    sb.busy = true;
    return 0;
}

static int zk_dec_sub_finish(zk_ctx* c, int si, ZkSubDec& sb, const ZkDecCall& q) {
    ZkSlot& s = c->slot[si];
    if (!sb.busy) return 0;
    int32_t* status = q.status ? q.status + sb.first : nullptr;
    int rc = zk_decode_collect(&s.dws, s.stream, q.p, status);
    if (rc == ZK_ST_RETRY) {            // scratch was too small for this sub-batch: exact needs are known now
        rc = zk_dec_sub_enqueue(c, si, sb, q);
        if (rc) { sb.busy = false; return rc; }
        rc = zk_decode_collect(&s.dws, s.stream, q.p, status);
        if (rc == ZK_ST_RETRY) rc = ZK_ERR_ZSTD(ZKZ_MEMORY_ALLOCATION);
    }
    sb.busy = false;
    return rc;
}

extern "C" int32_t zk_decompress_frames(zk_ctx* c, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off,
                                        uint32_t n, uint8_t* dst, int32_t verify, int32_t* status) {
    return zk_decompress_frames_upto(c, comp, c_off, d_off, n, dst, nullptr, verify, status);
}

extern "C" int32_t zk_decompress_frames_upto(zk_ctx* c, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off,
                                             uint32_t n, uint8_t* dst, const uint32_t* d_need, int32_t verify, int32_t* status) {
    return zk_decompress_frames_prefix(c, comp, c_off, d_off, n, dst, d_need, verify, status, nullptr, 0);
}

extern "C" int32_t zk_decompress_frames_prefix(zk_ctx* c, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off, uint32_t n,
                                               uint8_t* dst, const uint32_t* d_need, int32_t verify, int32_t* status,
                                               const uint8_t* prefix, size_t prefix_len) {
    if (!c) return ZK_ERR_INVALID_ARG;
    ZkDecCall q = {comp, c_off, d_off, dst, verify, status, ZkDecodeParams()};
    int32_t rc = zk_upload_prefix(c, prefix, prefix_len, &q.p.prefix, &q.p.prefix_len);
    if (rc) return rc;
    if (n && (!comp || !c_off || !d_off || !dst)) return ZK_ERR_INVALID_ARG;
    if (n == 0) return 0;
    ZK_CUDA_OK(cudaSetDevice(c->device));
    const size_t sub_bytes = zk_env_size("ZK_HOST_SUB_BYTES", (size_t)128 << 20);     // tuning knob (tools/e2e_sweep2.sh sweeps it)
    q.p.need = d_need;
    q.p.share = (int)zk_env_size("ZK_HOST_SHARE", 3);
    q.p.side = zk_env_size("ZK_HOST_SIDE", 1) != 0;
    q.p.up = c->up; q.p.down = c->down;
    ZkSubDec sub[ZK_SLOTS];
    const int NS = zk_host_slots(false);
    const uint32_t ramp = (uint32_t)zk_env_size("ZK_HOST_RAMP", 0);            // the first `ramp` sub-batches are 1/2^ramp ... 1/2 of the full size
    int32_t worst = 0;
    uint32_t k = 0;
    ZkTrace tr; tr.begin(c->slot[0].stream);
    for (uint32_t first = 0; first < n; k++) {
        int si = (int)(k % NS);
        rc = zk_dec_sub_finish(c, si, sub[si], q);
        if (rc && !worst) worst = rc;
        // ZK_HOST_RAMP=r (default 0): the first r sub-batches are 1/2^r ... 1/2 of the full size, so that the output copy could start
        // earlier.  It gave no gain when it was tried: a sub-batch of any size spends about one frame latency in
        // K-D2, so a small first sub-batch is not done much sooner than a full one
        const size_t this_sub = k < ramp ? sub_bytes >> (ramp - k) : sub_bytes;
        uint32_t end = zk_next_sub(d_off, first, n, this_sub, 1u << 20);
        sub[si].first = first; sub[si].count = end - first;
        rc = zk_dec_sub_enqueue(c, si, sub[si], q, &tr, (int)k);
        if (rc) { if (!worst) worst = rc; break; }
        first = end;
    }
    for (int si = 0; si < ZK_SLOTS; si++) {
        rc = zk_dec_sub_finish(c, si, sub[si], q);
        if (rc && !worst) worst = rc;
    }
    tr.end("dec");
    return worst;
}

// ---------------------------------------------------------------------------------------------
// compress: every entry point describes its call as a ZkCompressReq, and zk_compress runs it
// ---------------------------------------------------------------------------------------------
enum ZkPolicy { ZK_FRAMES_UNIFORM, ZK_FRAMES_SIZED, ZK_FRAMES_COMPRESSED, ZK_FRAMES_CONTENT };

struct ZkCompressReq {
    ZkPolicy policy = ZK_FRAMES_UNIFORM;
    uint32_t size = 0;                                      // uniform: the frame size; Compressed: the target; ContentDefined: the size
    const uint32_t* sizes = nullptr; uint32_t count = 0;    // sized: the caller's frame sizes
    const uint8_t* src = nullptr; size_t n = 0;
    bool host = true;                                       // src and dst in host memory; else device memory, worked on `stream`
    cudaStream_t stream = nullptr;                          // nullptr: slot 0's
    const uint8_t* prefix = nullptr; size_t prefix_len = 0; // host memory
    ZkEncodeParams params;                                  // its prefix: the device copy of `prefix`
    int32_t final_ = 1;                                     // Compressed / ContentDefined: no more input follows this call's
    uint8_t* dst = nullptr; size_t dst_cap = 0;
    uint32_t* c_sizes = nullptr; uint32_t* d_sizes = nullptr; uint32_t frames_cap = 0; uint32_t* n_frames = nullptr;
    size_t* dst_len = nullptr; size_t* consumed = nullptr;
};

// device-resident input and output: sub-batches of at most sub_bytes input (which bound the scratch, about 4x that) one after the other on st
static int32_t zk_compress_dev_subs(zk_ctx* c, const ZkFrames& fr, const uint8_t* d_src, const ZkEncodeParams& p, uint8_t* d_dst,
                                    size_t dst_cap, uint32_t* c_sizes, size_t* dst_len, cudaStream_t st, size_t sub_bytes) {
    size_t out_pos = 0, in_off = 0;
    for (uint32_t f0 = 0; f0 < fr.count;) {
        size_t in_len = 0;
        const uint32_t end = fr.next_sub(f0, sub_bytes, &in_len);
        size_t produced = 0;
        int rc = zk_encode_enqueue(&c->slot[0].ews, st, d_src + in_off, fr.sub(f0, end - f0, in_len), p, d_dst + out_pos, dst_cap - out_pos);
        if (!rc) rc = zk_encode_collect(&c->slot[0].ews, st, c_sizes ? c_sizes + f0 : nullptr, &produced);
        if (rc) return rc;
        out_pos += produced; in_off += in_len; f0 = end;
    }
    *dst_len = out_pos;
    return 0;
}

struct ZkSubEnc { uint32_t f0 = 0, cnt = 0; size_t in_off = 0, in_len = 0, out_pos = 0; bool busy = false; };

// host input and output: sub-batches on up to ZK_HOST_SLOTS_ENC slots, output placed in order
static int32_t zk_compress_host_run(zk_ctx* c, const ZkFrames& fr, const ZkCompressReq& q, size_t sub_bytes, size_t* dst_len) {
    ZkEncodeParams p = q.params;
    p.side = zk_env_size("ZK_HOST_SIDE", 1) != 0;
    // The compressed size of a sub-batch is only known when it completes, so output positions are assigned in
    // order at completion time: H2D and kernels of later sub-batches overlap the D2H of earlier ones.
    ZkSubEnc sub[ZK_SLOTS];
    size_t out_pos = 0, in_off = 0; int32_t err = 0;
    std::vector<uint32_t> tmp_sizes(q.c_sizes ? 0 : fr.count);
    ZkTrace tr; tr.begin(c->slot[0].stream);
    int sub_k[ZK_SLOTS] = {0};
    auto finish = [&](int si) -> int {
        ZkSubEnc& sb = sub[si]; ZkSlot& s = c->slot[si];
        if (!sb.busy) return 0;
        sb.busy = false;
        size_t produced = 0;
        int rc = zk_encode_collect(&s.ews, s.stream, (q.c_sizes ? q.c_sizes : tmp_sizes.data()) + sb.f0, &produced);
        if (rc) return rc;
        if (out_pos + produced > q.dst_cap) return ZK_ERR_ZSTD(ZKZ_DST_TOO_SMALL);
        tr.mark(s.stream, sub_k[si], 3);
        if (cudaMemcpyAsync(q.dst + out_pos, s.d_out, produced, cudaMemcpyDeviceToHost, s.stream) != cudaSuccess) return ZK_ERR_CUDA;
        tr.mark(s.stream, sub_k[si], 4);
        out_pos += produced;
        return 0;
    };
    uint32_t k = 0;
    const int NS = zk_host_slots(true);
    int n_inflight = 0;                                     // completion must follow submission order
    for (uint32_t f0 = 0; f0 < fr.count && !err; k++) {
        const int si = (int)(k % NS);
        if (n_inflight == NS) {                             // oldest in flight is exactly slot si
            err = finish(si); n_inflight--;
            if (err) break;
        }
        ZkSlot& s = c->slot[si]; ZkSubEnc& sb = sub[si];
        if (cudaStreamSynchronize(s.stream) != cudaSuccess) { err = ZK_ERR_CUDA; break; }   // its previous D2H must be done before d_out is reused
        const uint32_t end = fr.next_sub(f0, sub_bytes, &sb.in_len);
        sb.f0 = f0; sb.cnt = end - f0; sb.in_off = in_off;
        const ZkFrames sf = fr.sub(f0, sb.cnt, sb.in_len);
        const size_t bound = sf.bound();
        int rc = zk_slot_ensure(&s, sb.in_len + 32, bound + 32);
        if (rc) { err = rc; break; }
        sub_k[si] = (int)k; tr.mark(s.stream, (int)k, 0);
        if (sb.in_len && cudaMemcpyAsync(s.d_in, q.src + sb.in_off, sb.in_len, cudaMemcpyHostToDevice, s.stream) != cudaSuccess) { err = ZK_ERR_CUDA; break; }
        tr.mark(s.stream, (int)k, 1);
        rc = zk_encode_enqueue(&s.ews, s.stream, s.d_in, sf, p, s.d_out, bound);
        if (rc) { err = rc; break; }
        tr.mark(s.stream, (int)k, 2);
        sb.busy = true; n_inflight++;
        f0 = end; in_off += sb.in_len;
    }
    // drain in submission order
    for (uint32_t j = 0; j < (uint32_t)NS && !err; j++) {
        const int si = (int)((k + j) % NS);                // oldest first
        int rc = finish(si);
        if (rc) err = rc;
    }
    for (int si = 0; si < ZK_SLOTS; si++) cudaStreamSynchronize(c->slot[si].stream);
    tr.end("enc");
    if (err) return err;
    *dst_len = out_pos;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// Frame sizes decided on the GPU (FrameSizePolicy::Compressed and ::ContentDefined): passes over the input, each starting at the first
// byte the previous one left in an open frame.  A pass starts at the encode sub-batch size and doubles while it closes no frame, up to
// grow_to, a pass length at which the policy always closes one.  step(d_in, len, at_end, d_out, cap, &r) cuts one pass and compresses the
// frames it closes to d_out.  min_frame: the fewest bytes of any frame but the last, which bounds a pass's output.  The host paths run
// unpipelined on slot 0.
// ---------------------------------------------------------------------------------------------
struct ZkPassOut {
    uint32_t n_frames = 0;
    size_t consumed = 0, total = 0;                         // input bytes the frames cover; bytes written
    const uint32_t* c_sizes = nullptr; const uint32_t* d_sizes = nullptr;
};

template <class Step>
static int32_t zk_frame_passes(zk_ctx* c, const ZkCompressReq& q, cudaStream_t st, size_t first_pass, size_t grow_to, uint32_t min_frame,
                               const Step& step) {
    const size_t block = 32768, max_pass = ZK_SEEKABLE_MAX_FRAME_SIZE;
    first_pass = first_pass / block * block;
    if (first_pass < block) first_pass = block;
    if (first_pass > max_pass) first_pass = max_pass;
    ZkSlot& s = c->slot[0];
    size_t pos = 0, out = 0, pass = first_pass;
    uint32_t nf = 0;
    while (pos < q.n) {
        const size_t len = q.n - pos < pass ? q.n - pos : pass;
        const int at_end = pos + len == q.n;
        const uint8_t* d_in = q.src + pos; uint8_t* d_out = q.dst + out; size_t cap = q.dst_cap - out;
        if (q.host) {
            cap = zk_encode_bound(len, min_frame);
            int rc = zk_slot_ensure(&s, len + 32, cap + 32);
            if (rc) return rc;
            ZK_CUDA_OK(cudaMemcpyAsync(s.d_in, q.src + pos, len, cudaMemcpyHostToDevice, st));
            d_in = s.d_in; d_out = s.d_out;
        }
        ZkPassOut r;
        int rc = step(d_in, len, at_end, d_out, cap, &r);
        if (rc) return rc;
        if (r.n_frames == 0) {
            if (at_end) break;
            pass = 2 * pass < grow_to ? 2 * pass : grow_to;
            continue;
        }
        if (r.n_frames > q.frames_cap - nf) return ZK_ERR_ZSTD(ZKZ_DST_TOO_SMALL);
        if (q.host) {
            if (r.total > q.dst_cap - out) return ZK_ERR_ZSTD(ZKZ_DST_TOO_SMALL);
            ZK_CUDA_OK(cudaMemcpy(q.dst + out, s.d_out, r.total, cudaMemcpyDeviceToHost));
        }
        if (q.c_sizes) memcpy(q.c_sizes + nf, r.c_sizes, (size_t)r.n_frames * 4);
        if (q.d_sizes) memcpy(q.d_sizes + nf, r.d_sizes, (size_t)r.n_frames * 4);
        nf += r.n_frames; out += r.total; pos += r.consumed;
        pass = first_pass;
    }
    if (q.n_frames) *q.n_frames = nf;
    if (q.dst_len) *q.dst_len = out;
    if (q.consumed) *q.consumed = pos;
    return 0;
}

// Compressed(target) (zk_encode_csize): the cut and the frames in one step; frames start at 32 KiB blocks
static int32_t zk_csize_passes(zk_ctx* c, const ZkCompressReq& q, cudaStream_t st, size_t first_pass) {
    auto step = [&](const uint8_t* d_in, size_t len, int at_end, uint8_t* d_out, size_t cap, ZkPassOut* o) -> int32_t {
        ZkCsizeOut r;
        const int rc = zk_encode_csize(&c->slot[0].ews, st, d_in, len, q.size, q.params, q.final_, at_end, d_out, cap, &r);
        if (rc) return rc;
        o->n_frames = r.n_frames; o->consumed = r.consumed; o->total = r.total; o->c_sizes = r.c_sizes; o->d_sizes = r.d_sizes;
        return 0;
    };
    return zk_frame_passes(c, q, st, first_pass, ZK_SEEKABLE_MAX_FRAME_SIZE, 32768u, step);
}

// ContentDefined(size): each pass is cut on the GPU (zk_encode_cdc), then its closed frames are compressed from the same device memory by
// the sized path, in sub-batches of at most the first pass's length.  A pass of mx bytes always closes a frame.
// ZK_CDC_CAP (tests): candidate positions kept per pass (default pass / 64 + 1); fewer only makes a pass cover less.
static int32_t zk_cdc_passes(zk_ctx* c, const ZkCompressReq& q, cudaStream_t st, size_t first_pass) {
    const ZkCdcRule rule = zk_cdc_rule(q.size);
    const uint32_t cand_cap = (uint32_t)zk_env_size("ZK_CDC_CAP", 0);
    std::vector<uint32_t> ds, cs;
    auto step = [&](const uint8_t* d_in, size_t len, int at_end, uint8_t* d_out, size_t cap, ZkPassOut* o) -> int32_t {
        ZkCdcOut r;
        int32_t rc = zk_encode_cdc(&c->slot[0].ews, st, d_in, len, q.size, q.final_, at_end, cand_cap, &r);
        if (rc || r.n_frames == 0) return rc;
        ds.assign(r.sizes, r.sizes + r.n_frames);
        cs.resize(r.n_frames);
        const ZkFrames fr = {ds.data(), r.consumed, 0, r.n_frames};
        rc = zk_compress_dev_subs(c, fr, d_in, q.params, d_out, cap, cs.data(), &o->total, st, first_pass);
        if (rc) return rc;
        o->n_frames = r.n_frames; o->consumed = r.consumed; o->c_sizes = cs.data(); o->d_sizes = ds.data();
        return 0;
    };
    return zk_frame_passes(c, q, st, first_pass, rule.mx, rule.mn, step);
}

// One compress call: the argument checks of its policy, the prefix upload, then the pipeline of its policy and memory.  The order of the
// checks decides which error a call with several faults reports, so each policy keeps its own.
static int32_t zk_compress(zk_ctx* c, ZkCompressReq q) {
    ZkFrames fr = {};
    int32_t rc = 0;
    if (q.policy == ZK_FRAMES_UNIFORM) {
        if (!c) return ZK_ERR_INVALID_ARG;
        if ((rc = zk_upload_prefix(c, q.prefix, q.prefix_len, &q.params.prefix, &q.params.prefix_len))) return rc;
        if (!q.dst || (q.n && !q.src) || q.size == 0) return ZK_ERR_INVALID_ARG;
        if (q.size > ZK_SEEKABLE_MAX_FRAME_SIZE) q.size = ZK_SEEKABLE_MAX_FRAME_SIZE;       // encode.rs:531-534
        if ((q.n + q.size - 1) / q.size > ZK_SEEKABLE_MAX_FRAMES) return ZK_ERR_FRAME_INDEX_TOO_LARGE;
        // no input: one empty frame, as Encoder::finish() always closes one (encode.rs:755-756)
        fr = {nullptr, q.n, q.size, q.n ? (uint32_t)((q.n + q.size - 1) / q.size) : 1u};
        if (fr.count > q.frames_cap) return ZK_ERR_ZSTD(ZKZ_DST_TOO_SMALL);
    } else if (q.policy == ZK_FRAMES_SIZED) {
        if (!c || (q.count && (!q.sizes || !q.dst))) return ZK_ERR_INVALID_ARG;
        if (q.count > ZK_SEEKABLE_MAX_FRAMES) return ZK_ERR_FRAME_INDEX_TOO_LARGE;
        for (uint32_t f = 0; f < q.count; f++) {
            if (q.sizes[f] > ZK_SEEKABLE_MAX_FRAME_SIZE) return ZK_ERR_ZSTD(ZKZ_PARAM_OUT_OF_BOUND);
            q.n += q.sizes[f];
        }
        if (q.n && !q.src) return ZK_ERR_INVALID_ARG;
        if (q.dst_len) *q.dst_len = 0;
        if (q.count == 0) return 0;                         // (no frame, unlike the uniform layout of no input)
        if ((rc = zk_upload_prefix(c, q.prefix, q.prefix_len, &q.params.prefix, &q.params.prefix_len))) return rc;
        fr = {q.sizes, q.n, 0, q.count};
    } else {
        if (!c || !q.dst || (q.n && !q.src)) return ZK_ERR_INVALID_ARG;
        if (q.consumed) *q.consumed = 0;
        if (q.n == 0) {                                     // one empty frame, as the uniform layout makes of no input
            if (!q.final_) { if (q.n_frames) *q.n_frames = 0; if (q.dst_len) *q.dst_len = 0; return 0; }
            q.policy = ZK_FRAMES_UNIFORM; q.size = 1;
            return zk_compress(c, q);
        }
        if ((rc = zk_upload_prefix(c, q.prefix, q.prefix_len, &q.params.prefix, &q.params.prefix_len))) return rc;
    }
    ZK_CUDA_OK(cudaSetDevice(c->device));
    const cudaStream_t st = q.stream ? q.stream : c->slot[0].stream;
    // tuning knobs: input bytes per sub-batch, and the first pass of the cut policies (tools/knobs_round.sh sweeps the host one)
    const size_t sub_bytes = q.host ? zk_env_size("ZK_HOST_SUB_BYTES_ENC", (size_t)96 << 20) : zk_env_size("ZK_DEV_SUB_BYTES", (size_t)1 << 30);
    if (!q.host) cudaEventRecord(c->ev0, st);
    size_t out_len = 0;
    if (q.policy == ZK_FRAMES_COMPRESSED) rc = zk_csize_passes(c, q, st, sub_bytes);
    else if (q.policy == ZK_FRAMES_CONTENT) rc = zk_cdc_passes(c, q, st, sub_bytes);
    else if (q.host) rc = zk_compress_host_run(c, fr, q, sub_bytes, &out_len);
    else rc = zk_compress_dev_subs(c, fr, q.src, q.params, q.dst, q.dst_cap, q.c_sizes, &out_len, st, sub_bytes);
    if (rc) return rc;
    if (!q.host) {                                          // zk_ctx_last_device_ms: the device paths only
        cudaEventRecord(c->ev1, st);
        cudaEventSynchronize(c->ev1);
        cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1);
    }
    if (q.policy == ZK_FRAMES_UNIFORM || q.policy == ZK_FRAMES_SIZED) { if (q.dst_len) *q.dst_len = out_len; }
    if (q.policy == ZK_FRAMES_UNIFORM) {
        if (q.d_sizes) for (uint32_t f = 0; f < fr.count; f++) q.d_sizes[f] = fr.size(f);
        if (q.n_frames) *q.n_frames = fr.count;
    }
    return 0;
}

extern "C" int32_t zk_compress_frames(zk_ctx* c, const uint8_t* src, size_t n, uint32_t frame_size, int32_t level, int32_t checksum,
                                      uint8_t* dst, size_t dst_cap, uint32_t* c_sizes, uint32_t* d_sizes, uint32_t frames_cap,
                                      uint32_t* n_frames, size_t* dst_len) {
    return zk_compress_frames_prefix(c, src, n, frame_size, level, checksum, nullptr, 0, dst, dst_cap, c_sizes, d_sizes, frames_cap, n_frames,
                                     dst_len);
}

extern "C" int32_t zk_compress_frames_prefix(zk_ctx* c, const uint8_t* src, size_t n, uint32_t frame_size, int32_t level, int32_t checksum,
                                             const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap, uint32_t* c_sizes,
                                             uint32_t* d_sizes, uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len) {
    ZkCompressReq q;
    q.size = frame_size; q.src = src; q.n = n; q.prefix = prefix; q.prefix_len = prefix_len;
    q.params.level = level; q.params.checksum = checksum;
    q.dst = dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.d_sizes = d_sizes; q.frames_cap = frames_cap; q.n_frames = n_frames; q.dst_len = dst_len;
    return zk_compress(c, q);
}

extern "C" int32_t zk_compress_frames_dev(zk_ctx* c, const void* d_src, size_t n, uint32_t frame_size, int32_t level, int32_t checksum,
                                          void* d_dst, size_t dst_cap, uint32_t* c_sizes, uint32_t* d_sizes, uint32_t frames_cap,
                                          uint32_t* n_frames, size_t* dst_len, void* cuda_stream) {
    ZkCompressReq q;
    q.size = frame_size; q.src = (const uint8_t*)d_src; q.n = n; q.host = false; q.stream = (cudaStream_t)cuda_stream;
    q.params.level = level; q.params.checksum = checksum;
    q.dst = (uint8_t*)d_dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.d_sizes = d_sizes; q.frames_cap = frames_cap; q.n_frames = n_frames;
    q.dst_len = dst_len;
    return zk_compress(c, q);
}

extern "C" size_t zk_compress_bound_sized(const uint32_t* frame_sizes, uint32_t n_frames) {
    return frame_sizes || n_frames == 0 ? zk_encode_bound_sized(frame_sizes, n_frames) : 0;
}

// caller-chosen frame sizes (Encoder::end_frame at any byte, encode.rs:438-472, as one batch): frame f is what zk_compress_frames_prefix
// writes for its bytes alone with frame_size = max(size, 1)
extern "C" int32_t zk_compress_frames_sized(zk_ctx* c, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                            int32_t checksum, const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap,
                                            uint32_t* c_sizes, size_t* dst_len) {
    ZkCompressReq q;
    q.policy = ZK_FRAMES_SIZED; q.sizes = frame_sizes; q.count = n_frames; q.src = src; q.prefix = prefix; q.prefix_len = prefix_len;
    q.params.level = level; q.params.checksum = checksum;
    q.dst = dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.dst_len = dst_len;
    return zk_compress(c, q);
}

extern "C" int32_t zk_compress_frames_sized_dev(zk_ctx* c, const void* d_src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                                int32_t checksum, void* d_dst, size_t dst_cap, uint32_t* c_sizes, size_t* dst_len,
                                                void* cuda_stream) {
    ZkCompressReq q;
    q.policy = ZK_FRAMES_SIZED; q.sizes = frame_sizes; q.count = n_frames; q.src = (const uint8_t*)d_src; q.host = false;
    q.stream = (cudaStream_t)cuda_stream; q.params.level = level; q.params.checksum = checksum;
    q.dst = (uint8_t*)d_dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.dst_len = dst_len;
    return zk_compress(c, q);
}

// ---------------------------------------------------------------------------------------------
// long-distance matching (the reference CLI's patch mode: WindowLog + EnableLongDistanceMatching on the CCtx it hands to with_cctx,
// cli/src/compress.rs:31-37): the prefix calls with K-C1h matching every frame against the whole prefix (zk_ldm.inc)
// ---------------------------------------------------------------------------------------------
extern "C" int32_t zk_compress_frames_ldm(zk_ctx* c, const uint8_t* src, size_t n, uint32_t frame_size, int32_t level, int32_t checksum,
                                          const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap, uint32_t* c_sizes,
                                          uint32_t* d_sizes, uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len) {
    ZkCompressReq q;
    q.size = frame_size; q.src = src; q.n = n; q.prefix = prefix; q.prefix_len = prefix_len;
    q.params.level = level; q.params.checksum = checksum; q.params.ldm = true;
    q.dst = dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.d_sizes = d_sizes; q.frames_cap = frames_cap; q.n_frames = n_frames; q.dst_len = dst_len;
    return zk_compress(c, q);
}

extern "C" int32_t zk_compress_frames_sized_ldm(zk_ctx* c, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                                int32_t checksum, const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap,
                                                uint32_t* c_sizes, size_t* dst_len) {
    ZkCompressReq q;
    q.policy = ZK_FRAMES_SIZED; q.sizes = frame_sizes; q.count = n_frames; q.src = src; q.prefix = prefix; q.prefix_len = prefix_len;
    q.params.level = level; q.params.checksum = checksum; q.params.ldm = true;
    q.dst = dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.dst_len = dst_len;
    return zk_compress(c, q);
}

// ---------------------------------------------------------------------------------------------
// long mode (zstd --long): the calls above with K-C1h also matching every frame against its own bytes up to 2^27 back (zk_ldm.inc),
// and against the whole prefix as the _ldm calls do
// ---------------------------------------------------------------------------------------------
extern "C" int32_t zk_compress_frames_long(zk_ctx* c, const uint8_t* src, size_t n, uint32_t frame_size, int32_t level, int32_t checksum,
                                           const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap, uint32_t* c_sizes,
                                           uint32_t* d_sizes, uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len) {
    ZkCompressReq q;
    q.size = frame_size; q.src = src; q.n = n; q.prefix = prefix; q.prefix_len = prefix_len;
    q.params.level = level; q.params.checksum = checksum; q.params.long_mode = true;
    q.dst = dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.d_sizes = d_sizes; q.frames_cap = frames_cap; q.n_frames = n_frames; q.dst_len = dst_len;
    return zk_compress(c, q);
}

extern "C" int32_t zk_compress_frames_sized_long(zk_ctx* c, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                                 int32_t checksum, const uint8_t* prefix, size_t prefix_len, uint8_t* dst, size_t dst_cap,
                                                 uint32_t* c_sizes, size_t* dst_len) {
    ZkCompressReq q;
    q.policy = ZK_FRAMES_SIZED; q.sizes = frame_sizes; q.count = n_frames; q.src = src; q.prefix = prefix; q.prefix_len = prefix_len;
    q.params.level = level; q.params.checksum = checksum; q.params.long_mode = true;
    q.dst = dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.dst_len = dst_len;
    return zk_compress(c, q);
}

extern "C" int32_t zk_compress_frames_long_dev(zk_ctx* c, const void* d_src, size_t n, uint32_t frame_size, int32_t level, int32_t checksum,
                                               void* d_dst, size_t dst_cap, uint32_t* c_sizes, uint32_t* d_sizes, uint32_t frames_cap,
                                               uint32_t* n_frames, size_t* dst_len, void* cuda_stream) {
    ZkCompressReq q;
    q.size = frame_size; q.src = (const uint8_t*)d_src; q.n = n; q.host = false; q.stream = (cudaStream_t)cuda_stream;
    q.params.level = level; q.params.checksum = checksum; q.params.long_mode = true;
    q.dst = (uint8_t*)d_dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.d_sizes = d_sizes; q.frames_cap = frames_cap; q.n_frames = n_frames;
    q.dst_len = dst_len;
    return zk_compress(c, q);
}

extern "C" int32_t zk_compress_frames_sized_long_dev(zk_ctx* c, const void* d_src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                                     int32_t checksum, void* d_dst, size_t dst_cap, uint32_t* c_sizes, size_t* dst_len,
                                                     void* cuda_stream) {
    ZkCompressReq q;
    q.policy = ZK_FRAMES_SIZED; q.sizes = frame_sizes; q.count = n_frames; q.src = (const uint8_t*)d_src; q.host = false;
    q.stream = (cudaStream_t)cuda_stream; q.params.level = level; q.params.checksum = checksum; q.params.long_mode = true;
    q.dst = (uint8_t*)d_dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.dst_len = dst_len;
    return zk_compress(c, q);
}

// ---------------------------------------------------------------------------------------------
// Frame sizes decided on the GPU: FrameSizePolicy::Compressed(target) and ::ContentDefined(size)
// ---------------------------------------------------------------------------------------------
extern "C" int32_t zk_compress_frames_csize(zk_ctx* c, const uint8_t* src, size_t n, uint32_t target, int32_t level, int32_t checksum,
                                            const uint8_t* prefix, size_t prefix_len, int32_t final_, uint8_t* dst, size_t dst_cap,
                                            uint32_t* c_sizes, uint32_t* d_sizes, uint32_t frames_cap, uint32_t* n_frames,
                                            size_t* dst_len, size_t* consumed) {
    ZkCompressReq q;
    q.policy = ZK_FRAMES_COMPRESSED; q.size = target; q.src = src; q.n = n; q.prefix = prefix; q.prefix_len = prefix_len;
    q.params.level = level; q.params.checksum = checksum; q.final_ = final_;
    q.dst = dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.d_sizes = d_sizes; q.frames_cap = frames_cap; q.n_frames = n_frames;
    q.dst_len = dst_len; q.consumed = consumed;
    return zk_compress(c, q);
}

extern "C" int32_t zk_compress_frames_csize_dev(zk_ctx* c, const void* d_src, size_t n, uint32_t target, int32_t level, int32_t checksum,
                                                int32_t final_, void* d_dst, size_t dst_cap, uint32_t* c_sizes, uint32_t* d_sizes,
                                                uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len, size_t* consumed, void* cuda_stream) {
    ZkCompressReq q;
    q.policy = ZK_FRAMES_COMPRESSED; q.size = target; q.src = (const uint8_t*)d_src; q.n = n; q.host = false;
    q.stream = (cudaStream_t)cuda_stream; q.params.level = level; q.params.checksum = checksum; q.final_ = final_;
    q.dst = (uint8_t*)d_dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.d_sizes = d_sizes; q.frames_cap = frames_cap; q.n_frames = n_frames;
    q.dst_len = dst_len; q.consumed = consumed;
    return zk_compress(c, q);
}

extern "C" int32_t zk_compress_frames_cdc(zk_ctx* c, const uint8_t* src, size_t n, uint32_t size, int32_t level, int32_t checksum,
                                          const uint8_t* prefix, size_t prefix_len, int32_t final_, uint8_t* dst, size_t dst_cap,
                                          uint32_t* c_sizes, uint32_t* d_sizes, uint32_t frames_cap, uint32_t* n_frames,
                                          size_t* dst_len, size_t* consumed) {
    ZkCompressReq q;
    q.policy = ZK_FRAMES_CONTENT; q.size = size; q.src = src; q.n = n; q.prefix = prefix; q.prefix_len = prefix_len;
    q.params.level = level; q.params.checksum = checksum; q.final_ = final_;
    q.dst = dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.d_sizes = d_sizes; q.frames_cap = frames_cap; q.n_frames = n_frames;
    q.dst_len = dst_len; q.consumed = consumed;
    return zk_compress(c, q);
}

extern "C" int32_t zk_compress_frames_cdc_dev(zk_ctx* c, const void* d_src, size_t n, uint32_t size, int32_t level, int32_t checksum,
                                              int32_t final_, void* d_dst, size_t dst_cap, uint32_t* c_sizes, uint32_t* d_sizes,
                                              uint32_t frames_cap, uint32_t* n_frames, size_t* dst_len, size_t* consumed, void* cuda_stream) {
    ZkCompressReq q;
    q.policy = ZK_FRAMES_CONTENT; q.size = size; q.src = (const uint8_t*)d_src; q.n = n; q.host = false;
    q.stream = (cudaStream_t)cuda_stream; q.params.level = level; q.params.checksum = checksum; q.final_ = final_;
    q.dst = (uint8_t*)d_dst; q.dst_cap = dst_cap; q.c_sizes = c_sizes; q.d_sizes = d_sizes; q.frames_cap = frames_cap; q.n_frames = n_frames;
    q.dst_len = dst_len; q.consumed = consumed;
    return zk_compress(c, q);
}
