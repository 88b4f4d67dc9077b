// zk_api.cu -- the batch half of the C ABI (include/zeekstd_b200.h): context + zk_{de,}compress_frames[_dev].
// The API-mirror half (SeekTable / RawEncoder / Encoder / Decoder) lives in zk_host.cpp and is built on
// top of these entry points only.
#include "zk_ctx.h"
#include "../../include/zeekstd_b200.h"
#include <stdio.h>
#include <time.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <set>
#include <unordered_map>
#include <unordered_set>
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
        c->slot[i].dws.order = zk_env_size("ZK_DEC_ORDER", 1) != 0 ? 1u : 0u;
        c->slot[i].ews.sm_count = c->sm_count;
    }
    cudaEventCreate(&c->ev0); cudaEventCreate(&c->ev1);
    cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming);
    for (int i = 0; i < ZK_SLOTS; i++) cudaEventCreateWithFlags(&c->ev_join[i], cudaEventDisableTiming);
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
    for (unsigned i = 0; i < ZK_CHAIN_MAX_DEPTH - 1; i++) if (c->d_level[i]) cudaFree(c->d_level[i]);
    for (int i = 0; i < 4; i++) if (c->d_reuse[i]) cudaFree(c->d_reuse[i]);
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    if (c->ev_fork) cudaEventDestroy(c->ev_fork);
    for (int i = 0; i < ZK_SLOTS; i++) if (c->ev_join[i]) cudaEventDestroy(c->ev_join[i]);
    if (c->d_chain) cudaFree(c->d_chain);
    delete c;
}

extern "C" uint64_t zk_ctx_kernel_launches(const zk_ctx* c) { return c ? c->launches() : 0; }
extern "C" uint64_t zk_ctx_decode_segments(const zk_ctx* c) {
    unsigned long long n = 0;
    for (int i = 0; c && i < ZK_SLOTS; i++) n += c->slot[i].dws.segments;
    return n;
}
extern "C" float zk_ctx_last_device_ms(const zk_ctx* c) { return c ? c->last_ms : 0.f; }
extern "C" uint64_t zk_ctx_prefix_bytes_uploaded(const zk_ctx* c) { return c ? c->prefix_uploaded : 0; }
extern "C" uint64_t zk_ctx_reference_entries_decoded(const zk_ctx* c) { return c ? c->ref_decoded : 0; }
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
    c->prefix_uploaded += len;
    *d_prefix = (const uint8_t*)c->d_prefix; *d_len = (uint32_t)len;
    return 0;
}
// the same for a prefix already in device memory (a reference archive decoded into the prefix arena): nothing is copied
static int32_t zk_device_prefix(const uint8_t* prefix, size_t len, const uint8_t** d_prefix, uint32_t* d_len) {
    *d_prefix = nullptr; *d_len = 0;
    if (!prefix || len == 0) return 0;
    if (len > 0x7FFFFFFFull) return ZK_ERR_INVALID_ARG;
    *d_prefix = prefix; *d_len = (uint32_t)len;
    return 0;
}

// per-frame prefixes: n ranges [ranges[2i], ranges[2i + 1]) of a prefix buffer of len bytes -> *out (two words per range); NULL: none (every
// frame has the whole buffer)
static int32_t zk_prefix_ranges(const uint64_t* ranges, uint32_t n, size_t len, std::vector<uint32_t>* out) {
    out->clear();
    if (!ranges) return 0;
    if (len > 0x7FFFFFFFull) return ZK_ERR_INVALID_ARG;
    out->resize(2 * (size_t)n);
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t lo = ranges[2 * i], hi = ranges[2 * i + 1];
        if (lo > hi || hi > len) return ZK_ERR_INVALID_ARG;
        (*out)[2 * i] = (uint32_t)lo; (*out)[2 * i + 1] = (uint32_t)hi;
    }
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

// Device-pointer calls run their sub-batches on the first ns slot streams: those start after the work the caller's stream st holds so far
// (zk_dev_fork), and st continues after all of theirs (zk_dev_join)
static int32_t zk_dev_fork(zk_ctx* c, cudaStream_t st, int ns) {
    ZK_CUDA_OK(cudaEventRecord(c->ev_fork, st));
    for (int i = 0; i < ns; i++) if (c->slot[i].stream != st) ZK_CUDA_OK(cudaStreamWaitEvent(c->slot[i].stream, c->ev_fork, 0));
    return 0;
}
static int32_t zk_dev_join(zk_ctx* c, cudaStream_t st, int ns) {
    for (int i = 0; i < ns; i++) {
        if (c->slot[i].stream == st) continue;
        ZK_CUDA_OK(cudaEventRecord(c->ev_join[i], c->slot[i].stream));
        ZK_CUDA_OK(cudaStreamWaitEvent(st, c->ev_join[i], 0));
    }
    return 0;
}

// input (compress) or output (decompress) bytes per sub-batch of the device-pointer paths, and the sub-batches in flight (tuning knobs,
// swept by tools/pipeline_probe.py; DESIGN §6).  Compress runs four sub-batches of 256 MiB at once: the drain of each stage of one overlaps
// the kernels of the others.  Decompress keeps one sub-batch of up to 1 GiB: concurrent sub-batches were slower than it at every size.
// The passes of the cut policies, each of which ends in a host synchronisation, start at the decompress size
static size_t zk_dev_sub_bytes(bool enc) { return zk_env_size("ZK_DEV_SUB_BYTES", enc ? (size_t)256 << 20 : (size_t)1 << 30); }
static int zk_dev_slots(bool enc) {
    const size_t v = zk_env_size("ZK_DEV_SLOTS", enc ? 4 : 1);
    return (int)(v < 1 ? 1 : (v > ZK_SLOTS ? ZK_SLOTS : v));
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

// one decompress call
struct ZkDecCall {
    const uint8_t* comp; const uint64_t* c_off; const uint64_t* d_off; uint8_t* dst; int verify; int32_t* status;
    ZkDecodeParams p;                                       // p.need: the whole call's
    bool host = true;                                       // comp and dst in host memory, copied through the slots; else device memory
};
struct ZkSubDec { uint32_t first = 0, count = 0; std::vector<uint64_t> c_rel, d_rel; bool busy = false; };

static int zk_dec_sub_enqueue(zk_ctx* c, int si, ZkSubDec& sb, const ZkDecCall& q, ZkTrace* tr = nullptr, int k = 0) {
    ZkSlot& s = c->slot[si];
    uint32_t f = sb.first, cnt = sb.count;
    const uint64_t* c_off = q.c_off; const uint64_t* d_off = q.d_off;
    if (!q.host) {                                          // decoded in place: the offsets stay those of the whole call
        const int rc = zk_decode_enqueue(&s.dws, s.stream, q.comp, c_off + f, d_off + f, cnt, q.dst, q.verify, q.p);
        sb.busy = rc == 0;
        return rc;
    }
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
    if (p.ranges) p.ranges += 2 * (size_t)f;
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

static int32_t zk_dec_run(zk_ctx* c, const ZkDecCall& q, uint32_t n, size_t sub_bytes, int ns, uint32_t ramp);

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
    return zk_decompress_frames_prefixes(c, comp, c_off, d_off, n, dst, d_need, verify, status, prefix, prefix_len, nullptr);
}

// ZK_PATCH_GROUP_BYTES (tests; default 1 GiB): the most prefix bytes one group of entries of the ranged calls uploads at once
static uint64_t zk_patch_group_bytes() { return zk_env_size("ZK_PATCH_GROUP_BYTES", (size_t)1 << 30); }

// The ranged calls work on groups of consecutive entries: from f0 on, as many as keep the hull of their non-empty ranges within `group`
// bytes, at least one -> the group's end; *hlo, *hhi: the hull (equal: every range of the group is empty)
static uint32_t zk_hull_group(const uint64_t* ranges, uint32_t f0, uint32_t n, uint64_t group, uint64_t* hlo, uint64_t* hhi) {
    uint64_t lo = 0, hi = 0;
    bool any = false;
    uint32_t f = f0;
    for (; f < n; f++) {
        const uint64_t a = ranges[2 * (size_t)f], b = ranges[2 * (size_t)f + 1];
        if (a == b) continue;
        const uint64_t nlo = any && lo < a ? lo : a, nhi = any && hi > b ? hi : b;
        if (f > f0 && any && nhi - nlo > group) break;
        lo = nlo; hi = nhi; any = true;
    }
    *hlo = lo; *hhi = hi;
    return f;
}
// the ranges of entries [f0, end) rebased to the hull that starts at hlo (an empty range becomes (0, 0))
static void zk_rebase_ranges(const uint64_t* ranges, uint32_t f0, uint32_t end, uint64_t hlo, std::vector<uint64_t>* out) {
    out->assign(2 * (size_t)(end - f0), 0);
    for (uint32_t f = f0; f < end; f++) {
        const uint64_t a = ranges[2 * (size_t)f], b = ranges[2 * (size_t)f + 1];
        if (a != b) { (*out)[2 * (size_t)(f - f0)] = a - hlo; (*out)[2 * (size_t)(f - f0) + 1] = b - hlo; }
    }
}

// entry e decoded against its own range [ranges[2e], ranges[2e + 1]) of a prefix of prefix_len bytes (ranges == NULL: all of it), which
// is already in device memory at d_prefix (nullptr: no prefix, the ranges are only checked)
static int32_t zk_decompress_prefixes_one(zk_ctx* c, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off, uint32_t n, uint8_t* dst,
                                          const uint32_t* d_need, int32_t verify, int32_t* status, const uint8_t* d_prefix, size_t prefix_len,
                                          const uint64_t* ranges) {
    ZkDecCall q = {comp, c_off, d_off, dst, verify, status, ZkDecodeParams()};
    std::vector<uint32_t> rw;
    int32_t rc = zk_prefix_ranges(ranges, n, prefix_len, &rw);
    if (!rc) rc = zk_device_prefix(d_prefix, prefix_len, &q.p.prefix, &q.p.prefix_len);
    if (rc) return rc;
    if (q.p.prefix && ranges) q.p.ranges = rw.data();
    if (n && (!comp || !c_off || !d_off || !dst)) return ZK_ERR_INVALID_ARG;
    if (n == 0) return 0;
    ZK_CUDA_OK(cudaSetDevice(c->device));
    const size_t sub_bytes = zk_env_size("ZK_HOST_SUB_BYTES", (size_t)128 << 20);     // tuning knob (tools/e2e_sweep2.sh sweeps it)
    q.p.need = d_need;
    q.p.share = (int)zk_env_size("ZK_HOST_SHARE", 3);
    q.p.side = zk_env_size("ZK_HOST_SIDE", 1) != 0;
    q.p.up = c->up; q.p.down = c->down;
    // ZK_HOST_RAMP=r (default 0): the first r sub-batches are 1/2^r ... 1/2 of the full size, so that the output copy could start
    // earlier.  It gave no gain when it was tried: a sub-batch of any size spends about one frame latency in
    // K-D2, so a small first sub-batch is not done much sooner than a full one
    return zk_dec_run(c, q, n, sub_bytes, zk_host_slots(false), (uint32_t)zk_env_size("ZK_HOST_RAMP", 0));
}

// the sub-batches of a decompress call, dealt round-robin over ns slots; the first `ramp` are 1/2^ramp ... 1/2 of sub_bytes.  Returns 0
// or the first failure in the order of the entries
static int32_t zk_dec_run(zk_ctx* c, const ZkDecCall& q, uint32_t n, size_t sub_bytes, int ns, uint32_t ramp) {
    ZkSubDec sub[ZK_SLOTS];
    int32_t worst = 0, rc;
    uint32_t k = 0;
    ZkTrace tr; tr.begin(c->slot[0].stream);
    for (uint32_t first = 0; first < n; k++) {
        int si = (int)(k % ns);
        rc = zk_dec_sub_finish(c, si, sub[si], q);
        if (rc && !worst) worst = rc;
        const size_t this_sub = k < ramp ? sub_bytes >> (ramp - k) : sub_bytes;
        uint32_t end = zk_next_sub(q.d_off, first, n, this_sub, 1u << 20);
        sub[si].first = first; sub[si].count = end - first;
        rc = zk_dec_sub_enqueue(c, si, sub[si], q, &tr, (int)k);
        if (rc) { if (!worst) worst = rc; break; }
        first = end;
    }
    for (uint32_t j = 0; j < (uint32_t)ns; j++) {         // oldest first
        rc = zk_dec_sub_finish(c, (int)((k + j) % ns), sub[(k + j) % ns], q);
        if (rc && !worst) worst = rc;
    }
    tr.end("dec");
    return worst;
}

// device-resident archive and output: sub-batches decoded in place on the slot streams, between the caller stream's work before and after
extern "C" int32_t zk_decompress_frames_dev(zk_ctx* c, const void* d_comp, const uint64_t* c_off, const uint64_t* d_off,
                                            uint32_t n, void* d_dst, int32_t verify, int32_t* status, void* cuda_stream) {
    if (!c || (n && (!d_comp || !c_off || !d_off || !d_dst))) return ZK_ERR_INVALID_ARG;
    if (n == 0) return 0;
    ZK_CUDA_OK(cudaSetDevice(c->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : c->slot[0].stream;
    ZkDecCall q = {(const uint8_t*)d_comp, c_off, d_off, (uint8_t*)d_dst, verify, status, ZkDecodeParams(), false};
    const int ns = zk_dev_slots(false);
    q.p.side = zk_env_size("ZK_DEV_SIDE", 1) != 0;
    q.p.share = (int)zk_env_size("ZK_DEV_SHARE", 1);
    ZK_CUDA_OK(cudaEventRecord(c->ev0, st));
    int32_t rc = zk_dev_fork(c, st, ns);
    const int32_t worst = rc ? rc : zk_dec_run(c, q, n, zk_dev_sub_bytes(false), ns, 0);
    if ((rc = zk_dev_join(c, st, ns))) return rc;
    ZK_CUDA_OK(cudaEventRecord(c->ev1, st));
    ZK_CUDA_OK(cudaEventSynchronize(c->ev1));
    cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1);
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
    bool prefix_dev = false;                                // sized: `prefix` is device memory already (zk_device_prefix), not uploaded
    const uint64_t* ranges = nullptr;                       // sized: frame f's prefix is prefix[ranges[2f], ranges[2f + 1]) (NULL: all of it)
    ZkEncodeParams params;                                  // its prefix: the device copy of `prefix`, and the ranges as 32-bit words
    int32_t final_ = 1;                                     // Compressed / ContentDefined: no more input follows this call's
    uint8_t* dst = nullptr; size_t dst_cap = 0;
    uint32_t* c_sizes = nullptr; uint32_t* d_sizes = nullptr; uint32_t frames_cap = 0; uint32_t* n_frames = nullptr;
    size_t* dst_len = nullptr; size_t* consumed = nullptr;
};

struct ZkSubEnc { uint32_t f0 = 0, cnt = 0; size_t in_off = 0, in_len = 0, out_pos = 0; bool busy = false; };

// Long-distance matching indexes every distinct prefix range of a sub-batch once, at about one byte of scratch per indexed byte (the last
// min(length, 2^27 - 1) bytes of the range): the sub-batch [f0, end) ends early where the ranges it indexes would pass max(sub_bytes, 2^27)
// bytes.  It keeps at least one frame, so a frame with a prefix of any length runs.  *in_len: the input bytes of what is kept
static uint32_t zk_ldm_sub_end(const ZkFrames& fr, const uint32_t* ranges, uint32_t f0, uint32_t end, size_t sub_bytes, size_t* in_len) {
    const size_t reach = (1u << 27) - 1u, budget = sub_bytes > reach + 1 ? sub_bytes : reach + 1;
    std::set<unsigned long long> seen;
    size_t indexed = 0, bytes = 0;
    uint32_t f = f0;
    for (; f < end; f++) {
        const uint32_t lo = ranges[2 * (size_t)f], hi = ranges[2 * (size_t)f + 1];
        if (hi > lo && seen.insert((unsigned long long)lo << 32 | hi).second) {
            const size_t add = hi - lo < reach ? hi - lo : reach;
            if (f > f0 && indexed + add > budget) break;
            indexed += add;
        }
        bytes += fr.size(f);
    }
    *in_len = bytes;
    return f;
}

// The sub-batches of a compress call (at most sub_bytes of input each, which bounds the scratch at about 4x that), dealt round-robin over ns
// slots.  A sub-batch's compressed size is only known when it completes.  host: src and dst in host memory; each sub-batch is copied up to
// its slot and its frames back at the position the ones before it end, assigned in order as they complete, so the copies of one overlap
// the kernels of others.  Else device memory: the slots start after the work of the caller's stream st, and every sub-batch writes its
// frames to dst itself, at the offset the frame scan of the one before left on the device (ZkEncodeParams::chain), so only that scan
// waits for the sub-batch before; st continues after all of them
static int32_t zk_compress_run(zk_ctx* c, const ZkFrames& fr, const uint8_t* src, const ZkEncodeParams& p, uint8_t* dst, size_t dst_cap,
                               uint32_t* c_sizes, bool host, size_t sub_bytes, int ns, cudaStream_t st, size_t* dst_len) {
    unsigned long long* chain = nullptr;
    if (!host) {
        if (const int rc = zk_grow(&c->d_chain, &c->cap_chain, ((size_t)fr.count + 1) * 8, 1)) return rc;
        chain = (unsigned long long*)c->d_chain;
        ZK_CUDA_OK(cudaMemsetAsync(chain, 0, 8, st));
        if (const int rc = zk_dev_fork(c, st, ns)) return rc;
    }
    ZkSubEnc sub[ZK_SLOTS];
    size_t out_pos = 0, in_off = 0; int32_t err = 0;
    ZkTrace tr; tr.begin(c->slot[0].stream);
    int sub_k[ZK_SLOTS] = {0};
    auto finish = [&](int si) -> int {
        ZkSubEnc& sb = sub[si]; ZkSlot& s = c->slot[si];
        if (!sb.busy) return 0;
        sb.busy = false;
        size_t produced = 0;
        int rc = zk_encode_collect(&s.ews, s.stream, c_sizes ? c_sizes + sb.f0 : nullptr, &produced);
        if (rc) return rc;
        if (host) {
            if (out_pos + produced > dst_cap) return ZK_ERR_ZSTD(ZKZ_DST_TOO_SMALL);
            tr.mark(s.stream, sub_k[si], 3);
            if (cudaMemcpyAsync(dst + out_pos, s.d_out, produced, cudaMemcpyDeviceToHost, s.stream) != cudaSuccess) return ZK_ERR_CUDA;
            tr.mark(s.stream, sub_k[si], 4);
        }
        out_pos += produced;
        return 0;
    };
    uint32_t k = 0;
    int n_inflight = 0;                                     // completion must follow submission order
    for (uint32_t f0 = 0; f0 < fr.count && !err; k++) {
        const int si = (int)(k % ns);
        if (n_inflight == ns) {                             // oldest in flight is exactly slot si
            err = finish(si); n_inflight--;
            if (err) break;
        }
        ZkSlot& s = c->slot[si]; ZkSubEnc& sb = sub[si];
        if (cudaStreamSynchronize(s.stream) != cudaSuccess) { err = ZK_ERR_CUDA; break; }   // its previous D2H must be done before d_out is reused
        uint32_t end = fr.next_sub(f0, sub_bytes, &sb.in_len);
        if (p.ranges && (p.ldm || p.long_mode)) end = zk_ldm_sub_end(fr, p.ranges, f0, end, sub_bytes, &sb.in_len);
        ZkEncodeParams sp = p;
        if (p.ranges) sp.ranges = p.ranges + 2 * (size_t)f0;
        sb.f0 = f0; sb.cnt = end - f0; sb.in_off = in_off;
        const ZkFrames sf = fr.sub(f0, sb.cnt, sb.in_len);
        int rc = 0;
        if (host) {
            const size_t bound = sf.bound();
            rc = zk_slot_ensure(&s, sb.in_len + 32, bound + 32);
            if (rc) { err = rc; break; }
            sub_k[si] = (int)k; tr.mark(s.stream, (int)k, 0);
            if (sb.in_len && cudaMemcpyAsync(s.d_in, src + sb.in_off, sb.in_len, cudaMemcpyHostToDevice, s.stream) != cudaSuccess) { err = ZK_ERR_CUDA; break; }
            tr.mark(s.stream, (int)k, 1);
            rc = zk_encode_enqueue(&s.ews, s.stream, s.d_in, sf, sp, s.d_out, bound);
        } else {
            sp.chain = chain + k;
            sp.chain_wait = k ? c->slot[(k - 1) % ns].ews.ev_chain : nullptr;
            rc = zk_encode_enqueue(&s.ews, s.stream, src + sb.in_off, sf, sp, dst, dst_cap);
        }
        if (rc) { err = rc; break; }
        tr.mark(s.stream, (int)k, 2);
        sb.busy = true; n_inflight++;
        f0 = end; in_off += sb.in_len;
    }
    // drain in submission order
    for (uint32_t j = 0; j < (uint32_t)ns && !err; j++) {
        const int si = (int)((k + j) % ns);                // oldest first
        int rc = finish(si);
        if (rc) err = rc;
    }
    for (int si = 0; si < ZK_SLOTS; si++) cudaStreamSynchronize(c->slot[si].stream);
    if (!host && !err) err = zk_dev_join(c, st, ns);
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
            cap = q.dst ? zk_encode_bound(len, min_frame) : 0;     // no dst: a cut without compression (zk_cut_frames_cdc)
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
            if (r.total) ZK_CUDA_OK(cudaMemcpy(q.dst + out, s.d_out, r.total, cudaMemcpyDeviceToHost));
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
// the sized path, in sub-batches of at most sub_bytes (q.dst == nullptr: not at all, zk_cut_frames_cdc).  A pass of mx
// bytes always closes a frame.
// ZK_CDC_CAP (tests): candidate positions kept per pass (default pass / 64 + 1); fewer only makes a pass cover less.
static int32_t zk_cdc_passes(zk_ctx* c, const ZkCompressReq& q, cudaStream_t st, size_t first_pass, size_t sub_bytes) {
    const ZkCdcRule rule = zk_cdc_rule(q.size);
    const uint32_t cand_cap = (uint32_t)zk_env_size("ZK_CDC_CAP", 0);
    std::vector<uint32_t> ds, cs;
    auto step = [&](const uint8_t* d_in, size_t len, int at_end, uint8_t* d_out, size_t cap, ZkPassOut* o) -> int32_t {
        ZkCdcOut r;
        int32_t rc = zk_encode_cdc(&c->slot[0].ews, st, d_in, len, q.size, q.final_, at_end, cand_cap, &r);
        if (rc || r.n_frames == 0) return rc;
        if (!q.dst) { o->n_frames = r.n_frames; o->consumed = r.consumed; o->d_sizes = r.sizes; return 0; }    // the cut alone
        ds.assign(r.sizes, r.sizes + r.n_frames);
        cs.resize(r.n_frames);
        const ZkFrames fr = {ds.data(), r.consumed, 0, r.n_frames};
        rc = zk_compress_run(c, fr, d_in, q.params, d_out, cap, cs.data(), false, sub_bytes, zk_dev_slots(true), st, &o->total);
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
    std::vector<uint32_t> range_words;
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
        if ((rc = zk_prefix_ranges(q.ranges, q.count, q.prefix_len, &range_words))) return rc;
        rc = q.prefix_dev ? zk_device_prefix(q.prefix, q.prefix_len, &q.params.prefix, &q.params.prefix_len)
                          : zk_upload_prefix(c, q.prefix, q.prefix_len, &q.params.prefix, &q.params.prefix_len);
        if (rc) return rc;
        if (q.params.prefix && q.ranges) q.params.ranges = range_words.data();
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
    const size_t sub_bytes = q.host ? zk_env_size("ZK_HOST_SUB_BYTES_ENC", (size_t)96 << 20) : zk_dev_sub_bytes(true);
    if (!q.host) cudaEventRecord(c->ev0, st);
    size_t out_len = 0;
    const size_t first_pass = q.host ? sub_bytes : zk_dev_sub_bytes(false);
    if (q.policy == ZK_FRAMES_COMPRESSED) rc = zk_csize_passes(c, q, st, first_pass);
    else if (q.policy == ZK_FRAMES_CONTENT) rc = zk_cdc_passes(c, q, st, first_pass, sub_bytes);
    else {
        ZkEncodeParams p = q.params;
        if (q.host) p.side = zk_env_size("ZK_HOST_SIDE", 1) != 0;
        rc = zk_compress_run(c, fr, q.src, p, q.dst, q.dst_cap, q.c_sizes, q.host, sub_bytes, q.host ? zk_host_slots(true) : zk_dev_slots(true), st,
                             &out_len);
    }
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

// frames of caller-chosen sizes, frame f against its own range of one prefix buffer: what the sized call (or its _ldm / _long variant)
// writes for frame f alone with that range as its prefix
extern "C" int32_t zk_compress_frames_sized_prefixes(zk_ctx* c, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                                     int32_t checksum, const uint8_t* prefix, size_t prefix_len, const uint64_t* ranges, int32_t ldm,
                                                     int32_t long_mode, uint8_t* dst, size_t dst_cap, uint32_t* c_sizes, size_t* dst_len) {
    ZkCompressReq q;
    q.policy = ZK_FRAMES_SIZED; q.sizes = frame_sizes; q.count = n_frames; q.src = src; q.prefix = prefix; q.prefix_len = prefix_len;
    q.ranges = ranges;
    q.params.level = level; q.params.checksum = checksum; q.params.ldm = ldm != 0; q.params.long_mode = long_mode != 0;
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

// the content-defined cut alone: the d_sizes and consumed of zk_compress_frames_cdc, from the same passes (zk_cdc_passes) without dst
extern "C" int32_t zk_cut_frames_cdc(zk_ctx* c, const uint8_t* src, size_t n, uint32_t size, int32_t final_, uint32_t* frame_sizes,
                                     uint32_t frames_cap, uint32_t* n_frames, size_t* consumed) {
    if (!c || (n && !src)) return ZK_ERR_INVALID_ARG;
    if (consumed) *consumed = 0;
    if (n_frames) *n_frames = 0;
    if (n == 0) {                                           // one empty frame when final, as zk_compress_frames_cdc makes of no input
        if (!final_) return 0;
        if (frames_cap < 1 || !frame_sizes) return frames_cap < 1 ? ZK_ERR_ZSTD(ZKZ_DST_TOO_SMALL) : ZK_ERR_INVALID_ARG;
        frame_sizes[0] = 0;
        if (n_frames) *n_frames = 1;
        return 0;
    }
    if (!frame_sizes) return ZK_ERR_INVALID_ARG;
    ZK_CUDA_OK(cudaSetDevice(c->device));
    ZkCompressReq q;
    q.policy = ZK_FRAMES_CONTENT; q.size = size; q.src = src; q.n = n; q.final_ = final_;
    q.d_sizes = frame_sizes; q.frames_cap = frames_cap; q.n_frames = n_frames; q.consumed = consumed;
    const size_t pass = zk_env_size("ZK_HOST_SUB_BYTES_ENC", (size_t)96 << 20);
    return zk_cdc_passes(c, q, c->slot[0].stream, pass, pass);
}

// ---------------------------------------------------------------------------------------------
// Reuse (DESIGN §3.8): compress a new version against the previous archive.  Frame f copies the lowest-index old entry of its size,
// checksum flag and key when the entry's decoded bytes equal f's bytes (compared on the GPU); every other frame is compressed by the sized
// path.  Unpipelined, on slot 0.
//   pass A  the old entries whose decoded size is some new frame's size (and whose flag matches), decoded in sub-batches of at most
//           ZK_HOST_SUB_BYTES of output: their keys go into a host map (size, key) -> lowest index
//   pass B  per sub-batch of at most ZK_HOST_SUB_BYTES_ENC of input: the frames' keys, the candidates decoded again and compared, the
//           changed frames gathered and compressed, the output assembled in frame order and copied down
// ---------------------------------------------------------------------------------------------
struct ZkReuseKey {
    uint32_t size; unsigned long long key;
    bool operator==(const ZkReuseKey& o) const { return size == o.size && key == o.key; }
};
struct ZkReuseKeyHash {
    size_t operator()(const ZkReuseKey& k) const { return (size_t)(k.key ^ (unsigned long long)k.size * 0x9E3779B97F4A7C15ull); }
};

static uint32_t zk_le32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }

// the Content_Checksum_flag of the first zstd frame of an entry (skippable frames before it are passed over): 0 or 1, -1 if it has none
static int zk_entry_checksum_flag(const uint8_t* p, size_t len) {
    size_t pos = 0;
    while (pos + 5 <= len) {
        const uint32_t magic = zk_le32(p + pos);
        if (magic == ZK_MAGIC) return (p[pos + 4] >> 2) & 1;
        if ((magic & ZK_SKIPPABLE_MASK) != ZK_SKIPPABLE_MAGIC || pos + 8 > len) return -1;
        pos += 8 + (size_t)zk_le32(p + pos + 4);
    }
    return -1;
}

// a device buffer of the context's reuse staging, grown to at least `need` bytes plus padding
static int32_t zk_reuse_buf(zk_ctx* c, int i, size_t need, uint8_t** out) {
    const int rc = zk_grow(&c->d_reuse[i], &c->cap_reuse[i], need + 64, 1);
    *out = (uint8_t*)c->d_reuse[i];
    return rc;
}

// entries list[0, m) of a host archive copied back to back into device memory d on st, entry list[k] at d + c_rel[k]: a run of
// consecutive entries in one copy
static int32_t zk_upload_entries(const zk_reference_archive& r, const uint32_t* list, uint32_t m, const uint64_t* c_rel, uint8_t* d,
                                 cudaStream_t st) {
    for (uint32_t k0 = 0; k0 < m;) {
        uint32_t k1 = k0 + 1;
        while (k1 < m && list[k1] == list[k1 - 1] + 1) k1++;
        const size_t bytes = (size_t)(c_rel[k1] - c_rel[k0]);
        if (bytes) ZK_CUDA_OK(cudaMemcpyAsync(d + c_rel[k0], r.comp + r.c_off[list[k0]], bytes, cudaMemcpyHostToDevice, st));
        k0 = k1;
    }
    return 0;
}

// old entries list[0, m): their bytes uploaded back to back into buffer 0 and decoded, with checksum verification, into buffer 1
// -> *c_rel / *d_rel (m + 1 offsets in those buffers), per-entry statuses in *status
static int32_t zk_reuse_decode(zk_ctx* c, const zk_reference_archive& o, const uint32_t* list, uint32_t m, std::vector<uint64_t>* c_rel,
                               std::vector<uint64_t>* d_rel, std::vector<int32_t>* status, uint8_t** comp, uint8_t** dec) {
    c_rel->assign(m + 1, 0); d_rel->assign(m + 1, 0); status->assign(m, 0);
    for (uint32_t k = 0; k < m; k++) {
        const uint32_t g = list[k];
        (*c_rel)[k + 1] = (*c_rel)[k] + (o.c_off[g + 1] - o.c_off[g]);
        (*d_rel)[k + 1] = (*d_rel)[k] + (o.d_off[g + 1] - o.d_off[g]);
    }
    int32_t rc = zk_reuse_buf(c, 0, (*c_rel)[m], comp);
    if (!rc) rc = zk_reuse_buf(c, 1, (*d_rel)[m], dec);
    if (rc || m == 0) return rc;
    ZkSlot& s = c->slot[0];
    if ((rc = zk_upload_entries(o, list, m, c_rel->data(), *comp, s.stream))) return rc;
    rc = zk_decode_batch(&s.dws, s.stream, *comp, c_rel->data(), d_rel->data(), m, *dec, 1, ZkDecodeParams(), status->data());
    if (rc == ZK_INT_CUDA || rc == -(int)ZKZ_MEMORY_ALLOCATION) return rc;
    return 0;                                               // an entry that fails to decode is only not a candidate
}

extern "C" int32_t zk_compress_frames_sized_reuse(zk_ctx* c, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                                  int32_t checksum, int32_t long_mode, const uint8_t* old_comp, size_t old_len,
                                                  const uint64_t* old_c_off, const uint64_t* old_d_off, uint32_t old_n, uint8_t* dst,
                                                  size_t dst_cap, uint32_t* c_sizes, uint32_t* reused, size_t* dst_len) {
    // the argument checks of zk_compress_frames_sized, then the old archive's
    if (!c || (n_frames && (!frame_sizes || !dst))) return ZK_ERR_INVALID_ARG;
    if (n_frames > ZK_SEEKABLE_MAX_FRAMES) return ZK_ERR_FRAME_INDEX_TOO_LARGE;
    size_t n = 0;
    for (uint32_t f = 0; f < n_frames; f++) {
        if (frame_sizes[f] > ZK_SEEKABLE_MAX_FRAME_SIZE) return ZK_ERR_ZSTD(ZKZ_PARAM_OUT_OF_BOUND);
        n += frame_sizes[f];
    }
    if (n && !src) return ZK_ERR_INVALID_ARG;
    if (dst_len) *dst_len = 0;
    if (old_n && (!old_comp || !old_c_off || !old_d_off)) return ZK_ERR_INVALID_ARG;
    if (old_c_off && old_d_off) {
        for (uint32_t g = 0; g < old_n; g++)
            if (old_c_off[g + 1] < old_c_off[g] || old_d_off[g + 1] < old_d_off[g]) return ZK_ERR_INVALID_ARG;
        if (old_c_off[old_n] > old_len) return ZK_ERR_INVALID_ARG;
    }
    if (n_frames == 0) return 0;
    ZK_CUDA_OK(cudaSetDevice(c->device));
    ZkSlot& s = c->slot[0];
    const cudaStream_t st = s.stream;
    const zk_reference_archive o = {old_comp, old_len, old_c_off, old_d_off, old_n};
    const size_t bits = zk_env_size("ZK_REUSE_KEY_BITS", 64);          // tests: keep only the key's low bits (0: every key is equal)
    const unsigned long long kmask = bits >= 64 ? ~0ull : (1ull << bits) - 1;
    const bool trace = getenv("ZK_E2E_TRACE") != nullptr;
    double t_index = 0, t_match = 0, t_comp = 0, t_asm = 0, t = ZkTrace::now();
    auto lap = [&](double* acc) { const double u = ZkTrace::now(); *acc += u - t; t = u; };
    int32_t rc = 0;
    std::vector<uint64_t> c_rel, d_rel;
    std::vector<int32_t> status;
    std::vector<ZkReuseSpan> spans;
    uint8_t *b_comp = nullptr, *b_dec = nullptr, *b_gather = nullptr, *b_out = nullptr;

    // pass A: index the old entries that could match a new frame
    std::unordered_set<uint32_t> want(frame_sizes, frame_sizes + n_frames);
    std::vector<uint32_t> sel;
    for (uint32_t g = 0; g < old_n; g++) {
        const uint64_t d = old_d_off[g + 1] - old_d_off[g];
        if (d <= ZK_SEEKABLE_MAX_FRAME_SIZE && want.count((uint32_t)d) &&
            zk_entry_checksum_flag(old_comp + old_c_off[g], (size_t)(old_c_off[g + 1] - old_c_off[g])) == (checksum ? 1 : 0))
            sel.push_back(g);
    }
    std::unordered_map<ZkReuseKey, uint32_t, ZkReuseKeyHash> index;
    const size_t dec_sub = zk_env_size("ZK_HOST_SUB_BYTES", (size_t)128 << 20);
    std::vector<unsigned long long> keys;
    for (size_t i0 = 0; i0 < sel.size();) {
        size_t i1 = i0 + 1, bytes = (size_t)(old_d_off[sel[i0] + 1] - old_d_off[sel[i0]]);
        while (i1 < sel.size() && i1 - i0 < (1u << 20) && bytes + (old_d_off[sel[i1] + 1] - old_d_off[sel[i1]]) <= dec_sub)
            bytes += (size_t)(old_d_off[sel[i1] + 1] - old_d_off[sel[i1]]), i1++;
        const uint32_t m = (uint32_t)(i1 - i0);
        if ((rc = zk_reuse_decode(c, o, &sel[i0], m, &c_rel, &d_rel, &status, &b_comp, &b_dec))) return rc;
        spans.clear();
        std::vector<uint32_t> ok;
        for (uint32_t k = 0; k < m; k++)
            if (status[k] == 0) { spans.push_back({d_rel[k], 0, (uint32_t)(d_rel[k + 1] - d_rel[k])}); ok.push_back(k); }
        keys.resize(spans.size());
        if ((rc = zk_reuse_run(&s.ews, st, ZK_REUSE_KEYS, b_dec, nullptr, spans.data(), (uint32_t)spans.size(), keys.data()))) return rc;
        for (size_t j = 0; j < ok.size(); j++) index.emplace(ZkReuseKey{spans[j].len, keys[j] & kmask}, sel[i0 + ok[j]]);   // lowest index kept
        i0 = i1;
    }
    lap(&t_index);

    // pass B: the new frames, sub-batch by sub-batch
    ZkEncodeParams p;
    p.level = level; p.checksum = checksum; p.long_mode = long_mode != 0;
    p.side = zk_env_size("ZK_HOST_SIDE", 1) != 0;
    const ZkFrames fr = {frame_sizes, n, 0, n_frames};
    const size_t enc_sub = zk_env_size("ZK_HOST_SUB_BYTES_ENC", (size_t)96 << 20);
    const uint32_t NONE = 0xFFFFFFFFu;
    std::vector<uint32_t> fo, cand, list, eq, chg_sizes, chg_cs, flags;
    size_t in_off = 0, out_pos = 0;
    for (uint32_t f0 = 0; f0 < n_frames;) {
        size_t in_len = 0;
        const uint32_t end = fr.next_sub(f0, enc_sub, &in_len), cnt = end - f0;
        if ((rc = zk_slot_ensure(&s, in_len + 64, 0))) return rc;
        if (in_len) ZK_CUDA_OK(cudaMemcpyAsync(s.d_in, src + in_off, in_len, cudaMemcpyHostToDevice, st));
        // the frames' keys, and each one's candidate
        fo.assign(cnt + 1, 0);
        spans.resize(cnt);
        for (uint32_t k = 0; k < cnt; k++) { fo[k + 1] = fo[k] + frame_sizes[f0 + k]; spans[k] = {fo[k], 0, frame_sizes[f0 + k]}; }
        keys.resize(cnt);
        if ((rc = zk_reuse_run(&s.ews, st, ZK_REUSE_KEYS, s.d_in, nullptr, spans.data(), cnt, keys.data()))) return rc;
        cand.assign(cnt, NONE); list.clear();
        for (uint32_t k = 0; k < cnt; k++) {
            const auto it = index.find(ZkReuseKey{frame_sizes[f0 + k], keys[k] & kmask});
            if (it != index.end()) { cand[k] = (uint32_t)list.size(); list.push_back(it->second); }
        }
        // the candidates decoded and compared with their frames
        if ((rc = zk_reuse_decode(c, o, list.data(), (uint32_t)list.size(), &c_rel, &d_rel, &status, &b_comp, &b_dec))) return rc;
        spans.clear();
        for (uint32_t k = 0; k < cnt; k++)
            if (cand[k] != NONE) spans.push_back({d_rel[cand[k]], fo[k], frame_sizes[f0 + k]});
        flags.resize(spans.size());
        if ((rc = zk_reuse_run(&s.ews, st, ZK_REUSE_COMPARE, b_dec, s.d_in, spans.data(), (uint32_t)spans.size(), flags.data()))) return rc;
        eq.assign(cnt, 0); chg_sizes.clear();
        size_t chg_bytes = 0;
        for (uint32_t k = 0, j = 0; k < cnt; k++) {
            if (cand[k] != NONE) { eq[k] = flags[j] != 0 && status[cand[k]] == 0; j++; }
            if (!eq[k]) { chg_sizes.push_back(frame_sizes[f0 + k]); chg_bytes += frame_sizes[f0 + k]; }
        }
        lap(&t_match);
        // the changed frames gathered (unless all of them changed) and compressed
        const uint32_t n_chg = (uint32_t)chg_sizes.size();
        size_t produced = 0;
        chg_cs.assign(n_chg, 0);
        if (n_chg) {
            const uint8_t* from = s.d_in;
            if (n_chg < cnt) {
                if ((rc = zk_reuse_buf(c, 2, chg_bytes, &b_gather))) return rc;
                spans.clear();
                size_t pos = 0;
                for (uint32_t k = 0; k < cnt; k++)
                    if (!eq[k]) { spans.push_back({fo[k], pos, frame_sizes[f0 + k]}); pos += frame_sizes[f0 + k]; }
                if ((rc = zk_reuse_run(&s.ews, st, ZK_REUSE_COPY, s.d_in, b_gather, spans.data(), (uint32_t)spans.size(), nullptr))) return rc;
                from = b_gather;
            }
            const ZkFrames cf = {chg_sizes.data(), chg_bytes, 0, n_chg};
            const size_t bound = cf.bound();
            if ((rc = zk_slot_ensure(&s, in_len + 64, bound + 64))) return rc;
            rc = zk_encode_enqueue(&s.ews, st, from, cf, p, s.d_out, bound);
            if (!rc) rc = zk_encode_collect(&s.ews, st, chg_cs.data(), &produced);
            if (rc) return rc;
        }
        lap(&t_comp);
        // the output in frame order: old entries from their staged bytes, the rest from the compressed changed frames
        size_t sub_out = 0;
        for (uint32_t k = 0, j = 0; k < cnt; k++) {
            const uint32_t f = f0 + k;
            const uint32_t cs = eq[k] ? (uint32_t)(c_rel[cand[k] + 1] - c_rel[cand[k]]) : chg_cs[j++];
            if (c_sizes) c_sizes[f] = cs;
            if (reused) reused[f] = eq[k] ? list[cand[k]] : NONE;
            sub_out += cs;
        }
        if (sub_out > dst_cap - out_pos) return ZK_ERR_ZSTD(ZKZ_DST_TOO_SMALL);
        const uint8_t* down = s.d_out;
        if (n_chg < cnt) {
            if ((rc = zk_reuse_buf(c, 3, sub_out, &b_out))) return rc;
            std::vector<ZkReuseSpan> from_new;                // one launch per source buffer
            spans.clear();
            size_t pos = 0, cpos = 0;
            for (uint32_t k = 0, j = 0; k < cnt; k++) {
                const uint32_t cs = eq[k] ? (uint32_t)(c_rel[cand[k] + 1] - c_rel[cand[k]]) : chg_cs[j++];
                if (eq[k]) spans.push_back({c_rel[cand[k]], pos, cs});
                else { from_new.push_back({cpos, pos, cs}); cpos += cs; }
                pos += cs;
            }
            if ((rc = zk_reuse_run(&s.ews, st, ZK_REUSE_COPY, b_comp, b_out, spans.data(), (uint32_t)spans.size(), nullptr))) return rc;
            if ((rc = zk_reuse_run(&s.ews, st, ZK_REUSE_COPY, s.d_out, b_out, from_new.data(), (uint32_t)from_new.size(), nullptr))) return rc;
            down = b_out;
        }
        if (sub_out) ZK_CUDA_OK(cudaMemcpy(dst + out_pos, down, sub_out, cudaMemcpyDeviceToHost));
        lap(&t_asm);
        out_pos += sub_out; in_off += in_len; f0 = end;
    }
    if (dst_len) *dst_len = out_pos;
    if (trace) fprintf(stderr, "reuse index %.3f match %.3f compress %.3f assemble %.3f ms\n", t_index, t_match, t_comp, t_asm);
    return 0;
}

// ---------------------------------------------------------------------------------------------
// Seekable patches (DESIGN §3.4): every frame of NEW against the slice of OLD its content anchors point at (zk_patch.inc), for an OLD of any
// size.  OLD and NEW stream through slot 0 in pieces; only the anchor tables and one group's hull of OLD are ever on the device.
// ---------------------------------------------------------------------------------------------
// ZK_PATCH_PIECE_BYTES (tests; default 1 GiB): the bytes of OLD or NEW one anchor pass uploads; pieces overlap by 63 bytes
static size_t zk_patch_piece_bytes() {
    const size_t v = zk_env_size("ZK_PATCH_PIECE_BYTES", (size_t)1 << 30);
    return v < 4096 ? 4096 : (v > ((size_t)1 << 30) ? (size_t)1 << 30 : v);
}

// the anchors of len bytes of host memory, piece by piece on slot 0
static int32_t zk_patch_scan(zk_ctx* c, const uint8_t* src, uint64_t len, std::vector<unsigned long long>* keys,
                             std::vector<unsigned long long>* pos) {
    ZkSlot& s = c->slot[0];
    const size_t piece = zk_patch_piece_bytes();
    for (uint64_t s0 = 0; s0 < len;) {
        const uint64_t e = len - s0 < piece ? len : s0 + piece;
        const size_t n = (size_t)(e - s0);
        int32_t rc = zk_slot_ensure(&s, n + 32, 0);
        if (rc) return rc;
        ZK_CUDA_OK(cudaMemcpyAsync(s.d_in, src + s0, n, cudaMemcpyHostToDevice, s.stream));
        if ((rc = zk_patch_anchors(&s.ews, s.stream, s.d_in, n, s0, keys, pos))) return rc;
        if (e == len) break;
        s0 = e - 63;                                          // the next piece's first anchor is at e: its hash needs the 63 bytes before
    }
    return 0;
}

// the slice frame (a skippable frame at the start of entry 0): magic, payload size, "ZKSLICE1", u64 old_len, u32 n, n x (u64 lo, u64 hi)
static const uint8_t zk_slice_tag[8] = {'Z', 'K', 'S', 'L', 'I', 'C', 'E', '1'};
static void zk_put_le(uint8_t* p, uint64_t v, int bytes) { for (int i = 0; i < bytes; i++) p[i] = (uint8_t)(v >> (8 * i)); }
static uint64_t zk_get_le(const uint8_t* p, int bytes) { uint64_t v = 0; for (int i = 0; i < bytes; i++) v |= (uint64_t)p[i] << (8 * i); return v; }

extern "C" size_t zk_patch_slices_size(uint32_t n_frames) { return 8 + 20 + 16 * (size_t)n_frames; }

extern "C" int32_t zk_patch_slices_write(uint64_t old_len, const uint64_t* ranges, uint32_t n_frames, uint8_t* dst, size_t dst_cap,
                                         size_t* written) {
    if ((n_frames && !ranges) || !dst || n_frames > ZK_SEEKABLE_MAX_FRAMES) return ZK_ERR_INVALID_ARG;
    for (uint32_t f = 0; f < n_frames; f++)
        if (ranges[2 * (size_t)f] > ranges[2 * (size_t)f + 1] || ranges[2 * (size_t)f + 1] > old_len) return ZK_ERR_INVALID_ARG;
    const size_t total = zk_patch_slices_size(n_frames);
    if (dst_cap < total) return ZK_ERR_ZSTD(ZKZ_DST_TOO_SMALL);
    zk_put_le(dst, ZK_PATCH_SLICES_MAGIC, 4);
    zk_put_le(dst + 4, total - 8, 4);
    memcpy(dst + 8, zk_slice_tag, 8);
    zk_put_le(dst + 16, old_len, 8);
    zk_put_le(dst + 24, n_frames, 4);
    for (size_t i = 0; i < 2 * (size_t)n_frames; i++) zk_put_le(dst + 28 + 8 * i, ranges[i], 8);
    if (written) *written = total;
    return 0;
}

extern "C" int32_t zk_patch_slices_read(const uint8_t* src, size_t len, uint32_t n_frames, uint64_t* old_len, uint64_t* ranges,
                                        size_t* frame_len) {
    if (!src || len < 28 || n_frames > ZK_SEEKABLE_MAX_FRAMES) return ZK_ERR_INVALID_ARG;
    const size_t total = zk_patch_slices_size(n_frames);
    if (zk_get_le(src, 4) != ZK_PATCH_SLICES_MAGIC || zk_get_le(src + 4, 4) != total - 8 || len < total) return ZK_ERR_INVALID_ARG;
    if (memcmp(src + 8, zk_slice_tag, 8) != 0 || zk_get_le(src + 24, 4) != n_frames) return ZK_ERR_INVALID_ARG;
    const uint64_t ol = zk_get_le(src + 16, 8);
    for (uint32_t f = 0; f < n_frames; f++) {
        const uint64_t lo = zk_get_le(src + 28 + 16 * (size_t)f, 8), hi = zk_get_le(src + 36 + 16 * (size_t)f, 8);
        if (lo > hi || hi > ol) return ZK_ERR_INVALID_ARG;
        if (ranges) { ranges[2 * (size_t)f] = lo; ranges[2 * (size_t)f + 1] = hi; }
    }
    if (old_len) *old_len = ol;
    if (frame_len) *frame_len = total;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// The reference of a seekable patch (DESIGN §3.4.1-§3.4.3): OLD is the content of the head of a reference chain R_0 <- R_1 <- ... <- R_{d-1}.
// The root R_0 is OLD's raw bytes in host memory (the raw calls, d = 1) or a plain archive; every other level is a seekable patch of the
// level below.  Every call works on groups of its entries (zk_hull_group) in one loop, zk_ref_groups: Need(head, hull) makes the group's
// hull resident in the prefix arena (c->d_prefix), and the prefix machinery reads it from there (zk_device_prefix).  Need of a raw root
// copies the hull up.  Need of an archive decodes, on slot 0, the entries whose output overlaps the hull, the last one only as far as the
// hull's end.  Need of a patch level runs the same loop on its own entries against the level below; each level below the head has its own
// arena (c->d_level).  The anchor pass reads OLD whole instead: a raw root in pieces, any other head decoded in runs of whole entries.
// The _archive calls are the chain of one level.
// ---------------------------------------------------------------------------------------------

// decoded content starts this far into a level's arena: the anchor pass puts the 63 bytes before a run in front of it
#define ZK_REF_HEAD 64u

// one level of a chain, and what the latest zk_ref_decode of it left in its arena
struct ZkRefLevel {
    zk_reference_archive r = {};
    bool raw = false;                                       // a raw root: r.comp holds OLD's r.len bytes, and r has no entries
    std::vector<uint64_t> slices;                           // a patch level: entry g reads [slices[2g], slices[2g + 1]) of the level below
    void** arena = nullptr; size_t* cap = nullptr;          // the level's device arena
    std::vector<uint32_t> list;                             // the entries decoded last, in order,
    std::vector<int32_t> status;                            // their statuses (a failure below them included),
    uint64_t base = 0;                                      // and the content offset of arena byte ZK_REF_HEAD (a raw root: of byte 0)
};
typedef std::vector<ZkRefLevel> ZkChain;

// R's offsets: never decreasing, content starting at 0, entries within R's bytes -> 0 or ZK_ERR_INVALID_ARG.  *len: the decoded length
static int32_t zk_ref_check(const zk_reference_archive& r, uint64_t* len) {
    if (!r.c_off || !r.d_off || (r.n && !r.comp) || r.d_off[0] != 0) return ZK_ERR_INVALID_ARG;
    for (uint32_t g = 0; g < r.n; g++)
        if (r.c_off[g + 1] < r.c_off[g] || r.d_off[g + 1] < r.d_off[g]) return ZK_ERR_INVALID_ARG;
    if (r.c_off[r.n] > r.len) return ZK_ERR_INVALID_ARG;
    *len = r.d_off[r.n];
    return 0;
}

// R starts with a slice frame: a seekable patch
static bool zk_ref_is_patch(const zk_reference_archive& r) {
    return r.c_off[r.n] - r.c_off[0] >= 4 && zk_le32(r.comp + r.c_off[0]) == ZK_PATCH_SLICES_MAGIC;
}

// chain[0, depth) checked and read (the slice frame of every patch level) -> *ch; *old_len: the head's decoded length.  ZK_ERR_INVALID_ARG:
// a depth of 0 or above ZK_CHAIN_MAX_DEPTH, a level with bad offsets, a root that is a patch, a patch level without a valid slice frame of
// its entry count or whose old_len is not the decoded length of the level below
static int32_t zk_chain_open(zk_ctx* c, const zk_reference_archive* chain, uint32_t depth, ZkChain* ch, uint64_t* old_len) {
    if (!chain || depth == 0 || depth > ZK_CHAIN_MAX_DEPTH) return ZK_ERR_INVALID_ARG;
    ch->assign(depth, ZkRefLevel());
    uint64_t below = 0;
    for (uint32_t i = 0; i < depth; i++) {
        ZkRefLevel& l = (*ch)[i];
        l.r = chain[i];
        uint64_t len = 0, ol = 0;
        int32_t rc = zk_ref_check(l.r, &len);
        if (rc) return rc;
        if (i == 0 ? zk_ref_is_patch(l.r) : !zk_ref_is_patch(l.r)) return ZK_ERR_INVALID_ARG;
        if (i > 0) {
            l.slices.assign(2 * (size_t)l.r.n, 0);
            rc = zk_patch_slices_read(l.r.comp + l.r.c_off[0], (size_t)(l.r.c_off[l.r.n] - l.r.c_off[0]), l.r.n, &ol, l.slices.data(), nullptr);
            if (rc || ol != below) return ZK_ERR_INVALID_ARG;
        }
        l.arena = i + 1 == depth ? &c->d_prefix : &c->d_level[i];
        l.cap = i + 1 == depth ? &c->cap_prefix : &c->cap_level[i];
        below = len;
    }
    *old_len = below;
    return 0;
}

// OLD's old_len bytes in host memory -> *ch, the chain of one raw root, resident in the prefix arena
static void zk_chain_raw(zk_ctx* c, const uint8_t* old, uint64_t old_len, ZkChain* ch) {
    ch->assign(1, ZkRefLevel());
    ZkRefLevel& l = ch->front();
    l.r.comp = old; l.r.len = (size_t)old_len; l.raw = true;
    l.arena = &c->d_prefix; l.cap = &c->cap_prefix;
}

// the first entry of l.list (decoded by zk_ref_decode) with a non-zero status whose output overlaps [lo, hi) -> that status, else 0 (a raw
// root has no entries: always 0)
static int32_t zk_ref_failure(const ZkRefLevel& l, uint64_t lo, uint64_t hi) {
    for (size_t k = 0; k < l.list.size(); k++)
        if (l.status[k] && l.r.d_off[l.list[k] + 1] > lo && l.r.d_off[l.list[k]] < hi) return l.status[k];
    return 0;
}

// entries l.list[a, b) uploaded back to back through slot 0 and decoded into the level's arena, entry list[k] at d_rel[k], against p's
// prefix; need: one per entry of the list (empty: every entry whole) -> l.status[a, b).  Returns 0 or a failure of the call itself (an entry
// that fails to decode: its status)
static int32_t zk_ref_run(zk_ctx* c, ZkRefLevel& l, uint32_t a, uint32_t b, const std::vector<uint64_t>& d_rel, int verify,
                          const std::vector<uint32_t>& need, ZkDecodeParams p) {
    const zk_reference_archive& r = l.r;
    const uint32_t m = b - a;
    std::vector<uint64_t> c_rel(m + 1, 0);
    for (uint32_t k = 0; k < m; k++) c_rel[k + 1] = c_rel[k] + (r.c_off[l.list[a + k] + 1] - r.c_off[l.list[a + k]]);
    ZkSlot& s = c->slot[0];
    int32_t rc = zk_slot_ensure(&s, (size_t)c_rel[m] + 32, 0);
    if (!rc) rc = zk_upload_entries(r, l.list.data() + a, m, c_rel.data(), s.d_in, s.stream);
    if (rc) return rc;
    if (!need.empty()) p.need = need.data() + a;
    rc = zk_decode_batch(&s.dws, s.stream, s.d_in, c_rel.data(), d_rel.data() + a, m, (uint8_t*)*l.arena + ZK_REF_HEAD, verify, p,
                         l.status.data() + a);
    c->ref_decoded += m;
    if (rc == ZK_INT_CUDA || rc == -(int)ZKZ_MEMORY_ALLOCATION) return rc;
    return 0;
}

static int32_t zk_ref_decode(zk_ctx* c, ZkChain& ch, uint32_t i, uint64_t lo, uint64_t hi, int verify);

// The group loop of every call on a reference: entries [0, n), entry k reading [ranges[2k], ranges[2k + 1]) of level i's content, in groups
// (zk_hull_group).  Per group, Need(i, hull) runs when the hull is not empty; then run(a, b, prefix, len, rebased) gets each run [a, b) of
// the group's entries with the hull on the device (prefix, len; nullptr, 0 for an empty hull) and the run's ranges rebased to it.
// status: an entry whose range overlaps a failed entry of level i takes that status there and is in no run.  status == nullptr: a failed
// entry anywhere under the hull fails the call, and the group is one run.  Returns 0 or a failure of the call itself (run's included)
template <class Run>
static int32_t zk_ref_groups(zk_ctx* c, ZkChain& ch, uint32_t i, const uint64_t* ranges, uint32_t n, int verify, int32_t* status,
                             const Run& run) {
    const ZkRefLevel& below = ch[i];
    const uint64_t group = zk_patch_group_bytes();
    std::vector<uint64_t> rb;
    std::vector<int32_t> fail;
    int32_t rc;
    for (uint32_t f0 = 0; f0 < n;) {
        uint64_t hlo, hhi;
        const uint32_t end = zk_hull_group(ranges, f0, n, group, &hlo, &hhi);
        zk_rebase_ranges(ranges, f0, end, hlo, &rb);
        const uint8_t* prefix = nullptr;
        fail.assign(end - f0, 0);
        if (hhi > hlo) {
            if ((rc = zk_ref_decode(c, ch, i, hlo, hhi, verify))) return rc;
            prefix = (const uint8_t*)*below.arena + (below.raw ? 0 : ZK_REF_HEAD) + (hlo - below.base);
            if (!status && (rc = zk_ref_failure(below, hlo, hhi))) return rc;
            for (uint32_t f = f0; status && f < end; f++)
                if (ranges[2 * (size_t)f] < ranges[2 * (size_t)f + 1]) fail[f - f0] = zk_ref_failure(below, ranges[2 * (size_t)f], ranges[2 * (size_t)f + 1]);
        }
        for (uint32_t a = f0; a < end;) {
            if (fail[a - f0]) { status[a] = fail[a - f0]; a++; continue; }
            uint32_t b = a + 1;
            while (b < end && !fail[b - f0]) b++;
            if ((rc = run(a, b, prefix, hhi - hlo, rb.data() + 2 * (size_t)(a - f0)))) return rc;
            a = b;
        }
        f0 = end;
    }
    return 0;
}

// Need(i, [lo, hi)), lo < hi: level i's content [lo, hi) made resident in its arena from ZK_REF_HEAD on (l.base: the content offset there).
// A raw root uploads it as any prefix (zk_upload_prefix: at the arena's start, with the 64 bytes of padding the kernels' wide loads read
// past its end); it has no entries, so nothing of it fails to decode.  Any other level decodes its non-empty entries whose output overlaps
// it, l.list, the last one only as far as hi (need: no checksum on it); a patch level decodes them in the group loop against level i - 1,
// its entries' slices as their ranges.  Returns 0 or a failure of the call itself.  Device memory, per level: a raw root's hull, or the
// decoded bytes from the first entry's start to hi, plus the rest of the block that holds hi (the decoder stops at a block's end)
static int32_t zk_ref_decode(zk_ctx* c, ZkChain& ch, uint32_t i, uint64_t lo, uint64_t hi, int verify) {
    ZkRefLevel& l = ch[i];
    const zk_reference_archive& r = l.r;
    if (l.raw) {                                            // the arena is c->d_prefix
        const uint8_t* d_prefix; uint32_t d_len;
        l.base = lo;
        return zk_upload_prefix(c, r.comp + lo, (size_t)(hi - lo), &d_prefix, &d_len);
    }
    l.list.clear();
    uint32_t g = (uint32_t)(std::upper_bound(r.d_off, r.d_off + r.n + 1, lo) - r.d_off) - 1;    // the entry that holds lo
    for (; g < r.n && r.d_off[g] < hi; g++)
        if (r.d_off[g + 1] > r.d_off[g]) l.list.push_back(g);
    const uint32_t m = (uint32_t)l.list.size();
    const uint32_t last = l.list[m - 1];
    l.base = r.d_off[l.list[0]];
    std::vector<uint64_t> d_rel(m + 1);
    for (uint32_t k = 0; k < m; k++) d_rel[k] = r.d_off[l.list[k]] - l.base;
    d_rel[m] = r.d_off[last + 1] - l.base;
    std::vector<uint32_t> need;
    if (r.d_off[last + 1] > hi) { need.assign(m, 0xFFFFFFFFu); need[m - 1] = (uint32_t)(hi - r.d_off[last]); }
    const uint64_t block = 128u << 10, end = r.d_off[last + 1] - hi > block ? hi + block : r.d_off[last + 1];
    for (int k = 0; k < ZK_SLOTS; k++) if (c->slot[k].stream) cudaStreamSynchronize(c->slot[k].stream);    // nobody reads the arena any more
    int32_t rc = zk_grow(l.arena, l.cap, ZK_REF_HEAD + (size_t)(end - l.base) + 64, 1);
    if (rc) return rc;
    l.status.assign(m, 0);
    if (i == 0) return zk_ref_run(c, l, 0, m, d_rel, verify, need, ZkDecodeParams());
    std::vector<uint64_t> sl(2 * (size_t)m);
    for (uint32_t k = 0; k < m; k++) { sl[2 * (size_t)k] = l.slices[2 * (size_t)l.list[k]]; sl[2 * (size_t)k + 1] = l.slices[2 * (size_t)l.list[k] + 1]; }
    std::vector<uint32_t> rw;
    auto run = [&](uint32_t a, uint32_t b, const uint8_t* prefix, uint64_t len, const uint64_t* rb) -> int32_t {
        ZkDecodeParams p;
        int32_t rc = zk_device_prefix(prefix, (size_t)len, &p.prefix, &p.prefix_len);
        if (!rc && p.prefix && !(rc = zk_prefix_ranges(rb, b - a, (size_t)len, &rw))) p.ranges = rw.data();
        return rc ? rc : zk_ref_run(c, l, a, b, d_rel, verify, need, p);
    };
    return zk_ref_groups(c, ch, i - 1, sl.data(), m, verify, l.status.data(), run);
}

// the decompress calls with ranges of a non-empty OLD: a call failure leaves `status` as it was
static int32_t zk_ref_decompress(zk_ctx* c, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off, uint32_t n, uint8_t* dst,
                                 const uint32_t* d_need, int32_t verify, int32_t* status, ZkChain& ch, uint64_t old_len, const uint64_t* ranges) {
    for (uint32_t i = 0; i < n; i++)
        if (ranges[2 * (size_t)i] > ranges[2 * (size_t)i + 1] || ranges[2 * (size_t)i + 1] > old_len) return ZK_ERR_INVALID_ARG;
    if (n && (!comp || !c_off || !d_off || !dst)) return ZK_ERR_INVALID_ARG;
    if (n == 0) return 0;
    ZK_CUDA_OK(cudaSetDevice(c->device));
    std::vector<int32_t> st(n, 0);
    int32_t worst = 0;                                      // a failure with no entry status (decode scratch that could not grow)
    auto run = [&](uint32_t a, uint32_t b, const uint8_t* prefix, uint64_t len, const uint64_t* rb) -> int32_t {
        const int32_t rc = zk_decompress_prefixes_one(c, comp, c_off + a, d_off + a, b - a, dst, d_need ? d_need + a : nullptr, verify,
                                                      st.data() + a, prefix, (size_t)len, rb);
        if (rc && !ZK_IS_ZSTD_ERR(rc)) return rc;           // the call failed; a frame's status does not stop the other groups
        if (rc && !worst) worst = rc;
        return 0;
    };
    const int32_t rc = zk_ref_groups(c, ch, (uint32_t)ch.size() - 1, ranges, n, verify, st.data(), run);
    if (rc) return rc;
    if (status) memcpy(status, st.data(), (size_t)n * 4);
    for (uint32_t i = 0; i < n; i++) if (st[i]) return st[i];
    return worst;
}

// entry e decoded against its own range of the prefix buffer; ranges == NULL: every entry against the whole buffer.  With ranges, the
// entries run in groups, each with only the hull of its ranges on the device, so the buffer may be of any size
extern "C" int32_t zk_decompress_frames_prefixes(zk_ctx* c, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off, uint32_t n,
                                                 uint8_t* dst, const uint32_t* d_need, int32_t verify, int32_t* status,
                                                 const uint8_t* prefix, size_t prefix_len, const uint64_t* ranges) {
    if (!c) return ZK_ERR_INVALID_ARG;
    if (!ranges || !prefix || prefix_len == 0) {
        const uint8_t* d_prefix; uint32_t d_len;
        const int32_t rc = zk_upload_prefix(c, prefix, prefix_len, &d_prefix, &d_len);
        return rc ? rc : zk_decompress_prefixes_one(c, comp, c_off, d_off, n, dst, d_need, verify, status, d_prefix, prefix_len, ranges);
    }
    ZkChain ch;
    zk_chain_raw(c, prefix, prefix_len, &ch);
    return zk_ref_decompress(c, comp, c_off, d_off, n, dst, d_need, verify, status, ch, prefix_len, ranges);
}

extern "C" int32_t zk_decompress_frames_prefixes_chain(zk_ctx* c, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off, uint32_t n,
                                                       uint8_t* dst, const uint32_t* d_need, int32_t verify, int32_t* status,
                                                       const zk_reference_archive* chain, uint32_t depth, const uint64_t* ranges) {
    if (!c) return ZK_ERR_INVALID_ARG;
    ZkChain ch;
    uint64_t old_len = 0;
    const int32_t rc = zk_chain_open(c, chain, depth, &ch, &old_len);
    if (rc) return rc;
    std::vector<uint64_t> whole;                            // no ranges: every entry against all of OLD
    if (!ranges) {
        whole.assign(2 * (size_t)n, 0);
        for (uint32_t i = 0; i < n; i++) whole[2 * (size_t)i + 1] = old_len;
        ranges = whole.data();
    }
    return zk_ref_decompress(c, comp, c_off, d_off, n, dst, d_need, verify, status, ch, old_len, ranges);
}

extern "C" int32_t zk_decompress_frames_prefixes_archive(zk_ctx* c, const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off, uint32_t n,
                                                         uint8_t* dst, const uint32_t* d_need, int32_t verify, int32_t* status,
                                                         const uint8_t* ref_comp, size_t ref_len, const uint64_t* ref_c_off,
                                                         const uint64_t* ref_d_off, uint32_t ref_n, const uint64_t* ranges) {
    const zk_reference_archive r = {ref_comp, ref_len, ref_c_off, ref_d_off, ref_n};
    return zk_decompress_frames_prefixes_chain(c, comp, c_off, d_off, n, dst, d_need, verify, status, &r, 1, ranges);
}

// frames of NEW against their ranges of OLD, group by group: each group is one zk_compress_frames_sized_prefixes call (ldm = 1) on its hull,
// with the ranges rebased, so no frame's bytes depend on the grouping.  A group whose ranges are all empty is level 16's plain frames, which
// is what that call writes for a frame with an empty range.  A reference entry that fails under a hull fails the call
static int32_t zk_ref_compress(zk_ctx* c, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level, int32_t checksum,
                               ZkChain& ch, uint64_t old_len, const uint64_t* ranges, uint8_t* dst, size_t dst_cap, uint32_t* c_sizes,
                               size_t* dst_len) {
    if (dst_len) *dst_len = 0;
    for (uint32_t f = 0; f < n_frames; f++)
        if (ranges[2 * (size_t)f] > ranges[2 * (size_t)f + 1] || ranges[2 * (size_t)f + 1] > old_len) return ZK_ERR_INVALID_ARG;
    if (n_frames) ZK_CUDA_OK(cudaSetDevice(c->device));
    std::vector<uint32_t> cs(n_frames);
    size_t out = 0, in = 0;
    auto run = [&](uint32_t a, uint32_t b, const uint8_t* prefix, uint64_t len, const uint64_t* rb) -> int32_t {
        size_t got = 0, bytes = 0;
        for (uint32_t f = a; f < b; f++) bytes += frame_sizes[f];
        int32_t rc;
        if (prefix) {
            ZkCompressReq q;
            q.policy = ZK_FRAMES_SIZED; q.sizes = frame_sizes + a; q.count = b - a; q.src = src ? src + in : nullptr;
            q.prefix = prefix; q.prefix_len = (size_t)len; q.prefix_dev = true; q.ranges = rb;
            q.params.level = level; q.params.checksum = checksum; q.params.ldm = true;
            q.dst = dst + out; q.dst_cap = dst_cap - out; q.c_sizes = cs.data() + a; q.dst_len = &got;
            rc = zk_compress(c, q);
        } else {
            rc = zk_compress_frames_sized(c, src ? src + in : nullptr, frame_sizes + a, b - a, 16, checksum, nullptr, 0, dst + out, dst_cap - out,
                                          cs.data() + a, &got);
        }
        out += got; in += bytes;
        return rc;
    };
    const int32_t rc = zk_ref_groups(c, ch, (uint32_t)ch.size() - 1, ranges, n_frames, 1, nullptr, run);
    if (rc) return rc;
    if (c_sizes && n_frames) memcpy(c_sizes, cs.data(), (size_t)n_frames * 4);
    if (dst_len) *dst_len = out;
    return 0;
}

extern "C" int32_t zk_compress_frames_patch(zk_ctx* c, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                            int32_t checksum, const uint8_t* old, uint64_t old_len, const uint64_t* ranges, uint8_t* dst,
                                            size_t dst_cap, uint32_t* c_sizes, size_t* dst_len) {
    if (!c || (n_frames && (!frame_sizes || !ranges || !dst)) || (old_len && !old)) return ZK_ERR_INVALID_ARG;
    ZkChain ch;
    zk_chain_raw(c, old, old_len, &ch);
    return zk_ref_compress(c, src, frame_sizes, n_frames, level, checksum, ch, old_len, ranges, dst, dst_cap, c_sizes, dst_len);
}

extern "C" int32_t zk_compress_frames_patch_chain(zk_ctx* c, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                                  int32_t checksum, const zk_reference_archive* chain, uint32_t depth, const uint64_t* ranges,
                                                  uint8_t* dst, size_t dst_cap, uint32_t* c_sizes, size_t* dst_len) {
    if (!c || (n_frames && (!frame_sizes || !ranges || !dst))) return ZK_ERR_INVALID_ARG;
    ZkChain ch;
    uint64_t old_len = 0;
    const int32_t rc = zk_chain_open(c, chain, depth, &ch, &old_len);
    if (rc) return rc;
    return zk_ref_compress(c, src, frame_sizes, n_frames, level, checksum, ch, old_len, ranges, dst, dst_cap, c_sizes, dst_len);
}

extern "C" int32_t zk_compress_frames_patch_archive(zk_ctx* c, const uint8_t* src, const uint32_t* frame_sizes, uint32_t n_frames, int32_t level,
                                                    int32_t checksum, const uint8_t* ref_comp, size_t ref_len, const uint64_t* ref_c_off,
                                                    const uint64_t* ref_d_off, uint32_t ref_n, const uint64_t* ranges, uint8_t* dst,
                                                    size_t dst_cap, uint32_t* c_sizes, size_t* dst_len) {
    const zk_reference_archive r = {ref_comp, ref_len, ref_c_off, ref_d_off, ref_n};
    return zk_compress_frames_patch_chain(c, src, frame_sizes, n_frames, level, checksum, &r, 1, ranges, dst, dst_cap, c_sizes, dst_len);
}

// the anchors of OLD = the head's decoded content: the head in runs of whole entries of at most ZK_PATCH_PIECE_BYTES (a larger entry
// alone), each run decoded into the prefix arena with the 63 bytes of OLD before it copied in front, so every anchor is found once, as
// the raw pass finds it
static int32_t zk_patch_scan_archive(zk_ctx* c, ZkChain& ch, std::vector<unsigned long long>* keys, std::vector<unsigned long long>* pos) {
    ZkSlot& s = c->slot[0];
    const zk_reference_archive& r = ch.back().r;
    const size_t piece = zk_patch_piece_bytes();
    const size_t most = (size_t)1 << 30;                    // zk_patch_anchors' largest piece
    int32_t rc = zk_slot_ensure(&s, 0, ZK_REF_HEAD);        // d_out: the tail of the run before, kept while the arena is reused
    if (rc) return rc;
    size_t ov = 0;
    for (uint32_t g0 = 0; g0 < r.n;) {
        uint32_t g1 = g0 + 1;
        while (g1 < r.n && r.d_off[g1 + 1] - r.d_off[g0] <= piece) g1++;
        const uint64_t lo = r.d_off[g0], hi = r.d_off[g1];
        g0 = g1;
        if (hi == lo) continue;
        rc = zk_ref_decode(c, ch, (uint32_t)ch.size() - 1, lo, hi, 1);
        if (rc || (rc = zk_ref_failure(ch.back(), lo, hi))) return rc;
        uint8_t* run = (uint8_t*)c->d_prefix + ZK_REF_HEAD;
        if (ov) ZK_CUDA_OK(cudaMemcpyAsync(run - ov, s.d_out, ov, cudaMemcpyDeviceToDevice, s.stream));
        const uint64_t n = ov + (hi - lo);
        for (uint64_t s0 = 0;;) {
            const uint64_t e = n - s0 < most ? n : s0 + most;
            if ((rc = zk_patch_anchors(&s.ews, s.stream, run - ov + s0, (size_t)(e - s0), lo - ov + s0, keys, pos))) return rc;
            if (e == n) break;
            s0 = e - 63;
        }
        const size_t nov = n < 63 ? (size_t)n : 63;
        ZK_CUDA_OK(cudaMemcpyAsync(s.d_out, run + (hi - lo) - nov, nov, cudaMemcpyDeviceToDevice, s.stream));
        ov = nov;
    }
    return zk_sync_check(s.stream);
}

// the anchors of OLD and NEW, then their join.  OLD's anchors: a raw root's bytes piece by piece through slot 0 (zk_patch_scan; not prefix
// bytes), any other head decoded (zk_patch_scan_archive)
static int32_t zk_ref_ranges(zk_ctx* c, ZkChain& ch, uint64_t old_len, const uint8_t* new_src, const uint32_t* frame_sizes, uint32_t n_frames,
                             uint64_t margin, uint64_t* ranges) {
    if (old_len >= (1ull << 62) || margin >= (1ull << 62)) return ZK_ERR_INVALID_ARG;
    ZkPatchTables t;
    t.fa.assign((size_t)n_frames + 1, 0);
    for (uint32_t f = 0; f < n_frames; f++) t.fa[f + 1] = t.fa[f] + frame_sizes[f];
    const uint64_t n = t.fa[n_frames];
    if (n && !new_src) return ZK_ERR_INVALID_ARG;
    if (n_frames == 0) return 0;
    ZK_CUDA_OK(cudaSetDevice(c->device));
    const ZkRefLevel& h = ch.back();
    int32_t rc = h.raw ? zk_patch_scan(c, h.r.comp, old_len, &t.okeys, &t.opos) : zk_patch_scan_archive(c, ch, &t.okeys, &t.opos);
    if (!rc) rc = zk_patch_scan(c, new_src, n, &t.nkeys, &t.npos);
    if (rc) return rc;
    if (t.okeys.size() > 0xFFFFFFF0ull || t.nkeys.size() > 0xFFFFFFF0ull) return ZK_ERR_INVALID_ARG;
    t.fanc.assign((size_t)n_frames + 1, 0);
    for (uint32_t f = 0, i = 0; f <= n_frames; f++) {
        while (i < t.npos.size() && t.npos[i] < t.fa[f]) i++;
        t.fanc[f] = f == n_frames ? (uint32_t)t.npos.size() : i;
    }
    return zk_patch_join(&c->slot[0].ews, c->slot[0].stream, t, n_frames, old_len, margin, (unsigned long long*)ranges);
}

extern "C" int32_t zk_patch_ranges(zk_ctx* c, const uint8_t* new_src, const uint32_t* frame_sizes, uint32_t n_frames, const uint8_t* old,
                                   uint64_t old_len, uint64_t margin, uint64_t* ranges) {
    if (!c || (n_frames && (!frame_sizes || !ranges)) || (old_len && !old)) return ZK_ERR_INVALID_ARG;
    ZkChain ch;
    zk_chain_raw(c, old, old_len, &ch);
    return zk_ref_ranges(c, ch, old_len, new_src, frame_sizes, n_frames, margin, ranges);
}

extern "C" int32_t zk_patch_ranges_chain(zk_ctx* c, const uint8_t* new_src, const uint32_t* frame_sizes, uint32_t n_frames,
                                         const zk_reference_archive* chain, uint32_t depth, uint64_t margin, uint64_t* ranges) {
    if (!c || (n_frames && (!frame_sizes || !ranges))) return ZK_ERR_INVALID_ARG;
    ZkChain ch;
    uint64_t old_len = 0;
    const int32_t rc = zk_chain_open(c, chain, depth, &ch, &old_len);
    if (rc) return rc;
    return zk_ref_ranges(c, ch, old_len, new_src, frame_sizes, n_frames, margin, ranges);
}

extern "C" int32_t zk_patch_ranges_archive(zk_ctx* c, const uint8_t* new_src, const uint32_t* frame_sizes, uint32_t n_frames,
                                           const uint8_t* ref_comp, size_t ref_len, const uint64_t* ref_c_off, const uint64_t* ref_d_off,
                                           uint32_t ref_n, uint64_t margin, uint64_t* ranges) {
    const zk_reference_archive r = {ref_comp, ref_len, ref_c_off, ref_d_off, ref_n};
    return zk_patch_ranges_chain(c, new_src, frame_sizes, n_frames, &r, 1, margin, ranges);
}
