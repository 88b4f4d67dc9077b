// tests/emul/cuda_emul.h -- TEST INFRASTRUCTURE ONLY.
//
// A tiny "CUDA on one CPU thread" execution model so that the *device* code of zeekstd_b200
// (zeekstd_b200/csrc/*.cu) can be exercised bit-for-bit on a machine without a GPU before it runs
// on an H100.  The kernels are compiled unmodified by g++ (-x c++ -DZK_EMUL
// -include cuda_emul.h); every CUDA thread of a CTA becomes a ucontext coroutine, CTAs run one
// after another, and the warp/block collectives (__shfl_*_sync, __ballot_sync, __syncwarp,
// __syncthreads) are rendez-vous points between those coroutines.  Scheduling order is
// pseudo-random (seed: env ZK_EMUL_SEED) so missing barriers show up as wrong results.
//
// This is NOT a product path: the emulated library is built into tests/emul/_build/ and is only
// ever loaded explicitly by tests; the shipped zeekstd_b200/libzeekstd_b200.so contains nvcc-built
// sm_90a code only and refuses to run without a GPU.
#pragma once
#ifndef ZK_EMUL
#error "cuda_emul.h is only for the ZK_EMUL test build"
#endif

#include <ucontext.h>
#include <sys/mman.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>
#include <algorithm>

// ----------------------------------------------------------------------------- keywords
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __shared__ static
#define __constant__ static const
#define __launch_bounds__(...)
#define __align__(n) alignas(n)

struct uint3_e { unsigned x, y, z; };
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct uint2 { unsigned x, y; };
struct uint4 { unsigned x, y, z, w; };
struct alignas(16) int4 { int x, y, z, w; };
struct ulonglong2 { unsigned long long x, y; };
static inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }

namespace emu {

constexpr size_t kStack = 256 * 1024;

enum State : uint8_t { RUNNABLE, WAIT_BLOCK, WAIT_WARP, DONE };

struct Thread {
    ucontext_t ctx;
    State st;
    uint8_t* stack;
};

struct WarpColl {            // one in-flight collective per (warp, mask)
    uint32_t mask = 0, arrived = 0;
    uint64_t slot[32], out[32];
    uint32_t gen = 0;
};

struct Cta {
    unsigned nthreads = 0;
    std::vector<Thread> th;
    std::vector<WarpColl> coll;      // 4 per warp
    unsigned bar_arrived = 0, bar_gen = 0;
    unsigned live = 0;
    ucontext_t sched;
    std::function<void()> body;
};

inline Cta g_cta;
inline unsigned g_cur = 0;
inline uint3_e threadIdx, blockIdx;
inline dim3 blockDim, gridDim;
inline uint8_t* g_dyn_smem = nullptr;
inline size_t g_dyn_smem_cap = 0;
inline uint64_t g_rng = 0x9E3779B97F4A7C15ull;
inline bool g_rng_init = false;
inline unsigned long long g_launches = 0;

inline uint32_t rnd() {
    g_rng ^= g_rng << 13; g_rng ^= g_rng >> 7; g_rng ^= g_rng << 17;
    return (uint32_t)(g_rng >> 32);
}

inline void set_thread_idx(unsigned t) {
    g_cur = t;
    threadIdx.x = t % blockDim.x;
    threadIdx.y = (t / blockDim.x) % blockDim.y;
    threadIdx.z = t / (blockDim.x * blockDim.y);
}

// switch from the running CUDA thread back to the scheduler
inline void to_sched() {
    unsigned me = g_cur;
    swapcontext(&g_cta.th[me].ctx, &g_cta.sched);
    set_thread_idx(me);
}

inline void yield() { to_sched(); }     // stays RUNNABLE

inline void trampoline() {
    g_cta.body();
    g_cta.th[g_cur].st = DONE;
    g_cta.live--;
    // a thread that exits counts as arrived for a pending __syncthreads (matches hardware behaviour)
    if (g_cta.bar_arrived && g_cta.bar_arrived == g_cta.live) {
        g_cta.bar_arrived = 0; g_cta.bar_gen++;
        for (auto& t : g_cta.th) if (t.st == WAIT_BLOCK) t.st = RUNNABLE;
    }
    swapcontext(&g_cta.th[g_cur].ctx, &g_cta.sched);
}

inline void run_cta(unsigned nthreads) {
    Cta& c = g_cta;
    if (c.th.size() < nthreads) {
        size_t old = c.th.size();
        c.th.resize(nthreads);
        for (size_t i = old; i < nthreads; i++) {
            c.th[i].stack = (uint8_t*)mmap(nullptr, kStack, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
            if (c.th[i].stack == MAP_FAILED) { perror("emu: mmap"); abort(); }
        }
    }
    c.nthreads = nthreads; c.live = nthreads; c.bar_arrived = 0;
    c.coll.assign(((nthreads + 31) / 32) * 4, WarpColl());
    for (unsigned i = 0; i < nthreads; i++) {
        getcontext(&c.th[i].ctx);
        c.th[i].ctx.uc_stack.ss_sp = c.th[i].stack;
        c.th[i].ctx.uc_stack.ss_size = kStack;
        c.th[i].ctx.uc_link = nullptr;
        makecontext(&c.th[i].ctx, (void (*)())trampoline, 0);
        c.th[i].st = RUNNABLE;
    }
    // scheduler: warp-granular pseudo-random order (run a random runnable warp's lanes in order)
    unsigned nwarps = (nthreads + 31) / 32;
    while (c.live) {
        bool progressed = false;
        unsigned w0 = rnd() % nwarps;
        for (unsigned wi = 0; wi < nwarps; wi++) {
            unsigned w = (w0 + wi) % nwarps;
            unsigned l0 = rnd() & 31;
            for (unsigned li = 0; li < 32; li++) {
                unsigned t = w * 32 + ((l0 + li) & 31);
                if (t >= nthreads || c.th[t].st != RUNNABLE) continue;
                set_thread_idx(t);
                swapcontext(&c.sched, &c.th[t].ctx);
                progressed = true;
            }
        }
        if (!progressed && c.live) {
            fprintf(stderr, "emu: DEADLOCK in block (%u,%u): %u live threads, none runnable\n", blockIdx.x, blockIdx.y, c.live);
            for (unsigned t = 0; t < nthreads; t++)
                if (c.th[t].st != DONE) fprintf(stderr, "  thread %u state %d\n", t, (int)c.th[t].st);
            abort();
        }
    }
}

template <class F>
inline void launch(dim3 grid, dim3 block, size_t smem, F&& f) {
    if (!g_rng_init) {
        g_rng_init = true;
        const char* s = getenv("ZK_EMUL_SEED");
        if (s) g_rng ^= strtoull(s, nullptr, 10) * 0xD1B54A32D192ED03ull;
    }
    g_launches++;
    if (smem > g_dyn_smem_cap) {
        free(g_dyn_smem);
        g_dyn_smem = (uint8_t*)aligned_alloc(128, (smem + 127) & ~size_t(127));
        g_dyn_smem_cap = smem;
    }
    gridDim = grid; blockDim = block;
    g_cta.body = std::function<void()>(f);
    unsigned nthreads = block.x * block.y * block.z;
    for (unsigned bz = 0; bz < grid.z; bz++)
        for (unsigned by = 0; by < grid.y; by++)
            for (unsigned bx = 0; bx < grid.x; bx++) {
                blockIdx.x = bx; blockIdx.y = by; blockIdx.z = bz;
                if (smem) memset(g_dyn_smem, 0xCD, smem);     // poison: smem is uninitialised on hardware
                run_cta(nthreads);
            }
}

inline void block_barrier() {
    Cta& c = g_cta;
    c.bar_arrived++;
    if (c.bar_arrived == c.live) {
        c.bar_arrived = 0; c.bar_gen++;
        for (auto& t : c.th) if (t.st == WAIT_BLOCK) t.st = RUNNABLE;
        return;
    }
    unsigned gen = c.bar_gen;
    c.th[g_cur].st = WAIT_BLOCK;
    while (c.bar_gen == gen) to_sched();
}

// generic warp rendez-vous: every lane named in `mask` deposits v; returns pointer to the 32 values
inline const uint64_t* warp_exchange(uint32_t mask, uint64_t v) {
    unsigned warp = g_cur / 32, lane = g_cur % 32;
    if (!((mask >> lane) & 1)) { fprintf(stderr, "emu: lane %u not in its own mask %08x\n", lane, mask); abort(); }
    WarpColl* wc = nullptr;
    for (int k = 0; k < 4; k++) { WarpColl& c = g_cta.coll[warp * 4 + k]; if (c.arrived && c.mask == mask) { wc = &c; break; } }
    if (!wc) for (int k = 0; k < 4; k++) { WarpColl& c = g_cta.coll[warp * 4 + k]; if (!c.arrived) { wc = &c; wc->mask = mask; break; } }
    if (!wc) { fprintf(stderr, "emu: too many concurrent sub-warp collectives\n"); abort(); }
    if ((wc->arrived >> lane) & 1) { fprintf(stderr, "emu: lane %u arrived twice (mask %08x)\n", lane, mask); abort(); }
    wc->slot[lane] = v; wc->arrived |= 1u << lane;
    if (wc->arrived == mask) {
        memcpy(wc->out, wc->slot, sizeof wc->out);
        wc->arrived = 0; wc->gen++;
        for (unsigned l = 0; l < 32; l++) {
            unsigned t = warp * 32 + l;
            if (((mask >> l) & 1) && t < g_cta.nthreads && g_cta.th[t].st == WAIT_WARP) g_cta.th[t].st = RUNNABLE;
        }
        return wc->out;
    }
    unsigned gen = wc->gen;
    g_cta.th[g_cur].st = WAIT_WARP;
    while (wc->gen == gen) to_sched();
    return wc->out;
}

}  // namespace emu

using emu::threadIdx; using emu::blockIdx; using emu::blockDim; using emu::gridDim;
constexpr int warpSize = 32;

// ----------------------------------------------------------------------------- collectives
static inline void __syncthreads() { emu::block_barrier(); }
static inline void __syncwarp(unsigned mask = 0xFFFFFFFFu) { emu::warp_exchange(mask, 0); }
static inline unsigned __ballot_sync(unsigned mask, int pred) {
    const uint64_t* o = emu::warp_exchange(mask, pred ? 1 : 0);
    unsigned r = 0;
    for (int l = 0; l < 32; l++) if (((mask >> l) & 1) && o[l]) r |= 1u << l;
    return r;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __all_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) == mask; }

template <class T> static inline uint64_t emu_pack(T v) { uint64_t u = 0; static_assert(sizeof(T) <= 8, ""); memcpy(&u, &v, sizeof(T)); return u; }
template <class T> static inline T emu_unpack(uint64_t u) { T v; memcpy(&v, &u, sizeof(T)); return v; }

template <class T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
    const uint64_t* o = emu::warp_exchange(mask, emu_pack(v));
    int lane = emu::g_cur % 32;
    int s = (lane & ~(width - 1)) | (src & (width - 1));
    return emu_unpack<T>(o[s]);
}
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    const uint64_t* o = emu::warp_exchange(mask, emu_pack(v));
    int lane = emu::g_cur % 32;
    int s = lane - (int)delta;
    if (s < (lane & ~(width - 1))) s = lane;
    return emu_unpack<T>(o[s]);
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    const uint64_t* o = emu::warp_exchange(mask, emu_pack(v));
    int lane = emu::g_cur % 32;
    int s = lane + (int)delta;
    if (s > (lane | (width - 1))) s = lane;
    return emu_unpack<T>(o[s]);
}
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int x, int width = 32) {
    const uint64_t* o = emu::warp_exchange(mask, emu_pack(v));
    int lane = emu::g_cur % 32;
    int s = lane ^ x;
    if ((s & ~(width - 1)) != (lane & ~(width - 1))) s = lane;
    return emu_unpack<T>(o[s]);
}
static inline unsigned __match_any_sync(unsigned mask, unsigned v) {
    const uint64_t* o = emu::warp_exchange(mask, v); unsigned r = 0;
    for (int l = 0; l < 32; l++) if (((mask >> l) & 1) && (unsigned)o[l] == v) r |= 1u << l;
    return r;
}
static inline unsigned __reduce_add_sync(unsigned mask, unsigned v) {
    const uint64_t* o = emu::warp_exchange(mask, v); unsigned r = 0;
    for (int l = 0; l < 32; l++) if ((mask >> l) & 1) r += (unsigned)o[l];
    return r;
}
static inline unsigned __reduce_max_sync(unsigned mask, unsigned v) {
    const uint64_t* o = emu::warp_exchange(mask, v); unsigned r = 0;
    for (int l = 0; l < 32; l++) if ((mask >> l) & 1) r = std::max(r, (unsigned)o[l]);
    return r;
}
static inline unsigned __reduce_min_sync(unsigned mask, unsigned v) {
    const uint64_t* o = emu::warp_exchange(mask, v); unsigned r = 0xFFFFFFFFu;
    for (int l = 0; l < 32; l++) if ((mask >> l) & 1) r = std::min(r, (unsigned)o[l]);
    return r;
}
static inline unsigned __reduce_or_sync(unsigned mask, unsigned v) {
    const uint64_t* o = emu::warp_exchange(mask, v); unsigned r = 0;
    for (int l = 0; l < 32; l++) if ((mask >> l) & 1) r |= (unsigned)o[l];
    return r;
}

// ----------------------------------------------------------------------------- bit / int intrinsics
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __ffsll(long long x) { return __builtin_ffsll(x); }
static inline unsigned __brev(unsigned x) { unsigned r = 0; for (int i = 0; i < 32; i++) r |= ((x >> i) & 1u) << (31 - i); return r; }
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) { uint64_t v = ((uint64_t)hi << 32) | lo; return (unsigned)(v >> (s & 31)); }
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned s) { uint64_t v = ((uint64_t)hi << 32) | lo; return (unsigned)((v << (s & 31)) >> 32); }
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned sel) {
    uint64_t v = ((uint64_t)b << 32) | a; unsigned r = 0;
    for (int i = 0; i < 4; i++) { unsigned s = (sel >> (4 * i)) & 7; r |= (unsigned)((v >> (8 * s)) & 0xFF) << (8 * i); }
    return r;
}
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((uint64_t)a * b) >> 32); }
static inline unsigned long long __umul64hi(unsigned long long a, unsigned long long b) { return (unsigned long long)(((unsigned __int128)a * b) >> 64); }
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcs(const T* p) { return *p; }
template <class T> static inline void __stcs(T* p, T v) { *p = v; }
template <class T> static inline void __stcg(T* p, T v) { *p = v; }
template <class T> static inline T __ldcg(const T* p) { return *p; }
static inline void __threadfence() {}
static inline void __threadfence_block() {}
static inline void __nanosleep(unsigned) { emu::yield(); }
static inline long long clock64() { return 0; }
using std::min; using std::max;

// ----------------------------------------------------------------------------- atomics (single OS thread)
template <class T, class U> static inline T atomicAdd(T* p, U v) { T o = *p; *p = (T)(o + (T)v); return o; }
template <class T, class U> static inline T atomicSub(T* p, U v) { T o = *p; *p = (T)(o - (T)v); return o; }
template <class T, class U> static inline T atomicMax(T* p, U v) { T o = *p; if ((T)v > o) *p = (T)v; return o; }
template <class T, class U> static inline T atomicMin(T* p, U v) { T o = *p; if ((T)v < o) *p = (T)v; return o; }
template <class T, class U> static inline T atomicOr(T* p, U v) { T o = *p; *p = (T)(o | (T)v); return o; }
template <class T, class U> static inline T atomicAnd(T* p, U v) { T o = *p; *p = (T)(o & (T)v); return o; }
template <class T, class U> static inline T atomicExch(T* p, U v) { T o = *p; *p = (T)v; return o; }
template <class T, class U, class V> static inline T atomicCAS(T* p, U cmp, V v) { T o = *p; if (o == (T)cmp) *p = (T)v; return o; }

// ----------------------------------------------------------------------------- runtime API subset
typedef int cudaError_t;
typedef struct emu_stream* cudaStream_t;
typedef struct emu_event* cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorInvalidValue = 1, cudaErrorNoDevice = 100 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaHostAllocDefault = 0, cudaHostRegisterDefault = 0 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct cudaDeviceProp { char name[256]; int multiProcessorCount; int major, minor; size_t totalGlobalMem; size_t sharedMemPerBlockOptin; };

static inline cudaError_t cudaMalloc(void** p, size_t n) {
    *p = aligned_alloc(256, (n + 255 + 64) & ~size_t(255));   // +64: device code may read a few bytes past the end like the real allocator allows
    if (*p) memset(*p, 0xA5, n);
    return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
static inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMallocHost(void** p, size_t n) { *p = aligned_alloc(256, (n + 255) & ~size_t(255)); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
static inline cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { return cudaMallocHost(p, n); }
static inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaHostRegister(void*, size_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaHostUnregister(void*) { return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (cudaStream_t)malloc(1); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, unsigned, int) { *s = (cudaStream_t)malloc(1); return cudaSuccess; }
static inline cudaError_t cudaDeviceGetStreamPriorityRange(int* least, int* greatest) { *least = 0; *greatest = -5; return cudaSuccess; }
static inline cudaError_t cudaStreamCreate(cudaStream_t* s) { *s = (cudaStream_t)malloc(1); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = (cudaEvent_t)malloc(1); return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = (cudaEvent_t)malloc(1); return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
static inline const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
    memset(p, 0, sizeof *p); strcpy(p->name, "ZK_EMUL (CPU coroutine emulation)");
    p->multiProcessorCount = 4; p->major = 10; p->minor = 0; p->totalGlobalMem = size_t(8) << 30; p->sharedMemPerBlockOptin = 227 * 1024;
    return cudaSuccess;
}
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
