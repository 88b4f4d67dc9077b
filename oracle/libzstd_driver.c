/*
 * oracle/libzstd_driver.c -- TEST / BASELINE INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The reference (rorosen/zeekstd) is Rust and cannot be built here (no cargo,
 * no network); all of its codec arithmetic is the third-party libzstd
 * (zstd-sys 2.0.16+zstd.1.5.7, Cargo.lock:1192-1198) which is absent from
 * the reference tree as source but present on the system as a shared object.
 * This driver dlopen()s that shared object and replays the reference's exact
 * libzstd call sequences:
 *
 *   compress   lib/src/encode.rs:340-346  compress_stream2(out,in,ZSTD_e_continue)
 *              lib/src/encode.rs:442-464  compress_stream2(out,empty,ZSTD_e_end) until 0
 *              lib/src/encode.rs:504-506  CCtx reset(SessionOnly) between frames
 *              lib/src/encode.rs:281-284  set CompressionLevel / ChecksumFlag
 *              lib/src/encode.rs:599      staging buffer = ZSTD_CStreamOutSize()
 *   decompress lib/src/decode.rs:221-256  decompress_stream with DStreamInSize /
 *              DStreamOutSize staging buffers (decode.rs:181-184)
 *   prefix     lib/src/encode.rs:332-338  cctx.ref_prefix(pref) when frame_d_size == 0 (start of every frame)
 *              lib/src/decode.rs:211-214  dctx.ref_prefix(pref) before the first frame,
 *              lib/src/decode.rs:246-255  reset(SessionOnly) + ref_prefix(pref) after every frame end (n == 0)
 *
 * plus ZSTD_compress() one-shot frames (Single_Segment / Frame_Content_Size headers: what other
 * libzstd producers emit and the Decoder must accept, SURVEY.md 8a) for the coverage fixtures.
 *
 * so it is (a) the oracle every parity test compares against ("bit-exact vs
 * the reference Decoder" == equality with ZSTD_decompressStream output) and
 * (b) the CPU baseline bench.py times on the GPU box's host cores.
 * No zstd.h exists in the image: prototypes are declared by hand from the
 * stable ABI (SURVEY.md Appendix B).
 */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <pthread.h>
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

typedef struct { const void* src; size_t size; size_t pos; } ZSTD_inBuffer;
typedef struct { void* dst; size_t size; size_t pos; } ZSTD_outBuffer;

static struct {
    void* h;
    void* (*createCCtx)(void);
    size_t (*freeCCtx)(void*);
    size_t (*CCtx_setParameter)(void*, int, int);
    size_t (*CCtx_reset)(void*, int);
    size_t (*compressStream2)(void*, ZSTD_outBuffer*, ZSTD_inBuffer*, int);
    void* (*createDCtx)(void);
    size_t (*freeDCtx)(void*);
    size_t (*DCtx_reset)(void*, int);
    size_t (*decompressStream)(void*, ZSTD_outBuffer*, ZSTD_inBuffer*);
    size_t (*CStreamOutSize)(void);
    size_t (*DStreamInSize)(void);
    size_t (*DStreamOutSize)(void);
    unsigned (*isError)(size_t);
    int (*getErrorCode)(size_t);
    const char* (*versionString)(void);
    size_t (*compressBound)(size_t);
    size_t (*compress)(void*, size_t, const void*, size_t, int);
    size_t (*CCtx_refPrefix)(void*, const void*, size_t);
    size_t (*DCtx_refPrefix)(void*, const void*, size_t);
} Z;

#define ZSTD_c_compressionLevel 100
#define ZSTD_c_checksumFlag 201
#define ZSTD_reset_session_only 1
#define ZSTD_e_continue 0
#define ZSTD_e_end 2

#define LOAD(field, name) do { *(void**)(&Z.field) = dlsym(Z.h, name); if (!Z.field) return -2; } while (0)

int zkr_open(const char* path) {
    if (Z.h) return 0;
    Z.h = dlopen(path ? path : "libzstd.so.1", RTLD_NOW | RTLD_LOCAL);
    if (!Z.h) return -1;
    LOAD(createCCtx, "ZSTD_createCCtx"); LOAD(freeCCtx, "ZSTD_freeCCtx");
    LOAD(CCtx_setParameter, "ZSTD_CCtx_setParameter"); LOAD(CCtx_reset, "ZSTD_CCtx_reset");
    LOAD(compressStream2, "ZSTD_compressStream2");
    LOAD(createDCtx, "ZSTD_createDCtx"); LOAD(freeDCtx, "ZSTD_freeDCtx");
    LOAD(DCtx_reset, "ZSTD_DCtx_reset"); LOAD(decompressStream, "ZSTD_decompressStream");
    LOAD(CStreamOutSize, "ZSTD_CStreamOutSize"); LOAD(DStreamInSize, "ZSTD_DStreamInSize");
    LOAD(DStreamOutSize, "ZSTD_DStreamOutSize"); LOAD(isError, "ZSTD_isError");
    LOAD(getErrorCode, "ZSTD_getErrorCode"); LOAD(versionString, "ZSTD_versionString");
    LOAD(compressBound, "ZSTD_compressBound");
    LOAD(compress, "ZSTD_compress"); LOAD(CCtx_refPrefix, "ZSTD_CCtx_refPrefix"); LOAD(DCtx_refPrefix, "ZSTD_DCtx_refPrefix");
    return 0;
}
const char* zkr_version(void) { return Z.h ? Z.versionString() : "unloaded"; }
size_t zkr_compress_bound(size_t n) { return Z.compressBound(n); }

/* Compress ONE frame the way RawEncoder does (encode.rs:311-354 + 438-472).
 * Returns compressed size or -(libzstd error code). */
static int64_t compress_one_frame(void* cctx, const uint8_t* src, size_t n, uint8_t* dst, size_t cap,
                                  uint8_t* stage, size_t stage_sz, const uint8_t* prefix, size_t prefix_len) {
    ZSTD_inBuffer in = { src, n, 0 };
    size_t written = 0;
    if (prefix && n) {                         /* encode.rs:332-338: only once input arrives (frame_d_size == 0 at the first compress call) */
        size_t r = Z.CCtx_refPrefix(cctx, prefix, prefix_len);
        if (Z.isError(r)) return -(int64_t)Z.getErrorCode(r);
    }
    while (in.pos < n) {                       /* Encoder::compress_with_prefix loop, encode.rs:648-661 */
        ZSTD_outBuffer out = { stage, stage_sz, 0 };
        while (in.pos < n && out.pos < out.size) {   /* encode.rs:340-346 */
            size_t r = Z.compressStream2(cctx, &out, &in, ZSTD_e_continue);
            if (Z.isError(r)) return -(int64_t)Z.getErrorCode(r);
        }
        if (written + out.pos > cap) return -70;
        memcpy(dst + written, stage, out.pos); written += out.pos;   /* flush_out_buf, encode.rs:779-787 */
    }
    for (;;) {                                  /* end_frame, encode.rs:438-464 */
        ZSTD_inBuffer empty = { "", 0, 0 };
        ZSTD_outBuffer out = { stage, stage_sz, 0 };
        size_t r = Z.compressStream2(cctx, &out, &empty, ZSTD_e_end);
        if (Z.isError(r)) return -(int64_t)Z.getErrorCode(r);
        if (written + out.pos > cap) return -70;
        memcpy(dst + written, stage, out.pos); written += out.pos;
        if (r == 0) break;
    }
    Z.CCtx_reset(cctx, ZSTD_reset_session_only);  /* reset_frame, encode.rs:501-507 */
    return (int64_t)written;
}

/* Decompress ONE seek-table entry's bytes as Decoder::decompress does (decode.rs:221-256). */
static int64_t decompress_one_frame(void* dctx, const uint8_t* src, size_t n, uint8_t* dst, size_t cap,
                                    size_t in_chunk, size_t out_chunk, const uint8_t* prefix, size_t prefix_len) {
    size_t ipos = 0, opos = 0;
    size_t last = 1;
    if (prefix) {                               /* decode.rs:211-214 */
        size_t r = Z.DCtx_refPrefix(dctx, prefix, prefix_len);
        if (Z.isError(r)) return -(int64_t)Z.getErrorCode(r);
    }
    while (ipos < n) {
        size_t take = n - ipos < in_chunk ? n - ipos : in_chunk;    /* src.read(&mut in_buf), decode.rs:222-225 */
        ZSTD_inBuffer in = { src + ipos, take, 0 };
        while (in.pos < take) {
            size_t room = cap - opos < out_chunk ? cap - opos : out_chunk;
            ZSTD_outBuffer out = { dst + opos, room, 0 };
            size_t before = in.pos;
            last = Z.decompressStream(dctx, &out, &in);             /* decode.rs:243-245 */
            if (Z.isError(last)) { Z.DCtx_reset(dctx, ZSTD_reset_session_only); return -(int64_t)Z.getErrorCode(last); }
            opos += out.pos;
            if (last == 0 && prefix) {                              /* frame end: decode.rs:246-255 */
                Z.DCtx_reset(dctx, ZSTD_reset_session_only);
                size_t r = Z.DCtx_refPrefix(dctx, prefix, prefix_len);
                if (Z.isError(r)) return -(int64_t)Z.getErrorCode(r);
                continue;
            }
            if (out.pos == 0 && in.pos == before) {                 /* no progress: output exhausted */
                Z.DCtx_reset(dctx, ZSTD_reset_session_only); return room == 0 ? -70 : -72;
            }
        }
        ipos += take;
    }
    /* drain anything libzstd still holds back */
    while (last != 0 && opos < cap) {
        ZSTD_inBuffer in = { src, 0, 0 };
        size_t room = cap - opos < out_chunk ? cap - opos : out_chunk;
        ZSTD_outBuffer out = { dst + opos, room, 0 };
        size_t r = Z.decompressStream(dctx, &out, &in);
        if (Z.isError(r)) { Z.DCtx_reset(dctx, ZSTD_reset_session_only); return -(int64_t)Z.getErrorCode(r); }
        if (out.pos == 0) break;
        opos += out.pos; last = r;
    }
    if (last != 0) { Z.DCtx_reset(dctx, ZSTD_reset_session_only); return -72; } /* truncated input */
    return (int64_t)opos;
}

typedef struct {
    int tid, nthreads;
    const uint8_t* src; size_t n; uint32_t frame_size; int level, checksum;
    uint8_t* dst; size_t slot;            /* compress: per-frame output slots of `slot` bytes */
    const uint64_t* c_off; const uint64_t* d_off; size_t dst_cap;   /* decompress */
    uint32_t n_frames; int64_t* sizes; int64_t err;
    const uint8_t* prefix; size_t prefix_len;
} job;

static void* compress_worker(void* arg) {
    job* j = (job*)arg;
    void* cctx = Z.createCCtx();
    Z.CCtx_setParameter(cctx, ZSTD_c_compressionLevel, j->level);   /* encode.rs:281-284 */
    Z.CCtx_setParameter(cctx, ZSTD_c_checksumFlag, j->checksum);
    size_t stage_sz = Z.CStreamOutSize();
    uint8_t* stage = (uint8_t*)malloc(stage_sz);
    /* contiguous frame ranges per thread, as a fair parallel CPU user would do */
    uint32_t per = (j->n_frames + j->nthreads - 1) / j->nthreads;
    uint32_t lo = per * j->tid, hi = lo + per > j->n_frames ? j->n_frames : lo + per;
    for (uint32_t f = lo; f < hi; f++) {
        size_t off = (size_t)f * j->frame_size;
        size_t len = j->n - off < j->frame_size ? j->n - off : j->frame_size;
        int64_t r = compress_one_frame(cctx, j->src + off, len, j->dst + (size_t)f * j->slot, j->slot, stage, stage_sz, j->prefix, j->prefix_len);
        j->sizes[f] = r;
        if (r < 0) { j->err = r; break; }
    }
    free(stage); Z.freeCCtx(cctx);
    return NULL;
}

static void* decompress_worker(void* arg) {
    job* j = (job*)arg;
    void* dctx = Z.createDCtx();
    size_t in_chunk = Z.DStreamInSize(), out_chunk = Z.DStreamOutSize();
    uint32_t per = (j->n_frames + j->nthreads - 1) / j->nthreads;
    uint32_t lo = per * j->tid, hi = lo + per > j->n_frames ? j->n_frames : lo + per;
    for (uint32_t f = lo; f < hi; f++) {
        int64_t r = decompress_one_frame(dctx, j->src + j->c_off[f], (size_t)(j->c_off[f + 1] - j->c_off[f]),
                                         j->dst + j->d_off[f], (size_t)(j->d_off[f + 1] - j->d_off[f]), in_chunk, out_chunk, j->prefix, j->prefix_len);
        j->sizes[f] = r;
        if (r < 0 && !j->err) j->err = r;
    }
    Z.freeDCtx(dctx);
    return NULL;
}

static void run(void* (*fn)(void*), job* proto, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    job* jobs = (job*)calloc((size_t)nthreads, sizeof(job));
    pthread_t* th = (pthread_t*)calloc((size_t)nthreads, sizeof(pthread_t));
    for (int t = 0; t < nthreads; t++) { jobs[t] = *proto; jobs[t].tid = t; jobs[t].nthreads = nthreads; }
    if (nthreads == 1) fn(&jobs[0]);
    else {
        for (int t = 0; t < nthreads; t++) pthread_create(&th[t], NULL, fn, &jobs[t]);
        for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
    }
    for (int t = 0; t < nthreads; t++) if (jobs[t].err && !proto->err) proto->err = jobs[t].err;
    free(jobs); free(th);
}

/*
 * Compress src into ceil(n/frame_size) independent frames (FrameSizePolicy::Uncompressed,
 * encode.rs:528-544).  Frame f lands at dst + f*slot (slot >= zkr_compress_bound(frame_size));
 * sizes[f] = compressed size.  Returns 0 or -(libzstd code).
 */
int64_t zkr_compress_frames(const uint8_t* src, size_t n, uint32_t frame_size, int level, int checksum,
                            uint8_t* dst, size_t slot, int64_t* sizes, uint32_t n_frames, int nthreads) {
    job j; memset(&j, 0, sizeof j);
    j.src = src; j.n = n; j.frame_size = frame_size; j.level = level; j.checksum = checksum;
    j.dst = dst; j.slot = slot; j.sizes = sizes; j.n_frames = n_frames;
    run(compress_worker, &j, nthreads);
    return j.err;
}

/* Decompress frames described by cumulative offsets (the seek table's N+1 entries, seek_table.rs:97-101).
 * sizes[f] = bytes produced or -(code).  Returns 0 or first error. */
int64_t zkr_decompress_frames(const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off, uint32_t n_frames,
                              uint8_t* dst, int64_t* sizes, int nthreads) {
    job j; memset(&j, 0, sizeof j);
    j.src = comp; j.c_off = c_off; j.d_off = d_off; j.n_frames = n_frames; j.dst = dst; j.sizes = sizes;
    run(decompress_worker, &j, nthreads);
    return j.err;
}

/* Decompress an arbitrary buffer of concatenated frames into dst (cap bytes); returns size or -(code). */
int64_t zkr_decompress_any(const uint8_t* comp, size_t n, uint8_t* dst, size_t cap) {
    void* dctx = Z.createDCtx();
    int64_t r = decompress_one_frame(dctx, comp, n, dst, cap, Z.DStreamInSize(), Z.DStreamOutSize(), NULL, 0);
    Z.freeDCtx(dctx);
    return r;
}

/* The two frame loops again, every frame with the same raw-content prefix (compress_with_prefix / decompress_with_prefix). */
int64_t zkr_compress_frames_prefix(const uint8_t* src, size_t n, uint32_t frame_size, int level, int checksum,
                                   uint8_t* dst, size_t slot, int64_t* sizes, uint32_t n_frames, int nthreads,
                                   const uint8_t* prefix, size_t prefix_len) {
    job j; memset(&j, 0, sizeof j);
    j.src = src; j.n = n; j.frame_size = frame_size; j.level = level; j.checksum = checksum;
    j.dst = dst; j.slot = slot; j.sizes = sizes; j.n_frames = n_frames; j.prefix = prefix; j.prefix_len = prefix_len;
    run(compress_worker, &j, nthreads);
    return j.err;
}
int64_t zkr_decompress_frames_prefix(const uint8_t* comp, const uint64_t* c_off, const uint64_t* d_off, uint32_t n_frames,
                                     uint8_t* dst, int64_t* sizes, int nthreads, const uint8_t* prefix, size_t prefix_len) {
    job j; memset(&j, 0, sizeof j);
    j.src = comp; j.c_off = c_off; j.d_off = d_off; j.n_frames = n_frames; j.dst = dst; j.sizes = sizes;
    j.prefix = prefix; j.prefix_len = prefix_len;
    run(decompress_worker, &j, nthreads);
    return j.err;
}

/* ZSTD_compress(): one-shot frame with a pledged size -> Frame_Content_Size (and Single_Segment when it fits the window). */
int64_t zkr_compress_simple(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int level) {
    size_t r = Z.compress(dst, cap, src, n, level);
    if (Z.isError(r)) return -(int64_t)Z.getErrorCode(r);
    return (int64_t)r;
}
