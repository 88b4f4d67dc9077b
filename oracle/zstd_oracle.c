/*
 * oracle/zstd_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C, serial, readable restatement of the Zstandard frame decoder
 * (RFC 8878) -- the arithmetic that rorosen/zeekstd reaches through
 *   lib/src/decode.rs:243-245   dctx.decompress_stream(...)
 * i.e. libzstd 1.5.7 (zstd-sys 2.0.16+zstd.1.5.7, Cargo.lock:1192-1198),
 * whose sources are NOT in the reference tree.  It is written from the format
 * rules restated in SURVEY.md Appendix A and pinned (tests/test_oracle.py)
 * against the real libzstd in the image (oracle/libzstd_driver.c) on the
 * reference's own fixture (assets/dickens.txt -> tests/golden/) and on
 * generated corpora.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline leg may link or call this file.  The product library
 * (zeekstd_b200/csrc) never does.
 *
 * Error convention: functions return >= 0 on success or -(libzstd error code)
 * so results can be compared with ZSTD_getErrorCode():
 *   10 prefix_unknown, 14 frameParameter_unsupported, 16 windowTooLarge,
 *   20 corruption_detected, 22 checksum_wrong, 32 dictionary_wrong,
 *   70 dstSize_tooSmall, 72 srcSize_wrong.
 */
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <stdlib.h>

#define ZE_PREFIX_UNKNOWN 10
#define ZE_FRAMEPARAM_UNSUPPORTED 14
#define ZE_WINDOW_TOO_LARGE 16
#define ZE_CORRUPTION 20
#define ZE_CHECKSUM_WRONG 22
#define ZE_DICT_CORRUPTED 30   /* libzstd: Treeless literals with no Huffman table yet (ZSTD_decodeLiteralsBlock: litEntropy == 0) */
#define ZE_DICT_WRONG 32
#define ZE_DST_TOO_SMALL 70
#define ZE_SRC_SIZE_WRONG 72

#define FAIL(code) return -(int64_t)(code)

/* ------------------------------------------------------------------ XXH64 */
/* SURVEY.md A.8; seed-0 content checksum of a frame = low 32 bits. */
static const uint64_t P1 = 0x9E3779B185EBCA87ULL, P2 = 0xC2B2AE3D27D4EB4FULL,
                      P3 = 0x165667B19E3779F9ULL, P4 = 0x85EBCA77C2B2AE63ULL,
                      P5 = 0x27D4EB2F165667C5ULL;
static uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
static uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
static uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint64_t xx_round(uint64_t acc, uint64_t in) { return rotl64(acc + in * P2, 31) * P1; }
static uint64_t xx_merge(uint64_t h, uint64_t v) { return (h ^ xx_round(0, v)) * P1 + P4; }

uint64_t zko_xxh64(const uint8_t* p, size_t len, uint64_t seed) {
    const uint8_t* end = p + len;
    uint64_t h;
    if (len >= 32) {
        uint64_t v1 = seed + P1 + P2, v2 = seed + P2, v3 = seed, v4 = seed - P1;
        const uint8_t* lim = end - 32;
        do {
            v1 = xx_round(v1, rd64(p));      v2 = xx_round(v2, rd64(p + 8));
            v3 = xx_round(v3, rd64(p + 16)); v4 = xx_round(v4, rd64(p + 24));
            p += 32;
        } while (p <= lim);
        h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
        h = xx_merge(h, v1); h = xx_merge(h, v2); h = xx_merge(h, v3); h = xx_merge(h, v4);
    } else {
        h = seed + P5;
    }
    h += (uint64_t)len;
    while (p + 8 <= end) { h ^= xx_round(0, rd64(p)); h = rotl64(h, 27) * P1 + P4; p += 8; }
    if (p + 4 <= end) { h ^= (uint64_t)rd32(p) * P1; h = rotl64(h, 23) * P2 + P3; p += 4; }
    while (p < end) { h ^= (*p) * P5; h = rotl64(h, 11) * P1; p++; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

/* ------------------------------------------------- backward bit reader A.7 */
typedef struct {
    const uint8_t* base; /* first byte of the stream */
    int64_t pos;         /* number of unread bits below the cursor; may go < 0 */
} bbits;

/* bit i of the stream (i < 0 reads as 0: over-read yields zeros) */
static inline uint32_t bb_bit(const bbits* b, int64_t i) {
    if (i < 0) return 0;
    return (b->base[i >> 3] >> (i & 7)) & 1u;
}
/* returns 0 on success */
static int bb_init(bbits* b, const uint8_t* p, size_t n) {
    if (n == 0) return -1;
    uint8_t last = p[n - 1];
    if (last == 0) return -1;
    int hb = 7; while (!((last >> hb) & 1)) hb--;
    b->base = p; b->pos = (int64_t)(n - 1) * 8 + hb;
    return 0;
}
static inline uint32_t bb_peek(const bbits* b, int n) { /* n <= 32; top n bits below cursor */
    uint32_t v = 0;
    for (int k = 0; k < n; k++) v = (v << 1) | bb_bit(b, b->pos - 1 - k);
    return v;
}
static inline uint32_t bb_read(bbits* b, int n) { uint32_t v = bb_peek(b, n); b->pos -= n; return v; }

/* --------------------------------------------------- forward bit reader A.6 */
typedef struct { const uint8_t* p; size_t n; size_t bit; } fbits;
static inline uint32_t fb_peek(const fbits* f, int n) {
    uint32_t v = 0;
    for (int k = 0; k < n; k++) {
        size_t i = f->bit + k;
        uint32_t bit = (i >> 3) < f->n ? (f->p[i >> 3] >> (i & 7)) & 1u : 0;
        v |= bit << k;
    }
    return v;
}

/* ------------------------------------------------------------ FSE tables A.6 */
typedef struct { uint8_t sym; uint8_t nb; uint16_t base; } fse_cell;
typedef struct { int log; fse_cell cell[512]; } fse_table;

/* Parse a normalized-count description. Returns bytes consumed or <0. */
static int64_t fse_read_ncount(const uint8_t* p, size_t n, int max_log, int max_sym,
                               int16_t* count, int* nsym, int* log_out) {
    fbits f = { p, n, 0 };
    if (n < 1) FAIL(ZE_CORRUPTION);
    int al = 5 + (int)fb_peek(&f, 4); f.bit += 4;
    if (al > max_log) FAIL(ZE_CORRUPTION);
    int remaining = (1 << al) + 1, threshold = 1 << al, nb = al + 1, s = 0;
    while (remaining > 1 && s <= max_sym) {
        int max = 2 * threshold - 1 - remaining, v;
        uint32_t lo = fb_peek(&f, nb - 1);
        if ((int)lo < max) { v = (int)lo; f.bit += nb - 1; }
        else {
            v = (int)fb_peek(&f, nb);
            if (v >= threshold) v -= max;
            f.bit += nb;
        }
        int c = v - 1;
        remaining -= c < 0 ? -c : c;
        count[s++] = (int16_t)c;
        if (c == 0) {
            for (;;) {
                int r = (int)fb_peek(&f, 2); f.bit += 2;
                for (int k = 0; k < r && s <= max_sym; k++) count[s++] = 0;
                if (r != 3) break;
            }
        }
        while (remaining < threshold) { nb--; threshold >>= 1; }
        if ((f.bit >> 3) > n) FAIL(ZE_CORRUPTION);
    }
    if (remaining != 1) FAIL(ZE_CORRUPTION);
    if (s > max_sym + 1) FAIL(ZE_CORRUPTION);
    size_t used = (f.bit + 7) >> 3;
    if (used > n) FAIL(ZE_CORRUPTION);
    *nsym = s; *log_out = al;
    return (int64_t)used;
}

static int fse_build(fse_table* t, const int16_t* count, int nsym, int log) {
    int S = 1 << log, high = S - 1;
    uint16_t next[256];
    uint8_t symof[512];
    for (int s = 0; s < nsym; s++) {
        if (count[s] == -1) { symof[high--] = (uint8_t)s; next[s] = 1; }
        else next[s] = (uint16_t)count[s];
    }
    int step = (S >> 1) + (S >> 3) + 3, pos = 0;
    for (int s = 0; s < nsym; s++) {
        for (int k = 0; k < count[s]; k++) {
            symof[pos] = (uint8_t)s;
            do { pos = (pos + step) & (S - 1); } while (pos > high);
        }
    }
    if (pos != 0) return -1;
    t->log = log;
    for (int u = 0; u < S; u++) {
        int s = symof[u];
        uint32_t x = next[s]++;
        int hb = 31; while (!((x >> hb) & 1)) hb--;
        int nb = log - hb;
        t->cell[u].sym = (uint8_t)s;
        t->cell[u].nb = (uint8_t)nb;
        t->cell[u].base = (uint16_t)((x << nb) - S);
    }
    return 0;
}
static void fse_build_rle(fse_table* t, int sym) {
    t->log = 0; t->cell[0].sym = (uint8_t)sym; t->cell[0].nb = 0; t->cell[0].base = 0;
}

/* ---------------------------------------------------------- Huffman A.4 */
typedef struct { int max_bits; uint8_t sym[2048]; uint8_t nb[2048]; int valid; } huf_table;

static int64_t huf_read_table(huf_table* h, const uint8_t* p, size_t n) {
    uint8_t w[256]; int nw = 0;
    if (n < 1) FAIL(ZE_CORRUPTION);
    int hb = p[0]; size_t used;
    if (hb >= 128) {
        nw = hb - 127; used = 1 + (size_t)(nw + 1) / 2;
        if (used > n) FAIL(ZE_CORRUPTION);
        for (int i = 0; i < nw; i++) {
            uint8_t b = p[1 + i / 2];
            w[i] = (i & 1) ? (b & 15) : (b >> 4);
        }
    } else {
        used = 1 + (size_t)hb;
        if (hb == 0 || used > n) FAIL(ZE_CORRUPTION);
        int16_t cnt[16]; int ns, log;
        int64_t r = fse_read_ncount(p + 1, (size_t)hb, 6, 12, cnt, &ns, &log);
        if (r < 0) return r;
        fse_table t;
        if (fse_build(&t, cnt, ns, log)) FAIL(ZE_CORRUPTION);
        bbits b;
        if (bb_init(&b, p + 1 + r, (size_t)hb - (size_t)r)) FAIL(ZE_CORRUPTION);
        uint32_t s1 = bb_read(&b, log), s2 = bb_read(&b, log);
        for (;;) { /* two interleaved states; over-read detection per A.4 */
            if (nw >= 254) FAIL(ZE_CORRUPTION);
            w[nw++] = t.cell[s1].sym;
            s1 = t.cell[s1].base + bb_read(&b, t.cell[s1].nb);
            if (b.pos < 0) { w[nw++] = t.cell[s2].sym; break; }
            if (nw >= 255) FAIL(ZE_CORRUPTION);
            w[nw++] = t.cell[s2].sym;
            s2 = t.cell[s2].base + bb_read(&b, t.cell[s2].nb);
            if (b.pos < 0) { w[nw++] = t.cell[s1].sym; break; }
        }
    }
    uint32_t total = 0;
    for (int i = 0; i < nw; i++) { if (w[i] > 11) FAIL(ZE_CORRUPTION); if (w[i]) total += 1u << (w[i] - 1); }
    if (total == 0) FAIL(ZE_CORRUPTION);
    int max_bits = 0; while ((1u << max_bits) <= total) max_bits++;   /* bit_length(total) */
    if (max_bits > 11) FAIL(ZE_CORRUPTION);
    uint32_t left = (1u << max_bits) - total;
    if (left == 0 || (left & (left - 1))) FAIL(ZE_CORRUPTION);
    int lw = 0; while ((1u << lw) < left) lw++;
    w[nw++] = (uint8_t)(lw + 1);
    /* fill: weight ascending, symbols in natural order */
    int pos = 0;
    for (int wt = 1; wt <= max_bits; wt++)
        for (int s = 0; s < nw; s++)
            if (w[s] == wt) {
                int len = 1 << (wt - 1);
                for (int k = 0; k < len; k++) { h->sym[pos + k] = (uint8_t)s; h->nb[pos + k] = (uint8_t)(max_bits + 1 - wt); }
                pos += len;
            }
    if (pos != (1 << max_bits)) FAIL(ZE_CORRUPTION);
    h->max_bits = max_bits; h->valid = 1;
    return (int64_t)used;
}

static int huf_decode_stream(const huf_table* h, const uint8_t* p, size_t n, uint8_t* out, size_t count) {
    bbits b;
    if (bb_init(&b, p, n)) return -1;
    for (size_t i = 0; i < count; i++) {
        uint32_t idx = bb_peek(&b, h->max_bits);
        out[i] = h->sym[idx];
        b.pos -= h->nb[idx];
    }
    return b.pos == 0 ? 0 : -1;
}

/* ------------------------------------------------------- sequence codes A.5 */
static const uint32_t LL_BASE[36] = {0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,18,20,22,24,28,32,40,48,64,128,256,512,1024,2048,4096,8192,16384,32768,65536};
static const uint8_t LL_BITS[36] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,6,7,8,9,10,11,12,13,14,15,16};
static const uint32_t ML_BASE[53] = {3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,19,20,21,22,23,24,25,26,27,28,29,30,31,32,33,34,35,37,39,41,43,47,51,59,67,83,99,131,259,515,1027,2051,4099,8195,16387,32771,65539};
static const uint8_t ML_BITS[53] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,4,5,7,8,9,10,11,12,13,14,15,16};
static const int16_t LL_DEFAULT[36] = {4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1};
static const int16_t ML_DEFAULT[53] = {1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1};
static const int16_t OF_DEFAULT[29] = {1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1};

/* Sequence-level statistics of a decode (tests: which repeat-offset cases / offset ranges an archive exercises). */
typedef struct {
    uint64_t rep_idx[4];        /* repeat-offset uses by resolved index: 0 rep1, 1 rep2, 2 rep3, 3 rep1-1 (code 3 with litLen == 0) */
    uint64_t rep_ll0;           /* repeat codes met with litLen == 0 (index shifted by one) */
    uint64_t overlap;           /* matches with offset < matchLength */
    uint64_t explicit_offsets;
    uint64_t max_offset;        /* largest match distance */
    uint64_t prefix_matches;    /* matches reaching before the start of the frame (only legal with a prefix) */
} zko_seq_stats;
static __thread zko_seq_stats* g_ss = NULL;
static __thread const uint8_t* g_prefix = NULL; static __thread size_t g_prefix_len = 0;

/* per-frame decoding context (entropy tables persist across blocks of a frame) */
typedef struct {
    huf_table huf;
    fse_table ll, of, ml;
    int have_ll, have_of, have_ml;
    uint32_t rep[3];
    uint64_t window;
    const uint8_t* prefix; size_t prefix_len;   /* raw-content prefix (ZSTD_DCtx_refPrefix; decode.rs:211-214): history before the frame */
} frame_ctx;

static int64_t read_seq_table(fse_table* t, int* have, int mode, const uint8_t* p, size_t n,
                              int max_log, int max_sym, const int16_t* def, int def_n, int def_log) {
    int16_t cnt[64]; int ns, log;
    switch (mode) {
    case 0: if (fse_build(t, def, def_n, def_log)) FAIL(ZE_CORRUPTION); *have = 1; return 0;
    case 1: if (n < 1) FAIL(ZE_CORRUPTION); if (p[0] > max_sym) FAIL(ZE_CORRUPTION);
            fse_build_rle(t, p[0]); *have = 1; return 1;
    case 2: {
        int64_t r = fse_read_ncount(p, n, max_log, max_sym, cnt, &ns, &log);
        if (r < 0) return r;
        if (fse_build(t, cnt, ns, log)) FAIL(ZE_CORRUPTION);
        *have = 1; return r;
    }
    default: if (!*have) FAIL(ZE_CORRUPTION); return 0;
    }
}

/* Decode one Compressed block. out_base = start of this frame's output. */
static int64_t decode_compressed_block(frame_ctx* fc, const uint8_t* p, size_t n,
                                       uint8_t* out_base, size_t out_pos, size_t out_cap) {
    static uint8_t litbuf[1 << 17];
    if (n < 2) FAIL(ZE_CORRUPTION);
    /* --- literals section A.3 */
    int ltype = p[0] & 3, sf = (p[0] >> 2) & 3;
    size_t hdr, regen, comp = 0; int streams = 1;
    if (ltype < 2) {
        if (sf == 0 || sf == 2) { hdr = 1; regen = p[0] >> 3; }
        else if (sf == 1) { hdr = 2; regen = ((size_t)p[0] >> 4) | ((size_t)p[1] << 4); }
        else { if (n < 3) FAIL(ZE_CORRUPTION); hdr = 3; regen = ((size_t)p[0] >> 4) | ((size_t)p[1] << 4) | ((size_t)p[2] << 12); }
    } else {
        if (n < 5) FAIL(ZE_CORRUPTION);
        uint64_t v = (uint64_t)p[0] | ((uint64_t)p[1] << 8) | ((uint64_t)p[2] << 16) | ((uint64_t)p[3] << 24) | ((uint64_t)p[4] << 32);
        if (sf == 0) { hdr = 3; streams = 1; regen = (v >> 4) & 0x3FF; comp = (v >> 14) & 0x3FF; }
        else if (sf == 1) { hdr = 3; streams = 4; regen = (v >> 4) & 0x3FF; comp = (v >> 14) & 0x3FF; }
        else if (sf == 2) { hdr = 4; streams = 4; regen = (v >> 4) & 0x3FFF; comp = (v >> 18) & 0x3FFF; }
        else { hdr = 5; streams = 4; regen = (v >> 4) & 0x3FFFF; comp = (v >> 22) & 0x3FFFF; }
    }
    if (regen > (1u << 17)) FAIL(ZE_CORRUPTION);
    const uint8_t* lit; size_t lsec;
    if (ltype == 0) { lsec = hdr + regen; if (lsec > n) FAIL(ZE_CORRUPTION); lit = p + hdr; }
    else if (ltype == 1) { lsec = hdr + 1; if (lsec > n) FAIL(ZE_CORRUPTION); memset(litbuf, p[hdr], regen); lit = litbuf; }
    else {
        lsec = hdr + comp; if (lsec > n) FAIL(ZE_CORRUPTION);
        const uint8_t* q = p + hdr; size_t qn = comp;
        if (ltype == 2) {
            int64_t r = huf_read_table(&fc->huf, q, qn);
            if (r < 0) return r;
            q += r; qn -= (size_t)r;
        } else if (!fc->huf.valid) FAIL(ZE_DICT_CORRUPTED);
        if (streams == 1) {
            if (huf_decode_stream(&fc->huf, q, qn, litbuf, regen)) FAIL(ZE_CORRUPTION);
        } else {
            if (qn < 6) FAIL(ZE_CORRUPTION);
            size_t s1 = q[0] | (q[1] << 8), s2 = q[2] | (q[3] << 8), s3 = q[4] | (q[5] << 8);
            if (6 + s1 + s2 + s3 > qn) FAIL(ZE_CORRUPTION);
            size_t s4 = qn - 6 - s1 - s2 - s3, seg = (regen + 3) / 4;
            if (seg * 3 > regen) FAIL(ZE_CORRUPTION);
            const uint8_t* d = q + 6;
            if (huf_decode_stream(&fc->huf, d, s1, litbuf, seg)) FAIL(ZE_CORRUPTION);
            if (huf_decode_stream(&fc->huf, d + s1, s2, litbuf + seg, seg)) FAIL(ZE_CORRUPTION);
            if (huf_decode_stream(&fc->huf, d + s1 + s2, s3, litbuf + 2 * seg, seg)) FAIL(ZE_CORRUPTION);
            if (huf_decode_stream(&fc->huf, d + s1 + s2 + s3, s4, litbuf + 3 * seg, regen - 3 * seg)) FAIL(ZE_CORRUPTION);
        }
        lit = litbuf;
    }
    /* --- sequences section A.5 */
    const uint8_t* s = p + lsec; size_t sn = n - lsec;
    if (sn < 1) FAIL(ZE_CORRUPTION);
    size_t nseq, sh;
    if (s[0] < 128) { nseq = s[0]; sh = 1; }
    else if (s[0] < 255) { if (sn < 2) FAIL(ZE_CORRUPTION); nseq = ((size_t)(s[0] - 128) << 8) + s[1]; sh = 2; }
    else { if (sn < 3) FAIL(ZE_CORRUPTION); nseq = (size_t)s[1] + ((size_t)s[2] << 8) + 0x7F00; sh = 3; }
    size_t start = out_pos, lpos = 0;
    if (nseq == 0) {
        if (sh != sn) FAIL(ZE_CORRUPTION);
        if (out_pos + regen > out_cap) FAIL(ZE_DST_TOO_SMALL);
        memcpy(out_base + out_pos, lit, regen);
        return (int64_t)regen;
    }
    if (sn < sh + 1) FAIL(ZE_CORRUPTION);
    int modes = s[sh];
    if (modes & 3) FAIL(ZE_CORRUPTION);
    const uint8_t* t = s + sh + 1; size_t tn = sn - sh - 1;
    int64_t r;
    r = read_seq_table(&fc->ll, &fc->have_ll, (modes >> 6) & 3, t, tn, 9, 35, LL_DEFAULT, 36, 6); if (r < 0) return r; t += r; tn -= (size_t)r;
    r = read_seq_table(&fc->of, &fc->have_of, (modes >> 4) & 3, t, tn, 8, 31, OF_DEFAULT, 29, 5); if (r < 0) return r; t += r; tn -= (size_t)r;
    r = read_seq_table(&fc->ml, &fc->have_ml, (modes >> 2) & 3, t, tn, 9, 52, ML_DEFAULT, 53, 6); if (r < 0) return r; t += r; tn -= (size_t)r;
    bbits b;
    if (bb_init(&b, t, tn)) FAIL(ZE_CORRUPTION);
    uint32_t sl = bb_read(&b, fc->ll.log), so = bb_read(&b, fc->of.log), sm = bb_read(&b, fc->ml.log);
    if (b.pos < 0) FAIL(ZE_CORRUPTION);
    for (size_t i = 0; i < nseq; i++) {
        int oc = fc->of.cell[so].sym, mc = fc->ml.cell[sm].sym, lc = fc->ll.cell[sl].sym;
        if (oc > 31 || mc > 52 || lc > 35) FAIL(ZE_CORRUPTION);
        uint32_t ov = (1u << oc) + bb_read(&b, oc);
        uint32_t mlen = ML_BASE[mc] + bb_read(&b, ML_BITS[mc]);
        uint32_t llen = LL_BASE[lc] + bb_read(&b, LL_BITS[lc]);
        if (i + 1 < nseq) {
            sl = fc->ll.cell[sl].base + bb_read(&b, fc->ll.cell[sl].nb);
            sm = fc->ml.cell[sm].base + bb_read(&b, fc->ml.cell[sm].nb);
            so = fc->of.cell[so].base + bb_read(&b, fc->of.cell[so].nb);
        }
        if (b.pos < 0) FAIL(ZE_CORRUPTION);
        /* repeat offsets */
        uint32_t off;
        if (ov > 3) { off = ov - 3; fc->rep[2] = fc->rep[1]; fc->rep[1] = fc->rep[0]; fc->rep[0] = off; if (g_ss) g_ss->explicit_offsets++; }
        else {
            uint32_t idx = ov - 1 + (llen == 0);
            if (g_ss) { g_ss->rep_idx[idx]++; g_ss->rep_ll0 += llen == 0; }
            if (idx == 0) off = fc->rep[0];
            else {
                off = idx == 3 ? fc->rep[0] - 1 : fc->rep[idx];
                if (off == 0) FAIL(ZE_CORRUPTION);
                if (idx != 1) fc->rep[2] = fc->rep[1];
                fc->rep[1] = fc->rep[0]; fc->rep[0] = off;
            }
        }
        /* execute */
        if (lpos + llen > regen) FAIL(ZE_CORRUPTION);
        if (out_pos + llen + mlen > out_cap) FAIL(ZE_DST_TOO_SMALL);
        memcpy(out_base + out_pos, lit + lpos, llen); lpos += llen; out_pos += llen;
        if (off > out_pos + fc->prefix_len) FAIL(ZE_CORRUPTION);
        if (g_ss) { g_ss->overlap += off < mlen; if (off > g_ss->max_offset) g_ss->max_offset = off; g_ss->prefix_matches += off > out_pos; }
        for (uint32_t k = 0; k < mlen; k++) {
            size_t at = out_pos + k;
            out_base[at] = at >= off ? out_base[at - off] : fc->prefix[fc->prefix_len - (off - at)];
        }
        out_pos += mlen;
    }
    if (b.pos != 0) FAIL(ZE_CORRUPTION);
    size_t rest = regen - lpos;
    if (out_pos + rest > out_cap) FAIL(ZE_DST_TOO_SMALL);
    memcpy(out_base + out_pos, lit + lpos, rest); out_pos += rest;
    if (out_pos - start > (1u << 17)) FAIL(ZE_CORRUPTION);
    return (int64_t)(out_pos - start);
}

/* Decode ONE zstd frame at src. *consumed = compressed bytes used. Returns bytes written or <0. */
static int64_t decode_one_frame(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* consumed, int verify) {
    if (n < 5) FAIL(ZE_SRC_SIZE_WRONG);
    if (rd32(src) != 0xFD2FB528u) FAIL(ZE_PREFIX_UNKNOWN);
    uint8_t fhd = src[4];
    int fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, csum = (fhd >> 2) & 1, did = fhd & 3;
    if (fhd & 0x08) FAIL(ZE_FRAMEPARAM_UNSUPPORTED);
    size_t pos = 5;
    frame_ctx* fc = (frame_ctx*)calloc(1, sizeof(frame_ctx));
    if (!fc) FAIL(64);
    fc->rep[0] = 1; fc->rep[1] = 4; fc->rep[2] = 8;
    fc->prefix = g_prefix; fc->prefix_len = g_prefix ? g_prefix_len : 0;   /* re-applied to every frame (decode.rs:246-255) */
    int64_t rc = 0;
#define FFAIL(code) do { rc = -(int64_t)(code); goto done; } while (0)
    if (!single) {
        if (pos >= n) FFAIL(ZE_SRC_SIZE_WRONG);
        uint8_t wd = src[pos++];
        int wlog = 10 + (wd >> 3);
        if (wlog > 31) FFAIL(ZE_WINDOW_TOO_LARGE);
        fc->window = (1ULL << wlog) + ((1ULL << wlog) >> 3) * (wd & 7);
    }
    {
        static const int did_sz[4] = {0, 1, 2, 4};
        uint32_t dict = 0;
        if (pos + did_sz[did] > n) FFAIL(ZE_SRC_SIZE_WRONG);
        for (int k = 0; k < did_sz[did]; k++) dict |= (uint32_t)src[pos + k] << (8 * k);
        pos += did_sz[did];
        if (dict != 0) FFAIL(ZE_DICT_WRONG);
    }
    uint64_t fcs = 0; int have_fcs = 0;
    {
        int fsz = fcs_flag == 0 ? (single ? 1 : 0) : fcs_flag == 1 ? 2 : fcs_flag == 2 ? 4 : 8;
        if (pos + fsz > n) FFAIL(ZE_SRC_SIZE_WRONG);
        for (int k = 0; k < fsz; k++) fcs |= (uint64_t)src[pos + k] << (8 * k);
        if (fsz == 2) fcs += 256;
        pos += fsz; have_fcs = fsz > 0;
        if (single) fc->window = fcs;
        /* ZSTD_decompressStream with a default DCtx (what the reference's Decoder holds, decode.rs:130-133) refuses windows above
         * (1 << ZSTD_WINDOWLOG_LIMIT_DEFAULT) + 1 = 2^27 + 1 once the header is decoded */
        if (fc->window > (1ULL << 27) + 1) FFAIL(ZE_WINDOW_TOO_LARGE);
    }
    size_t out = 0;
    /* Block_Maximum_Size = min(Window_Size, 128 KiB), RFC 8878 3.1.1.2.3; libzstd: "Block Size Exceeds Maximum" for the content
     * of a block, "Decompressed Block Size Exceeds Maximum" for what it regenerates (ZSTD_decompressContinue) */
    const size_t bmax = fc->window < (1u << 17) ? (size_t)fc->window : (1u << 17);
    for (;;) {
        if (pos + 3 > n) FFAIL(ZE_SRC_SIZE_WRONG);
        uint32_t bh = src[pos] | (src[pos + 1] << 8) | ((uint32_t)src[pos + 2] << 16);
        pos += 3;
        int last = bh & 1, type = (bh >> 1) & 3; size_t bsz = bh >> 3;
        if (type == 3) FFAIL(ZE_CORRUPTION);
        if (type == 0) {
            if (bsz > bmax) FFAIL(ZE_CORRUPTION);
            if (pos + bsz > n) FFAIL(ZE_SRC_SIZE_WRONG);
            if (out + bsz > cap) FFAIL(ZE_DST_TOO_SMALL);
            memcpy(dst + out, src + pos, bsz); pos += bsz; out += bsz;
        } else if (type == 1) {
            if (bsz > bmax) FFAIL(ZE_CORRUPTION);
            if (pos + 1 > n) FFAIL(ZE_SRC_SIZE_WRONG);
            if (out + bsz > cap) FFAIL(ZE_DST_TOO_SMALL);
            memset(dst + out, src[pos], bsz); pos += 1; out += bsz;
        } else {
            if (bsz > bmax) FFAIL(ZE_CORRUPTION);
            if (pos + bsz > n) FFAIL(ZE_SRC_SIZE_WRONG);
            int64_t r = decode_compressed_block(fc, src + pos, bsz, dst, out, cap);
            if (r < 0) { rc = r; goto done; }
            if ((size_t)r > bmax) FFAIL(ZE_CORRUPTION);
            pos += bsz; out += (size_t)r;
        }
        if (last) break;
    }
    if (have_fcs && fcs != out) FFAIL(ZE_CORRUPTION);
    if (csum) {
        if (pos + 4 > n) FFAIL(ZE_SRC_SIZE_WRONG);
        if (verify && rd32(src + pos) != (uint32_t)zko_xxh64(dst, out, 0)) FFAIL(ZE_CHECKSUM_WRONG);
        pos += 4;
    }
    *consumed = pos; rc = (int64_t)out;
done:
    free(fc);
    return rc;
}

/*
 * Decode every frame (zstd or skippable) found in src[0..n).  This is what
 * ZSTD_decompressStream does when the reference feeds it one seek-table
 * entry's worth of bytes (decode.rs:221-256).  Returns bytes written or <0.
 */
int64_t zko_decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int verify_checksum) {
    size_t pos = 0, out = 0;
    while (pos < n) {
        if (n - pos < 4) FAIL(ZE_SRC_SIZE_WRONG);
        uint32_t magic = rd32(src + pos);
        if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {
            if (n - pos < 8) FAIL(ZE_SRC_SIZE_WRONG);
            uint64_t sz = rd32(src + pos + 4);
            if (sz + 8 > n - pos) FAIL(ZE_SRC_SIZE_WRONG);
            pos += 8 + (size_t)sz;
            continue;
        }
        size_t used = 0;
        int64_t r = decode_one_frame(src + pos, n - pos, dst + out, cap - out, &used, verify_checksum);
        if (r < 0) return r;
        pos += used; out += (size_t)r;
    }
    return (int64_t)out;
}

/* zko_decompress with a raw-content prefix for every frame (decompress_with_prefix, decode.rs:201-270) and/or
 * sequence statistics.  prefix / ss may be NULL. */
int64_t zko_decompress_ex(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int verify_checksum,
                          const uint8_t* prefix, size_t prefix_len, zko_seq_stats* ss) {
    if (ss) memset(ss, 0, sizeof *ss);
    g_ss = ss; g_prefix = prefix; g_prefix_len = prefix_len;
    int64_t r = zko_decompress(src, n, dst, cap, verify_checksum);
    g_ss = NULL; g_prefix = NULL; g_prefix_len = 0;
    return r;
}

/* Frame-structure statistics used by tests to confirm coverage of the format matrix (SURVEY.md 8a). */
typedef struct {
    uint32_t n_raw, n_rle, n_comp;              /* block types */
    uint32_t lit_raw, lit_rle, lit_huf, lit_treeless, lit_1stream, lit_4stream;
    uint32_t huf_direct, huf_fse;
    uint32_t mode_predef, mode_rle, mode_fse, mode_repeat; /* summed over LL/OF/ML */
    uint32_t nseq0_blocks;
    uint32_t checksum_frames, single_segment_frames, skippable_frames, zstd_frames;
    uint64_t n_seq;
} zko_stats;

int64_t zko_frame_stats(const uint8_t* src, size_t n, zko_stats* st) {
    memset(st, 0, sizeof *st);
    size_t pos = 0;
    while (pos < n) {
        if (n - pos < 4) FAIL(ZE_SRC_SIZE_WRONG);
        uint32_t magic = rd32(src + pos);
        if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {
            if (n - pos < 8) FAIL(ZE_SRC_SIZE_WRONG);
            uint64_t sz = rd32(src + pos + 4);
            if (sz + 8 > n - pos) FAIL(ZE_SRC_SIZE_WRONG);
            pos += 8 + (size_t)sz; st->skippable_frames++; continue;
        }
        if (magic != 0xFD2FB528u) FAIL(ZE_PREFIX_UNKNOWN);
        if (n - pos < 6) FAIL(ZE_SRC_SIZE_WRONG);
        st->zstd_frames++;
        uint8_t fhd = src[pos + 4];
        int fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, csum = (fhd >> 2) & 1, did = fhd & 3;
        static const int did_sz[4] = {0, 1, 2, 4};
        pos += 5 + (single ? 0 : 1) + did_sz[did] + (fcs_flag == 0 ? (single ? 1 : 0) : fcs_flag == 1 ? 2 : fcs_flag == 2 ? 4 : 8);
        st->checksum_frames += csum; st->single_segment_frames += single;
        for (;;) {
            if (pos + 3 > n) FAIL(ZE_SRC_SIZE_WRONG);
            uint32_t bh = src[pos] | (src[pos + 1] << 8) | ((uint32_t)src[pos + 2] << 16);
            pos += 3;
            int last = bh & 1, type = (bh >> 1) & 3; size_t bsz = bh >> 3;
            if (type == 0) { st->n_raw++; pos += bsz; }
            else if (type == 1) { st->n_rle++; pos += 1; }
            else if (type == 2) {
                st->n_comp++;
                if (pos + bsz > n) FAIL(ZE_SRC_SIZE_WRONG);
                const uint8_t* p = src + pos;
                int ltype = p[0] & 3, sf = (p[0] >> 2) & 3; size_t hdr, regen, comp = 0;
                if (ltype < 2) {
                    if (sf == 0 || sf == 2) { hdr = 1; regen = p[0] >> 3; }
                    else if (sf == 1) { hdr = 2; regen = (p[0] >> 4) | ((size_t)p[1] << 4); }
                    else { hdr = 3; regen = (p[0] >> 4) | ((size_t)p[1] << 4) | ((size_t)p[2] << 12); }
                    if (ltype == 0) { st->lit_raw++; comp = regen; } else { st->lit_rle++; comp = 1; }
                } else {
                    uint64_t v = (uint64_t)p[0] | ((uint64_t)p[1] << 8) | ((uint64_t)p[2] << 16) | ((uint64_t)p[3] << 24) | ((uint64_t)p[4] << 32);
                    if (sf == 0) { hdr = 3; comp = (v >> 14) & 0x3FF; st->lit_1stream++; }
                    else if (sf == 1) { hdr = 3; comp = (v >> 14) & 0x3FF; st->lit_4stream++; }
                    else if (sf == 2) { hdr = 4; comp = (v >> 18) & 0x3FFF; st->lit_4stream++; }
                    else { hdr = 5; comp = (v >> 22) & 0x3FFFF; st->lit_4stream++; }
                    if (ltype == 2) { st->lit_huf++; if (p[hdr] >= 128) st->huf_direct++; else st->huf_fse++; }
                    else st->lit_treeless++;
                }
                const uint8_t* s = p + hdr + comp;
                size_t nseq, sh;
                if (s[0] < 128) { nseq = s[0]; sh = 1; }
                else if (s[0] < 255) { nseq = ((size_t)(s[0] - 128) << 8) + s[1]; sh = 2; }
                else { nseq = (size_t)s[1] + ((size_t)s[2] << 8) + 0x7F00; sh = 3; }
                st->n_seq += nseq;
                if (nseq == 0) st->nseq0_blocks++;
                else {
                    int modes = s[sh];
                    for (int sft = 2; sft <= 6; sft += 2) {
                        int m = (modes >> sft) & 3;
                        if (m == 0) st->mode_predef++; else if (m == 1) st->mode_rle++; else if (m == 2) st->mode_fse++; else st->mode_repeat++;
                    }
                }
                pos += bsz;
            } else FAIL(ZE_CORRUPTION);
            if (pos > n) FAIL(ZE_SRC_SIZE_WRONG);
            if (last) break;
        }
        if (csum) pos += 4;
    }
    return 0;
}
