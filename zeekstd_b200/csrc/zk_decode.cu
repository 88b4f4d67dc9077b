// zk_decode.cu -- batched Zstandard frame decode for sm_90a.
//
// Replaces the reference's only decompression call into libzstd,
//   lib/src/decode.rs:243-245   self.dctx.decompress_stream(&mut out_buffer, &mut in_buffer)
// with these kernels over a whole batch of independent seek-table entries ("frames" of the
// seekable format, seekable_format.md:23-29):
//
//   K-D0 zk_scan_kernel        one thread / entry   : walk frame + block headers, carve scratch
//   K-D1s zk_seq2_kernel       one chain / block    : FSE sequence decode (4 chains per warp, TMA-staged bitstreams);
//         zk_seq2_full_kernel                       the same for blocks whose tables need more cells than zk_seq2_kernel holds
//   K-D1h zk_huf_kernel        one LANE  / stream   : Huffman literal decode (4 lanes per 4-stream block, two-level table)
//   K-D0o / K-D1o zk_order_kernel  one CTA / list   : the work lists of K-D1s / K-D1h (after K-D0) and of K-D2 (after K-D1p), heaviest first
//   K-D1p zk_plan_kernel       one warp / entry     : output positions, the serial walk's checks, execution segments
//   K-D2w zk_exec_warp_kernel  one warp / segment   : short segments, strictly in order through a per-warp window
//   K-D2 zk_exec_kernel[_w5]   one CTA  / segment   : long segments, sequence execution through a shared-memory ring
//   K-D3 zk_xxh64_kernel       one warp  / entry    : content checksum (only if requested & present)
// Both executors come in a prefix-mode build (template PREFIX): matches may reach into a raw-content prefix before
// every zstd frame.
//
// Format rules: RFC 8878 as restated in SURVEY.md Appendix A (the arithmetic is not in the
// reference tree).  All integer/byte work; no tensor cores.
#include "zk_common.cuh"
#include "zk_decode.h"
#include <stdio.h>
#include <stdlib.h>

// =============================================================================================
// K-D0: header scan
// =============================================================================================
struct ZkBlkInfo {
    uint32_t src, size; uint8_t type, flags;
    uint32_t lit_size, nseq, bmax; uint8_t lit_type, modes, lit_hdr; uint64_t fcs;
};

struct ZkLitHdr { uint32_t type, hdr, regen, comp, streams; };

// Literals_Section_Header (A.3).  n = bytes available. Returns false if truncated.
__device__ __forceinline__ bool zk_parse_lit_hdr(const uint8_t* p, uint32_t n, ZkLitHdr& h) {
    if (n < 1) return false;
    uint32_t b0 = p[0];
    h.type = b0 & 3; uint32_t sf = (b0 >> 2) & 3;
    h.comp = 0; h.streams = 1;
    if (h.type < 2) {
        if (sf == 0 || sf == 2) { h.hdr = 1; h.regen = b0 >> 3; }
        else if (sf == 1) { if (n < 2) return false; h.hdr = 2; h.regen = (b0 >> 4) | ((uint32_t)p[1] << 4); }
        else { if (n < 3) return false; h.hdr = 3; h.regen = (b0 >> 4) | ((uint32_t)p[1] << 4) | ((uint32_t)p[2] << 12); }
    } else {
        if (n < 5) return false;
        unsigned long long v = (unsigned long long)zk_ld_le32(p) | ((unsigned long long)p[4] << 32);
        if (sf == 0) { h.hdr = 3; h.streams = 1; h.regen = (uint32_t)(v >> 4) & 0x3FF; h.comp = (uint32_t)(v >> 14) & 0x3FF; }
        else if (sf == 1) { h.hdr = 3; h.streams = 4; h.regen = (uint32_t)(v >> 4) & 0x3FF; h.comp = (uint32_t)(v >> 14) & 0x3FF; }
        else if (sf == 2) { h.hdr = 4; h.streams = 4; h.regen = (uint32_t)(v >> 4) & 0x3FFF; h.comp = (uint32_t)(v >> 18) & 0x3FFF; }
        else { h.hdr = 5; h.streams = 4; h.regen = (uint32_t)(v >> 4) & 0x3FFFF; h.comp = (uint32_t)(v >> 22) & 0x3FFFF; }
    }
    return true;
}
__device__ __forceinline__ uint32_t zk_lit_section_size(const ZkLitHdr& h) {
    return h.hdr + (h.type == 0 ? h.regen : h.type == 1 ? 1u : h.comp);
}

// Sequences_Section_Header (A.5): number of sequences.  Returns header bytes (1..3) or 0 if truncated.
__device__ __forceinline__ uint32_t zk_parse_nseq(const uint8_t* s, uint32_t n, uint32_t& nseq) {
    if (n < 1) return 0;
    uint32_t b0 = s[0];
    if (b0 < 128) { nseq = b0; return 1; }
    if (b0 < 255) { if (n < 2) return 0; nseq = ((b0 - 128) << 8) + s[1]; return 2; }
    if (n < 3) return 0;
    nseq = (uint32_t)s[1] + ((uint32_t)s[2] << 8) + 0x7F00u; return 3;
}

// Walks every zstd / skippable frame inside one seek-table entry.  emit(info) is called per block.
template <class Emit>
__device__ int zk_walk_entry(const uint8_t* p, uint32_t n, Emit& emit) {
    uint32_t pos = 0;
    while (pos < n) {
        if (n - pos < 4) return ZKZ_SRC_SIZE_WRONG;
        uint32_t magic = zk_ld_le32(p + pos);
        if ((magic & ZK_SKIPPABLE_MASK) == ZK_SKIPPABLE_MAGIC) {
            if (n - pos < 8) return ZKZ_SRC_SIZE_WRONG;
            uint32_t sz = zk_ld_le32(p + pos + 4);
            if ((unsigned long long)sz + 8ull > (unsigned long long)(n - pos)) return ZKZ_SRC_SIZE_WRONG;
            pos += 8 + sz;
            continue;
        }
        if (magic != ZK_MAGIC) return ZKZ_PREFIX_UNKNOWN;
        if (n - pos < 5) return ZKZ_SRC_SIZE_WRONG;
        uint32_t fhd = p[pos + 4];
        uint32_t fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, csum = (fhd >> 2) & 1, did = fhd & 3;
        if (fhd & 0x08) return ZKZ_FRAMEPARAM_UNSUPPORTED;
        uint32_t did_sz = did == 3 ? 4u : did;
        uint32_t fcs_sz = fcs_flag == 0 ? single : (fcs_flag == 1 ? 2u : (fcs_flag == 2 ? 4u : 8u));
        uint32_t hsz = 5 + (single ? 0 : 1) + did_sz + fcs_sz;
        if (n - pos < hsz) return ZKZ_SRC_SIZE_WRONG;
        uint32_t q = pos + 5;
        unsigned long long window = 0;
        if (!single) {
            const uint32_t wd = p[q++], wlog = 10 + (wd >> 3);
            if (wlog > 31) return ZKZ_WINDOW_TOO_LARGE;                  // ZSTD_WINDOWLOG_MAX, refused while the header is parsed
            window = (1ull << wlog) + ((1ull << wlog) >> 3) * (wd & 7);
        }
        uint32_t dict = 0;
        for (uint32_t i = 0; i < did_sz; i++) dict |= (uint32_t)p[q + i] << (8 * i);
        q += did_sz;
        if (dict != 0) return ZKZ_DICT_WRONG;
        unsigned long long fcs = 0;
        for (uint32_t i = 0; i < fcs_sz; i++) fcs |= (unsigned long long)p[q + i] << (8 * i);
        if (fcs_sz == 2) fcs += 256;
        // the reference decodes with a default DCtx (decode.rs:130-133): streaming decompression refuses windows above
        // 2^ZSTD_WINDOWLOG_LIMIT_DEFAULT (+1), after the dictionary check -- a Single_Segment frame's window is its content size
        if (single) window = fcs;
        if (window > (1ull << 27) + 1) return ZKZ_WINDOW_TOO_LARGE;
        // Block_Maximum_Size = min(Window_Size, 128 KiB) (RFC 8878 3.1.1.2.3): libzstd refuses a block whose content or
        // regenerated size exceeds it (ZSTD_decompressContinue: "Block Size Exceeds Maximum", "Decompressed Block Size Exceeds Maximum")
        const uint32_t bsmax = window < ZK_BLOCK_MAX ? (uint32_t)window : ZK_BLOCK_MAX;
        pos += hsz;
        bool first = true;
        for (;;) {
            if (n - pos < 3) return ZKZ_SRC_SIZE_WRONG;
            uint32_t bh = zk_ld_le24(p + pos);
            uint32_t last = bh & 1, type = (bh >> 1) & 3, bsize = bh >> 3;
            if (type == 3) return ZKZ_CORRUPTION;
            if (bsize > bsmax) return ZKZ_CORRUPTION;
            uint32_t content = type == 1 ? 1u : bsize;
            if (n - pos - 3 < content) return ZKZ_SRC_SIZE_WRONG;
            ZkBlkInfo bi;
            bi.src = pos + 3; bi.size = bsize; bi.type = (uint8_t)type;
            bi.flags = (uint8_t)((first ? ZKB_FIRST : 0) | (last ? ZKB_LAST : 0) | ((last && csum) ? ZKB_HAS_CSUM : 0) |
                                 ((last && fcs_sz) ? ZKB_HAS_FCS : 0));
            bi.fcs = fcs; bi.bmax = bsmax; bi.lit_size = 0; bi.nseq = 0; bi.lit_type = 0; bi.modes = 0; bi.lit_hdr = 0;
            if (type == 2) {
                const uint8_t* b = p + pos + 3;
                if (bsize < 2) return ZKZ_CORRUPTION;
                ZkLitHdr lh;
                if (!zk_parse_lit_hdr(b, bsize, lh)) return ZKZ_CORRUPTION;
                if (lh.regen > bsmax) return ZKZ_CORRUPTION;
                uint32_t lsec = zk_lit_section_size(lh);
                if (lsec >= bsize) return ZKZ_CORRUPTION;          // at least the nseq byte must follow
                uint32_t nseq;
                uint32_t sh = zk_parse_nseq(b + lsec, bsize - lsec, nseq);
                if (sh == 0) return ZKZ_CORRUPTION;
                if (nseq == 0) { if (lsec + sh != bsize) return ZKZ_CORRUPTION; }
                else {
                    if (lsec + sh >= bsize) return ZKZ_CORRUPTION;
                    bi.modes = b[lsec + sh];
                    if (bi.modes & 3) return ZKZ_CORRUPTION;
                }
                bi.lit_size = lh.regen; bi.nseq = nseq; bi.lit_type = (uint8_t)lh.type; bi.lit_hdr = (uint8_t)lh.hdr;
            }
            int rc = emit(bi);
            if (rc) return rc;
            pos += 3 + content;
            first = false;
            if (last) break;
        }
        if (csum) { if (n - pos < 4) return ZKZ_SRC_SIZE_WRONG; pos += 4; }
    }
    return 0;
}

struct ZkCountEmit {
    uint32_t nb = 0, nlit = 0, nseq = 0, nhuf = 0, nsqb = 0;
    // Treeless literals / Repeat_Mode tables must refer to something defined earlier in the same zstd frame.  This is
    // checked HERE so that the fill pass (which reserves slots of huf_list / seq_list from these counts) cannot fail
    // after the count pass succeeded: every reserved work-list slot is always written.
    uint32_t have = 0;            // bit 0 Huffman tree, bits 1..3 LL / OF / ML table
    __device__ int operator()(const ZkBlkInfo& bi) {
        nb++;
        if (bi.flags & ZKB_FIRST) have = 0;
        if (bi.type == 2) {
            if (bi.lit_type == 3 && !(have & 1u)) return ZKZ_DICT_CORRUPTED;
            if (bi.lit_type == 2) have |= 1u;
            if (bi.lit_type >= 2) { nlit += (bi.lit_size + 15u) & ~15u; nhuf++; }
            if (bi.nseq) {
                const uint32_t ml_m = (bi.modes >> 2) & 3, of_m = (bi.modes >> 4) & 3, ll_m = (bi.modes >> 6) & 3;
                if (ll_m == 3) { if (!(have & 2u)) return ZKZ_CORRUPTION; } else have |= 2u;
                if (of_m == 3) { if (!(have & 4u)) return ZKZ_CORRUPTION; } else have |= 4u;
                if (ml_m == 3) { if (!(have & 8u)) return ZKZ_CORRUPTION; } else have |= 8u;
            }
            nseq += bi.nseq; nsqb += bi.nseq != 0;
        }
        return 0;
    }
};

struct ZkFillEmit {
    ZkBlock* blocks; const uint8_t* ebase; uint32_t* huf_list; uint32_t* seq_list; uint32_t entry, bidx, lit, seq, hufi, sqbi;
    int32_t huf_ref = -1, ll_ref = -1, of_ref = -1, ml_ref = -1;
    __device__ int operator()(const ZkBlkInfo& bi) {
        ZkBlock b;
        b.src = bi.src; b.size = bi.size; b.entry = entry; b.type = bi.type; b.flags = bi.flags;
        b.lit_kind = 0; b.lit_byte = 0; b.lit_base = lit; b.seq_base = seq; b.nseq = bi.nseq; b.lit_size = bi.lit_size;
        b.lit_src = 0; b.regen = bi.type == 2 ? 0 : bi.size; b.status = 0; b.lit_status = 0;
        b.rep_out[0] = ZK_SYM_MAKE(0, 0); b.rep_out[1] = ZK_SYM_MAKE(1, 0); b.rep_out[2] = ZK_SYM_MAKE(2, 0);
        b.fcs = bi.fcs; b.hash_start = 0; b.hash_len = 0; b.bmax = bi.bmax;
        b.back = bi.type == 2 && bi.nseq ? ZK_BACK_UNKNOWN : 0u;   // blocks without sequences read no earlier output
        b.out_pos = 0; b.frame_start = 0;
        if (bi.flags & ZKB_FIRST) { huf_ref = ll_ref = of_ref = ml_ref = -1; }
        b.huf_ref = -1; b.ll_ref = -1; b.of_ref = -1; b.ml_ref = -1;
        if (bi.type == 2) {
            if (bi.lit_type == 3) { if (huf_ref < 0) return ZKZ_DICT_CORRUPTED; b.huf_ref = huf_ref; }
            if (bi.lit_type == 2) huf_ref = (int32_t)bidx;
            if (bi.lit_type >= 2) { lit += (bi.lit_size + 15u) & ~15u; b.lit_kind = 2; huf_list[hufi++] = bidx; }
            else if (bi.lit_type == 0) { b.lit_kind = 0; b.lit_src = bi.src + bi.lit_hdr; }
            else { b.lit_kind = 1; b.lit_byte = ebase[bi.src + bi.lit_hdr]; }
            if (bi.nseq == 0) b.regen = bi.lit_size;         // literals-only block
            if (bi.nseq) {
                seq_list[sqbi++] = bidx;
                uint32_t ml_m = (bi.modes >> 2) & 3, of_m = (bi.modes >> 4) & 3, ll_m = (bi.modes >> 6) & 3;
                if (ll_m == 3) { if (ll_ref < 0) return ZKZ_CORRUPTION; b.ll_ref = ll_ref; } else ll_ref = (int32_t)bidx;
                if (of_m == 3) { if (of_ref < 0) return ZKZ_CORRUPTION; b.of_ref = of_ref; } else of_ref = (int32_t)bidx;
                if (ml_m == 3) { if (ml_ref < 0) return ZKZ_CORRUPTION; b.ml_ref = ml_ref; } else ml_ref = (int32_t)bidx;
                seq += bi.nseq;
            }
        }
        blocks[bidx++] = b;
        return 0;
    }
};

__global__ void __launch_bounds__(128) zk_scan_kernel(ZkDecodeArgs a) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n_entries) return;
    ZkEntry ent; ent.first_block = 0; ent.n_blocks = 0; ent.status = 0; ent.produced = 0; ent.run_blocks = 0; ent.segs_left = 0; ent.fail = ~0ull;
    unsigned long long c0 = a.c_off[e], c1 = a.c_off[e + 1];
    if (c1 < c0 || c1 - c0 > 0xFFFFFFFFull) { ent.status = -ZKZ_SRC_SIZE_WRONG; a.entries[e] = ent; return; }
    const uint8_t* p = a.comp + c0; uint32_t n = (uint32_t)(c1 - c0);
    ZkCountEmit ce;
    int rc = zk_walk_entry(p, n, ce);
    if (rc) { ent.status = -rc; atomicAdd(&a.counters->n_errors, 1u); a.entries[e] = ent; return; }
    unsigned long long b0 = atomicAdd(&a.counters->n_blocks, (unsigned long long)ce.nb);
    unsigned long long l0 = atomicAdd(&a.counters->n_lit, (unsigned long long)ce.nlit);
    unsigned long long s0 = atomicAdd(&a.counters->n_seq, (unsigned long long)ce.nseq);
    uint32_t h0 = atomicAdd(&a.counters->n_huf_blocks, ce.nhuf), q0 = atomicAdd(&a.counters->n_seq_blocks, ce.nsqb);
    if (b0 + ce.nb > a.cap_blocks || l0 + ce.nlit > a.cap_lit || s0 + ce.nseq > a.cap_seq) {
        atomicOr(&a.counters->overflow, 1u);
        ent.status = ZK_ST_RETRY; a.entries[e] = ent; return;
    }
    ZkFillEmit fe; fe.blocks = a.blocks; fe.entry = e; fe.bidx = (uint32_t)b0; fe.lit = (uint32_t)l0; fe.seq = (uint32_t)s0;
    fe.ebase = p; fe.huf_list = a.huf_list; fe.seq_list = a.seq_list; fe.hufi = h0; fe.sqbi = q0;   // lists have cap_blocks entries
    rc = zk_walk_entry(p, n, fe);
    ent.first_block = (uint32_t)b0; ent.n_blocks = ce.nb;
    if (rc) { ent.status = -rc; ent.n_blocks = 0; atomicAdd(&a.counters->n_errors, 1u); }
    a.entries[e] = ent;
}

// =============================================================================================
// K-D1s: FSE sequence decode tables.
//
// A sequence bitstream is one serial dependency chain (three interleaved FSE states sharing one
// backward bit cursor, A.5), so the only parallelism is across blocks.
// =============================================================================================

// Thin decoding cell: one 32-bit shared-memory load yields everything on the dependency chain of a sequence (bits to
// skip, bits of the next state, next-state baseline); the value baselines come from small per-CTA tables by symbol code,
// off the chain.  (The first version used libzstd's 8-byte cell: 11.7 KiB of tables per chain, 18 chains per SM.)
//   [0,9) next-state baseline   [9,13) nbBits   [13,18) extra bits   [18,24) symbol code
#define ZK_CELL(code, add, nb, base) ((uint32_t)(base) | ((uint32_t)(nb) << 9) | ((uint32_t)(add) << 13) | ((uint32_t)(code) << 18))
#define ZK_CELL_BASE(c) ((c) & 511u)
#define ZK_CELL_NB(c) (((c) >> 9) & 15u)
#define ZK_CELL_ADD(c) (((c) >> 13) & 31u)
#define ZK_CELL_CODE(c) (((c) >> 18) & 63u)

struct ZkSeqSlot {                            // what a block's three table descriptions parse to, and the build scratch
    int16_t cnt[3][64];
    uint16_t nxt[64];
    int tbl_log[3], tbl_nsym[3], tbl_mode[3];  // mode: 0 = counts in cnt[t], 1 = RLE (cnt[t][0] = symbol)
};
struct ZkSeqTabs { uint32_t ll_base[36], ml_base[53]; };

// A block's LL, OF and ML cells lie back to back in one array, each table as large as its log asks for.  The format allows
// up to 512 + 256 + 512 cells; this codec's encoder never writes a table above log 8, so its blocks need at most 768.
#define ZK_SEQ_CELLS_FULL 1280u
#define ZK_SEQ_CELLS_COMPACT 768u
__device__ __forceinline__ uint32_t zk_seq_cells(const ZkSeqSlot& sl, int t) { return sl.tbl_mode[t] == 1 ? 1u : 1u << sl.tbl_log[t]; }

// Locate the three table descriptions of a block (A.5) and parse those that are wanted into sl.cnt[t]
// (t: 0 LL, 1 OF, 2 ML).  Returns 0 or a zstd code.  *bits_off = start of the sequence bitstream.
__device__ int zk_locate_seq_tables(ZkSeqSlot& sl, const uint8_t* b, uint32_t bsize, bool w0, bool w1, bool w2, uint32_t* bits_off) {
    ZkLitHdr lh;
    if (!zk_parse_lit_hdr(b, bsize, lh)) return ZKZ_CORRUPTION;
    uint32_t lsec = zk_lit_section_size(lh);
    if (lsec >= bsize) return ZKZ_CORRUPTION;
    uint32_t nseq, sh = zk_parse_nseq(b + lsec, bsize - lsec, nseq);
    if (!sh || nseq == 0 || lsec + sh >= bsize) return ZKZ_CORRUPTION;
    uint32_t modes = b[lsec + sh], pos = lsec + sh + 1;
    for (int t = 0; t < 3; t++) {
        const bool want = t == 0 ? w0 : (t == 1 ? w1 : w2);
        const int max_log = t == 1 ? 8 : 9, max_sym = t == 0 ? 35 : (t == 1 ? 31 : 52);
        uint32_t m = (modes >> (6 - 2 * t)) & 3;
        if (m == 0) {
            if (want) {
                sl.tbl_mode[t] = 0;
                if (t == 0) { for (int i = 0; i < 36; i++) sl.cnt[0][i] = ZK_LL_DEFAULT[i]; sl.tbl_nsym[0] = 36; sl.tbl_log[0] = 6; }
                else if (t == 1) { for (int i = 0; i < 29; i++) sl.cnt[1][i] = ZK_OF_DEFAULT[i]; sl.tbl_nsym[1] = 29; sl.tbl_log[1] = 5; }
                else { for (int i = 0; i < 53; i++) sl.cnt[2][i] = ZK_ML_DEFAULT[i]; sl.tbl_nsym[2] = 53; sl.tbl_log[2] = 6; }
            }
        } else if (m == 1) {
            if (pos >= bsize) return ZKZ_CORRUPTION;
            if (want) {
                if (b[pos] > max_sym) return ZKZ_CORRUPTION;
                sl.tbl_mode[t] = 1; sl.cnt[t][0] = b[pos]; sl.tbl_log[t] = 0; sl.tbl_nsym[t] = 1;
            }
            pos += 1;
        } else if (m == 2) {
            int ns, lg;
            // an unwanted table is parsed into the (not yet used) nxt scratch just to learn its length
            uint32_t used = zk_fse_read_ncount(b + pos, bsize - pos, max_log, max_sym, want ? sl.cnt[t] : (int16_t*)sl.nxt, &ns, &lg);
            if (!used) return ZKZ_CORRUPTION;
            if (want) { sl.tbl_mode[t] = 0; sl.tbl_nsym[t] = ns; sl.tbl_log[t] = lg; }
            pos += used;
        } else {
            if (want) return ZKZ_CORRUPTION;   // Repeat is resolved through *_ref by the caller
        }
    }
    if (pos > bsize) return ZKZ_CORRUPTION;
    *bits_off = pos;
    return 0;
}

// Build one sequence decoding table from sl.cnt[t] (A.6) into cell[0, zk_seq_cells(sl, t)).  The symbol spread is written
// into the cell array itself and converted to cells in place.
__device__ int zk_build_seq_table(ZkSeqSlot& sl, int t, uint32_t* cell, uint16_t* nxt_scratch = nullptr) {
    if (sl.tbl_mode[t] == 1) {
        const uint32_t sy = (uint32_t)sl.cnt[t][0];
        const uint32_t add = t == 0 ? ZK_LL_BITS[sy] : (t == 1 ? sy : ZK_ML_BITS[sy]);
        cell[0] = ZK_CELL(sy, add, 0, 0);
        return 0;
    }
    int log = sl.tbl_log[t], S = 1 << log, nsym = sl.tbl_nsym[t], high = S - 1;
    uint16_t* nxt = nxt_scratch ? nxt_scratch : sl.nxt; const int16_t* cnt = sl.cnt[t];
    for (int s = 0; s < nsym; s++) {
        if (cnt[s] == -1) { cell[high--] = (uint32_t)s; nxt[s] = 1; }
        else nxt[s] = (uint16_t)cnt[s];
    }
    int step = (S >> 1) + (S >> 3) + 3, pos = 0;
    for (int s = 0; s < nsym; s++)
        for (int q = 0; q < cnt[s]; q++) {
            cell[pos] = (uint32_t)s;
            do { pos = (pos + step) & (S - 1); } while (pos > high);
        }
    if (pos != 0) return ZKZ_CORRUPTION;
    for (int u = 0; u < S; u++) {
        const uint32_t sy = cell[u];
        const uint32_t x = nxt[sy]++;
        const int nb = log - zk_highbit(x);
        const uint32_t add = t == 0 ? ZK_LL_BITS[sy] : (t == 1 ? sy : ZK_ML_BITS[sy]);
        cell[u] = ZK_CELL(sy, add, nb, (x << nb) - (uint32_t)S);
    }
    return 0;
}

// =============================================================================================
// K-D1s (second generation): the same decode, cut into what MUST be serial and what need not be.
//
// A sequence bitstream is one serial chain: the next FSE states depend on bits whose position depends on the current
// states' cells.  The first kernel ran the whole per-sequence work (~110 dependent instructions: extra-bit reads, value
// arithmetic, repeat-offset history, three stores, refills from global memory) on that chain -- about 1 000 cycles per
// sequence.  Here
//   * the bitstream is staged in shared memory by TMA bulk copies (cp.async.bulk + mbarrier, four 256-byte tiles per
//     chain, refilled ahead of the cursor), so a bit field anywhere near the cursor is two shared-memory loads and a
//     funnel shift -- no bit buffer, no refill branches, no global latency on the chain;
//   * a CHAIN LANE only walks the states: three cell loads, the sum of the extra-bit counts, one 32-bit window for the
//     three state updates, and one 16-byte record {cells, cursor} per sequence (~40 instructions);
//   * after every 32 steps ALL lanes turn the records into values: extra bits, literal / match lengths, two warp scans for
//     the cumulative ends, bounds checks, coalesced stores; the repeat-offset history -- a serial state machine -- is run
//     warp-uniformly over the FEW sequences that use a repeat code (explicit offsets just shift it).
// Four chains per warp (lanes 0, 8, 16, 24) share every issued instruction of the chain phase.
//
// Shared memory per chain decides how many chains an SM holds beside K-D1h, so the kernel comes in two layouts of the
// cell array: zk_seq2_kernel (768 cells, every block of this codec's encoder) and zk_seq2_full_kernel (1280, the format's
// largest tables).  The first kernel passes a block whose parsed tables need more cells than it has to the second, which
// runs after it on the same stream.
// =============================================================================================
#define ZK_S2_NCH 4
#define ZK_S2_TILE 256u
#define ZK_S2_RING_BYTES 1024u            // four tiles: the cursor's tile, the two below it (>= 512 bytes below the cursor,
                                          // more than a phase's 356), one being refilled
template <uint32_t NCELLS>
struct ZkSeq2Chain {
    uint32_t cells[NCELLS];                // thin cells: LL, OF, ML back to back (zk_seq_cells)
    ZkSeqSlot t;                           // build scratch (zk_locate_seq_tables / zk_build_seq_table)
    alignas(128) uint32_t ring[ZK_S2_RING_BYTES / 4];   // staged bitstream (bulk copies want 16-byte aligned shared addresses): byte at offset o from gbase lives at ring byte o & 1023
    uint4 rec[32];                         // per step: {LL cell, OF cell, ML cell, bit cursor before the extra bits}
    uint16_t nxt2[2][64];                  // build scratch of the OF / ML tables (LL uses t.nxt): the three tables are built side by side
    alignas(8) unsigned long long bar[4];  // one mbarrier per tile slot
    uint32_t lit_end, out_end, r0, r1, r2; // carries of the helper phase
    uint32_t back;                         // ... and the block's ZkBlock::back so far
    int st;
};

// the 32 bits just below bit position cur (MSB = bit cur - 1) of the staged stream
__device__ __forceinline__ uint32_t zk_s2_window(const uint32_t* ring, uint32_t cur) {
    const uint32_t t = cur - 1u, wi = t >> 5, sh = 31u - (t & 31u);
    return __funnelshift_l(ring[(wi - 1u) & (ZK_S2_RING_BYTES / 4 - 1)], ring[wi & (ZK_S2_RING_BYTES / 4 - 1)], sh);
}
__device__ __forceinline__ uint32_t zk_s2_bits(const uint32_t* ring, uint32_t cur, uint32_t n) {       // n in [0, 31]
    return __funnelshift_l(zk_s2_window(ring, cur), 0u, n);
}

template <uint32_t NCELLS>
__device__ __forceinline__ void zk_seq2_body(const ZkDecodeArgs& a) {
    constexpr bool full = NCELLS == ZK_SEQ_CELLS_FULL;                 // decodes the blocks the compact layout passed on
    ZK_DYN_SMEM(smem);
    ZkSeqTabs* tb = (ZkSeqTabs*)smem;
    ZkSeq2Chain<NCELLS>* chains = (ZkSeq2Chain<NCELLS>*)(smem + ((sizeof(ZkSeqTabs) + 127) & ~(size_t)127));
    const int lane = threadIdx.x & 31;
    const int myc = lane >> 3;                                     // the chain this lane belongs to ...
    const bool chain_lane = (lane & 7) == 0;                       // ... and whether it walks it
    for (int i = lane; i < 36; i += 32) tb->ll_base[i] = ZK_LL_BASE[i];
    for (int i = lane; i < 53; i += 32) tb->ml_base[i] = ZK_ML_BASE[i];
    if (chain_lane) for (int k = 0; k < 4; k++) zk_mbar_init(&chains[myc].bar[k], 1);
#ifndef ZK_EMUL
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
    __syncwarp();
    if (a.counters->overflow) return;
    const uint32_t n = full ? a.counters->n_seq_full : a.counters->n_seq_blocks;
    const uint32_t* list = full ? a.seq_list + a.cap_blocks : a.seq_list;
    uint32_t tile_uses = 0;                                        // tiles this chain lane has issued so far (slot = use & 3, parity = (use >> 2) & 1)
    for (;;) {
        uint32_t g = 0;
        if (lane == 0) g = atomicAdd(&a.work_counter[full ? 4 : 0], 1u);
        g = __shfl_sync(0xFFFFFFFFu, g, 0);
        const uint32_t first = g * ZK_S2_NCH;
        if (first >= n) break;
        ZkSeq2Chain<NCELLS>& ch = chains[myc];
        // ---------------- per chain: tables, stream geometry, first tiles, initial states (chain lanes, side by side)
        uint32_t bidx = 0, remaining = 0, done = 0, cur = 0, sb_bit = 0, s_l = 0, s_o = 0, s_m = 0, seq_base = 0, lit_size = 0, o_of = 0, o_ml = 0;
        const uint8_t* gbase = nullptr;
        int next_issue = -1, next_wait = -1, top_tile = 0; uint32_t stream_end_off = 0, use0 = 0;
        bool live = false, parsed = false;
        if (chain_lane) {
            ch.st = 0; ch.lit_end = 0; ch.out_end = 0; ch.back = 0; ch.r0 = ZK_SYM_MAKE(0, 0); ch.r1 = ZK_SYM_MAKE(1, 0); ch.r2 = ZK_SYM_MAKE(2, 0);
            const uint32_t my = first + (uint32_t)myc;
            if (my < n) {
                bidx = list[my];
                ZkBlock blk; blk.entry = 0xFFFFFFFFu;
                if (bidx < a.cap_blocks) blk = a.blocks[bidx];
                if (blk.entry < a.n_entries && a.entries[blk.entry].status == 0) {
                    live = true;
                    const uint8_t* ebase = a.comp + a.c_off[blk.entry];
                    const uint8_t* b = ebase + blk.src;
                    uint32_t bits_off = 0;
                    int st = zk_locate_seq_tables(ch.t, b, blk.size, blk.ll_ref < 0, blk.of_ref < 0, blk.ml_ref < 0, &bits_off);
                    if (!st && blk.ll_ref >= 0) { const ZkBlock& rb = a.blocks[blk.ll_ref]; uint32_t d; st = zk_locate_seq_tables(ch.t, ebase + rb.src, rb.size, true, false, false, &d); }
                    if (!st && blk.of_ref >= 0) { const ZkBlock& rb = a.blocks[blk.of_ref]; uint32_t d; st = zk_locate_seq_tables(ch.t, ebase + rb.src, rb.size, false, true, false, &d); }
                    if (!st && blk.ml_ref >= 0) { const ZkBlock& rb = a.blocks[blk.ml_ref]; uint32_t d; st = zk_locate_seq_tables(ch.t, ebase + rb.src, rb.size, false, false, true, &d); }
                    if (!st) { o_of = zk_seq_cells(ch.t, 0); o_ml = o_of + zk_seq_cells(ch.t, 1); }
                    if (!full && !st && o_ml + zk_seq_cells(ch.t, 2) > NCELLS) {
                        a.seq_list[a.cap_blocks + atomicAdd(&a.counters->n_seq_full, 1u)] = bidx;          // tables too large for these cells: the
                        live = false;                                                        // full layout decodes the block
                    } else {
                        ch.st = st; parsed = !st;
                        const uint8_t* sp = b + bits_off; const uint32_t sn = blk.size - bits_off;
                        if (!st && (sn == 0 || sp[sn - 1] == 0)) st = ZKZ_CORRUPTION;
                        if (!st) {
                            gbase = (const uint8_t*)((uintptr_t)sp & ~(uintptr_t)15);
                            sb_bit = (uint32_t)(sp - gbase) * 8u;
                            stream_end_off = (uint32_t)(sp - gbase) + sn;                       // byte offset of the end of the stream from gbase
                            cur = sb_bit + (sn - 1) * 8u + (uint32_t)zk_highbit(sp[sn - 1]);     // the end mark itself is not data
                            // tiles are staged from the CURSOR's tile downwards: when the end mark is the first byte of a tile, that tile holds
                            // no data (the mark was read above), and counting it would put five tiles in flight on four slots
                            top_tile = (int)(((cur ? cur - 1u : 0u) >> 3) / ZK_S2_TILE);
                            next_issue = top_tile; next_wait = top_tile; use0 = tile_uses;
                            remaining = blk.nseq; seq_base = blk.seq_base; lit_size = blk.lit_size;
                        }
                        ch.st = st;
                    }
                }
            }
        }
        // ---------------- the three decoding tables of every chain, built side by side by lanes 0..2 of the chain's lane group
        __syncwarp();
        {
            const bool go = __shfl_sync(0xFFFFFFFFu, (uint32_t)(parsed && ch.st == 0), myc * 8) != 0;
            const int t = lane & 7;
            int bst = 0;
            if (go && t < 3) {
                const uint32_t off = t == 0 ? 0u : (t == 1 ? zk_seq_cells(ch.t, 0) : zk_seq_cells(ch.t, 0) + zk_seq_cells(ch.t, 1));
                bst = zk_build_seq_table(ch.t, t, ch.cells + off, t == 0 ? nullptr : ch.nxt2[t - 1]);
            }
            const uint32_t failed = __ballot_sync(0xFFFFFFFFu, bst != 0);
            if (chain_lane && ((failed >> (myc * 8)) & 7u) && ch.st == 0) ch.st = ZKZ_CORRUPTION;
        }
        __syncwarp();
        // ---------------- tiles of 32 steps
        for (;;) {
            uint32_t cnt = 0;
            if (chain_lane && remaining && ch.st == 0) {
                // tiles: the cursor's tile jc and the two below it must have landed; everything above jc is dead (the records of
                // the previous steps were consumed), so the copies may run down to jc - 3
                const int jc = (int)(((cur ? cur - 1u : 0u) >> 3) / ZK_S2_TILE);
                while (next_issue >= 0 && next_issue >= jc - 3) {
                    const uint32_t off = (uint32_t)next_issue * ZK_S2_TILE;
                    uint32_t bytes = stream_end_off - off; bytes = bytes > ZK_S2_TILE ? ZK_S2_TILE : ((bytes + 15u) & ~15u);   // (16 readable bytes follow every buffer)
                    zk_bulk_g2s((uint8_t*)ch.ring + (off & (ZK_S2_RING_BYTES - 1)), gbase + off, bytes, &ch.bar[tile_uses & 3u]);
                    tile_uses++; next_issue--;
                }
                while (next_wait >= 0 && next_wait >= jc - 2) {
                    const uint32_t u = use0 + (uint32_t)(top_tile - next_wait);
                    if (!zk_mbar_wait(&ch.bar[u & 3u], (u >> 2) & 1u)) {
                        printf("zk_seq2: tile wait timed out: block %u tile %d top %d use %u use0 %u jc %d cur %u\n", bidx, next_wait, top_tile, u, use0, jc, cur);
                        ch.st = ZKZ_GENERIC;
                    }
                    next_wait--;
                }
                if (done == 0) {                                                          // initial states (A.5: LL, OF, ML)
                    const int ll_log = ch.t.tbl_log[0], of_log = ch.t.tbl_log[1], ml_log = ch.t.tbl_log[2];
                    if (cur < sb_bit + (uint32_t)(ll_log + of_log + ml_log)) ch.st = ZKZ_CORRUPTION;
                    else {
                        s_l = zk_s2_bits(ch.ring, cur, (uint32_t)ll_log); cur -= (uint32_t)ll_log;
                        s_o = zk_s2_bits(ch.ring, cur, (uint32_t)of_log); cur -= (uint32_t)of_log;
                        s_m = zk_s2_bits(ch.ring, cur, (uint32_t)ml_log); cur -= (uint32_t)ml_log;
                    }
                }
                if (ch.st == 0) {
                    cnt = remaining < 32u ? remaining : 32u;
                    const bool last_tile = cnt == remaining;
                    bool over = false;
                    const uint32_t* cof = ch.cells + o_of; const uint32_t* cml = ch.cells + o_ml;
                    for (uint32_t k = 0; k < cnt; k++) {
                        const uint32_t cl = ch.cells[s_l], co = cof[s_o], cm = cml[s_m];
                        ch.rec[k] = make_uint4(cl, co, cm, cur);
                        const uint32_t eb = ZK_CELL_CODE(co) + ZK_CELL_ADD(cm) + ZK_CELL_ADD(cl);
                        const uint32_t nl = ZK_CELL_NB(cl), nm = ZK_CELL_NB(cm), no = ZK_CELL_NB(co);
                        const bool upd = !(last_tile && k + 1 == cnt);                   // no state update after the block's last sequence
                        const uint32_t need_bits = eb + (upd ? nl + nm + no : 0u);
                        if (cur - sb_bit < need_bits) { over = true; cnt = k; break; }    // the stream is shorter than its sequences need
                        cur -= eb;
                        if (upd) {
                            const uint32_t w = zk_s2_window(ch.ring, cur);
                            s_l = ZK_CELL_BASE(cl) + __funnelshift_l(w, 0u, nl);
                            s_m = ZK_CELL_BASE(cm) + __funnelshift_l(w << nl, 0u, nm);
                            s_o = ZK_CELL_BASE(co) + __funnelshift_l(w << (nl + nm), 0u, no);
                            cur -= nl + nm + no;
                        }
                    }
                    if (over) ch.st = ZKZ_CORRUPTION;
                    remaining -= cnt; 
                    if (over) remaining = 0;
                }
            }
            __syncwarp();
            // ---------------- helper phase: every lane, one chain after the other
            uint32_t any = 0;
#pragma unroll 1
            for (int cc = 0; cc < ZK_S2_NCH; cc++) {
                const uint32_t ncc = __shfl_sync(0xFFFFFFFFu, cnt, cc * 8);
                if (ncc == 0) continue;
                any = 1;
                ZkSeq2Chain<NCELLS>& hc = chains[cc];
                const uint32_t sbase = __shfl_sync(0xFFFFFFFFu, seq_base, cc * 8), sdone = __shfl_sync(0xFFFFFFFFu, done, cc * 8);
                const uint32_t lsz = __shfl_sync(0xFFFFFFFFu, lit_size, cc * 8);
                const bool act = (uint32_t)lane < ncc;
                uint32_t llv = 0, mlv = 0, ofv = 4;                                       // inactive lanes: explicit offsets that push nothing (masked below)
                if (act) {
                    const uint4 r = hc.rec[lane];
                    const uint32_t ofc = ZK_CELL_CODE(r.y), mlb = ZK_CELL_ADD(r.z), llb = ZK_CELL_ADD(r.x);
                    uint32_t c = r.w;
                    ofv = (1u << ofc) + zk_s2_bits(hc.ring, c, ofc); c -= ofc;
                    mlv = tb->ml_base[ZK_CELL_CODE(r.z)] + zk_s2_bits(hc.ring, c, mlb); c -= mlb;
                    llv = tb->ll_base[ZK_CELL_CODE(r.x)] + zk_s2_bits(hc.ring, c, llb);
                }
                // cumulative ends: two inclusive warp scans on top of the chain's carries
                uint32_t le = llv, oe = llv + mlv;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, le, d), y = __shfl_up_sync(0xFFFFFFFFu, oe, d);
                    if (lane >= d) { le += x; oe += y; }
                }
                le += hc.lit_end; oe += hc.out_end;
                // bounded after EVERY sequence (a tile adds < 2^23, the carries are <= 2^17: no wrap can hide an overflow)
                const bool badv = act && (le > lsz || oe > ZK_BLOCK_MAX);
                // repeat-offset history (A.5), symbolic with respect to the state entering the block: explicit offsets only shift it,
                // so the serial part runs over the sequences that USE a repeat code
                uint32_t r0 = hc.r0, r1 = hc.r1, r2 = hc.r2, off = ofv - 3u;
                const uint32_t repm = __ballot_sync(0xFFFFFFFFu, act && ofv <= 3u);
                const uint32_t idxv = ofv - 1u + (llv == 0u ? 1u : 0u);                 // meaningful on repeat lanes only
                uint32_t m = repm; int lastpos = 0; bool badr = false;
                for (;;) {
                    const int j = m ? __ffs((int)m) - 1 : (int)ncc;                      // next repeat lane, or the end of the tile
                    const int cnte = j - lastpos;                                        // explicit offsets since the last repeat lane
                    if (cnte > 0) {
                        const uint32_t e1 = __shfl_sync(0xFFFFFFFFu, off, j - 1);
                        const uint32_t e2 = __shfl_sync(0xFFFFFFFFu, off, cnte > 1 ? j - 2 : 0), e3 = __shfl_sync(0xFFFFFFFFu, off, cnte > 2 ? j - 3 : 0);
                        const uint32_t o0 = r0, o1 = r1;
                        r0 = e1; r1 = cnte > 1 ? e2 : o0; r2 = cnte > 2 ? e3 : (cnte == 2 ? o0 : o1);
                    }
                    if (!m) break;
                    const uint32_t idx = __shfl_sync(0xFFFFFFFFu, idxv, j);
                    uint32_t o;
                    if (idx == 0) o = r0;
                    else {
                        if (idx == 3) { if (r0 & ZK_SYM) o = r0 + 1u; else { o = r0 - 1u; if (o == 0) badr = true; } }
                        else o = idx == 1 ? r1 : r2;
                        if (idx != 1) r2 = r1;
                        r1 = r0; r0 = o;
                    }
                    if (lane == j) off = o;
                    lastpos = j + 1; m &= m - 1;
                }
                uint32_t back = 0;                                                       // how far before the block's first byte this match reads
                if (act) {
                    const uint32_t at = sbase + sdone + (uint32_t)lane;
                    a.seq_lit_end[at] = le; a.seq_out_end[at] = oe; a.seq_off[at] = off;
                    const uint32_t md = oe - mlv;                                        // block-relative match destination
                    back = (off & ZK_SYM) ? ZK_BACK_UNKNOWN : (off > md ? min(off - md, ZK_BACK_UNKNOWN - 1u) : 0u);
                }
                back = __reduce_max_sync(0xFFFFFFFFu, back);
                const bool anybad = __any_sync(0xFFFFFFFFu, badv) || badr;
                if (lane == (int)ncc - 1) { hc.lit_end = le; hc.out_end = oe; }
                if (lane == 0) { hc.r0 = r0; hc.r1 = r1; hc.r2 = r2; hc.back = max(hc.back, back); if (anybad && hc.st == 0) hc.st = ZKZ_CORRUPTION; }
            }
            __syncwarp();
            if (chain_lane) { done += cnt; if (ch.st != 0) remaining = 0; }
            if (!any) break;
        }
        // ---------------- results of the block
        if (chain_lane) {     // copies issued ahead but never needed must have landed before the next block reuses the ring
            while (next_wait > next_issue) { const uint32_t u = use0 + (uint32_t)(top_tile - next_wait); zk_mbar_wait(&ch.bar[u & 3u], (u >> 2) & 1u); next_wait--; }
        }
        if (chain_lane && live) {
            int st = ch.st;
            if (!st && cur != sb_bit) st = ZKZ_CORRUPTION;                                // every bit of the stream is consumed, no more
            if (!st && ch.out_end + (lit_size - ch.lit_end) > a.blocks[bidx].bmax) st = ZKZ_CORRUPTION;
            a.blocks[bidx].rep_out[0] = ch.r0; a.blocks[bidx].rep_out[1] = ch.r1; a.blocks[bidx].rep_out[2] = ch.r2;
            a.blocks[bidx].regen = ch.out_end + (lit_size - ch.lit_end);
            a.blocks[bidx].status = st ? -st : 0;
            a.blocks[bidx].back = st ? ZK_BACK_UNKNOWN : ch.back;
        }
        __syncwarp();
    }
}
static_assert(ZK_SEQ_CELLS_FULL == 512 + 256 + 512, "the full layout holds the largest tables the format allows (LL, ML log 9; OF log 8)");

__global__ void __launch_bounds__(32) zk_seq2_kernel(ZkDecodeArgs a) { zk_seq2_body<ZK_SEQ_CELLS_COMPACT>(a); }
__global__ void __launch_bounds__(32) zk_seq2_full_kernel(ZkDecodeArgs a) { zk_seq2_body<ZK_SEQ_CELLS_FULL>(a); }

// =============================================================================================
// K-D1h: Huffman literal decode -- one LANE per Huffman stream (4 lanes per 4-stream block).
// =============================================================================================
#define ZK_HUF_SLOTS 8            // blocks per warp-CTA; 8 x 2 KiB of tables + 0.3 KiB of build scratch

// Two-level decoding table.  Cells are laid out weight ascending (A.4), so the codes of the two longest lengths occupy
// the first L <= 510 cells of the 2^maxBits index space, and everything above is replicated at least four times:
//   idx < L  -> low[idx]        (full resolution)        idx >= L -> l1[idx >> 2]      (2^(maxBits-2) <= 512 entries)
// 2 KiB instead of the flat 4 KiB table.  The kernel is bound by memory latency and runs beside K-D1s, so the shared
// memory a block holds decides how many blocks and how many K-D1s chains fit on an SM: the table is all a block keeps
// through its decode (L and maxBits live in registers).  Before the table is filled, the same memory holds the block's
// weights, decoded by one lane per block with the eight blocks side by side.
union ZkHufTab {
    struct { uint16_t l1[512], low[512]; } t;  // (nbBits << 8) | symbol
    struct {
        uint8_t weights[256];                  // explicit weights, as the tree description gives them
        uint8_t sym[64], nb[64]; uint16_t base[64];   // FSE table for compressed weights (log <= 6)
    } w;
};
// Build scratch, one per warp: the warp ranks the weights and fills the tables one block after another.
struct ZkHufScratch {
    uint8_t sorted[256];                       // the symbols by (weight, symbol): the order of their cells
    uint32_t cntw[16];                         // symbols per weight
};

// Huffman tree description -> hw.weights[0..*nw) without the implied last weight (A.4).  Serial (one lane per block).
// Returns bytes consumed or 0 on corruption.
__device__ uint32_t zk_read_huf_weights(ZkHufTab& hw, const uint8_t* p, uint32_t n, int* nw_out) {
    if (n < 1) return 0;
    uint32_t hb = p[0], used; int nw = 0;
    if (hb >= 128) {
        nw = (int)hb - 127; used = 1 + (uint32_t)(nw + 1) / 2;
        if (used > n) return 0;
        for (int i = 0; i < nw; i++) { uint32_t b = p[1 + i / 2]; hw.w.weights[i] = (uint8_t)((i & 1) ? (b & 15) : (b >> 4)); }
    } else {
        used = 1 + hb;
        if (hb == 0 || used > n) return 0;
        int16_t cnt[16]; int ns, lg;
        uint32_t r = zk_fse_read_ncount(p + 1, hb, 6, 12, cnt, &ns, &lg);
        if (!r) return 0;
        int S = 1 << lg, high = S - 1; uint16_t nx[16];
        for (int s = 0; s < ns; s++) { if (cnt[s] == -1) { hw.w.sym[high--] = (uint8_t)s; nx[s] = 1; } else nx[s] = (uint16_t)cnt[s]; }
        int step = (S >> 1) + (S >> 3) + 3, pos = 0;
        for (int s = 0; s < ns; s++)
            for (int q = 0; q < cnt[s]; q++) { hw.w.sym[pos] = (uint8_t)s; do { pos = (pos + step) & (S - 1); } while (pos > high); }
        if (pos != 0) return 0;
        for (int u = 0; u < S; u++) {
            int s = hw.w.sym[u]; uint32_t x = nx[s]++; int nb = lg - zk_highbit(x);
            hw.w.nb[u] = (uint8_t)nb; hw.w.base[u] = (uint16_t)((x << nb) - S);
        }
        ZkBackBits br;
        if (!br.init(p + 1 + r, hb - r)) return 0;
        br.refill();
        uint32_t s1 = br.read(lg), s2 = br.read(lg);
        if (br.bp < 0) return 0;
        for (;;) {   // two interleaved states, over-read terminates (A.4)
            if (nw >= 254) return 0;
            br.refill();
            hw.w.weights[nw++] = hw.w.sym[s1];
            s1 = hw.w.base[s1] + br.read(hw.w.nb[s1]);
            if (br.bp < 0) { hw.w.weights[nw++] = hw.w.sym[s2]; break; }
            hw.w.weights[nw++] = hw.w.sym[s2];
            s2 = hw.w.base[s2] + br.read(hw.w.nb[s2]);
            if (br.bp < 0) { hw.w.weights[nw++] = hw.w.sym[s1]; break; }
        }
        if (nw > 255) return 0;                    // at most 255 explicit weights (+ the implied one = 256 symbols)
    }
    *nw_out = nw;
    return used;
}

// The nw explicit weights in hw -> decoding table in the same memory, built by the whole warp (warp-uniform arguments,
// every lane returns the same).  Returns false on corruption; sets *n_low (L) and *bits (maxBits).  Symbol lane + 32k is
// this lane's k-th symbol: its weight and its rank among the symbols of that weight stay in registers.
__device__ bool zk_huf_build(ZkHufTab& hw, ZkHufScratch& sc, int nw, int lane, uint32_t* n_low, int* bits) {
    const uint32_t full = 0xFFFFFFFFu, lt = (1u << lane) - 1u;
    // 1. the implied last weight and libzstd's sanity rules (HUF_readStats)
    uint32_t w[8], total = 0, n_w1 = 0; bool bad = false;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const int s = lane + 32 * k;
        w[k] = s < nw ? hw.w.weights[s] : 0u;
        bad |= w[k] > 11;
        total += w[k] ? 1u << (w[k] - 1) : 0u;
        n_w1 += w[k] == 1;
    }
    if (__any_sync(full, bad)) return false;
    total = __reduce_add_sync(full, total); n_w1 = __reduce_add_sync(full, n_w1);
    if (total == 0) return false;
    const int max_bits = zk_highbit(total) + 1;
    if (max_bits > 11) return false;
    const uint32_t left = (1u << max_bits) - total;
    if (left & (left - 1)) return false;       // must be a power of two (left >= 1 by construction)
    const uint32_t lw = (uint32_t)zk_highbit(left) + 1;
#pragma unroll
    for (int k = 0; k < 8; k++) if (lane + 32 * k == nw) w[k] = lw;
    n_w1 += (lw == 1);
    if (n_w1 < 2 || (n_w1 & 1)) return false;
    // 2. symbols per weight, and each symbol's rank among those of its weight (natural order)
    if (lane < 16) sc.cntw[lane] = 0;
    __syncwarp();
    uint32_t occ[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint32_t m = __match_any_sync(full, w[k]);
        occ[k] = sc.cntw[w[k]] + (uint32_t)__popc(m & lt);
        __syncwarp();
        if (!(m & lt)) sc.cntw[w[k]] += (uint32_t)__popc(m);
        __syncwarp();
    }
    // lane w (1 <= w <= maxBits): first cell and first sorted index of weight w, by exclusive scans over 16 lanes
    const uint32_t cw = (lane >= 1 && lane <= max_bits) ? sc.cntw[lane] : 0u, own = lane >= 1 ? cw << (lane - 1) : 0u;
    uint32_t cells = own, cs = cw;
#pragma unroll
    for (int d = 1; d < 16; d <<= 1) {
        const uint32_t x = __shfl_up_sync(full, cells, d), y = __shfl_up_sync(full, cs, d);
        if (lane >= d) { cells += x; cs += y; }
    }
    const uint32_t acc = __shfl_sync(full, cells, 15), rank_start = cells - own, cstart = cs - cw;
    if (acc != (1u << max_bits)) return false;
    const uint32_t nl = __shfl_sync(full, cw, 1) + 2u * __shfl_sync(full, cw, 2);   // cells of the two longest code lengths
    if (nl > 512u) return false;
    // 3. symbols in cell order
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint32_t at = __shfl_sync(full, cstart, (int)w[k]) + occ[k];
        if (w[k]) sc.sorted[at] = (uint8_t)(lane + 32 * k);
    }
    __syncwarp();
    // 4. fill (the weights are in registers now): weight w owns the cells [rank_start, + count << (w-1)); w <= 2 -> low,
    //    one l1 entry per 4 cells above (L is a multiple of 4 whenever a weight >= 3 exists)
    for (int wt = 1; wt <= max_bits; wt++) {
        const uint32_t c = __shfl_sync(full, cw, wt), rs = __shfl_sync(full, rank_start, wt), c0 = __shfl_sync(full, cstart, wt);
        const uint32_t hi = (uint32_t)(max_bits + 1 - wt) << 8;
        if (wt <= 2) { for (uint32_t i = lane; i < (c << (wt - 1)); i += 32) hw.t.low[rs + i] = (uint16_t)(hi | sc.sorted[c0 + (i >> (wt - 1))]); }
        else { for (uint32_t i = lane; i < (c << (wt - 3)); i += 32) hw.t.l1[(rs >> 2) + i] = (uint16_t)(hi | sc.sorted[c0 + (i >> (wt - 3))]); }
    }
    *n_low = nl; *bits = max_bits;
    return true;
}

// Decode `cnt` Huffman symbols of one stream into out (A.4).  Returns false on corruption.
__device__ __forceinline__ uint32_t zk_huf_lookup(const ZkHufTab& t, uint32_t n_low, uint32_t idx) {
    return idx < n_low ? t.t.low[idx & 511u] : t.t.l1[idx >> 2];
}
__device__ bool zk_huf_decode_stream(const ZkHufTab& t, uint32_t n_low, int max_bits, const uint8_t* p, uint32_t n, uint8_t* out, uint32_t cnt) {
    ZkBackBits br;
    if (!br.init(p, n)) return false;
    uint32_t i = 0;
    while (i < cnt && ((uintptr_t)(out + i) & 3)) {
        br.refill();
        uint32_t e = zk_huf_lookup(t, n_low, br.peek(max_bits)); br.skip((int)(e >> 8)); out[i++] = (uint8_t)e;
    }
    for (; i + 4 <= cnt; i += 4) {
        br.refill();                                   // >= 33 bits: three codes of <= 11 bits
        uint32_t e0 = zk_huf_lookup(t, n_low, br.peek(max_bits)); br.skip((int)(e0 >> 8));
        uint32_t e1 = zk_huf_lookup(t, n_low, br.peek(max_bits)); br.skip((int)(e1 >> 8));
        uint32_t e2 = zk_huf_lookup(t, n_low, br.peek(max_bits)); br.skip((int)(e2 >> 8));
        br.refill();
        uint32_t e3 = zk_huf_lookup(t, n_low, br.peek(max_bits)); br.skip((int)(e3 >> 8));
        *(uint32_t*)(out + i) = (e0 & 0xFF) | ((e1 & 0xFF) << 8) | ((e2 & 0xFF) << 16) | ((e3 & 0xFF) << 24);
    }
    for (; i < cnt; i++) {
        br.refill();
        uint32_t e = zk_huf_lookup(t, n_low, br.peek(max_bits)); br.skip((int)(e >> 8)); out[i] = (uint8_t)e;
    }
    return br.bp == 0;
}

__global__ void __launch_bounds__(32) zk_huf_kernel(ZkDecodeArgs a) {
    ZK_DYN_SMEM(smem);
    ZkHufTab* tabs = (ZkHufTab*)smem;
    ZkHufScratch& sc = *(ZkHufScratch*)(smem + sizeof(ZkHufTab) * ZK_HUF_SLOTS);
    const int lane = threadIdx.x, si = lane >> 2, stream = lane & 3;
    if (a.counters->overflow) return;
    const uint32_t n = a.counters->n_huf_blocks;
    for (;;) {
        uint32_t g = 0;
        if (lane == 0) g = atomicAdd(&a.work_counter[1], 1u);
        g = __shfl_sync(0xFFFFFFFFu, g, 0);
        uint32_t first = g * ZK_HUF_SLOTS;
        if (first >= n) break;
        const uint32_t my = first + si;
        const bool active = my < n;
        uint32_t bidx = 0; ZkBlock blk; ZkLitHdr lh; const uint8_t* ebase = nullptr;
        const uint8_t* tree = nullptr; uint32_t tree_n = 0;
        bool live = false;
        if (active) {
            bidx = a.huf_list[my];
            if (bidx < a.cap_blocks) {                              // always: every reserved slot is written by the scan kernel
                blk = a.blocks[bidx];
                live = blk.entry < a.n_entries && a.entries[blk.entry].status == 0;
            }
            if (live) {
                ebase = a.comp + a.c_off[blk.entry];
                zk_parse_lit_hdr(ebase + blk.src, blk.size, lh);  // validated by the scan kernel
                if (lh.type == 2) { tree = ebase + blk.src + lh.hdr; tree_n = lh.comp; }
                else {                                              // Treeless: the tree of the block it refers to
                    const ZkBlock& rb = a.blocks[blk.huf_ref];
                    ZkLitHdr rh; zk_parse_lit_hdr(ebase + rb.src, rb.size, rh);
                    tree = ebase + rb.src + rh.hdr; tree_n = rh.comp;
                }
            }
        }
        // 1. tables: weights by one lane per block, the eight blocks side by side; ranks and cells by the whole warp, one
        //    block after another in the shared scratch
        int st = 0, huf_bits = 0, nw = 0; uint32_t n_low = 0, tree_bytes = 0;
        if (live && stream == 0) {
            const uint32_t used = zk_read_huf_weights(tabs[si], tree, tree_n, &nw);
            if (!used) st = ZKZ_CORRUPTION;
            tree_bytes = lh.type == 2 ? used : 0u;
        }
        __syncwarp();
        st = __shfl_sync(0xFFFFFFFFu, st, lane & ~3); tree_bytes = __shfl_sync(0xFFFFFFFFu, tree_bytes, lane & ~3);   // to the block's four lanes
        for (int b = 0; b < ZK_HUF_SLOTS; b++) {
            if (!__shfl_sync(0xFFFFFFFFu, (int)live && st == 0, 4 * b)) continue;
            uint32_t nl = 0; int bits = 0;
            const bool built = zk_huf_build(tabs[b], sc, __shfl_sync(0xFFFFFFFFu, nw, 4 * b), lane, &nl, &bits);
            __syncwarp();
            if (si == b) { st = built ? 0 : ZKZ_CORRUPTION; n_low = nl; huf_bits = bits; }
        }
        // 2. decode: one lane per stream
        const ZkHufTab& tb = tabs[si];
        bool ok = true;
        if (live && st == 0) {
            const uint8_t* q = ebase + blk.src + lh.hdr + tree_bytes;
            uint32_t qn = lh.comp - tree_bytes;
            uint8_t* out = a.lit + blk.lit_base;
            if (lh.streams == 1) {
                if (stream == 0) ok = zk_huf_decode_stream(tb, n_low, huf_bits, q, qn, out, lh.regen);
            } else {
                uint32_t seg = (lh.regen + 3) / 4;
                if (qn < 10 || lh.regen < 6 || seg * 3 > lh.regen) ok = false;   // jump table + 4 non-empty streams; libzstd rejects regen < 6
                else {
                    uint32_t s1 = zk_ld_le16(q), s2 = zk_ld_le16(q + 2), s3 = zk_ld_le16(q + 4);
                    if (6 + s1 + s2 + s3 >= qn) ok = false;
                    else {
                        uint32_t s4 = qn - 6 - s1 - s2 - s3;
                        uint32_t off = stream == 0 ? 0 : (stream == 1 ? s1 : (stream == 2 ? s1 + s2 : s1 + s2 + s3));
                        uint32_t len = stream == 0 ? s1 : (stream == 1 ? s2 : (stream == 2 ? s3 : s4));
                        uint32_t cnt = stream < 3 ? seg : lh.regen - 3 * seg;
                        ok = zk_huf_decode_stream(tb, n_low, huf_bits, q + 6 + off, len, out + stream * seg, cnt);
                    }
                }
            }
        }
        uint32_t bad = __ballot_sync(0xFFFFFFFFu, !ok);
        if (live && stream == 0) {
            if (!st && ((bad >> (si * 4)) & 0xFu)) st = ZKZ_CORRUPTION;
            a.blocks[bidx].lit_status = st ? -st : 0;
        }
        __syncwarp();
    }
}

// =============================================================================================
// K-D0o / K-D1o: work order -- heaviest item first.
//
// Every persistent decode stage pulls its items from a work counter, so it lasts about as long as its heaviest item plus
// however late that item was pulled.  Handing out the items by cost, heaviest first (LPT), bounds a stage near the larger
// of its longest item and the mean load per worker, and gives the 4 chains of a K-D1s warp and the 8 blocks of a K-D1h
// warp similar costs.  The key is bucketed into quarter octaves of log2(1 + cost) and the list counting-sorted, one CTA
// per list; the order inside a bucket is whatever the shared-memory atomics give, which no output depends on.
//   K-D0o (after the scan):  seq_list by nseq, huf_list by lit_size
//   K-D1o (after the plan):  both halves of seg_list by seg_key
// The ordered lists keep the layout of the ones they are made from and are what the consumers receive as their lists.
// =============================================================================================
#define ZK_ORD_ALPHA 16u            // segment cost: ZK_ORD_ALPHA x sequences + output bytes
#define ZK_ORD_BUCKETS 128u         // 4 per octave of a 32-bit key
#define ZK_ORD_THREADS 1024u
#define ZK_ORD_UNROLL 4u

__device__ __forceinline__ uint32_t zk_ord_bucket(uint32_t cost) {
    const unsigned long long v = (unsigned long long)cost + 1u;
    const uint32_t hb = 63u - (uint32_t)__clzll((long long)v);
    const uint32_t frac = hb >= 2 ? (uint32_t)(v >> (hb - 2)) & 3u : (uint32_t)(v << (2 - hb)) & 3u;
    const uint32_t b = 4u * hb + frac;
    return b < ZK_ORD_BUCKETS ? b : ZK_ORD_BUCKETS - 1u;
}

// src / dst: the list, item i at base + dir * i; key of item i: keys ? keys[base + dir * i] : the field of blocks[src item]
template <int FIELD>
__device__ void zk_order_list(const ZkDecodeArgs& a, const uint32_t* src, uint32_t* dst, const uint32_t* keys, uint32_t n,
                              uint64_t base, int dir) {
    __shared__ uint32_t hist[ZK_ORD_BUCKETS];
    for (uint32_t b = threadIdx.x; b < ZK_ORD_BUCKETS; b += blockDim.x) hist[b] = 0;
    __syncthreads();
    auto bucket = [&](uint32_t i) -> uint32_t {
        const uint64_t at = base + (int64_t)dir * i;
        if (keys) return zk_ord_bucket(keys[at]);
        const uint32_t bidx = src[at];
        if (bidx >= a.cap_blocks) return 0;            // (every reserved slot is written by the scan kernel)
        return zk_ord_bucket(FIELD == 0 ? a.blocks[bidx].nseq : a.blocks[bidx].lit_size);
    };
    for (uint32_t i0 = threadIdx.x; i0 < n; i0 += ZK_ORD_UNROLL * blockDim.x) {
        uint32_t bk[ZK_ORD_UNROLL];
#pragma unroll
        for (uint32_t u = 0; u < ZK_ORD_UNROLL; u++) { const uint32_t i = i0 + u * blockDim.x; bk[u] = i < n ? bucket(i) : 0u; }
#pragma unroll
        for (uint32_t u = 0; u < ZK_ORD_UNROLL; u++) if (i0 + u * blockDim.x < n) atomicAdd(&hist[bk[u]], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 32) {                            // exclusive scan from the heaviest bucket down: where each bucket starts
        const uint32_t lane = threadIdx.x, per = ZK_ORD_BUCKETS / 32u;
        uint32_t h[ZK_ORD_BUCKETS / 32u], sum = 0;
        for (uint32_t k = 0; k < per; k++) { h[k] = hist[ZK_ORD_BUCKETS - 1u - (lane * per + k)]; sum += h[k]; }
        uint32_t incl = sum;
        for (int d = 1; d < 32; d <<= 1) { const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, incl, d); if ((int)lane >= d) incl += x; }
        uint32_t run = incl - sum;
        for (uint32_t k = 0; k < per; k++) { hist[ZK_ORD_BUCKETS - 1u - (lane * per + k)] = run; run += h[k]; }
    }
    __syncthreads();
    for (uint32_t i0 = threadIdx.x; i0 < n; i0 += ZK_ORD_UNROLL * blockDim.x) {
        uint32_t bk[ZK_ORD_UNROLL];
#pragma unroll
        for (uint32_t u = 0; u < ZK_ORD_UNROLL; u++) { const uint32_t i = i0 + u * blockDim.x; bk[u] = i < n ? bucket(i) : 0u; }
#pragma unroll
        for (uint32_t u = 0; u < ZK_ORD_UNROLL; u++) {
            const uint32_t i = i0 + u * blockDim.x;
            if (i >= n) continue;
            const uint32_t pos = atomicAdd(&hist[bk[u]], 1u);
            dst[base + (int64_t)dir * pos] = src[base + (int64_t)dir * i];
        }
    }
}

// Two CTAs: the lists of one stage side by side.  o holds the ordered lists (ZkDecodeWs::ord_list).
__global__ void __launch_bounds__(ZK_ORD_THREADS) zk_order_kernel(ZkDecodeArgs a, ZkDecodeArgs o, int segs) {
    if (a.counters->overflow) return;
    if (segs) {
        if (blockIdx.x == 0) zk_order_list<2>(a, a.seg_list, o.seg_list, a.seg_key, a.counters->n_long, 0, 1);
        else zk_order_list<2>(a, a.seg_list, o.seg_list, a.seg_key, a.counters->n_short, a.cap_blocks - 1, -1);
    } else {
        if (blockIdx.x == 0) zk_order_list<0>(a, a.seq_list, o.seq_list, nullptr, a.counters->n_seq_blocks, 0, 1);
        else zk_order_list<1>(a, a.huf_list, o.huf_list, nullptr, a.counters->n_huf_blocks, 0, 1);
    }
}

// =============================================================================================
// K-D1p: execution plan -- one warp per entry.
//
// The serial walk over an entry's blocks is cut into SEGMENTS: runs of consecutive blocks that read nothing written
// before their first block.  Segments are independent, so K-D2 runs them on different CTAs, and no CTA ever waits for
// another.  Block b starts a segment iff it is the entry's first block, or
//   * no match of b or of any later block (up to where the walk stops) reads before b's first byte -- which also rules
//     out symbolic offsets from b on (ZkBlock::back is unknown for those), and
//   * b starts a zstd frame, or its outgoing repeat offsets are concrete,
// so every repeat offset inside a segment resolves from state created inside it.  The checks the serial walk made as it
// went (a failed entropy stage, output overflow, Frame_Content_Size, the final size, the wanted prefix of a range read)
// are made here: they only need the regenerated sizes.  The walk stops at the first of them; the failure is kept as a key
// ordered like the serial walk (block, then check), and K-D2 adds the bad offsets it meets by atomicMin.
// =============================================================================================
__device__ void zk_entry_finish(const ZkDecodeArgs& a, uint32_t e) {
    ZkEntry& en = a.entries[e];
    const unsigned long long f = *(volatile unsigned long long*)&en.fail;
    if (f == ~0ull) { en.status = 0; return; }
    const uint32_t bi = (uint32_t)(f >> 32), stage = (uint32_t)(f >> 16) & 0xFFu;
    en.status = -(int32_t)(f & 0xFFFFu);
    if (bi < en.n_blocks) {             // the walk stopped before the failing block, or after it for a frame size mismatch
        const ZkBlock& b = a.blocks[en.first_block + bi];
        en.produced = b.out_pos + (stage == ZK_FAIL_FCS ? b.regen : 0u);
    }
    atomicAdd(&a.counters->n_errors, 1u);
}

__global__ void __launch_bounds__(128) zk_plan_kernel(ZkDecodeArgs a) {
    const int lane = threadIdx.x & 31;
    const uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (e >= a.n_entries || a.counters->overflow) return;
    const ZkEntry ent = a.entries[e];
    if (ent.status != 0) return;
    ZkBlock* blocks = a.blocks + ent.first_block;
    const unsigned long long cap64 = a.d_off[e + 1] - a.d_off[e];
    const unsigned long long cap = cap64 > 0xFFFFFFFFull ? 0xFFFFFFFFull : cap64;
    const unsigned long long need = a.d_need ? a.d_need[e] : 0xFFFFFFFFull;
    // ---- forward: output positions, frame starts, where the walk stops
    unsigned long long pos = 0, zs = 0, fail = ~0ull;
    uint32_t run = ent.n_blocks;
    bool stopped = false;
    for (uint32_t t = 0; t < ent.n_blocks; t += 32) {
        const uint32_t bi = t + (uint32_t)lane;
        const bool in = bi < ent.n_blocks;
        uint32_t regen = 0, flags = 0; int32_t st = 0; unsigned long long fcs = 0;
        if (in) { const ZkBlock& b = blocks[bi]; regen = b.regen; flags = b.flags; st = b.status ? b.status : b.lit_status; fcs = b.fcs; }
        unsigned long long end = regen, fs = in && (flags & ZKB_FIRST) ? 1ull + bi : 0ull;   // fs: 1 + index of the frame's first block
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long x = __shfl_up_sync(0xFFFFFFFFu, end, d), y = __shfl_up_sync(0xFFFFFFFFu, fs, d);
            if (lane >= d) { end += x; fs = fs > y ? fs : y; }
        }
        end += pos;
        const unsigned long long p = end - regen;
        // the frame start is the position of that first block: p of its lane, or the carry from an earlier tile
        const unsigned long long fsp = __shfl_sync(0xFFFFFFFFu, p, fs > t ? (int)(fs - 1 - t) : 0);
        const unsigned long long z = fs > t ? fsp : zs;
        uint32_t stage = 0, code = 0;
        bool ev = false;
        if (in) {
            if (p >= need) ev = true;                                                    // the wanted prefix is complete
            else if (st) { ev = true; stage = ZK_FAIL_STATUS; code = (uint32_t)-st; }
            else if (end > cap) { ev = true; stage = ZK_FAIL_DST; code = ZKZ_DST_TOO_SMALL; }
            else if ((flags & ZKB_LAST) && (flags & ZKB_HAS_FCS) && fcs != end - z) { ev = true; stage = ZK_FAIL_FCS; code = ZKZ_CORRUPTION; }
        }
        const uint32_t evm = __ballot_sync(0xFFFFFFFFu, ev);
        const int first = evm ? __ffs((int)evm) - 1 : 32;
        if (in && lane <= first) {
            ZkBlock& b = blocks[bi];
            b.out_pos = (uint32_t)p; b.frame_start = (uint32_t)z;
            if ((flags & ZKB_LAST) && !ev) { b.hash_start = (uint32_t)z; b.hash_len = (uint32_t)(end - z); }
        }
        if (evm) {
            if (lane == first) {
                if (code) fail = ZK_FAIL_KEY(bi, stage, code);
                else stopped = true;
                run = stage == ZK_FAIL_FCS ? bi + 1 : bi;
                pos = p;
            }
            fail = __shfl_sync(0xFFFFFFFFu, fail, first); stopped = __shfl_sync(0xFFFFFFFFu, (uint32_t)stopped, first) != 0;
            run = __shfl_sync(0xFFFFFFFFu, run, first); pos = __shfl_sync(0xFFFFFFFFu, pos, first);
            break;
        }
        pos = __shfl_sync(0xFFFFFFFFu, end, 31); zs = __shfl_sync(0xFFFFFFFFu, z, 31);
    }
    if (fail == ~0ull && !stopped && pos != cap64)                                      // tagged after the last block
        fail = ZK_FAIL_KEY(ent.n_blocks, ZK_FAIL_STATUS, pos < cap64 ? ZKZ_SRC_SIZE_WRONG : ZKZ_DST_TOO_SMALL);
    // ---- backward over the blocks that run: suffix minimum of the lowest position read, segment starts
    long long low = 0x7FFFFFFFFFFFFFFFll;                                                // lowest position read by the blocks after this tile
    uint32_t nseg = 0;
    __syncwarp();
    uint32_t seg_end = run ? blocks[run - 1].out_pos + blocks[run - 1].regen : 0u;      // output end of the first segment after this tile
    uint32_t seg_send = run ? blocks[run - 1].seq_base + blocks[run - 1].nseq : 0u;    // and its sequence end (seq_base runs on per entry)
    for (uint32_t t = run ? (run - 1) & ~31u : 0; run; t -= 32) {
        const uint32_t bi = t + (uint32_t)lane;
        const bool in = bi < run;
        long long lo = 0x7FFFFFFFFFFFFFFFll;
        uint32_t flags = 0, op = 0, sb = 0; bool conc = false;
        if (in) {
            const ZkBlock& b = blocks[bi];
            flags = b.flags; op = b.out_pos; sb = b.seq_base;
            lo = b.back == ZK_BACK_UNKNOWN ? -0x7FFFFFFFFFFFFFFFll : (long long)op - (long long)b.back;
            conc = !((b.rep_out[0] | b.rep_out[1] | b.rep_out[2]) & ZK_SYM);
        }
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const long long x = __shfl_down_sync(0xFFFFFFFFu, lo, d);
            if (lane + d < 32 && x < lo) lo = x;
        }
        if (low < lo) lo = low;
        const bool start = in && (bi == 0 || (lo >= (long long)op && ((flags & ZKB_FIRST) || conc)));
        if (in) blocks[bi].flags = (uint8_t)(start ? flags | ZKB_SEG : flags & ~ZKB_SEG);
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, start);
        if (m) {
            // a segment ends where the next one starts (in this tile, else seg_end); short ones go to the single-warp list
            const uint32_t later = m & (0xFFFFFFFEu << lane);
            const uint32_t nxp = __shfl_sync(0xFFFFFFFFu, op, later ? __ffs((int)later) - 1 : 0);
            const uint32_t nxs = __shfl_sync(0xFFFFFFFFu, sb, later ? __ffs((int)later) - 1 : 0);
            const uint32_t end = later ? nxp : seg_end, send = later ? nxs : seg_send;
            const unsigned long long cost = (unsigned long long)ZK_ORD_ALPHA * (send - sb) + (end - op);
            const uint32_t key = cost > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)cost;
            const uint32_t ms = __ballot_sync(0xFFFFFFFFu, start && a.exec_short && end - op <= a.exec_short), mlong = m & ~ms;
            uint32_t base_l = 0, base_s = 0;
            if (lane == 0) {
                if (mlong) base_l = atomicAdd(&a.counters->n_long, (uint32_t)__popc(mlong));
                if (ms) base_s = atomicAdd(&a.counters->n_short, (uint32_t)__popc(ms));
            }
            base_l = __shfl_sync(0xFFFFFFFFu, base_l, 0); base_s = __shfl_sync(0xFFFFFFFFu, base_s, 0);
            const uint32_t below = (1u << lane) - 1u;
            if (start) {
                const uint64_t at = ((ms >> lane) & 1u) ? a.cap_blocks - 1 - (base_s + __popc(ms & below)) : base_l + __popc(mlong & below);
                a.seg_list[at] = ent.first_block + bi; a.seg_key[at] = key;
            }
            nseg += __popc(m);
            seg_end = __shfl_sync(0xFFFFFFFFu, op, __ffs((int)m) - 1);
            seg_send = __shfl_sync(0xFFFFFFFFu, sb, __ffs((int)m) - 1);
        }
        low = __shfl_sync(0xFFFFFFFFu, lo, 0);
        if (t == 0) break;
    }
    if (lane == 0) {
        ZkEntry& en = a.entries[e];
        en.run_blocks = run; en.produced = (uint32_t)pos; en.fail = fail; en.segs_left = nseg;
        if (nseg == 0) zk_entry_finish(a, e);
    }
}

// =============================================================================================
// K-D2: ordered sequence execution with a shared-memory window.
//
// One CTA per seek-table entry, W warps.  The entry's sequences are cut into chunks of 32 (one per
// lane); chunk c belongs to warp c % W.  The last R bytes of output live in a shared-memory ring:
// every copy writes into the ring, dependent (recent) match sources are read from the ring
// (~30-cycle latency instead of an L2 round trip -- the first version spent 60 % of its samples
// waiting on those), and each finished chunk is flushed to HBM with 16-byte stores.
//   * done_pos / done_chunk : in-order publication of finished chunks (everything below done_pos
//     is final AND flushed to HBM);
//   * a chunk may start once its end lies within R/2 of done_pos, so the in-flight region never
//     laps the ring; a source at distance < R/2 from the chunk start is therefore still resident;
//   * chunks larger than R/2, Raw/RLE blocks and literal-only blocks run alone ("direct" path:
//     HBM to HBM, then the ring is re-synchronised from HBM).
// =============================================================================================
#define ZK_LONG 48u     // literal runs / matches at least this long are copied by the whole warp

#define ZK_D2_META 64u          // chunk descriptors kept in shared memory (chunks between the oldest unflushed and the newest started)

struct ZkD2Smem {
    // in-order prefixes, advanced co-operatively by whoever polls ("helping"); nobody ever waits for a predecessor to publish
    uint32_t done_pos, done_chunk;         // every byte below done_pos is final (readable from the ring); chunks [0, done_chunk) are done
    uint32_t flushed_pos, flushed_chunk;   // ... and below flushed_pos it is in HBM too
    int abort_code;
    uint32_t abort_block;                  // the earliest block (entry-relative) at which a warp aborted
    uint32_t seg;                          // the segment this CTA runs now (index into seg_list)
    // per-chunk descriptors, slot = chunk & (ZK_D2_META-1); a field is valid for chunk k iff its tag == k + 1
    uint32_t started[ZK_D2_META], start[ZK_D2_META], end[ZK_D2_META], done[ZK_D2_META], flushed[ZK_D2_META];
    // per-SEQUENCE completion inside a chunk (the dependency chain of a frame runs sequence to sequence, not chunk to chunk):
    uint32_t oe[ZK_D2_META][32];          // end position of each of the chunk's 32 sequences (non-decreasing; lanes past the last = chunk end)
    uint32_t dmask[ZK_D2_META];           // bit j: sequence j is completely written (literals + match)
    uint32_t litdone[ZK_D2_META];         // tag: every literal run of the chunk is in place
};
#define ZK_VOL(x) (*(volatile uint32_t*)&(x))

__device__ __forceinline__ void zk_d2_abort(ZkD2Smem& sm, int code, uint32_t block) { atomicCAS(&sm.abort_code, 0, code); atomicMin(&sm.abort_block, block); }
// warp-uniform view of the abort flag (every lane must take the same branch around collectives)
__device__ __forceinline__ bool zk_d2_aborted(ZkD2Smem& sm) { return __any_sync(0xFFFFFFFFu, *(volatile int*)&sm.abort_code != 0); }

// advance the in-order prefixes as far as the per-chunk flags allow (any thread may do this at any time)
__device__ __noinline__ void zk_d2_help(ZkD2Smem& sm) {
    uint32_t dc = ZK_VOL(sm.done_chunk), dc0 = dc, dp = 0;
    while (ZK_VOL(sm.done[dc & (ZK_D2_META - 1)]) == dc + 1) { dp = ZK_VOL(sm.end[dc & (ZK_D2_META - 1)]); dc++; }
    if (dc != dc0) { atomicMax(&sm.done_pos, dp); __threadfence_block(); atomicMax(&sm.done_chunk, dc); }
    uint32_t fc = ZK_VOL(sm.flushed_chunk), fc0 = fc, fp = 0;
    while (ZK_VOL(sm.flushed[fc & (ZK_D2_META - 1)]) == fc + 1) { fp = ZK_VOL(sm.end[fc & (ZK_D2_META - 1)]); fc++; }
    if (fc != fc0) { atomicMax(&sm.flushed_pos, fp); __threadfence_block(); atomicMax(&sm.flushed_chunk, fc); }
}

// warp-cooperative copy of n bytes HBM -> HBM, non-overlapping (or src entirely before dst with distance >= n)
__device__ __noinline__ void zk_warp_copy(uint8_t* dst, const uint8_t* src, uint32_t n, int lane) {
    uint32_t head = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
    if (head > n) head = n;
    if (lane < (int)head) dst[lane] = src[lane];
    dst += head; src += head; n -= head;
    uint32_t nvec = n >> 4;
    uint32_t mis = (uint32_t)((uintptr_t)src & 3);
    if (mis == 0) {
        if (((uintptr_t)src & 15) == 0) {
            for (uint32_t i = lane; i < nvec; i += 32) ((uint4*)dst)[i] = ((const uint4*)src)[i];
        } else {
            for (uint32_t i = lane; i < nvec; i += 32) {
                const uint32_t* s = (const uint32_t*)src + 4 * i;
                ((uint4*)dst)[i] = make_uint4(s[0], s[1], s[2], s[3]);
            }
        }
    } else {
        const uint32_t* sa = (const uint32_t*)(src - mis);
        uint32_t sh = mis * 8;
        for (uint32_t i = lane; i < nvec; i += 32) {
            const uint32_t* s = sa + 4 * i;
            uint32_t w0 = s[0], w1 = s[1], w2 = s[2], w3 = s[3], w4 = s[4];
            ((uint4*)dst)[i] = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh),
                                          __funnelshift_r(w2, w3, sh), __funnelshift_r(w3, w4, sh));
        }
    }
    uint32_t done = nvec << 4;
    for (uint32_t i = done + lane; i < n; i += 32) dst[i] = src[i];
}

__device__ __noinline__ void zk_warp_fill(uint8_t* dst, uint32_t byte, uint32_t n, int lane) {
    uint32_t head = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
    if (head > n) head = n;
    if (lane < (int)head) dst[lane] = (uint8_t)byte;
    dst += head; n -= head;
    uint32_t w = byte * 0x01010101u, nvec = n >> 4;
    for (uint32_t i = lane; i < nvec; i += 32) ((uint4*)dst)[i] = make_uint4(w, w, w, w);
    for (uint32_t i = (nvec << 4) + lane; i < n; i += 32) dst[i] = (uint8_t)byte;
}

// warp-cooperative match copy in HBM: dst[0..n) = dst[-off ..), overlap allowed (period doubling)
__device__ __noinline__ void zk_warp_match(uint8_t* dst, uint32_t off, uint32_t n, int lane) {
    const uint8_t* src = dst - off;
    if (off >= n) { zk_warp_copy(dst, src, n, lane); return; }
    uint32_t have = off, done = 0;            // [src, src+have) is final periodic data
    while (done < n) {
        uint32_t c = n - done < have ? n - done : have;
        zk_warp_copy(dst + done, src, c, lane);
        __syncwarp();
        done += c; have += c;
    }
}

// the low min(k, 8) bytes of (lo, hi) -> p[0..): predicated byte stores at immediate offsets (k >= 1)
__device__ __forceinline__ void zk_st_bytes8(uint8_t* p, uint32_t lo, uint32_t hi, uint32_t k) {
    p[0] = (uint8_t)lo;
    if (k > 1) p[1] = (uint8_t)(lo >> 8);
    if (k > 2) p[2] = (uint8_t)(lo >> 16);
    if (k > 3) p[3] = (uint8_t)(lo >> 24);
    if (k > 4) p[4] = (uint8_t)hi;
    if (k > 5) p[5] = (uint8_t)(hi >> 8);
    if (k > 6) p[6] = (uint8_t)(hi >> 16);
    if (k > 7) p[7] = (uint8_t)(hi >> 24);
}

// per-CTA view of the ring: position p (entry-relative) lives at ring[(p + mis) & mask], mis = (out address & 15)
// so that 16-byte groups of the ring line up with 16-byte groups of HBM.
struct ZkRing {
    uint8_t* ring; uint32_t mask, mis; uint8_t* out;
    __device__ __forceinline__ uint8_t& at(uint32_t p) const { return ring[(p + mis) & mask]; }
    // unaligned 8-byte read of positions [p, p+8) (three aligned word reads, wrap-safe)
    __device__ __forceinline__ unsigned long long ld8(uint32_t p) const {
        const uint32_t idx = (p + mis) & mask, wi = idx & ~3u, sh = (idx & 3u) * 8u;
        const uint32_t w0 = *(const uint32_t*)(ring + wi), w1 = *(const uint32_t*)(ring + ((wi + 4) & mask)), w2 = *(const uint32_t*)(ring + ((wi + 8) & mask));
        return (unsigned long long)__funnelshift_r(w0, w1, sh) | ((unsigned long long)__funnelshift_r(w1, w2, sh) << 32);
    }
    // lane-local match copy inside the ring, 8 bytes per step when the period allows it.  This copy sits on the dependency
    // chain of the frame AND was 40 % of all instructions of the kernel when it stored byte by byte through at() (address
    // arithmetic, 64-bit shifts and loop control per byte: ~12 instructions a byte); without a wrap on either side it is three
    // word loads, two funnel shifts and predicated byte stores at immediate offsets.
    __device__ __forceinline__ void copy_near(uint32_t dst, uint32_t src, uint32_t n) const {
        const uint32_t size = mask + 1, di = (dst + mis) & mask, si = (src + mis) & mask;
        if (dst - src >= 8) {
            if (di + n <= size && si + n + 12 <= size) {
                uint8_t* dp = ring + di; const uint32_t* sp = (const uint32_t*)(ring + (si & ~3u)); const uint32_t sh = (si & 3u) * 8u;
                for (uint32_t i = 0; i < n; i += 8) {
                    const uint32_t w0 = sp[0], w1 = sp[1], w2 = sp[2];
                    zk_st_bytes8(dp, __funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), n - i);
                    dp += 8; sp += 2;
                }
            } else {
                for (uint32_t i = 0; i < n; i += 8) {
                    unsigned long long v = ld8(src + i);
                    const uint32_t k = n - i < 8 ? n - i : 8;
                    for (uint32_t q = 0; q < k; q++) { at(dst + i + q) = (uint8_t)v; v >>= 8; }
                }
            }
        } else for (uint32_t i = 0; i < n; i++) at(dst + i) = at(src + i);
    }
    // store the low min(k, 8) bytes of (lo, hi) at positions [p, p + k) of the entry
    __device__ __forceinline__ void st8(uint32_t p, uint32_t lo, uint32_t hi, uint32_t k) const {
        const uint32_t di = (p + mis) & mask;
        if (di + 8 <= mask + 1) zk_st_bytes8(ring + di, lo, hi, k);
        else { unsigned long long v = (unsigned long long)lo | ((unsigned long long)hi << 32); for (uint32_t q = 0; q < k && q < 8; q++) { at(p + q) = (uint8_t)v; v >>= 8; } }
    }
};

// flush [s, e) ring -> HBM: full 16-byte groups with vector stores, the ragged head and tail (neighbours own the rest of those
// groups) byte-parallel by lanes 0..15 / 16..31
__device__ __forceinline__ void zk_ring_flush(const ZkRing& rg, uint32_t s, uint32_t e, int lane) {
    if (e <= s) return;
    const uint32_t sb = s + rg.mis, eb = e + rg.mis;                       // shifted positions: 16-byte groups line up with HBM
    const uint32_t uf0 = (sb + 15) >> 4, uf1 = eb >> 4;                    // full groups [uf0, uf1)
    for (uint32_t u = uf0 + lane; u < uf1; u += 32) { const uint32_t g = u << 4; *(uint4*)(rg.out + (g - rg.mis)) = *(const uint4*)(rg.ring + (g & rg.mask)); }
    const uint32_t head_end = (uf0 << 4) < eb ? (uf0 << 4) : eb;
    if (lane < 16) { const uint32_t q = sb + (uint32_t)lane; if (q < head_end) rg.out[q - rg.mis] = rg.ring[q & rg.mask]; }
    else if (uf1 >= uf0) { const uint32_t q = (uf1 << 4) + (uint32_t)lane - 16u; if (q < eb) rg.out[q - rg.mis] = rg.ring[q & rg.mask]; }
}

// reload [s, e) HBM -> ring (after a direct HBM-to-HBM block)
__device__ __noinline__ void zk_ring_reload(const ZkRing& rg, uint32_t s, uint32_t e, int tid, int nthr) {
    if (e <= s) return;
    const uint32_t u0 = (s + rg.mis) >> 4, u1 = (e + rg.mis - 1) >> 4;
    for (uint32_t u = u0 + tid; u <= u1; u += nthr) {
        const uint32_t g = u << 4;
        const uint32_t lo = g > s + rg.mis ? g : s + rg.mis, hi = g + 16 < e + rg.mis ? g + 16 : e + rg.mis;
        if (hi - lo == 16) *(uint4*)(rg.ring + (g & rg.mask)) = *(const uint4*)(rg.out + (g - rg.mis));
        else for (uint32_t q = lo; q < hi; q++) rg.ring[q & rg.mask] = rg.out[q - rg.mis];
    }
}

// unaligned 8-byte little-endian load from HBM (three aligned 4-byte loads issued back to back)
__device__ __forceinline__ unsigned long long zk_ld8_unaligned(const uint8_t* p) {
    uintptr_t a = (uintptr_t)p; uint32_t mis = (uint32_t)(a & 3);
    const uint32_t* q = (const uint32_t*)(a - mis);
    uint32_t w0 = q[0], w1 = q[1];
    if (mis == 0) return (unsigned long long)w0 | ((unsigned long long)w1 << 32);
    uint32_t w2 = q[2], sh = mis * 8;
    return (unsigned long long)__funnelshift_r(w0, w1, sh) | ((unsigned long long)__funnelshift_r(w1, w2, sh) << 32);
}

// Place the literal runs of one chunk.  The runs are CONTIGUOUS in the block's literal buffer ([lit_lo, lit_hi)), so the
// warp reads them with coalesced loads, 32 bytes a step, and every byte finds its destination by a 5-step search over the
// lanes' cumulative literal ends (le is non-decreasing across lanes).  A per-lane byte loop paid one HBM round trip per
// byte and was the real bottleneck of the first exec kernels.  TO_RING: destination is the ring, else HBM directly.
template <bool TO_RING>
__device__ __forceinline__ void zk_chunk_literals(const ZkRing& rg, const uint8_t* lit, int lit_kind, uint32_t lit_byte, uint32_t le, uint32_t le_prev,
                                                  uint32_t o_lit, int lane) {
    const uint32_t lit_lo = __shfl_sync(0xFFFFFFFFu, le_prev, 0), lit_hi = __shfl_sync(0xFFFFFFFFu, le, 31);
    for (uint32_t base = lit_lo; base < lit_hi; base += 256) {
        // issue up to eight coalesced 32-byte loads first (one memory latency for 256 literal bytes), then place them
        uint32_t bytes[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const uint32_t t = base + u * 32 + lane;
            bytes[u] = lit_byte;
            if (t < lit_hi && lit_kind != 1) bytes[u] = lit[t];
        }
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const uint32_t t = base + u * 32 + lane;
            if (base + u * 32 >= lit_hi) break;           // warp-uniform
            const bool active = t < lit_hi;
            int lo = 0, hi = 31;                          // owner = first lane whose le > t
#pragma unroll
            for (int step = 0; step < 5; step++) {
                const int mid = (lo + hi) >> 1;
                const uint32_t v = __shfl_sync(0xFFFFFFFFu, le, mid);
                if (v > t) hi = mid; else lo = mid + 1;
            }
            const uint32_t d0 = __shfl_sync(0xFFFFFFFFu, o_lit, lo), l0 = __shfl_sync(0xFFFFFFFFu, le_prev, lo);
            if (active) {
                const uint32_t dest = d0 + (t - l0);
                if (TO_RING) rg.at(dest) = (uint8_t)bytes[u]; else rg.out[dest] = (uint8_t)bytes[u];
            }
        }
    }
}

// Prefix mode: the prefix of an entry's zstd frames, its range of the prefix buffer (ZkDecodeArgs::pranges): `len` bytes that end at `end`
struct ZkPrefixSlice { const uint8_t* end; uint32_t len; };
__device__ __forceinline__ ZkPrefixSlice zk_entry_prefix(const ZkDecodeArgs& a, uint32_t e) {
    const uint32_t lo = a.pranges[2 * e], hi = a.pranges[2 * e + 1];
    return {a.prefix + hi, hi - lo};
}

// Prefix mode: the part of a match that lies before its frame's first byte (zstart) comes from the raw-content prefix that
// precedes every zstd frame of the entry.  That part is constant data with no dependency, copied at once by its lane; what is left
// of the match, if anything, starts at the frame's first byte with the same offset and is an ordinary match.  TO_RING: destination
// is the ring, else HBM directly.
template <bool TO_RING>
__device__ __forceinline__ void zk_prefix_part(const ZkRing& rg, const ZkPrefixSlice& px, bool valid, uint32_t zstart, uint32_t off,
                                               uint32_t& md, uint32_t& ml) {
    if (valid && ml > 0 && off > md - zstart) {
        const uint32_t back = off - (md - zstart), la = ml < back ? ml : back;
        const uint8_t* ps = px.end - back;
        for (uint32_t i = 0; i < la; i++) { if (TO_RING) rg.at(md + i) = ps[i]; else rg.out[md + i] = ps[i]; }
        md += la; ml -= la;
    }
}

// ---------------------------------------------------------------------------------------------
// The work both segment executors (zk_exec_segment, zk_exec_warp_segment) share: repeat offsets, loading and checking the
// sequences of a chunk, blocks without sequences, trailing literals, direct chunks, match copies into the ring and the end
// of a segment.  A bound check that reached one executor only would accept a corrupt frame on some segment lengths only.
// ---------------------------------------------------------------------------------------------

// R0..R2 while a segment's blocks execute in order
struct ZkRepOffsets {
    uint32_t r0 = 1, r1 = 4, r2 = 8;
    __device__ __forceinline__ void reset() { r0 = 1; r1 = 4; r2 = 8; }        // a zstd frame starts
    // the incoming slot a symbolic value (ZK_SYM) names; the value is that minus its ZK_SYM_DELTA
    __device__ __forceinline__ uint32_t slot(uint32_t v) const { const uint32_t sl = ZK_SYM_SLOT(v); return sl == 0 ? r0 : (sl == 1 ? r1 : r2); }
    // the state after a block with sequences: its rep_out, symbolic values resolved against the state before it
    __device__ __forceinline__ void advance(const ZkBlock& blk) {
        uint32_t n[3];
        for (int q = 0; q < 3; q++) { const uint32_t v = blk.rep_out[q]; n[q] = (v & ZK_SYM) ? slot(v) - ZK_SYM_DELTA(v) : v; }
        r0 = n[0]; r1 = n[1]; r2 = n[2];
    }
};

// One lane's sequence of a chunk of 32: the literal run lit[le_prev, le) goes to [o_lit, md), then a match of ml bytes at md
// from md - off (entry-relative positions; PREFIX: md / ml shrink to the in-frame part).  le / oe are the cumulative literal
// / output ends of the block's sequences; lanes past the block's last sequence repeat its ends (zero-length runs; keeps `le`
// monotone across the lanes).
struct ZkLaneSeq {
    bool valid;
    uint32_t le, oe, le_prev, oe_prev, ll, ml, o_lit, md, off;
};

// Load lane `lane`'s sequence of chunk j of a block (sequences seq_base + [32j, 32j + 32) of nseq); le0 / oe0 are lane 0's
// predecessor ends (those of sequence 32j - 1, 0 for the first chunk).  Resolves a symbolic offset and checks the offset
// against the output of the frame before it (and the entry's prefix, px).  Returns, on every lane, whether some lane's offset is bad.
template <bool PREFIX>
__device__ __forceinline__ bool zk_lane_seq(ZkLaneSeq& q, const ZkDecodeArgs& a, uint32_t seq_base, uint32_t nseq, const ZkRepOffsets& rep,
                                            uint32_t j, uint32_t pos, uint32_t zstart, uint32_t le0, uint32_t oe0, int lane,
                                            const ZkPrefixSlice& px) {
    const uint32_t s = j * 32 + lane;
    q.valid = s < nseq;
    const uint32_t sc = q.valid ? s : nseq - 1;
    q.le = a.seq_lit_end[seq_base + sc]; q.oe = a.seq_out_end[seq_base + sc];
    const uint32_t offv = q.valid ? a.seq_off[seq_base + s] : 0u;
    q.le_prev = __shfl_up_sync(0xFFFFFFFFu, q.le, 1); q.oe_prev = __shfl_up_sync(0xFFFFFFFFu, q.oe, 1);
    if (lane == 0) { q.le_prev = le0; q.oe_prev = oe0; }
    q.ll = q.le - q.le_prev; q.ml = (q.oe - q.oe_prev) - q.ll;
    q.o_lit = pos + q.oe_prev; q.md = q.o_lit + q.ll;
    q.off = offv;
    bool bad = false;
    if (q.valid) {
        if (offv & ZK_SYM) {
            const uint32_t r = rep.slot(offv), dl = ZK_SYM_DELTA(offv);
            bad = r <= dl; q.off = r - dl;
        }
        if (q.off == 0 || q.off > q.md - zstart + (PREFIX ? px.len : 0u)) bad = true;
    }
    return __any_sync(0xFFFFFFFFu, bad);
}

__device__ __forceinline__ const uint8_t* zk_block_lit(const ZkDecodeArgs& a, const ZkBlock& blk, const uint8_t* ebase) {
    return blk.lit_kind == 0 ? ebase + blk.lit_src : a.lit + blk.lit_base;
}

// A Raw block, an RLE block or a compressed block without sequences: HBM to HBM at [pos, pos + regen), then the ring is
// reloaded with the last half ring of it (nothing before pos0: that output belongs to another warp or CTA).
__device__ __forceinline__ void zk_direct_block(const ZkRing& rg, const ZkDecodeArgs& a, const ZkBlock& blk, const uint8_t* ebase,
                                                uint32_t pos, uint32_t pos0, uint32_t half, int lane) {
    uint8_t* d = rg.out + pos;
    const uint32_t en = pos + blk.regen;
    if (blk.type == 0) zk_warp_copy(d, ebase + blk.src, blk.size, lane);
    else if (blk.type == 1) zk_warp_fill(d, ebase[blk.src], blk.size, lane);
    else if (blk.lit_kind == 1) zk_warp_fill(d, blk.lit_byte, blk.lit_size, lane);
    else zk_warp_copy(d, zk_block_lit(a, blk, ebase), blk.lit_size, lane);
    __syncwarp();
    zk_ring_reload(rg, en - pos0 > half ? en - half : pos0, en, lane, 32);
}

// The literals after a block's last sequence, lit[le, le + n) to [st0, en): more than half a ring HBM to HBM, then the ring is
// reloaded (the caller runs them alone); else into the ring, and the caller flushes [st0, en).
__device__ __forceinline__ void zk_trailing_literals(const ZkRing& rg, uint32_t lit_kind, uint32_t lit_byte, const uint8_t* lit, uint32_t le, uint32_t n,
                                                     uint32_t st0, uint32_t en, uint32_t half, int lane) {
    if (n > half) {
        if (lit_kind == 1) zk_warp_fill(rg.out + st0, lit_byte, n, lane);
        else zk_warp_copy(rg.out + st0, lit + le, n, lane);
        __syncwarp();
        zk_ring_reload(rg, en - half, en, lane, 32);
    } else {
        for (uint32_t i = lane; i < n; i += 32) rg.at(st0 + i) = lit_kind == 1 ? lit_byte : lit[le + i];
    }
}

// A chunk larger than half a ring: built HBM to HBM while everything before it is final (the CTA kernel runs it alone), then
// the ring is reloaded with its last half ring.  Literal runs of 256 bytes or more are copied by the whole warp, shorter ones
// byte-parallel; within the chunk, a match goes once every earlier match that its source overlaps is written.
template <bool PREFIX>
__device__ __forceinline__ void zk_direct_chunk(const ZkRing& rg, const ZkPrefixSlice& px, uint32_t lit_kind, uint32_t lit_byte, const uint8_t* lit, ZkLaneSeq& q,
                                                uint32_t zstart, uint32_t chunk_end, uint32_t half, int lane) {
    uint8_t* out = rg.out;
    uint32_t longlit = __ballot_sync(0xFFFFFFFFu, q.valid && q.ll >= 256);
    if (!longlit) zk_chunk_literals<false>(rg, lit, lit_kind, lit_byte, q.le, q.le_prev, q.o_lit, lane);
    else {
        if (q.valid && q.ll < 256) {
            uint8_t* d = out + q.o_lit;
            if (lit_kind == 1) for (uint32_t i = 0; i < q.ll; i++) d[i] = lit_byte;
            else { const uint8_t* sp = lit + q.le_prev; for (uint32_t i = 0; i < q.ll; i++) d[i] = sp[i]; }
        }
        while (longlit) {
            int l = __ffs((int)longlit) - 1; longlit &= longlit - 1;
            uint32_t n = __shfl_sync(0xFFFFFFFFu, q.ll, l), d = __shfl_sync(0xFFFFFFFFu, q.o_lit, l), sp = __shfl_sync(0xFFFFFFFFu, q.le_prev, l);
            if (lit_kind == 1) zk_warp_fill(out + d, lit_byte, n, lane);
            else zk_warp_copy(out + d, lit + sp, n, lane);
        }
    }
    if (PREFIX) zk_prefix_part<false>(rg, px, q.valid, zstart, q.off, q.md, q.ml);
    __syncwarp();
    const uint32_t need_end = q.md - q.off + (q.ml < q.off ? q.ml : q.off);
    uint32_t pending = __ballot_sync(0xFFFFFFFFu, q.valid && q.ml > 0);
    while (pending) {
        const int first = __ffs((int)pending) - 1;
        const uint32_t frontier = __shfl_sync(0xFFFFFFFFu, q.md, first);
        const bool mine = (pending >> lane) & 1;
        const bool ready = mine && (need_end <= frontier || lane == first);
        const uint32_t rmask = __ballot_sync(0xFFFFFFFFu, ready);
        if (ready && q.ml < ZK_LONG) {
            uint8_t* d = out + q.md; const uint8_t* sp = d - q.off;
            for (uint32_t i = 0; i < q.ml; i++) d[i] = sp[i];
        }
        uint32_t longm = __ballot_sync(0xFFFFFFFFu, ready && q.ml >= ZK_LONG);
        while (longm) {
            int l = __ffs((int)longm) - 1; longm &= longm - 1;
            uint32_t n = __shfl_sync(0xFFFFFFFFu, q.ml, l), d = __shfl_sync(0xFFFFFFFFu, q.md, l), o = __shfl_sync(0xFFFFFFFFu, q.off, l);
            zk_warp_match(out + d, o, n, lane);
        }
        __syncwarp();
        pending &= ~rmask;
    }
    zk_ring_reload(rg, chunk_end - half, chunk_end, lane, 32);
}

// The matches of the `ready` lanes, built in the ring.  A short one is copied by its lane: from the ring if its source is near
// (less than half a ring before the chunk start, so all of it is resident), else from HBM, where it is final and never
// overlaps, 8 bytes per round trip.  A long one (>= ZK_LONG) is copied by the whole warp.
__device__ __forceinline__ void zk_ring_matches(const ZkRing& rg, bool ready, bool near_src, uint32_t md, uint32_t off, uint32_t ml, int lane) {
    if (ready && ml < ZK_LONG) {
        if (near_src) rg.copy_near(md, md - off, ml);
        else {
            const uint8_t* sp = rg.out + (md - off);
            for (uint32_t i = 0; i < ml; i += 8) {
                const unsigned long long v = zk_ld8_unaligned(sp + i);
                rg.st8(md + i, (uint32_t)v, (uint32_t)(v >> 32), ml - i < 8 ? ml - i : 8);
            }
        }
    }
    uint32_t longm = __ballot_sync(0xFFFFFFFFu, ready && ml >= ZK_LONG);
    while (longm) {
        const int l = __ffs((int)longm) - 1; longm &= longm - 1;
        const uint32_t n = __shfl_sync(0xFFFFFFFFu, ml, l), d = __shfl_sync(0xFFFFFFFFu, md, l), o = __shfl_sync(0xFFFFFFFFu, off, l);
        const bool nr = __shfl_sync(0xFFFFFFFFu, (uint32_t)near_src, l) != 0;
        if (!nr) { const uint8_t* sp = rg.out + (d - o); for (uint32_t i = lane; i < n; i += 32) rg.at(d + i) = sp[i]; }
        else if (o >= n) { for (uint32_t i = lane; i < n; i += 32) rg.at(d + i) = rg.at(d - o + i); }
        else if (o >= 32) {           // overlapping, period >= 32: 32 bytes per step are already final
            for (uint32_t i0 = 0; i0 < n; i0 += 32) { const uint32_t i = i0 + lane; if (i < n) rg.at(d + i) = rg.at(d - o + i); __syncwarp(); }
        } else {                      // short period: replicate the pattern
            for (uint32_t i = lane; i < n; i += 32) rg.at(d + i) = rg.at(d - o + (i % o));
        }
    }
}

// One thread, once a segment is done: record its failure (a bad offset at entry-relative block fail_block; code 0 = none)
// and, if it was the entry's last segment, write the entry's status.
__device__ __forceinline__ void zk_segment_end(const ZkDecodeArgs& a, uint32_t e, uint32_t fail_block, int code) {
    ZkEntry& en = a.entries[e];
    if (code) atomicMin(&en.fail, ZK_FAIL_KEY(fail_block, ZK_FAIL_EXEC, code));
    __threadfence();
    if (atomicSub(&en.segs_left, 1u) == 1u) { __threadfence(); zk_entry_finish(a, e); }   // the entry's last segment
}

// chunk c's bytes are final in the ring: dependants may read them
__device__ __forceinline__ void zk_d2_mark_done(ZkD2Smem& sm, uint32_t c, int lane) {
    __threadfence_block();
    __syncwarp();
    if (lane == 0) {
        const uint32_t e = c & (ZK_D2_META - 1);
        ZK_VOL(sm.dmask[e]) = 0xFFFFFFFFu; ZK_VOL(sm.litdone[e]) = c + 1; ZK_VOL(sm.done[e]) = c + 1;
        zk_d2_help(sm);
    }
    __syncwarp();
}
// ... and now they are in HBM as well (far readers and ring reuse depend on this one)
__device__ __forceinline__ void zk_d2_mark_flushed(ZkD2Smem& sm, uint32_t c, int lane) {
    __threadfence_block();
    __syncwarp();
    if (lane == 0) { ZK_VOL(sm.flushed[c & (ZK_D2_META - 1)]) = c + 1; zk_d2_help(sm); }
    __syncwarp();
}

// announce chunk c = [start_pos, end_pos) and the end position of each of its sequences (seq_end per lane)
__device__ __forceinline__ void zk_d2_announce(ZkD2Smem& sm, uint32_t c, uint32_t start_pos, uint32_t end_pos, uint32_t seq_end, uint32_t premask, int lane) {
    const uint32_t e = c & (ZK_D2_META - 1);
    ZK_VOL(sm.oe[e][lane]) = seq_end;
    if (lane == 0) { ZK_VOL(sm.start[e]) = start_pos; ZK_VOL(sm.end[e]) = end_pos; ZK_VOL(sm.dmask[e]) = premask; }
    __threadfence_block();
    __syncwarp();
    if (lane == 0) ZK_VOL(sm.started[e]) = c + 1;
    __syncwarp();
}
// sequences `mask` of chunk c are completely written
__device__ __forceinline__ void zk_d2_progress(ZkD2Smem& sm, uint32_t c, uint32_t mask, int lane) {
    __threadfence_block();
    __syncwarp();
    if (lane == 0 && mask) atomicOr(&sm.dmask[c & (ZK_D2_META - 1)], mask);
}

// warp-uniform wait until chunk c = [start_pos, end_pos) may start.  Returns false if the CTA aborted.
// exclusive == false: its end lies within `window` of flushed_pos (the in-flight region never laps the ring);
// exclusive == true: every earlier chunk is done and flushed (the chunk then runs alone, HBM to HBM).
__device__ __forceinline__ bool zk_d2_wait_start(ZkD2Smem& sm, uint32_t c, uint32_t start_pos, uint32_t end_pos, uint32_t window, bool exclusive, int lane) {
    for (;;) {
        uint32_t ok = 0, ab = 0;
        if (lane == 0) {
            ab = *(volatile int*)&sm.abort_code != 0;
            uint32_t fc = ZK_VOL(sm.flushed_chunk), fp = ZK_VOL(sm.flushed_pos);
            ok = exclusive ? (fc == c) : (fc == c || (end_pos - fp <= window && c - fc < ZK_D2_META - 2));
            if (!ok) {           // only then is it worth walking the flags (the walk was 6 % of the kernel's instructions when done on every entry)
                zk_d2_help(sm);
                fc = ZK_VOL(sm.flushed_chunk); fp = ZK_VOL(sm.flushed_pos);
                ok = exclusive ? (fc == c) : (fc == c || (end_pos - fp <= window && c - fc < ZK_D2_META - 2));
            }
            __threadfence_block();
        }
        ok = __shfl_sync(0xFFFFFFFFu, ok, 0); ab = __shfl_sync(0xFFFFFFFFu, ab, 0);
        __syncwarp();
        if (ab) return false;
        if (ok) return true;
        ZK_SPIN();
    }
}

// One segment (K-D1p) of an entry: blocks [first block, next segment start or run_blocks), from the segment's output
// position on.  The ring and the in-order state start at that position; a segment's first block either starts a zstd
// frame or uses no repeat offset it did not set itself, so R0..R2 need no incoming state.  The checks that need only
// block sizes were made by the plan kernel, which also stopped the walk where the serial one stopped.
template <bool PREFIX>
__device__ __forceinline__ void zk_exec_segment(ZkD2Smem& sm, const ZkDecodeArgs& a, uint32_t ring_bytes, uint32_t first_bidx) {
    ZK_DYN_SMEM(ring_mem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;
    const ZkBlock head = a.blocks[first_bidx];
    const uint32_t e = head.entry;
    const ZkPrefixSlice px = PREFIX ? zk_entry_prefix(a, e) : ZkPrefixSlice{nullptr, 0u};
    const ZkEntry ent = a.entries[e];
    const uint32_t pos0 = head.out_pos;
    if (threadIdx.x == 0) { sm.done_pos = pos0; sm.done_chunk = 0; sm.flushed_pos = pos0; sm.flushed_chunk = 0; sm.abort_code = 0; sm.abort_block = 0xFFFFFFFFu; }
    for (uint32_t i = threadIdx.x; i < ZK_D2_META; i += blockDim.x) { sm.started[i] = 0; sm.done[i] = 0; sm.flushed[i] = 0; sm.litdone[i] = 0; }
    __syncthreads();
    uint8_t* out = a.dst + a.d_off[e];
    const uint8_t* ebase = a.comp + a.c_off[e];
    ZkRing rg; rg.ring = ring_mem; rg.mask = ring_bytes - 1; rg.mis = (uint32_t)((uintptr_t)out & 15); rg.out = out;
    const uint32_t half = ring_bytes >> 1;

    uint32_t pos = pos0, zstart = head.frame_start, chunk_base = 0;
    ZkRepOffsets rep;
    uint32_t preannounced = 0xFFFFFFFFu;          // chunk id this warp has already announced ahead of time
    for (uint32_t bi = first_bidx - ent.first_block; bi < ent.run_blocks; bi++) {
        if (zk_d2_aborted(sm)) break;
        const uint32_t bidx = ent.first_block + bi;
        const ZkBlock blk = a.blocks[bidx];
        if (bidx != first_bidx && (blk.flags & ZKB_SEG)) break;
        if (blk.flags & ZKB_FIRST) { rep.reset(); zstart = pos; }
        const bool has_seq = blk.type == 2 && blk.nseq > 0;
        const uint32_t nchunks = has_seq ? (blk.nseq + 31) / 32 + 1 : 1;
        // first chunk index of this block that belongs to this warp
        uint32_t c = chunk_base + ((uint32_t)warp + W - (chunk_base % W)) % W;
        for (; c < chunk_base + nchunks; c += W) {
            const uint32_t j = c - chunk_base;
            if (!has_seq) {
                // ---------------- Raw block / RLE block / literals-only compressed block: direct path, runs alone
                if (!zk_d2_wait_start(sm, c, pos, pos + blk.regen, 0, true, lane)) break;
                zk_d2_announce(sm, c, pos, pos + blk.regen, pos + blk.regen, 0u, lane);
                zk_direct_block(rg, a, blk, ebase, pos, pos0, half, lane);
                zk_d2_mark_done(sm, c, lane);
                zk_d2_mark_flushed(sm, c, lane);
                continue;
            }
            const uint32_t* s_lit = a.seq_lit_end + blk.seq_base;
            const uint32_t* s_out = a.seq_out_end + blk.seq_base;
            const uint8_t* lit = zk_block_lit(a, blk, ebase);
            if (j == nchunks - 1) {
                // ---------------- trailing literals of the block
                const uint32_t le = s_lit[blk.nseq - 1], oe = s_out[blk.nseq - 1];
                const uint32_t n = blk.lit_size - le, st0 = pos + oe, en = pos + blk.regen;
                const bool direct = n > half;
                if (!zk_d2_wait_start(sm, c, st0, en, half, direct, lane)) break;
                zk_d2_announce(sm, c, st0, en, en, 0u, lane);
                zk_trailing_literals(rg, blk.lit_kind, blk.lit_byte, lit, le, n, st0, en, half, lane);
                zk_d2_mark_done(sm, c, lane);
                if (!direct) zk_ring_flush(rg, st0, en, lane);
                zk_d2_mark_flushed(sm, c, lane);
                continue;
            }
            // ---------------- 32 sequences, one per lane
            uint32_t le0 = 0, oe0 = 0;
            if (lane == 0 && j) { le0 = s_lit[j * 32 - 1]; oe0 = s_out[j * 32 - 1]; }
            ZkLaneSeq q;
            if (zk_lane_seq<PREFIX>(q, a, blk.seq_base, blk.nseq, rep, j, pos, zstart, le0, oe0, lane, px)) { zk_d2_abort(sm, ZKZ_CORRUPTION, bi); break; }
            const uint32_t chunk_start = pos + __shfl_sync(0xFFFFFFFFu, q.oe_prev, 0);
            const uint32_t chunk_end = pos + __shfl_sync(0xFFFFFFFFu, q.oe, min(31u, blk.nseq - 1 - j * 32));
            const bool direct = chunk_end - chunk_start > half;
            if (!zk_d2_wait_start(sm, c, chunk_start, chunk_end, half, direct, lane)) break;
            if (preannounced != c) zk_d2_announce(sm, c, chunk_start, chunk_end, pos + q.oe, 0u, lane);
            // Announce this warp's NEXT chunk of the block right away (its sequence ends are one coalesced load away): chunks of
            // other warps that depend on it can then resolve their producers without waiting for this warp to get there.
            {
                const uint32_t jn = j + (uint32_t)W;
                if (jn < nchunks - 1) {
                    uint32_t okp = 0;
                    if (lane == 0) okp = (c + (uint32_t)W) - ZK_VOL(sm.flushed_chunk) < ZK_D2_META - 2;
                    if (__shfl_sync(0xFFFFFFFFu, okp, 0)) {
                        const uint32_t sn = jn * 32 + lane, scn = sn < blk.nseq ? sn : blk.nseq - 1;
                        const uint32_t oen = s_out[scn];
                        uint32_t stn = 0;
                        if (lane == 0) stn = s_out[jn * 32 - 1];
                        stn = __shfl_sync(0xFFFFFFFFu, stn, 0);
                        const uint32_t enn = __shfl_sync(0xFFFFFFFFu, oen, 31);
                        zk_d2_announce(sm, c + (uint32_t)W, pos + stn, pos + enn, pos + oen, 0u, lane);
                        preannounced = c + (uint32_t)W;
                    }
                }
            }

            if (direct) {
                // ======== huge chunk: HBM -> HBM, alone in flight (it is the oldest chunk)
                zk_direct_chunk<PREFIX>(rg, px, blk.lit_kind, blk.lit_byte, lit, q, zstart, chunk_end, half, lane);
                zk_d2_mark_done(sm, c, lane);
                zk_d2_mark_flushed(sm, c, lane);
                continue;
            }

            // ======== normal chunk: build the output in the ring, then flush
            // literal runs: no dependencies (HBM scratch -> ring)
            zk_chunk_literals<true>(rg, lit, blk.lit_kind, blk.lit_byte, q.le, q.le_prev, q.o_lit, lane);
            if (PREFIX) zk_prefix_part<true>(rg, px, q.valid, zstart, q.off, q.md, q.ml);
            {   // all literal runs are in place: sequences without a match (and the lanes past the last one) are complete
                const uint32_t withm = __ballot_sync(0xFFFFFFFFu, q.valid && q.ml > 0);
                zk_d2_progress(sm, c, ~withm, lane);
                if (lane == 0) ZK_VOL(sm.litdone[c & (ZK_D2_META - 1)]) = c + 1;
            }
            __syncwarp();

            // matches.  near: the whole source is still resident in the ring (distance < R/2 from the chunk start);
            // far: it is read from HBM and must be published (done_pos).  A lane may go once its source is final.
            const uint32_t src0 = q.md - q.off;
            const bool near_src = src0 + half >= chunk_start;          // src0 >= chunk_start - R/2
            const uint32_t need_end = src0 + (q.ml < q.off ? q.ml : q.off);
            uint32_t pending = __ballot_sync(0xFFFFFFFFu, q.valid && q.ml > 0);
            bool aborted = false;
            // dataflow readiness: a match may go as soon as the bytes of its source are final -- the part that lies before this
            // chunk is tracked per chunk (descriptors in shared memory), the part inside this chunk by lane order.  Sources older
            // than R/2 are in HBM by construction of the start rule (flushed_pos >= chunk_end - R/2 > any far source).
            // Step 1 (once): which in-flight chunks [klo, khi] produce my source?  Step 2 (poll): are they done?  The poll loop is
            // the critical link of the frame's dependency chain, so it only reads those few flags.
            uint32_t klo = 1, khi = 0;                                  // empty range: nothing to wait for outside this chunk
            uint32_t mask_lo = 0, mask_hi = 0;                          // which sequences of chunk klo / khi produce my source
            {
                bool resolved = !(q.valid && q.ml > 0) || !near_src || src0 >= chunk_start;
                const uint32_t ne = need_end < chunk_start ? need_end : chunk_start;
                for (;;) {
                    if (!resolved) {
                        // chunk ids are consecutive and their start positions increase with the id: two binary searches over
                        // the in-flight chunks [dc, c) find the chunks holding src0 and ne-1 (a linear walk cost one shared-memory
                        // round trip per chunk of distance and dominated the kernel)
                        const uint32_t dp = ZK_VOL(sm.done_pos), dc = ZK_VOL(sm.done_chunk);
                        if (ne <= dp || dc >= c) { resolved = true; klo = 1; khi = 0; }
                        else {
                            bool ok = true;
                            uint32_t lo = dc, hi = c - 1;                       // khi = largest k with start[k] < ne (start[dc] == done_pos < ne)
                            while (lo < hi) {
                                const uint32_t mid = (lo + hi + 1) >> 1, e = mid & (ZK_D2_META - 1);
                                if (ZK_VOL(sm.started[e]) != mid + 1) { ok = false; break; }
                                if (ZK_VOL(sm.start[e]) < ne) lo = mid; else hi = mid - 1;
                            }
                            const uint32_t kh = lo;
                            lo = dc; hi = kh;                                   // klo = largest k <= khi with start[k] <= src0, else dc
                            while (ok && lo < hi) {
                                const uint32_t mid = (lo + hi + 1) >> 1, e = mid & (ZK_D2_META - 1);
                                if (ZK_VOL(sm.started[e]) != mid + 1) { ok = false; break; }
                                if (ZK_VOL(sm.start[e]) <= src0) lo = mid; else hi = mid - 1;
                            }
                            const uint32_t kl = lo;
                            if (ok && (ZK_VOL(sm.started[kl & (ZK_D2_META - 1)]) != kl + 1 || ZK_VOL(sm.started[kh & (ZK_D2_META - 1)]) != kh + 1)) ok = false;
                            if (ok) {
                                resolved = true; klo = kl; khi = kh;
                                // first sequence of klo whose end lies beyond src0; last sequence of khi that starts before ne
                                int a = 0, b = 0;
                                { const uint32_t e = klo & (ZK_D2_META - 1); int lo2 = 0, hi2 = 31;
                                  for (int st = 0; st < 5; st++) { int mid = (lo2 + hi2) >> 1; if (ZK_VOL(sm.oe[e][mid]) > src0) hi2 = mid; else lo2 = mid + 1; } a = lo2; }
                                { const uint32_t e = khi & (ZK_D2_META - 1); int lo2 = 0, hi2 = 31;
                                  for (int st = 0; st < 5; st++) { int mid = (lo2 + hi2) >> 1; if (ZK_VOL(sm.oe[e][mid]) >= ne) hi2 = mid; else lo2 = mid + 1; } b = lo2; }
                                mask_lo = 0xFFFFFFFFu << a;
                                mask_hi = b >= 31 ? 0xFFFFFFFFu : ((2u << b) - 1u);
                                if (klo == khi) { mask_lo &= mask_hi; mask_hi = mask_lo; }
                            }
                        }
                    }
                    if (__all_sync(0xFFFFFFFFu, resolved)) break;
                    if (zk_d2_aborted(sm)) { aborted = true; break; }
                    ZK_SPIN();
                }
            }
            while (pending && !aborted) {
                const bool mine = (pending >> lane) & 1;
                bool ext_ok = true;
                if (mine && khi >= klo) {
                    const uint32_t dc = ZK_VOL(sm.done_chunk);
                    for (uint32_t k = khi + 1; k-- > klo;) {
                        if (k < dc) break;                                                   // it and everything older is done
                        const uint32_t e = k & (ZK_D2_META - 1);
                        const uint32_t need = k == khi ? mask_hi : (k == klo ? mask_lo : 0xFFFFFFFFu);
                        if (ZK_VOL(sm.started[e]) != k + 1 || ZK_VOL(sm.litdone[e]) != k + 1 || (ZK_VOL(sm.dmask[e]) & need) != need) { ext_ok = false; break; }
                    }
                    if (ext_ok) khi = 0, klo = 1;                       // sticky
                }
                const int first = __ffs((int)pending) - 1;
                const uint32_t md_first = __shfl_sync(0xFFFFFFFFu, q.md, first);   // inside this chunk everything below it is final
                const bool ready = mine && ext_ok && (need_end <= md_first || lane == first);
                const uint32_t rmask = __ballot_sync(0xFFFFFFFFu, ready);
                if (!rmask) { if (zk_d2_aborted(sm)) { aborted = true; break; } ZK_SPIN(); continue; }
                __threadfence_block();             // acquire: the flags were read before the data is
                zk_ring_matches(rg, ready, near_src, q.md, q.off, q.ml, lane);
                zk_d2_progress(sm, c, rmask, lane);    // dependants of these sequences may go now (not only when the whole chunk is done)
                __syncwarp();
                pending &= ~rmask;
            }
            if (aborted) break;
            zk_d2_mark_done(sm, c, lane);                          // dependants can read the ring now ...
            zk_ring_flush(rg, chunk_start, chunk_end, lane);       // ... while the HBM flush happens off the critical chain
            zk_d2_mark_flushed(sm, c, lane);
        }
        // advance to the next block
        if (has_seq) rep.advance(blk);
        pos += blk.regen;
        chunk_base += nchunks;
    }
    __syncthreads();
    if (threadIdx.x == 0) zk_segment_end(a, e, sm.abort_block, sm.abort_code);
}

// CTAs are persistent: each pulls segments from a work counter until none is left.  Segments never wait for each other,
// so a CTA that is not resident holds nobody up.
template <bool PREFIX>
__device__ __forceinline__ void zk_exec_body(ZkD2Smem& sm, const ZkDecodeArgs& a, uint32_t ring_bytes) {
    if (a.counters->overflow) return;
    const uint32_t nseg = a.counters->n_long;
    for (;;) {
        if (threadIdx.x == 0) sm.seg = atomicAdd(&a.work_counter[2], 1u);
        __syncthreads();
        const uint32_t s = sm.seg;
        if (s >= nseg) break;
        zk_exec_segment<PREFIX>(sm, a, ring_bytes, a.seg_list[s]);
        __syncthreads();                          // every warp is done with the segment before its state is reset
    }
}

// =============================================================================================
// K-D2w: short segments, one warp each.
//
// A segment is one serial chain that no other warp can shorten, so a warp runs it alone, strictly chunk after chunk:
// when a chunk starts, everything before it is final, and none of the CTA kernel's cross-warp bookkeeping (descriptors,
// completion masks, announcements, helping) is needed.  The warp keeps its last ZK_XW_WIN bytes of output in a private
// shared-memory window with the CTA kernel's discipline: a chunk of at most half a window is built there and flushed to
// HBM, so a source less than half a window before the chunk is still in the window ("near") and an older one is in HBM
// ("far", flushed by this warp earlier: __syncwarp orders it).  Larger chunks, Raw / RLE and literal-only blocks are
// copied HBM to HBM and the window is reloaded.  Inside a chunk, matches go in ballot rounds: a lane copies once every
// earlier lane whose destination overlaps its source is done.  Every store lies inside the segment's output range, which no other warp or
// CTA writes.  Repeat offsets, the offset check, direct chunks, copies and the failure key are the helpers zk_exec_segment calls.
// =============================================================================================
#define ZK_XW_WARPS 4u          // warps per CTA; __launch_bounds__ below asks for 8 CTAs (32 warps) per SM, i.e. <= 64 registers
#define ZK_XW_WIN 4096u         // window bytes per warp (H100, bench mix: 2 KiB ran as fast, 8 KiB 9 % slower)

template <bool PREFIX>
__device__ __forceinline__ void zk_exec_warp_segment(const ZkDecodeArgs& a, uint8_t* win, uint32_t first_bidx, int lane) {
    const ZkBlock& head = a.blocks[first_bidx];
    const uint32_t e = head.entry, pos0 = head.out_pos;
    const ZkPrefixSlice px = PREFIX ? zk_entry_prefix(a, e) : ZkPrefixSlice{nullptr, 0u};
    const ZkEntry ent = a.entries[e];
    uint8_t* out = a.dst + a.d_off[e];
    const uint8_t* ebase = a.comp + a.c_off[e];
    ZkRing rg; rg.ring = win; rg.mask = ZK_XW_WIN - 1; rg.mis = (uint32_t)((uintptr_t)out & 15); rg.out = out;
    const uint32_t half = ZK_XW_WIN >> 1;
    uint32_t pos = pos0, zstart = head.frame_start;
    ZkRepOffsets rep;
    uint32_t bad_block = 0xFFFFFFFFu;
    for (uint32_t bi = first_bidx - ent.first_block; bi < ent.run_blocks && bad_block == 0xFFFFFFFFu; bi++) {
        const uint32_t bidx = ent.first_block + bi;
        const ZkBlock& blk = a.blocks[bidx];
        const uint32_t flags = blk.flags, nseq = blk.nseq, regen = blk.regen;
        if (bidx != first_bidx && (flags & ZKB_SEG)) break;
        if (flags & ZKB_FIRST) { rep.reset(); zstart = pos; }
        if (!(blk.type == 2 && nseq > 0)) {
            // ---------------- Raw block / RLE block / literals-only compressed block: HBM to HBM
            zk_direct_block(rg, a, blk, ebase, pos, pos0, half, lane);
            pos += regen;
            __syncwarp();
            continue;
        }
        const uint32_t seq_base = blk.seq_base, lit_kind = blk.lit_kind, lit_byte = blk.lit_byte;
        const uint8_t* lit = zk_block_lit(a, blk, ebase);
        uint32_t le_last = 0, oe_last = 0;            // cumulative literal / output ends of the sequences before the chunk
        for (uint32_t j = 0; j * 32 < nseq; j++) {
            // ---------------- 32 sequences, one per lane
            ZkLaneSeq q;
            if (zk_lane_seq<PREFIX>(q, a, seq_base, nseq, rep, j, pos, zstart, le_last, oe_last, lane, px)) { bad_block = bi; break; }
            le_last = __shfl_sync(0xFFFFFFFFu, q.le, 31); oe_last = __shfl_sync(0xFFFFFFFFu, q.oe, 31);
            const uint32_t chunk_start = pos + __shfl_sync(0xFFFFFFFFu, q.oe_prev, 0), chunk_end = pos + oe_last;
            if (chunk_end - chunk_start > half) {
                zk_direct_chunk<PREFIX>(rg, px, lit_kind, lit_byte, lit, q, zstart, chunk_end, half, lane);
                __syncwarp();
                continue;
            }
            if (PREFIX) zk_prefix_part<true>(rg, px, q.valid, zstart, q.off, q.md, q.ml);
            const uint32_t src0 = q.md - q.off, need_end = src0 + (q.ml < q.off ? q.ml : q.off);
            const bool near_src = src0 + half >= chunk_start;
            zk_chunk_literals<true>(rg, lit, lit_kind, lit_byte, q.le, q.le_prev, q.o_lit, lane);
            __syncwarp();
            uint32_t pending = __ballot_sync(0xFFFFFFFFu, q.valid && q.ml > 0);
            while (pending) {
                // everything below the first pending match's destination is final
                const int first = __ffs((int)pending) - 1;
                const uint32_t md_first = __shfl_sync(0xFFFFFFFFu, q.md, first);
                const bool ready = ((pending >> lane) & 1u) && (need_end <= md_first || lane == first);
                const uint32_t rmask = __ballot_sync(0xFFFFFFFFu, ready);
                zk_ring_matches(rg, ready, near_src, q.md, q.off, q.ml, lane);
                __syncwarp();
                pending &= ~rmask;
            }
            zk_ring_flush(rg, chunk_start, chunk_end, lane);
            __syncwarp();
        }
        if (bad_block != 0xFFFFFFFFu) break;
        {   // ---------------- trailing literals of the block
            const uint32_t n = blk.lit_size - le_last, st0 = pos + oe_last, en = pos + regen;
            zk_trailing_literals(rg, lit_kind, lit_byte, lit, le_last, n, st0, en, half, lane);
            __syncwarp();
            if (n <= half) zk_ring_flush(rg, st0, en, lane);
            __syncwarp();
        }
        rep.advance(blk);
        pos += regen;
    }
    if (lane == 0) zk_segment_end(a, e, bad_block, bad_block != 0xFFFFFFFFu ? ZKZ_CORRUPTION : 0);
    __syncwarp();
}

// Persistent: every warp pulls short segments from its own work counter until none is left.
template <bool PREFIX>
__global__ void __launch_bounds__(32 * ZK_XW_WARPS, 8) zk_exec_warp_kernel(ZkDecodeArgs a) {
    ZK_DYN_SMEM(win_mem);
    if (a.counters->overflow) return;
    const int lane = threadIdx.x & 31;
    uint8_t* win = win_mem + (threadIdx.x >> 5) * ZK_XW_WIN;
    const uint32_t nshort = a.counters->n_short;
    for (;;) {
        uint32_t s = 0;
        if (lane == 0) s = atomicAdd(&a.work_counter[3], 1u);
        s = __shfl_sync(0xFFFFFFFFu, s, 0);
        if (s >= nshort) break;
        zk_exec_warp_segment<PREFIX>(a, win, a.seg_list[a.cap_blocks - 1 - s], lane);
    }
}

// Two register budgets for the same body: up to 16 warps per entry (<= 128 registers, few entries per SM), and a
// 5-warp variant compiled for 4 CTAs per SM (<= 102 registers) for large batches, where every entry of the batch should
// stay resident and the warps per SM are what hides the latency.
template <bool PREFIX>
__global__ void __launch_bounds__(512, 1) zk_exec_kernel(ZkDecodeArgs a, uint32_t ring_bytes) {
    __shared__ ZkD2Smem sm;
    zk_exec_body<PREFIX>(sm, a, ring_bytes);
}
template <bool PREFIX>
__global__ void __launch_bounds__(160, 4) zk_exec_kernel_w5(ZkDecodeArgs a, uint32_t ring_bytes) {
    __shared__ ZkD2Smem sm;
    zk_exec_body<PREFIX>(sm, a, ring_bytes);
}

// =============================================================================================
// K-D3: XXH64 content checksum (A.8), one warp per entry, lanes 0..3 carry the four accumulators
// =============================================================================================
__global__ void __launch_bounds__(128) zk_xxh64_kernel(ZkDecodeArgs a) {
    const int lane = threadIdx.x & 31;
    const uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (e >= a.n_entries) return;
    ZkEntry ent = a.entries[e];
    if (ent.status != 0 || a.counters->overflow) return;
    if (a.d_need && (unsigned long long)a.d_need[e] < a.d_off[e + 1] - a.d_off[e]) return;   // a prefix only: no checksum, as the reference (decode.rs:425-427)
    const uint8_t* out = a.dst + a.d_off[e];
    const uint8_t* ebase = a.comp + a.c_off[e];
    for (uint32_t bi = 0; bi < ent.n_blocks; bi++) {
        const ZkBlock* blk = &a.blocks[ent.first_block + bi];
        uint32_t flags = blk->flags;
        if ((flags & (ZKB_LAST | ZKB_HAS_CSUM)) != (ZKB_LAST | ZKB_HAS_CSUM)) continue;
        uint32_t content = blk->type == 1 ? 1u : blk->size;
        uint32_t want = zk_ld_le32(ebase + blk->src + content);
        unsigned long long h = zk_warp_xxh64(out + blk->hash_start, blk->hash_len, lane);
        if ((uint32_t)h != want) {
            if (lane == 0) { a.entries[e].status = -ZKZ_CHECKSUM_WRONG; atomicAdd(&a.counters->n_errors, 1u); }
            return;
        }
    }
}

// =============================================================================================
// host-side launcher
// =============================================================================================
#define ZK_WORK_COUNTERS 5

void zk_decode_ws_free(ZkDecodeWs* ws) {
    void* ptrs[] = { ws->blocks, ws->entries, ws->counters, ws->lit, ws->seq_lit_end, ws->seq_out_end, ws->seq_off, ws->c_off, ws->d_off,
                     ws->huf_list, ws->seq_list, ws->seg_list, ws->ord_list, ws->seg_key, ws->d_need, ws->d_pr };
    for (void* p : ptrs) if (p) cudaFree(p);
    if (ws->h_need) cudaFreeHost(ws->h_need);
    if (ws->h_pr) cudaFreeHost(ws->h_pr);
    if (ws->h_entries) cudaFreeHost(ws->h_entries);
    if (ws->h_counters) cudaFreeHost(ws->h_counters);
    if (ws->h_off) cudaFreeHost(ws->h_off);
    if (ws->side) cudaStreamDestroy(ws->side);
    if (ws->ev_scan) cudaEventDestroy(ws->ev_scan);
    if (ws->ev_huf) cudaEventDestroy(ws->ev_huf);
    if (ws->ev_up) cudaEventDestroy(ws->ev_up);
    if (ws->ev_done) cudaEventDestroy(ws->ev_done);
    if (ws->ev_down) cudaEventDestroy(ws->ev_down);
    ws->prof.destroy();
    *ws = ZkDecodeWs();
}

static int zk_decode_ensure(ZkDecodeWs* ws, uint32_t n, size_t need_blocks, size_t need_lit, size_t need_seq) {
    int rc;
    size_t cap;
    if (ws->cap_blocks < need_blocks || !ws->blocks) {
        size_t c1 = ws->cap_blocks, c2 = ws->cap_blocks, c3 = ws->cap_blocks, c4 = ws->cap_blocks, c5 = ws->cap_blocks, c6 = ws->cap_blocks;
        if ((rc = zk_grow((void**)&ws->blocks, &c1, need_blocks, sizeof(ZkBlock)))) return rc;
        if ((rc = zk_grow((void**)&ws->huf_list, &c2, need_blocks, 4))) return rc;
        if ((rc = zk_grow((void**)&ws->seq_list, &c3, 2 * need_blocks, 4))) return rc;   // two lists (ZkDecodeArgs::seq_list)
        c3 /= 2;
        if ((rc = zk_grow((void**)&ws->seg_list, &c4, need_blocks, 4))) return rc;
        if ((rc = zk_grow((void**)&ws->ord_list, &c5, 4 * need_blocks, 4))) return rc;   // ordered seq (two lists), huf, seg
        c5 /= 4;
        if ((rc = zk_grow((void**)&ws->seg_key, &c6, need_blocks, 4))) return rc;
        ws->cap_blocks = c1 < c2 ? (c1 < c3 ? c1 : c3) : (c2 < c3 ? c2 : c3);
        if (c4 < ws->cap_blocks) ws->cap_blocks = c4;
        if (c5 < ws->cap_blocks) ws->cap_blocks = c5;
        if (c6 < ws->cap_blocks) ws->cap_blocks = c6;
    }
    cap = ws->cap_lit; if ((rc = zk_grow((void**)&ws->lit, &cap, need_lit + 64, 1))) return rc; ws->cap_lit = cap;
    if (ws->cap_seq < need_seq || !ws->seq_off) {
        size_t c1 = ws->cap_seq, c2 = ws->cap_seq, c3 = ws->cap_seq;
        if ((rc = zk_grow((void**)&ws->seq_lit_end, &c1, need_seq, 4))) return rc;
        if ((rc = zk_grow((void**)&ws->seq_out_end, &c2, need_seq, 4))) return rc;
        if ((rc = zk_grow((void**)&ws->seq_off, &c3, need_seq, 4))) return rc;
        ws->cap_seq = c1 < c2 ? (c1 < c3 ? c1 : c3) : (c2 < c3 ? c2 : c3);
    }
    if (ws->cap_entries < n || !ws->entries) {
        size_t c = ws->cap_entries;
        if ((rc = zk_grow((void**)&ws->entries, &c, n, sizeof(ZkEntry)))) return rc;
        size_t c2 = 0, c3 = 0;
        if (ws->c_off) { cudaFree(ws->c_off); ws->c_off = nullptr; }
        if (ws->d_off) { cudaFree(ws->d_off); ws->d_off = nullptr; }
        if ((rc = zk_grow((void**)&ws->c_off, &c2, c + 1, 8))) return rc;
        if ((rc = zk_grow((void**)&ws->d_off, &c3, c + 1, 8))) return rc;
        if (ws->h_entries) cudaFreeHost(ws->h_entries);
        if (ws->h_off) cudaFreeHost(ws->h_off);
        if (cudaMallocHost((void**)&ws->h_entries, c * sizeof(ZkEntry)) != cudaSuccess) return -(int)ZKZ_MEMORY_ALLOCATION;
        if (cudaMallocHost((void**)&ws->h_off, 2 * (c + 1) * 8) != cudaSuccess) return -(int)ZKZ_MEMORY_ALLOCATION;
        if (ws->d_need) { cudaFree(ws->d_need); ws->d_need = nullptr; }
        if (ws->h_need) { cudaFreeHost(ws->h_need); ws->h_need = nullptr; }
        if (ws->d_pr) { cudaFree(ws->d_pr); ws->d_pr = nullptr; }
        if (ws->h_pr) { cudaFreeHost(ws->h_pr); ws->h_pr = nullptr; }
        if (cudaMalloc((void**)&ws->d_need, (c + 1) * 4) != cudaSuccess) return -(int)ZKZ_MEMORY_ALLOCATION;
        if (cudaMallocHost((void**)&ws->h_need, (c + 1) * 4) != cudaSuccess) return -(int)ZKZ_MEMORY_ALLOCATION;
        if (cudaMalloc((void**)&ws->d_pr, c * 8) != cudaSuccess) return -(int)ZKZ_MEMORY_ALLOCATION;
        if (cudaMallocHost((void**)&ws->h_pr, c * 8) != cudaSuccess) return -(int)ZKZ_MEMORY_ALLOCATION;
        ws->cap_entries = c;
    }
    if (!ws->counters) {
        if (cudaMalloc((void**)&ws->counters, sizeof(ZkCounters) + ZK_WORK_COUNTERS * 4) != cudaSuccess) return -(int)ZKZ_MEMORY_ALLOCATION;
        if (cudaMallocHost((void**)&ws->h_counters, sizeof(ZkCounters) + ZK_WORK_COUNTERS * 4) != cudaSuccess) return -(int)ZKZ_MEMORY_ALLOCATION;
    }
    return 0;
}

// Enqueue one batch on `stream` (scan, entropy, exec[, checksum], status read-back).  No host sync.
int zk_decode_enqueue(ZkDecodeWs* ws, cudaStream_t stream, const uint8_t* d_comp, const uint64_t* c_off, const uint64_t* d_off,
                      uint32_t n, uint8_t* d_dst, int verify_checksum, const ZkDecodeParams& p) {
    ws->pending_n = 0;
    if (n == 0) return 0;
    unsigned long long total_d = d_off[n] - d_off[0];
    // optimistic scratch sizing; the scan kernel reports exact needs and zk_decode_collect retries if exceeded
    size_t need_blocks = (size_t)(total_d / 32768u) + 4 * (size_t)n + 64;      // this codec's own encoder cuts 32 KiB blocks (libzstd: 128 KiB)
    size_t need_lit = (size_t)total_d + 16 * need_blocks;
    size_t need_seq = (size_t)(total_d / 4) + 1024;
    if (need_blocks < ws->want_blocks) need_blocks = ws->want_blocks;
    if (need_lit < ws->want_lit) need_lit = ws->want_lit;
    if (need_seq < ws->want_seq) need_seq = ws->want_seq;
    int sms = ws->sm_count > 0 ? ws->sm_count : 132;
    int rc = zk_decode_ensure(ws, n, need_blocks, need_lit, need_seq);
    if (rc) return rc;
    memcpy(ws->h_off, c_off, (size_t)(n + 1) * 8);
    memcpy(ws->h_off + (n + 1), d_off, (size_t)(n + 1) * 8);
    // Host pipelines hand in dedicated copy streams (p.up / p.down): copies of different compute streams otherwise share
    // copy-engine channels, where the upload of one sub-batch queues behind the status read-back of another that is still
    // waiting for its kernels (measured: sub-batch k + 4 started its upload when sub-batch k had finished its download).
    cudaStream_t us = p.up ? p.up : stream, ds = p.down ? p.down : stream;
    if (us != stream && !ws->ev_up) {
        ZK_CUDA_OK(cudaEventCreateWithFlags(&ws->ev_up, cudaEventDisableTiming)); ZK_CUDA_OK(cudaEventCreateWithFlags(&ws->ev_done, cudaEventDisableTiming));
        ZK_CUDA_OK(cudaEventCreateWithFlags(&ws->ev_down, cudaEventDisableTiming));
    }
    ZK_CUDA_OK(cudaMemcpyAsync(ws->c_off, ws->h_off, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, us));
    ZK_CUDA_OK(cudaMemcpyAsync(ws->d_off, ws->h_off + (n + 1), (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, us));
    ZK_CUDA_OK(cudaMemsetAsync(ws->counters, 0, sizeof(ZkCounters) + ZK_WORK_COUNTERS * 4, stream));
    ZkDecodeArgs a;
    a.comp = d_comp; a.c_off = (const unsigned long long*)ws->c_off; a.d_off = (const unsigned long long*)ws->d_off; a.dst = d_dst; a.n_entries = n;
    a.blocks = ws->blocks; a.entries = ws->entries; a.counters = ws->counters;
    a.work_counter = (uint32_t*)((uint8_t*)ws->counters + sizeof(ZkCounters));   // seq, huf, exec, single-warp exec, full-layout seq; zeroed with the struct
    a.lit = ws->lit; a.seq_lit_end = ws->seq_lit_end; a.seq_out_end = ws->seq_out_end; a.seq_off = ws->seq_off;
    a.huf_list = ws->huf_list; a.seq_list = ws->seq_list; a.seg_list = ws->seg_list;
    a.cap_blocks = ws->cap_blocks; a.cap_lit = ws->cap_lit - 64; a.cap_seq = ws->cap_seq;
    a.d_need = nullptr; a.seg_key = ws->seg_key;
    a.prefix = p.prefix; a.pranges = nullptr;
    if (p.prefix) {                              // every entry's range of the prefix buffer (the whole buffer without p.ranges)
        for (uint32_t i = 0; i < n; i++) {
            ws->h_pr[2 * i] = p.ranges ? p.ranges[2 * i] : 0u; ws->h_pr[2 * i + 1] = p.ranges ? p.ranges[2 * i + 1] : p.prefix_len;
        }
        ZK_CUDA_OK(cudaMemcpyAsync(ws->d_pr, ws->h_pr, (size_t)n * 8, cudaMemcpyHostToDevice, us));
        a.pranges = ws->d_pr;
    }
    if (p.need) {
        memcpy(ws->h_need, p.need, (size_t)n * 4);
        ZK_CUDA_OK(cudaMemcpyAsync(ws->d_need, ws->h_need, (size_t)n * 4, cudaMemcpyHostToDevice, us));
        a.d_need = ws->d_need;
    }
    if (us != stream) { ZK_CUDA_OK(cudaEventRecord(ws->ev_up, us)); ZK_CUDA_OK(cudaStreamWaitEvent(stream, ws->ev_up, 0)); }   // also orders the caller's upload of the compressed bytes
    // the consumers of the work lists get `o`: the lists as filled, or their copies ordered heaviest first (K-D0o, K-D1o)
    ZkDecodeArgs o = a;
    if (ws->order) { o.seq_list = ws->ord_list; o.huf_list = ws->ord_list + 2 * ws->cap_blocks; o.seg_list = ws->ord_list + 3 * ws->cap_blocks; }
    ws->prof.begin(0, stream);
    ZK_LAUNCH(zk_scan_kernel, (n + 127) / 128, 128, 0, stream, a);
    if (ws->order) ZK_LAUNCH(zk_order_kernel, 2, ZK_ORD_THREADS, 0, stream, a, o, 0);
    ws->prof.end(0, stream);
    // entropy stage: persistent warp-CTAs pulling groups of blocks from a work counter
    size_t est_blocks = (size_t)(total_d / ZK_BLOCK_MAX) + n;
    constexpr size_t huf_smem = sizeof(ZkHufTab) * ZK_HUF_SLOTS + sizeof(ZkHufScratch);
    static_assert(huf_smem <= 48 * 1024, "K-D1h launches without a shared-memory opt-in");
    const size_t seq2_smem = ((sizeof(ZkSeqTabs) + 127) & ~(size_t)127) + sizeof(ZkSeq2Chain<ZK_SEQ_CELLS_COMPACT>) * ZK_S2_NCH;
    const size_t seq2f_smem = ((sizeof(ZkSeqTabs) + 127) & ~(size_t)127) + sizeof(ZkSeq2Chain<ZK_SEQ_CELLS_FULL>) * ZK_S2_NCH;
    if (!ws->attr_set) {
        ZK_CUDA_OK(cudaFuncSetAttribute(zk_seq2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)seq2_smem));
        ZK_CUDA_OK(cudaFuncSetAttribute(zk_seq2_full_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)seq2f_smem));
        ZK_CUDA_OK(cudaFuncSetAttribute(zk_exec_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
        ZK_CUDA_OK(cudaFuncSetAttribute(zk_exec_kernel_w5<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
        ZK_CUDA_OK(cudaFuncSetAttribute(zk_exec_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
        ZK_CUDA_OK(cudaFuncSetAttribute(zk_exec_kernel_w5<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
        ws->attr_set = true;
    }
    if (!ws->huf_fit) {                          // K-D1h CTAs that fit on an SM by their shared memory
#ifndef ZK_EMUL
        int fit = 0;
        ZK_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, zk_huf_kernel, 32, huf_smem));
        ws->huf_fit = fit > 0 ? (uint32_t)fit : 1u;
#else
        ws->huf_fit = 16;                        // (no SM to fill)
#endif
    }
    // Half of them: K-D1s runs beside K-D1h, and the two only overlap when both fit on the SM (DESIGN §6).  K-D1s gets the CTAs
    // that fit in three quarters of an SM's shared memory (7 on H100: the best of 5-8 measured beside K-D1h's grid), at most
    // what the occupancy query allows; the CTAs of either kernel that do not fit beside the other's start as those finish.
    const uint32_t huf_ctas = ws->huf_fit > 1 ? ws->huf_fit / 2 : 1u;
    if (!ws->seq2_fit) {
#ifndef ZK_EMUL
        int dev = 0, fit = 0, sm_smem = 0, reserved = 0;
        ZK_CUDA_OK(cudaGetDevice(&dev));
        ZK_CUDA_OK(cudaDeviceGetAttribute(&sm_smem, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
        ZK_CUDA_OK(cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev));
        ZK_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, zk_seq2_kernel, 32, seq2_smem));
        const int share = (int)((size_t)sm_smem * 3 / 4 / (seq2_smem + (size_t)reserved));
        ws->seq2_fit = share < 1 ? 1u : (uint32_t)(share < fit ? share : fit);
#else
        ws->seq2_fit = 4;                        // (no SM to fill)
#endif
    }
    uint32_t gh = (uint32_t)sms * huf_ctas;      // persistent CTAs
    const size_t need_h = est_blocks / ZK_HUF_SLOTS + 1;
    if (need_h < gh) gh = (uint32_t)need_h;
    // the two entropy kernels are independent: run the Huffman one on a side stream
    if (!ws->side) {
        ZK_CUDA_OK(cudaStreamCreateWithPriority(&ws->side, cudaStreamNonBlocking, ws->prio));
        ZK_CUDA_OK(cudaEventCreateWithFlags(&ws->ev_scan, cudaEventDisableTiming));
        ZK_CUDA_OK(cudaEventCreateWithFlags(&ws->ev_huf, cudaEventDisableTiming));
    }
    const cudaStream_t hs = ws->side;
    ZK_CUDA_OK(cudaEventRecord(ws->ev_scan, stream));
    ZK_CUDA_OK(cudaStreamWaitEvent(hs, ws->ev_scan, 0));
    ws->prof.begin(2, hs);
    ZK_LAUNCH(zk_huf_kernel, gh, 32, huf_smem, hs, o);
    ws->prof.end(2, hs);
    ZK_CUDA_OK(cudaEventRecord(ws->ev_huf, hs));
    ws->prof.begin(1, stream);
    {
        uint32_t g2 = (uint32_t)sms * ws->seq2_fit;
        const size_t need2 = est_blocks / ZK_S2_NCH + 1;
        if (need2 < g2) g2 = (uint32_t)need2;
        ZK_LAUNCH(zk_seq2_kernel, g2, 32, seq2_smem, stream, o);
        // the blocks it passed on (none in this codec's own archives: the CTAs exit at their first work-counter read)
        ZK_LAUNCH(zk_seq2_full_kernel, (uint32_t)sms, 32, seq2f_smem, stream, o);
    }
    ws->prof.end(1, stream);
    ZK_CUDA_OK(cudaStreamWaitEvent(stream, ws->ev_huf, 0));
    // exec stage: ring size / warps per entry chosen from how many entries share the machine
    // Each entry is one serial dependency chain, so throughput comes from entries in flight: pick warps per
    // CTA and ring size such that (if possible) every entry of the batch is resident at once.
    // (`share` > 1: that many sub-batches of a host pipeline run concurrently on different streams)
    int per_sm = (int)(((unsigned long long)n * (unsigned)(p.share > 0 ? p.share : 1) + (uint32_t)sms - 1) / (uint32_t)sms);
    if (per_sm < 1) per_sm = 1;
    int W = (int)ws->exec_warps;
    a.exec_short = o.exec_short = ws->exec_short;
    ws->prof.begin(3, stream);                   // (the exec slot includes the plan kernel)
    ZK_LAUNCH(zk_plan_kernel, (n + 3) / 4, 128, 0, stream, a);
    if (ws->order) ZK_LAUNCH(zk_order_kernel, 2, ZK_ORD_THREADS, 0, stream, a, o, 1);
    // 126 registers/thread -> 16 warps per SM; from four entries per SM on, the 96-register build of the same body
    // (20 warps per SM, <= 5 per entry) keeps every entry of the batch resident with one more warp each.  One CTA per
    // entry; the CTAs then share the batch's segments (K-D1p).
    bool small_regs = false;
    if (W <= 0) {
        if (per_sm >= 4) { W = 20 / per_sm; if (W < 2) W = 2; small_regs = true; }
        else W = 16 / per_sm;
    } else small_regs = W <= 5 && per_sm >= 4;
    if (W > 16) W = 16;
    uint32_t ring = 128 * 1024;
    while (ring > 8 * 1024 && (size_t)ring * (size_t)per_sm > 200 * 1024) ring >>= 1;
    if (ws->ring_override) ring = ws->ring_override;
    // prefix mode: the same executors, built with the prefix split
    const bool prefix = a.prefix != nullptr;
    void (*cta_kernel)(ZkDecodeArgs, uint32_t) = small_regs ? (prefix ? zk_exec_kernel_w5<true> : zk_exec_kernel_w5<false>)
                                                            : (prefix ? zk_exec_kernel<true> : zk_exec_kernel<false>);
    // Long segments run on the side stream beside the short ones: segments never wait for each other, so the CTA executor's long serial
    // chains start with the warp executor's work instead of after its drain.  They are launched first, so their CTAs are resident first.
    // Without short segments every segment runs on the CTAs, on `stream`
    if (a.exec_short) {
        ZK_CUDA_OK(cudaEventRecord(ws->ev_scan, stream)); ZK_CUDA_OK(cudaStreamWaitEvent(hs, ws->ev_scan, 0));     // after the plan (and K-D1o)
        ZK_LAUNCH(cta_kernel, n, W * 32, ring, hs, o, ring);
        ZK_CUDA_OK(cudaEventRecord(ws->ev_huf, hs));
        // short segments on single warps; the CTAs pull only long ones
        uint32_t gw = (uint32_t)sms * 8u;
        const size_t need_w = est_blocks / ZK_XW_WARPS + 1;
        if (need_w < gw) gw = (uint32_t)need_w;
        void (*warp_kernel)(ZkDecodeArgs) = prefix ? zk_exec_warp_kernel<true> : zk_exec_warp_kernel<false>;
        ZK_LAUNCH(warp_kernel, gw, 32 * ZK_XW_WARPS, ZK_XW_WARPS * ZK_XW_WIN, stream, o);
        ZK_CUDA_OK(cudaStreamWaitEvent(stream, ws->ev_huf, 0));
    } else ZK_LAUNCH(cta_kernel, n, W * 32, ring, stream, o, ring);
    ws->prof.end(3, stream);
    if (verify_checksum) { ws->prof.begin(4, stream); ZK_LAUNCH(zk_xxh64_kernel, (n + 3) / 4, 128, 0, stream, a); ws->prof.end(4, stream); }
    if (ds != stream) { ZK_CUDA_OK(cudaEventRecord(ws->ev_done, stream)); ZK_CUDA_OK(cudaStreamWaitEvent(ds, ws->ev_done, 0)); }
    ZK_CUDA_OK(cudaMemcpyAsync(ws->h_entries, ws->entries, (size_t)n * sizeof(ZkEntry), cudaMemcpyDeviceToHost, ds));
    ZK_CUDA_OK(cudaMemcpyAsync(ws->h_counters, ws->counters, sizeof(ZkCounters), cudaMemcpyDeviceToHost, ds));
    ws->launches += 6 + (a.exec_short ? 1 : 0) + (verify_checksum ? 1 : 0) + (ws->order ? 2 : 0);
    ws->pending_n = n;
    return 0;
}

// Wait for the batch enqueued last on `stream`; returns 0, the first failing entry status, or ZK_ST_RETRY when the
// scratch was too small (ws->want_* then hold the exact needs: the caller re-enqueues the same batch).
int zk_decode_collect(ZkDecodeWs* ws, cudaStream_t stream, const ZkDecodeParams& p, int32_t* status_out) {
    uint32_t n = ws->pending_n;
    if (n == 0) return 0;
    // with a download stream: ev_down, recorded by the caller after the output copy on it
    if (const int rc = zk_sync_check(stream, p.down ? ws->ev_down : nullptr)) return rc;
    ws->pending_n = 0;
    ws->prof.harvest();
    if (ws->h_counters->overflow) {
        ws->want_blocks = (size_t)ws->h_counters->n_blocks; ws->want_lit = (size_t)ws->h_counters->n_lit; ws->want_seq = (size_t)ws->h_counters->n_seq;
        return ZK_ST_RETRY;
    }
    ws->segments += ws->h_counters->n_long + ws->h_counters->n_short;
    int worst = 0;
    for (uint32_t i = 0; i < n; i++) {
        int32_t st = ws->h_entries[i].status;
        if (st == ZK_ST_RETRY) st = -(int)ZKZ_MEMORY_ALLOCATION;
        if (status_out) status_out[i] = st;
        if (st && !worst) worst = st;
    }
    return worst;
}

int zk_decode_batch(ZkDecodeWs* ws, cudaStream_t stream, const uint8_t* d_comp, const uint64_t* c_off, const uint64_t* d_off,
                    uint32_t n, uint8_t* d_dst, int verify_checksum, const ZkDecodeParams& p, int32_t* status_out) {
    for (int attempt = 0; attempt < 2; attempt++) {
        int rc = zk_decode_enqueue(ws, stream, d_comp, c_off, d_off, n, d_dst, verify_checksum, p);
        if (rc) return rc;
        rc = zk_decode_collect(ws, stream, p, status_out);
        if (rc != ZK_ST_RETRY) return rc;
    }
    fprintf(stderr, "zeekstd_b200: decode scratch still too small after growing to the exact needs (blocks %zu lit %zu seq %zu; caps %zu %zu %zu)\n",
            ws->want_blocks, ws->want_lit, ws->want_seq, ws->cap_blocks, ws->cap_lit, ws->cap_seq);
    return -(int)ZKZ_MEMORY_ALLOCATION;
}
