// zk_encode.cu -- batched Zstandard frame compression for sm_90a.
//
// Replaces the reference's compression calls into libzstd,
//   lib/src/encode.rs:341-345   cctx.compress_stream2(out, in, ZSTD_e_continue)
//   lib/src/encode.rs:444-448   cctx.compress_stream2(out, empty, ZSTD_e_end)
// with kernels over a whole batch of independent frames (seekable_format.md:23-29); every frame is cut
// into zstd blocks of ZKC_BLOCK bytes and every block is one unit of work:
//
//   K-C1 zk_match_kernel<HLOG> one warp / block : LZ77 match finding (hash table in shared memory), greedy parse resolved
//                                               with ballots, repeat-offset codes, sequences + literals written per window
//   K-C2s zk_seq_enc_kernel  one warp / block : FSE sequences (three lanes run the state chains, 32 lanes pack the bits)
//   K-C2l zk_lit_enc_kernel  one warp / block : Huffman literals (tree build, FSE-coded weights, 4 streams packed by warp scan), 4 warps / CTA
//   K-C2f zk_block_finish_kernel              : joins the two sections of a block (coded on two streams), Raw fallback, header
//   K-C3 zk_frame_{hash,size,scan,gather}_kernel : optional XXH64, frame sizes, offsets, frame headers + block gather, over the
//                                               frame and block tables (zk_geo_*_kernel, or the cut of K-C3c zk_csize_*_kernel)
//
// Output is a standard Zstandard frame per seek-table entry (RFC 8878; SURVEY.md Appendix A), decodable
// by libzstd; the compressed bytes are NOT meant to equal libzstd's.
#include "zk_encode.h"
#include <string.h>
#include <map>
#include <vector>

#define ZKC_BLOCK 32768u                 // zstd block size used by this encoder (<= Block_Maximum_Size)
#define ZKC_HLOG_FAST 11                 // hash table per warp: 2048 x u16 at level 1 (40 warps / SM hide the two dependent loads per window),
#define ZKC_HLOG 12                      // 4096 x u16 from level 2 on (24 warps / SM, 0.3-3 % better ratio)
#define ZKC_MINMATCH 5
#define ZKC_MAXSEQ (ZKC_BLOCK / 4 + 8)   // every sequence covers at least 4 bytes (repeat matches may be 4 long); multiple of 8 for 16-byte chunked loads
#define ZKC_SLOT (ZKC_BLOCK + 64u)       // per-block staging slot for the compressed block
#define ZKC_FRAME_HDR 10u                // magic + FHD + window descriptor + 4-byte FCS

struct ZkcBlock {                        // per-block record in HBM
    uint32_t nseq, nlit;                 // K-C1
    uint32_t seq_hdr, seq_bits;          // K-C2s: bytes of the sequence-section header / bitstream (seq_hdr == 0: not encodable)
    uint32_t lit_bytes, last_flag;       // K-C2l: bytes staged so far (3-byte header gap + literals section; 0 = send the block Raw)
    uint32_t csize;                      // K-C2f: size of the staged block incl. its 3-byte header
    uint32_t out_off;                    // K-C3: offset of the block inside its frame
};
#define ZKC_SEQSEC 16384u                // per-block scratch for the sequence section: [0,256) header, [256,..) bitstream
#define ZKC_SEQHDR 256u

// The block geometry of a batch (DESIGN §2), built on the device by zk_geo_*_kernel from per-frame sizes (the caller's, or those of
// the uniform layout): every kernel reads a block's input range and its place in its frame, and a frame's range and blocks, from
// these two tables and nowhere else.  A frame of d bytes has max(1, ceil(d / ZKC_BLOCK)) blocks, cut from its first byte.
struct ZkcGeo {                          // per block, 24 bytes
    size_t lo;                           // first input byte; the frame starts at lo - k * ZKC_BLOCK
    uint32_t len;                        // input bytes (0 only in the one block of an empty frame)
    uint32_t frame, k;                   // frame index, block index inside the frame
    uint32_t last;                       // 1: the last block of its frame
};
struct ZkcFrame {                        // per frame, 40 bytes
    size_t start;                        // first input byte
    uint32_t size, first_block, n_blocks;
    uint32_t tail;                       // bytes of its prefix K-C1 and K-C1h stage in front of it: min(plen, ZKC_BLOCK), 0 without a prefix
    uint32_t plo, plen;                  // its prefix: prefix[plo, plo + plen) of the batch's prefix buffer
    unsigned long long vpre;             // the tails of the frames before it (K-C1h's virtual layout: the frame's tail starts at start + vpre)
};

struct ZkEncodeArgs {
    const uint8_t* src; size_t n; uint32_t n_frames; uint32_t n_blocks;
    const ZkcGeo* geo; const ZkcFrame* frames;
    int level, checksum;
    ZkcBlock* blocks;
    uint16_t* seq_ll; uint16_t* seq_ml; uint32_t* seq_off;      // ZKC_MAXSEQ per block
    uint8_t* lits;                                              // ZKC_BLOCK per block
    uint8_t* stage;                                             // ZKC_SLOT per block
    uint8_t* seqsec;                                            // ZKC_SEQSEC per block
    // K-C3 (the frame assembly).  res: the result area of the batch (ZKC_RES_HDR).  V: variants of every block (zk_encode_csize; 1
    // elsewhere): block b of the tables is variant v = min(geo[b].k, V - 1), its record at blocks[v * n_blocks + b] and its staged bytes
    // in slot v * n_blocks + b.  wmin, wmax, far: the window the frames announce (zkc_carve)
    uint32_t* res; unsigned long long* frame_off; uint32_t* frame_hash;
    uint8_t* dst; size_t dst_cap; uint32_t V, wmin, wmax, far;
    // raw-content prefix (RawEncoder::compress_with_prefix, encode.rs:311-338: re-applied at the start of EVERY frame): the buffer
    // every frame's prefix lies in (nullptr: no frame has one).  The last tail <= ZKC_BLOCK bytes of frame f's prefix (ZkcFrame) are
    // staged in front of a copy of its first block, so that block's match finder sees one contiguous history and needs no second pointer
    const uint8_t* prefix; uint8_t* pstage;
    // bytes of the frame before a block that K-C1 may search, on top of the tier's own limit: unlimited (~0) except in the size variants
    // of the wide tier (zk_encode_csize), where variant d must match the block d blocks into its frame
    size_t hist_cap;
    uint8_t* hc;                         // scratch of the high-level tier (zk_hc.inc), carved for its largest internal pass
};
// The result area of a batch, read back by one copy: [0] frames and [1] blocks K-C3 assembles, written on the device by whatever built
// the tables (n_frames / n_blocks bound them), [2] error, [4..5] the bytes written (u64); then the frames' compressed sizes and, where
// the frames were cut on the device, their input sizes
#define ZKC_RES_HDR 8u
#define ZKC_PSLOT (2u * ZKC_BLOCK + 64u)   // per-frame staging slot: [prefix tail | first block]

__device__ __forceinline__ ZkcGeo zkc_block_range(const ZkEncodeArgs& a, uint32_t b, size_t& lo, size_t& hi, size_t& fstart) {
    const ZkcGeo g = a.geo[b];
    lo = g.lo; hi = g.lo + g.len; fstart = g.lo - (size_t)g.k * ZKC_BLOCK;
    return g;
}

// The prefix of a frame of the batch: prefix[plo, plo + plen), of which the last min(plen, ZKC_BLOCK) bytes are staged (none when the
// batch has no prefix: pfx == 0)
__device__ __forceinline__ void zkc_frame_prefix(ZkcFrame& r, uint32_t pfx, uint32_t plo, uint32_t plen) {
    r.plo = plo; r.plen = plen; r.tail = pfx ? (plen < ZKC_BLOCK ? plen : ZKC_BLOCK) : 0u;
}

// uniform layout: frames of frame_size bytes, the last one shorter (n_frames = 1 and one empty frame when n == 0).  Every frame but the
// last is full, so frame f starts at block f * ceil(frame_size / ZKC_BLOCK).  Every frame's prefix is the whole buffer of plen bytes.
// count: the frames and the blocks they cover
__global__ void __launch_bounds__(256) zk_geo_uniform_kernel(ZkcFrame* fr, uint32_t* count, uint32_t n_frames, size_t n, uint32_t frame_size,
                                                             uint32_t pfx, uint32_t plen) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    const uint32_t bpf = (uint32_t)(((size_t)frame_size + ZKC_BLOCK - 1) / ZKC_BLOCK);
    const size_t start = (size_t)f * frame_size;
    const uint32_t size = (uint32_t)(n - start < frame_size ? n - start : frame_size);
    ZkcFrame r;
    r.start = start; r.size = size; r.first_block = f * bpf; r.n_blocks = size ? (size + ZKC_BLOCK - 1) / ZKC_BLOCK : 1u;
    zkc_frame_prefix(r, pfx, 0, plen);
    r.vpre = (unsigned long long)f * r.tail;
    fr[f] = r;
    if (f + 1 == n_frames) { count[0] = n_frames; count[1] = r.first_block + r.n_blocks; }
}

// caller-chosen sizes: frame starts, first blocks and the tails before each frame by one scan (one CTA, 1024 frames a round).  ranges:
// two per frame, its prefix [ranges[2f], ranges[2f + 1]) (nullptr: the whole buffer of plen bytes).  count as zk_geo_uniform_kernel
__global__ void __launch_bounds__(1024) zk_geo_sized_kernel(ZkcFrame* fr, uint32_t* count, const uint32_t* sizes, uint32_t n_frames,
                                                            const uint32_t* ranges, uint32_t pfx, uint32_t plen) {
    __shared__ unsigned long long wb[32], wt[32], cb, ct;
    __shared__ uint32_t wk[32], ck;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { cb = 0; ck = 0; ct = 0; }
    __syncthreads();
    for (uint32_t base = 0; base < n_frames; base += 1024) {
        const uint32_t f = base + threadIdx.x;
        const uint32_t d = f < n_frames ? sizes[f] : 0u;
        const uint32_t nb = f < n_frames ? (d ? (d + ZKC_BLOCK - 1) / ZKC_BLOCK : 1u) : 0u;
        ZkcFrame r;
        zkc_frame_prefix(r, f < n_frames ? pfx : 0u, ranges && f < n_frames ? ranges[2 * f] : 0u,
                         ranges && f < n_frames ? ranges[2 * f + 1] - ranges[2 * f] : plen);
        unsigned long long xb = d, xt = r.tail; uint32_t xk = nb;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
            const unsigned long long tb = __shfl_up_sync(0xFFFFFFFFu, xb, s), tt = __shfl_up_sync(0xFFFFFFFFu, xt, s);
            const uint32_t tk = __shfl_up_sync(0xFFFFFFFFu, xk, s);
            if (lane >= s) { xb += tb; xk += tk; xt += tt; }
        }
        if (lane == 31) { wb[warp] = xb; wk[warp] = xk; wt[warp] = xt; }
        __syncthreads();
        if (warp == 0) {
            unsigned long long yb = wb[lane], yt = wt[lane]; uint32_t yk = wk[lane];
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) {
                const unsigned long long tb = __shfl_up_sync(0xFFFFFFFFu, yb, s), tt = __shfl_up_sync(0xFFFFFFFFu, yt, s);
                const uint32_t tk = __shfl_up_sync(0xFFFFFFFFu, yk, s);
                if (lane >= s) { yb += tb; yk += tk; yt += tt; }
            }
            wb[lane] = yb; wk[lane] = yk; wt[lane] = yt;
        }
        __syncthreads();
        if (f < n_frames) {
            r.start = cb + (warp ? wb[warp - 1] : 0ull) + xb - d; r.size = d;
            r.first_block = ck + (warp ? wk[warp - 1] : 0u) + xk - nb; r.n_blocks = nb;
            r.vpre = ct + (warp ? wt[warp - 1] : 0ull) + xt - r.tail;
            fr[f] = r;
            if (f + 1 == n_frames) { count[0] = n_frames; count[1] = r.first_block + nb; }
        }
        __syncthreads();
        if (threadIdx.x == 0) { cb += wb[31]; ck += wk[31]; ct += wt[31]; }
        __syncthreads();
    }
}

// one thread per block of the count[1] the frame table covers: its frame is the last one whose first block is <= b (every frame has a
// block, so first blocks increase)
__global__ void __launch_bounds__(256) zk_geo_block_kernel(ZkcGeo* geo, const ZkcFrame* fr, const uint32_t* count) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= count[1]) return;
    uint32_t lo = 0, hi = count[0] - 1;
    while (lo < hi) { const uint32_t mid = lo + (hi - lo + 1) / 2; if (fr[mid].first_block <= b) lo = mid; else hi = mid - 1; }
    const ZkcFrame F = fr[lo];
    const uint32_t k = b - F.first_block, off = k * ZKC_BLOCK;
    ZkcGeo g;
    g.lo = F.start + off; g.len = F.size - off < ZKC_BLOCK ? F.size - off : ZKC_BLOCK;
    g.frame = lo; g.k = k; g.last = k + 1 == F.n_blocks ? 1u : 0u;
    geo[b] = g;
}

// unaligned 8-byte little-endian load from global memory
__device__ __forceinline__ unsigned long long zkc_ld8(const uint8_t* p) {
    uintptr_t a = (uintptr_t)p; uint32_t mis = (uint32_t)(a & 3);
    const uint32_t* q = (const uint32_t*)(a - mis);
    uint32_t w0 = q[0], w1 = q[1];
    if (mis == 0) return (unsigned long long)w0 | ((unsigned long long)w1 << 32);
    uint32_t w2 = q[2], sh = mis * 8;
    return (unsigned long long)__funnelshift_r(w0, w1, sh) | ((unsigned long long)__funnelshift_r(w1, w2, sh) << 32);
}
template <int HLOG>
__device__ __forceinline__ uint32_t zkc_hash5(unsigned long long v) {
    return (uint32_t)(((v << 24) * 889523592379ull) >> (64 - HLOG));
}
template <int HLOG>
__device__ __forceinline__ uint32_t zkc_hash8(unsigned long long v) {
    return (uint32_t)((v * 0xCF1BBCDCB7A56463ull) >> (64 - HLOG));
}

// =============================================================================================
// K-C1: match finding.  One warp per block; lane i examines position ip + i * stride.
//
// Every position is a 32-bit offset from `base` (the start of the searchable history, < 64 KiB before the end of the
// block), so the u16 hash table stores positions directly.  A window is always full (32 valid lanes): the last < 40
// bytes of a block are left as literals.  Matches are only taken from stride-1 windows -- when a wider window (used
// after runs of misses on incompressible data) sees a candidate, the window is simply redone at stride 1.  That makes
// literal emission a per-window register operation: a byte that no selected match covers is written from the lane that
// already holds it (ballot + popc rank), and sequences are staged one per lane and stored 32 at a time.
// =============================================================================================
#define ZKC_C1_WARPS 4

// a match whose first ml = 8 bytes agree, extended cooperatively: lane k compares bytes [8 + 8k, 16 + 8k) of it, 256 bytes a round
__device__ __forceinline__ void zkc_extend_fwd(const uint8_t* sb, uint32_t mpos, uint32_t off, uint32_t hi32, int lane, uint32_t& ml) {
    for (;;) {
        const uint32_t q = mpos + ml + (uint32_t)lane * 8u;
        uint32_t eq = 8;
        if (q + 8 <= hi32) { const unsigned long long x = zkc_ld8(sb + q) ^ zkc_ld8(sb + q - off); if (x) eq = (uint32_t)(__ffsll((long long)x) - 1) >> 3; }
        else { eq = 0; for (uint32_t t = q; t < hi32 && sb[t] == sb[t - off]; t++) eq++; }
        const uint32_t stop = __ballot_sync(0xFFFFFFFFu, eq < 8);
        if (stop) { const int g = __ffs((int)stop) - 1; ml += 8 * g + __shfl_sync(0xFFFFFFFFu, eq, g); break; }
        ml += 256;
    }
}

// Offset_Value of a sequence (A.5) for the fast tier, updating the repeat-offset history r0..r2 as the decoder will: the rule of
// zkc_match_block, which keeps its own inline copy.  As a call there it compiles to different code, and the level-1 kernel took 10.84-10.94
// ms per GiB of the bench mix instead of 10.68-10.77 (H100 80GB HBM3, 700 W)
__device__ __forceinline__ uint32_t zkc_offset_value(uint32_t off, uint32_t ll, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& known) {
    uint32_t ov = off + 3;
    if (off != r0 && off != r1 && off != r2 && off + 1 != r0) {           // the common case: an explicit offset
        r2 = r1; r1 = r0; r0 = off; known += known < 3;
    } else {
        bool hit0 = false, hit1 = false;
        if (known == 3) {
            const bool e0 = off == r0, e1 = off == r1, e2 = off == r2, em = r0 > 1 && off == r0 - 1;
            if (ll != 0) { if (e0) { ov = 1; hit0 = true; } else if (e1) { ov = 2; hit1 = true; } else if (e2) ov = 3; }
            else { if (e1) { ov = 1; hit1 = true; } else if (e2) ov = 2; else if (em) ov = 3; }
        } else known++;
        if (!hit0) { r2 = hit1 ? r2 : r1; r1 = r0; r0 = off; }
    }
    return ov;
}

// n bytes from s to d by one warp: 8 bytes per lane and round (the source is read as aligned words, never past the word holding s[n - 1])
__device__ __forceinline__ void zkc_warp_copy(uint8_t* __restrict__ d, const uint8_t* __restrict__ s, uint32_t n, int lane) {
    const uint32_t n8 = n & ~7u;
    for (uint32_t i = 8u * (uint32_t)lane; i < n8; i += 256) {
        const unsigned long long v = zkc_ld8(s + i);
#pragma unroll
        for (int q = 0; q < 8; q++) d[i + q] = (uint8_t)(v >> (8 * q));
    }
    if ((uint32_t)lane < n - n8) d[n8 + lane] = s[n8 + lane];
}

// prefix mode: [tail of frame f's prefix | first block of frame f] -> pstage slot f (one CTA per frame)
__global__ void __launch_bounds__(256) zk_prefix_stage_kernel(ZkEncodeArgs a) {
    const uint32_t f = blockIdx.x;
    const ZkcFrame F = a.frames[f];
    const uint32_t len = a.geo[F.first_block].len;
    uint8_t* d = a.pstage + (size_t)f * ZKC_PSLOT;
    const uint8_t* pt = a.prefix + (F.plo + F.plen - F.tail);
    for (uint32_t i = threadIdx.x; i < F.tail; i += blockDim.x) d[i] = pt[i];
    for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) d[F.tail + i] = a.src[F.start + i];
    for (uint32_t i = threadIdx.x; i < 64; i += blockDim.x) d[F.tail + len + i] = 0;
}

// inserts the history sb[0, lo32) into the table, and into the 8-byte table when DFAST, so that matches can reach into it.  Several
// lanes may hash to the same slot: the highest position wins, as sequential insertion would leave it (keeps the compressed bytes
// deterministic)
template <int HLOG, bool DFAST, typename PosT>
__device__ __forceinline__ void zkc_insert_history(const uint8_t* sb, uint32_t lo32, int lane, PosT* table, PosT* tableL = nullptr) {
    for (uint32_t p0 = 0; p0 < lo32; p0 += 32) {
        const uint32_t p = p0 + lane;
        const unsigned long long v8 = p < lo32 ? zkc_ld8(sb + p) : 0ull;
        const uint32_t hh = p < lo32 ? zkc_hash5<HLOG>(v8) : (0xFFFF0000u | (uint32_t)lane);
        const uint32_t same = __match_any_sync(0xFFFFFFFFu, hh);
        if (p < lo32 && lane == 31 - __clz((int)same)) table[hh] = (PosT)p;
        if (DFAST) {
            const uint32_t hl = p < lo32 ? zkc_hash8<HLOG>(v8) : (0xFFFF0000u | (uint32_t)lane);
            const uint32_t sameL = __match_any_sync(0xFFFFFFFFu, hl);
            if (p < lo32 && lane == 31 - __clz((int)sameL)) tableL[hl] = (PosT)p;
        }
    }
    __syncwarp();
}

// The match finder of levels 1-15, run by one warp on block b.  table: the warp's 2^HLOG-entry hash table; an entry is a position, an
// offset from the start of the history, so u16 entries need history + block < 64 KiB.  HIST_BYTES: how far before the block the history
// reaches.  DFAST (level >= 4): tableL, a second table of 2^HLOG entries indexed by a hash of EIGHT bytes, is probed first -- its candidates
// are long matches by construction, the 5-byte table catches the rest (the idea of zstd's double-fast strategy); tableL is not touched
// otherwise.
template <int HLOG, bool DFAST, typename PosT, uint32_t HIST_BYTES>
__device__ __forceinline__ void zkc_match_block(const ZkEncodeArgs& a, uint32_t b, int lane, PosT* table, PosT* tableL) {
    size_t lo, hi, fstart;
    const ZkcGeo g = zkc_block_range(a, b, lo, hi, fstart);
    // history: up to HIST_BYTES of the same frame before `lo` are searchable, capped by a.hist_cap; the first block of a frame
    // searches the tail of its prefix instead, through its staged copy
    const uint32_t ptail = a.prefix && lo == fstart ? a.frames[g.frame].tail : 0u;
    const bool pfx = ptail != 0;
    const size_t hist = a.hist_cap < HIST_BYTES ? a.hist_cap : HIST_BYTES;
    const size_t base = lo - fstart >= hist ? lo - hist : fstart;
    const uint8_t* sb = pfx ? a.pstage + (size_t)g.frame * ZKC_PSLOT : a.src + base;
    const uint32_t lo32 = pfx ? ptail : (uint32_t)(lo - base), hi32 = lo32 + (uint32_t)(hi - lo);
    for (int i = lane; i < ((DFAST ? 2 : 1) << HLOG); i += 32) table[i] = 0;
    __syncwarp();
    const uint32_t len = hi32 - lo32;
    uint16_t* o_ll = a.seq_ll + (size_t)b * ZKC_MAXSEQ; uint16_t* o_ml = a.seq_ml + (size_t)b * ZKC_MAXSEQ;
    uint32_t* o_off = a.seq_off + (size_t)b * ZKC_MAXSEQ;
    uint8_t* o_lit = a.lits + (size_t)b * ZKC_BLOCK;
    uint32_t nseq = 0, nlit = 0;
    uint32_t ip = lo32;                                     // every literal byte below ip has been written to o_lit
    if (len >= 16) {
        const uint32_t mflimit = hi32 - 8;                  // last position where 8 bytes can be read
        const uint32_t lt_mask = (1u << lane) - 1u;
        const bool lazy = a.level >= 2;
        // pre-insert the history so matches can reach into the previous block (or the prefix)
        if (a.level >= 2 || pfx) zkc_insert_history<HLOG, DFAST>(sb, lo32, lane, table, tableL);
        uint32_t anchor = lo32;
        uint32_t rep = 0;                                   // last emitted offset (0 = none)
        // repeat-offset history (A.5) as the decoder will hold it: blocks are coded independently, so repeat codes are used
        // only once three explicit offsets have been coded in this block (the history is then certain); the first block of a
        // frame starts from the known {1,4,8}.  o_off receives Offset_Values (1..3 = repeat codes, offset + 3 otherwise).
        uint32_t r0 = 1, r1 = 4, r2 = 8, known = lo == fstart ? 3u : 0u;
        uint32_t misses = 0;                                // consecutive windows without a match: widen the stride (incompressible data)
        uint32_t s_ll = 0, s_ml = 0, s_off = 0, flushed = 0; // staged sequences: slot nseq - flushed lives in that lane
        for (;;) {
            const uint32_t stride = 1u + min(misses >> 3, 3u);
            if (ip + 32u * stride > mflimit) {
                if (stride == 1) break;
                misses = 0; continue;                       // the tail may still fit a stride-1 window
            }
            const uint32_t wb = ip;
            const uint32_t p = wb + (uint32_t)lane * stride;
            if (lane < 2) zk_prefetch_l1(sb + min(wb + 256u + 128u * (uint32_t)lane, hi32 - 1u));
            const unsigned long long cur = zkc_ld8(sb + p);
            const uint32_t h = zkc_hash5<HLOG>(cur);
            const uint32_t cand = table[h];
            uint32_t hl = 0, candL = 0;
            if (DFAST) { hl = zkc_hash8<HLOG>(cur); candL = tableL[hl]; }
            __syncwarp();
            // several lanes may hash to the same slot: the highest position wins, as sequential insertion would leave it
            // (keeps the compressed bytes deterministic)
            const uint32_t same = __match_any_sync(0xFFFFFFFFu, h);
            if (lane == 31 - __clz((int)same)) table[h] = (PosT)p;
            if (DFAST) { const uint32_t sameL = __match_any_sync(0xFFFFFFFFu, hl); if (lane == 31 - __clz((int)sameL)) tableL[hl] = (PosT)p; }
            // candidate from the hash table(s), and the repeat-offset candidate
            uint32_t moff = 0, mlen0 = 0;
            if (cand < p) {
                const unsigned long long x = zkc_ld8(sb + cand) ^ cur;
                const uint32_t m = x ? (uint32_t)(__ffsll((long long)x) - 1) >> 3 : 8;
                if (m >= ZKC_MINMATCH) { moff = p - cand; mlen0 = m; }
            }
            if (DFAST && candL < p && candL != cand) {
                const unsigned long long x = zkc_ld8(sb + candL) ^ cur;
                const uint32_t m = x ? (uint32_t)(__ffsll((long long)x) - 1) >> 3 : 8;
                if (m >= ZKC_MINMATCH && m > mlen0) { moff = p - candL; mlen0 = m; }       // both 8 long: the nearer one (5-byte table) is kept
            }
            if (rep && p >= rep) {
                const unsigned long long x = zkc_ld8(sb + p - rep) ^ cur;
                const uint32_t m = x ? (uint32_t)(__ffsll((long long)x) - 1) >> 3 : 8;
                if (m >= 4 && m + 1 >= mlen0) { moff = rep; mlen0 = m; }
            }
            const uint32_t found = __ballot_sync(0xFFFFFFFFu, mlen0 != 0);
            if (stride > 1) {
                if (found) { misses = 0; continue; }        // compressible again: redo this window at stride 1
                // the whole window is literals, straight from the registers
                uint8_t* o = o_lit + nlit + (uint32_t)lane * stride;
                o[0] = (uint8_t)cur; o[1] = (uint8_t)(cur >> 8);
                if (stride > 2) o[2] = (uint8_t)(cur >> 16);
                if (stride > 3) o[3] = (uint8_t)(cur >> 24);
                nlit += 32u * stride; ip = wb + 32u * stride; misses++;
                continue;
            }
            if (!found) {
                o_lit[nlit + lane] = (uint8_t)cur;
                nlit += 32u; ip = wb + 32u; misses++;
                continue;
            }
            misses = 0;
            // take every non-overlapping match of this window, left to right (one memory round trip serves them all)
            const uint32_t packed = (moff << 4) | mlen0;
            // a stride-1 window yields at most 8 sequences (matches are >= 4 bytes): make room in the 32 staging lanes first
            if (nseq - flushed > 24u) {
                if ((uint32_t)lane < nseq - flushed) { const uint32_t at = flushed + (uint32_t)lane; o_ll[at] = (uint16_t)s_ll; o_ml[at] = (uint16_t)s_ml; o_off[at] = s_off; }
                flushed = nseq;
            }
            uint32_t next_lane = 0;
            bool cov = false;                               // this lane's byte is covered by a selected match
            while (next_lane < 32) {
                const uint32_t m = found & (0xFFFFFFFFu << next_lane);
                if (!m) break;
                int f = __ffs((int)m) - 1;
                uint32_t mo = __shfl_sync(0xFFFFFFFFu, packed, f);          // (offset << 4) | length
                // one step of lazy matching: a clearly longer match starting at the next position wins (one more literal)
                if (lazy && (mo & 15u) < 8 && f < 31 && ((found >> (f + 1)) & 1u)) {
                    const uint32_t mo2 = __shfl_sync(0xFFFFFFFFu, packed, f + 1);
                    if ((mo2 & 15u) > (mo & 15u) + 1) { f++; mo = mo2; }
                }
                uint32_t ml = mo & 15u;
                const uint32_t off = mo >> 4;
                const uint32_t mpos = wb + (uint32_t)f;
                if (ml == 8) zkc_extend_fwd(sb, mpos, off, hi32, lane, ml);
                // emit: literals [anchor, mpos) are already / will be placed by the windows that hold them
                const uint32_t ll = mpos - anchor;
                // after every sequence r0 == off; a repeat of r0 itself (ll != 0) leaves the history alone, every other
                // case shifts (r0 -> r1) and drops r2, except the r1 hit, which swaps the first two
                uint32_t ov = off + 3;
                if (off != r0 && off != r1 && off != r2 && off + 1 != r0) {           // the common case: an explicit offset
                    r2 = r1; r1 = r0; r0 = off; known += known < 3;
                } else {
                    bool hit0 = false, hit1 = false;
                    if (known == 3) {
                        const bool e0 = off == r0, e1 = off == r1, e2 = off == r2, em = r0 > 1 && off == r0 - 1;
                        if (ll != 0) { if (e0) { ov = 1; hit0 = true; } else if (e1) { ov = 2; hit1 = true; } else if (e2) ov = 3; }
                        else { if (e1) { ov = 1; hit1 = true; } else if (e2) ov = 2; else if (em) ov = 3; }
                    } else known++;
                    if (!hit0) { r2 = hit1 ? r2 : r1; r1 = r0; r0 = off; }
                }
                if (lane == (int)(nseq - flushed)) { s_ll = ll; s_ml = ml - 3; s_off = ov; }
                nseq++;
                cov = cov || (p - mpos < ml);               // unsigned: mpos <= p < mpos + ml
                anchor = mpos + ml; rep = off;
                next_lane = anchor - wb;                    // >= 32: the match runs past the window
            }
            const uint32_t lm = __ballot_sync(0xFFFFFFFFu, !cov);
            if (!cov) o_lit[nlit + __popc(lm & lt_mask)] = (uint8_t)cur;
            nlit += (uint32_t)__popc(lm);
            ip = anchor > wb + 32u ? anchor : wb + 32u;
        }
        if ((uint32_t)lane < nseq - flushed) {
            const uint32_t at = flushed + (uint32_t)lane;
            o_ll[at] = (uint16_t)s_ll; o_ml[at] = (uint16_t)s_ml; o_off[at] = s_off;
        }
    }
    const uint32_t rest = hi32 - ip;
    for (uint32_t i = lane; i < rest; i += 32) o_lit[nlit + i] = sb[ip + i];
    nlit += rest;
    if (lane == 0) { a.blocks[b].nseq = nseq; a.blocks[b].nlit = nlit; }
}

// levels 1-12: a history of one block, u16 positions, NW warps per CTA with their tables in static shared memory
template <int HLOG, int NW, bool DFAST>
__global__ void __launch_bounds__(NW * 32) zk_match_kernel(ZkEncodeArgs a) {
    __shared__ uint16_t tables[NW][(DFAST ? 2 : 1) << HLOG];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t b = blockIdx.x * NW + warp;
    if (b >= a.n_blocks) return;
    zkc_match_block<HLOG, DFAST, uint16_t, ZKC_BLOCK>(a, b, lane, tables[warp], tables[warp] + (1 << HLOG));
}

// Wide-history tier (level >= ZKC_WIDE_LEVEL): the same match finder with a history of ZKC_WIDE_HIST blocks of the frame instead of one -- the frame
// header then announces a 256 KiB window (zk_frame_gather_kernel) --, 32-bit positions, and one table of 2^HLOG entries in DYNAMIC shared memory
// (128 KiB at HLOG 15: one warp-CTA per SM).  Every block still finds its matches alone and pre-inserts its whole history first, so a block costs
// several times a level-3 block: a tier for ratio (2.50 on the reference's corpus against 2.40 in a 64 KiB window), not for speed.
#define ZKC_WIDE_LEVEL 13
#define ZKC_WIDE_HIST 7
#define ZKC_WIDE_HLOG 15
template <int HLOG>
__global__ void __launch_bounds__(32) zk_match_wide_kernel(ZkEncodeArgs a) {
    ZK_DYN_SMEM(wide_tab);
    const uint32_t b = blockIdx.x;
    if (b >= a.n_blocks) return;
    zkc_match_block<HLOG, false, uint32_t, ZKC_WIDE_HIST * ZKC_BLOCK>(a, b, threadIdx.x & 31, (uint32_t*)wide_tab, nullptr);
}

// Fast tier (level < 0, zstd's negative levels; acceleration A = -level): level 1's table, warps and history, with sparse probing.  Lane i of
// a window probes position ip + i * s, where s = A + 1 + (windows since the last match) / ZKC_FAST_GROW, so long stretches without a match
// are crossed ever faster.  Lanes whose probe lies past the last position where 8 bytes can be read idle for that window; only probed positions
// are inserted.  A hit is extended forward as in the other tiers and backward down to the end of the previous sequence, which recovers the
// start a sparse probe missed.  Literals are copied from the input when a sequence (or the block) ends.  The window setup and the sequence
// staging repeat zkc_match_block's: shared with it as functions, they made the level-1 kernel compile to different code that took 11.19-11.28
// ms per GiB of the bench mix instead of 10.64-10.67 (H100 80GB HBM3, 700 W).
#define ZKC_FAST_GROW 8
#define ZKC_MIN_LEVEL (-131072)          // ZSTD_minCLevel(): lower levels clamp to it
template <int HLOG, int NW>
__global__ void __launch_bounds__(NW * 32) zk_match_fast_kernel(ZkEncodeArgs a) {
    __shared__ uint16_t tables[NW][1 << HLOG];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t b = blockIdx.x * NW + warp;
    if (b >= a.n_blocks) return;
    uint16_t* table = tables[warp];
    size_t lo, hi, fstart;
    const ZkcGeo g = zkc_block_range(a, b, lo, hi, fstart);
    const uint32_t ptail = a.prefix && lo == fstart ? a.frames[g.frame].tail : 0u;
    const bool pfx = ptail != 0;
    const size_t hist = a.hist_cap < ZKC_BLOCK ? a.hist_cap : ZKC_BLOCK;
    const size_t base = lo - fstart >= hist ? lo - hist : fstart;
    const uint8_t* sb = pfx ? a.pstage + (size_t)g.frame * ZKC_PSLOT : a.src + base;
    const uint32_t lo32 = pfx ? ptail : (uint32_t)(lo - base), hi32 = lo32 + (uint32_t)(hi - lo);
    for (int i = lane; i < (1 << HLOG); i += 32) table[i] = 0;
    __syncwarp();
    uint16_t* o_ll = a.seq_ll + (size_t)b * ZKC_MAXSEQ; uint16_t* o_ml = a.seq_ml + (size_t)b * ZKC_MAXSEQ;
    uint32_t* o_off = a.seq_off + (size_t)b * ZKC_MAXSEQ;
    uint8_t* o_lit = a.lits + (size_t)b * ZKC_BLOCK;
    uint32_t nseq = 0, nlit = 0;
    uint32_t anchor = lo32;                                 // end of the last sequence: every literal byte below it is in o_lit
    if (hi32 - lo32 >= 16) {
        const uint32_t mflimit = hi32 - 8;                  // last position where 8 bytes can be read
        const uint32_t step0 = (uint32_t)(-a.level) + 1u;
        if (pfx) zkc_insert_history<HLOG, false>(sb, lo32, lane, table);       // the prefix tail, as at level 1
        uint32_t rep = 0, r0 = 1, r1 = 4, r2 = 8, known = lo == fstart ? 3u : 0u;
        uint32_t misses = 0;                                // windows since the last match
        uint32_t s_ll = 0, s_ml = 0, s_off = 0, flushed = 0; // staged sequences: slot nseq - flushed lives in that lane
        for (uint32_t ip = lo32; ip <= mflimit;) {
            const uint32_t s = step0 + misses / ZKC_FAST_GROW;
            const uint32_t wb = ip, p = wb + (uint32_t)lane * s;      // no overflow: s <= 2^17 + 65 (a block is <= 512 windows)
            const bool live = p <= mflimit;
            const unsigned long long cur = live ? zkc_ld8(sb + p) : 0ull;
            const uint32_t h = live ? zkc_hash5<HLOG>(cur) : (0xFFFF0000u | (uint32_t)lane);
            const uint32_t cand = live ? table[h] : 0u;
            __syncwarp();
            // several lanes may hash to the same slot: the highest position wins, as sequential insertion would leave it
            const uint32_t same = __match_any_sync(0xFFFFFFFFu, h);
            if (live && lane == 31 - __clz((int)same)) table[h] = (uint16_t)p;
            uint32_t moff = 0, mlen0 = 0;
            if (live && cand < p) {
                const unsigned long long x = zkc_ld8(sb + cand) ^ cur;
                const uint32_t m = x ? (uint32_t)(__ffsll((long long)x) - 1) >> 3 : 8;
                if (m >= ZKC_MINMATCH) { moff = p - cand; mlen0 = m; }
            }
            if (live && rep && p >= rep) {
                const unsigned long long x = zkc_ld8(sb + p - rep) ^ cur;
                const uint32_t m = x ? (uint32_t)(__ffsll((long long)x) - 1) >> 3 : 8;
                if (m >= 4 && m + 1 >= mlen0) { moff = rep; mlen0 = m; }
            }
            const uint32_t found = __ballot_sync(0xFFFFFFFFu, mlen0 != 0);
            ip = wb + 32u * s;
            if (!found) { misses++; continue; }
            misses = 0;
            const uint32_t packed = (moff << 4) | mlen0;
            // every hit at or after the end of the previous sequence, left to right
            for (uint32_t m = found; m;) {
                const int f = __ffs((int)m) - 1;
                const uint32_t mo = __shfl_sync(0xFFFFFFFFu, packed, f);
                const uint32_t off = mo >> 4;
                uint32_t mpos = wb + (uint32_t)f * s;
                uint32_t ml = mo & 15u;
                if (ml == 8) zkc_extend_fwd(sb, mpos, off, hi32, lane, ml);
                // backward, one byte per lane and round, down to the previous sequence (and the start of the history)
                const uint32_t lim = anchor > off ? anchor : off;
                for (;;) {
                    const bool eq = (uint32_t)lane < mpos - lim && sb[mpos - 1 - lane] == sb[mpos - 1 - lane - off];
                    const uint32_t ne = __ballot_sync(0xFFFFFFFFu, !eq);
                    const uint32_t k = ne ? (uint32_t)__ffs((int)ne) - 1 : 32u;
                    mpos -= k; ml += k;
                    if (k < 32) break;
                }
                const uint32_t ll = mpos - anchor;
                zkc_warp_copy(o_lit + nlit, sb + anchor, ll, lane);
                nlit += ll;
                const uint32_t ov = zkc_offset_value(off, ll, r0, r1, r2, known);
                if (nseq - flushed == 32) {
                    const uint32_t at = flushed + (uint32_t)lane; o_ll[at] = (uint16_t)s_ll; o_ml[at] = (uint16_t)s_ml; o_off[at] = s_off;
                    flushed = nseq;
                }
                if (lane == (int)(nseq - flushed)) { s_ll = ll; s_ml = ml - 3; s_off = ov; }
                nseq++;
                anchor = mpos + ml; rep = off;
                if (anchor >= ip) { ip = anchor; break; }
                const uint32_t first = (anchor - wb + s - 1) / s;           // the first lane whose probe lies at or after anchor
                if (first >= 32) break;
                m = found & (0xFFFFFFFFu << first);
            }
        }
        if ((uint32_t)lane < nseq - flushed) {
            const uint32_t at = flushed + (uint32_t)lane;
            o_ll[at] = (uint16_t)s_ll; o_ml[at] = (uint16_t)s_ml; o_off[at] = s_off;
        }
    }
    zkc_warp_copy(o_lit + nlit, sb + anchor, hi32 - anchor, lane);
    nlit += hi32 - anchor;
    if (lane == 0) { a.blocks[b].nseq = nseq; a.blocks[b].nlit = nlit; }
}

// =============================================================================================
// K-C2: entropy coding.  One warp per block.
// =============================================================================================
__constant__ uint8_t ZKC_LL_CODE[64] = {0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,16,17,17,18,18,19,19,20,20,20,20,21,21,21,21,
                                        22,22,22,22,22,22,22,22,23,23,23,23,23,23,23,23,24,24,24,24,24,24,24,24,24,24,24,24,24,24,24,24};
__constant__ uint8_t ZKC_ML_CODE[128] = {0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,19,20,21,22,23,24,25,26,27,28,29,30,31,
                                         32,32,33,33,34,34,35,35,36,36,36,36,37,37,37,37,38,38,38,38,38,38,38,38,39,39,39,39,39,39,39,39,
                                         40,40,40,40,40,40,40,40,40,40,40,40,40,40,40,40,41,41,41,41,41,41,41,41,41,41,41,41,41,41,41,41,
                                         42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42};
__device__ __forceinline__ uint32_t zkc_ll_code(uint32_t ll) { return ll < 64 ? ZKC_LL_CODE[ll] : (uint32_t)zk_highbit(ll) + 19; }
__device__ __forceinline__ uint32_t zkc_ml_code(uint32_t mlb) { return mlb < 128 ? ZKC_ML_CODE[mlb] : (uint32_t)zk_highbit(mlb) + 36; }

// forward bit writer (A.7 streams are written forward, read backward).  WORDS: the base is 4-byte aligned and full
// 32-bit words are stored at once (used when a lane streams straight into HBM).
template <bool WORDS>
struct ZkcBitWT {
    uint8_t* p; uint32_t cap, pos; unsigned long long acc; int nb; bool ovf;
    __device__ __forceinline__ void init(uint8_t* buf, uint32_t capacity) { p = buf; cap = capacity; pos = 0; acc = 0; nb = 0; ovf = false; }
    __device__ __forceinline__ void add(uint32_t v, int n) {          // n <= 32
        acc |= (unsigned long long)(v & (n == 32 ? 0xFFFFFFFFu : ((1u << n) - 1u))) << nb; nb += n;
        if (nb >= 32) {
            if (pos + 4 <= cap) {
                if (WORDS) *(uint32_t*)(p + pos) = (uint32_t)acc;
                else { p[pos] = (uint8_t)acc; p[pos + 1] = (uint8_t)(acc >> 8); p[pos + 2] = (uint8_t)(acc >> 16); p[pos + 3] = (uint8_t)(acc >> 24); }
            } else ovf = true;
            pos += 4; acc >>= 32; nb -= 32;
        }
    }
    // end mark + flush; returns total bytes or 0 on overflow
    __device__ __forceinline__ uint32_t finish() { add(1, 1); return finish_raw(); }
    // flush without end mark (FSE table descriptions, A.6)
    __device__ __forceinline__ uint32_t finish_raw() {
        while (nb > 0) { if (pos < cap) p[pos] = (uint8_t)acc; else ovf = true; pos++; acc >>= 8; nb -= 8; }
        return ovf ? 0 : pos;
    }
};
typedef ZkcBitWT<false> ZkcBitW;
typedef ZkcBitWT<true> ZkcBitWW;

// FSE compression table for one symbol alphabet (state values in [S, 2S))
// (table logs are capped at 8 by this encoder: 1 KiB per table lets twice as many block chains share an SM's shared memory)
struct ZkcFse {
    uint16_t state_tbl[256];
    uint32_t delta_nb[64];
    int16_t delta_find[64];
    int16_t norm[64];
    int8_t log, mode;                    // mode: 0 predefined, 1 RLE, 2 FSE-compressed
    uint8_t nsym, rle_sym;
};

// normalise counts to a sum of 2^log with every present symbol >= 1 (any such distribution is a valid header)
template <class CT>
__device__ void zkc_fse_normalize(ZkcFse& t, const CT* cnt, int nsym, uint32_t total, int log) {
    const uint32_t S = 1u << log;
    uint32_t sum = 0, best = 0; int besti = 0;
    for (int s = 0; s < nsym; s++) {
        uint32_t c = cnt[s], v = 0;
        if (c) { v = (uint32_t)(((unsigned long long)c * S + total / 2) / total); if (v == 0) v = 1; }
        t.norm[s] = (int16_t)v; sum += v;
        if (c > best) { best = c; besti = s; }
    }
    // give / take the rounding error to the largest symbols
    while (sum != S) {
        if (sum < S) { t.norm[besti] = (int16_t)(t.norm[besti] + (S - sum)); sum = S; }
        else {
            uint32_t over = sum - S;
            // take from the symbol with the largest normalised count that can afford it
            int bi = -1; int16_t bv = 1;
            for (int s = 0; s < nsym; s++) if (t.norm[s] > bv) { bv = t.norm[s]; bi = s; }
            if (bi < 0) break;
            uint32_t take = (uint32_t)(bv - 1) < over ? (uint32_t)(bv - 1) : over;
            t.norm[bi] = (int16_t)(bv - take); sum -= take;
        }
    }
    t.log = (int8_t)log; t.nsym = (uint8_t)nsym;
}

// build the encoding tables from t.norm (mirror of A.6 table build); symof: 2^log bytes of scratch, cumul: nsym + 1 entries
__device__ __forceinline__ void zkc_fse_build_in(ZkcFse& t, uint8_t* symof, uint16_t* cumul) {
    const int log = t.log, S = 1 << log, nsym = t.nsym;
    int high = S - 1;
    cumul[0] = 0;
    for (int s = 0; s < nsym; s++) {
        if (t.norm[s] == -1) { cumul[s + 1] = cumul[s] + 1; symof[high--] = (uint8_t)s; }
        else cumul[s + 1] = (uint16_t)(cumul[s] + t.norm[s]);
    }
    const int step = (S >> 1) + (S >> 3) + 3; int pos = 0;
    for (int s = 0; s < nsym; s++)
        for (int q = 0; q < t.norm[s]; q++) { symof[pos] = (uint8_t)s; do { pos = (pos + step) & (S - 1); } while (pos > high); }
    for (int u = 0; u < S; u++) { int s = symof[u]; t.state_tbl[cumul[s]++] = (uint16_t)(S + u); }
    int total = 0;
    for (int s = 0; s < nsym; s++) {
        int n = t.norm[s];
        if (n == 0) { t.delta_nb[s] = ((uint32_t)(log + 1) << 16) - (1u << log); t.delta_find[s] = 0; }
        else if (n == 1 || n == -1) { t.delta_nb[s] = ((uint32_t)log << 16) - (1u << log); t.delta_find[s] = (int16_t)(total - 1); total++; }
        else {
            uint32_t max_bits_out = (uint32_t)log - (uint32_t)zk_highbit((uint32_t)n - 1);
            uint32_t min_state_plus = (uint32_t)n << max_bits_out;
            t.delta_nb[s] = (max_bits_out << 16) - min_state_plus;
            t.delta_find[s] = (int16_t)(total - n); total += n;
        }
    }
}
__device__ void zkc_fse_build(ZkcFse& t, uint8_t* symof /* >= 512 bytes scratch */) { uint16_t cumul[65]; zkc_fse_build_in(t, symof, cumul); }

// write the normalised-count header (A.6); returns bytes written (0 on overflow)
__device__ uint32_t zkc_fse_write_ncount(const ZkcFse& t, uint8_t* out, uint32_t cap) {
    ZkcBitW w; w.init(out, cap);
    const int log = t.log; const int S = 1 << log;
    w.add((uint32_t)(log - 5), 4);
    int remaining = S + 1, threshold = S, nb = log + 1, s = 0; bool prev0 = false;
    while (s < t.nsym && remaining > 1) {
        if (prev0) {
            int start = s;
            while (s < t.nsym && t.norm[s] == 0) s++;
            if (s == t.nsym) break;
            while (s >= start + 3) { start += 3; w.add(3, 2); }
            w.add((uint32_t)(s - start), 2);
        }
        int count = t.norm[s++];
        const int mx = 2 * threshold - 1 - remaining;
        remaining -= count < 0 ? -count : count;
        count++;
        if (count >= threshold) count += mx;
        w.add((uint32_t)count, nb - (count < mx ? 1 : 0));
        prev0 = count == 1;
        if (remaining < 1) return 0;
        while (remaining < threshold) { nb--; threshold >>= 1; }
    }
    if (remaining != 1) return 0;
    return w.finish_raw();
}

__device__ __forceinline__ void zkc_fse_init_state(const ZkcFse& t, uint32_t sym, uint32_t& state) {
    if (t.mode == 1) { state = 0; return; }
    const uint32_t dnb = t.delta_nb[sym];
    const uint32_t nb_out = (dnb + (1u << 15)) >> 16;
    const uint32_t value = (nb_out << 16) - dnb;
    state = t.state_tbl[(value >> nb_out) + t.delta_find[sym]];
}
template <class W>
__device__ __forceinline__ void zkc_fse_encode(const ZkcFse& t, W& w, uint32_t sym, uint32_t& state) {
    if (t.mode == 1) return;
    const uint32_t nb_out = (state + t.delta_nb[sym]) >> 16;
    w.add(state, (int)nb_out);
    state = t.state_tbl[(state >> nb_out) + t.delta_find[sym]];
}
template <class W>
__device__ __forceinline__ void zkc_fse_flush(const ZkcFse& t, W& w, uint32_t state) {
    if (t.mode == 1) return;
    w.add(state, t.log);
}

__device__ void zkc_fse_set_predefined(ZkcFse& t, int which) {
    if (which == 0) { for (int i = 0; i < 36; i++) t.norm[i] = ZK_LL_DEFAULT[i]; t.nsym = 36; t.log = 6; }
    else if (which == 1) { for (int i = 0; i < 29; i++) t.norm[i] = ZK_OF_DEFAULT[i]; t.nsym = 29; t.log = 5; }
    else { for (int i = 0; i < 53; i++) t.norm[i] = ZK_ML_DEFAULT[i]; t.nsym = 53; t.log = 6; }
    t.mode = 0;
}

// =============================================================================================
// K-C2s: sequence section -- one WARP per block.
// The only serial part of coding a block's sequences is the FSE state chain (state -> bits out -> next state, A.6): four
// integer operations and one shared-memory load per symbol.  Three lanes run the three chains (LL, OF, ML) over a tile of
// 32 sequences; everything else is done by all 32 lanes, one sequence each: codes and histograms (pass A), the per-step
// (deltaNbBits, deltaFindState) operands of the chains, extra bits, a warp scan of the bit counts and the packing of each
// sequence's <= 87 bits into a shared-memory staging window that is flushed to HBM as whole words.  (The first version
// ran one LANE per block with all of that on the serial chain: ~400 dependent instructions per sequence.)
// The section is written to a per-block scratch ([0,256) header + table descriptions, [256,..) bitstream) and moved
// into place by the assembly kernel.  Offsets arrive as Offset_Values (repeat codes resolved by K-C1).
// =============================================================================================
#define ZKC_SW 8                   // warps per CTA = blocks in flight per CTA
struct ZkcTabs { uint32_t ll_base[36], ml_base[53]; uint8_t ll_bits[36], ml_bits[53], ll_code[64], ml_code[128]; };
__device__ __forceinline__ uint32_t zkc_llc(const ZkcTabs& tb, uint32_t ll) { return ll < 64 ? tb.ll_code[ll] : (uint32_t)zk_highbit(ll) + 19; }
__device__ __forceinline__ uint32_t zkc_mlc(const ZkcTabs& tb, uint32_t mlb) { return mlb < 128 ? tb.ml_code[mlb] : (uint32_t)zk_highbit(mlb) + 36; }

struct ZkcSeqWarp {
    ZkcFse fse[3];                                   // 0 LL, 1 OF, 2 ML
    uint32_t cnt[3][64];
    union {
        uint8_t symof[3][256];                       // table build scratch (lanes 0..2 build one table each)
        struct {
            uint2 tin[3][33];                        // per step: (deltaNbBits, deltaFindState) of the step's symbol (padded: the three chains hit different banks)
            uint16_t tout[3][34];                    // per step: (bits << 4) | nbBits written by the chain
            uint32_t stage[96];                      // bit staging: [0] carries the partial word of the previous tile
        } b;
    } u;
    uint8_t hdr[3][84];                              // table descriptions before they are concatenated
};

// one table (lane t of the warp): choose the mode, build the coding table, write its description.  -> false: not encodable
__device__ bool zkc_seq_table(ZkcFse& ft, const uint32_t* cnt, int t, uint32_t nseq, uint8_t* symof, uint8_t* hdr, uint32_t* mode, uint32_t* nbytes) {
    const int max_log = 8, nsym_all = t == 0 ? 36 : (t == 1 ? 32 : 53);
    int last = nsym_all - 1; while (last > 0 && cnt[last] == 0) last--;
    uint32_t distinct = 0; for (int q = 0; q <= last; q++) distinct += cnt[q] != 0;
    if (distinct == 1) {
        ft.mode = 1; ft.rle_sym = (uint8_t)last; ft.log = 0;
        ft.state_tbl[0] = 0; ft.delta_nb[last] = 0; ft.delta_find[last] = 0;             // the chain then idles at state 0, emitting no bits
        hdr[0] = (uint8_t)last; *mode = 1; *nbytes = 1;
        return true;
    }
    if (nseq < 48 && (t != 1 || last <= 28)) { zkc_fse_set_predefined(ft, t); zkc_fse_build(ft, symof); *mode = 0; *nbytes = 0; return true; }
    int lg = zk_highbit(nseq) - 1; if (lg < 5) lg = 5; if (lg > max_log) lg = max_log;
    int need = zk_highbit(distinct) + 1; if (lg < need) lg = need; if (lg > max_log) return false;
    zkc_fse_normalize(ft, cnt, last + 1, nseq, lg);
    ft.mode = 2;
    zkc_fse_build(ft, symof);
    const uint32_t hb = zkc_fse_write_ncount(ft, hdr, 84);
    if (!hb) return false;
    *mode = 2; *nbytes = hb;
    return true;
}

// whole warp; returns false if the section cannot be encoded within the scratch (the block then becomes a Raw block)
__device__ bool zkc_encode_sequences(ZkcSeqWarp& sw, const ZkcTabs& tb, const uint16_t* s_ll, const uint16_t* s_ml, const uint32_t* s_ov, uint32_t nseq,
                                     uint8_t* out, uint32_t* hdr_bytes, uint32_t* bits_bytes, int lane) {
    // ---- pass A: code histograms, one sequence per lane
    for (int i = lane; i < 3 * 64; i += 32) (&sw.cnt[0][0])[i] = 0;
    __syncwarp();
    for (uint32_t i = lane; i < nseq; i += 32) {
        atomicAdd(&sw.cnt[0][zkc_llc(tb, s_ll[i])], 1u); atomicAdd(&sw.cnt[1][zk_highbit(s_ov[i])], 1u); atomicAdd(&sw.cnt[2][zkc_mlc(tb, s_ml[i])], 1u);
    }
    __syncwarp();
    // ---- tables: lanes 0..2 build one each
    uint32_t mode = 0, nb_t = 0; bool ok = true;
    if (lane < 3) ok = zkc_seq_table(sw.fse[lane], sw.cnt[lane], lane, nseq, sw.u.symof[lane], sw.hdr[lane], &mode, &nb_t);
    if (!__all_sync(0xFFFFFFFFu, ok)) return false;
    uint32_t hp = 0;
    if (lane == 0) {
        if (nseq < 128) out[hp++] = (uint8_t)nseq;
        else if (nseq < 0x7F00) { out[hp++] = (uint8_t)((nseq >> 8) + 128); out[hp++] = (uint8_t)nseq; }
        else { out[hp++] = 255; out[hp++] = (uint8_t)(nseq - 0x7F00); out[hp++] = (uint8_t)((nseq - 0x7F00) >> 8); }
    }
    hp = __shfl_sync(0xFFFFFFFFu, hp, 0);
    {
        const uint32_t m0 = __shfl_sync(0xFFFFFFFFu, mode, 0), m1 = __shfl_sync(0xFFFFFFFFu, mode, 1), m2 = __shfl_sync(0xFFFFFFFFu, mode, 2);
        const uint32_t n0 = __shfl_sync(0xFFFFFFFFu, nb_t, 0), n1 = __shfl_sync(0xFFFFFFFFu, nb_t, 1), n2 = __shfl_sync(0xFFFFFFFFu, nb_t, 2);
        if (lane == 0) out[hp] = (uint8_t)((m0 << 6) | (m1 << 4) | (m2 << 2));
        hp++;
        if (hp + n0 + n1 + n2 > ZKC_SEQHDR - 6) return false;
        for (uint32_t i = lane; i < n0; i += 32) out[hp + i] = sw.hdr[0][i];
        for (uint32_t i = lane; i < n1; i += 32) out[hp + n0 + i] = sw.hdr[1][i];
        for (uint32_t i = lane; i < n2; i += 32) out[hp + n0 + n1 + i] = sw.hdr[2][i];
        hp += n0 + n1 + n2;
    }
    __syncwarp();                                    // the build scratch (union) is dead from here on
    // ---- pass B (backward): the bitstream, last sequence first (mirror of the decoder's order, A.5)
    uint32_t* const gw = (uint32_t*)(out + ZKC_SEQHDR);
    const uint32_t cap_words = (ZKC_SEQSEC - ZKC_SEQHDR) / 4;
    for (int i = lane; i < 96; i += 32) sw.u.b.stage[i] = 0;
    uint32_t st = 0;                                 // lanes 0..2: state of chain `lane`
    uint32_t bitpos = 0;                             // bits emitted so far
    bool first = true, ovf = false;
    const uint32_t lt_mask = (1u << lane) - 1u; (void)lt_mask;
    for (uint32_t hi_i = nseq; hi_i > 0;) {
        const uint32_t cntT = hi_i < 32u ? hi_i : 32u;
        const bool act = (uint32_t)lane < cntT;
        const uint32_t idx = act ? hi_i - 1u - (uint32_t)lane : 0u;       // step `lane` of this tile codes sequence idx
        const uint32_t llv = s_ll[idx], mlb = s_ml[idx], ov = s_ov[idx];
        const uint32_t llc = zkc_llc(tb, llv), mlc = zkc_mlc(tb, mlb), ofc = (uint32_t)zk_highbit(ov);
        if (act) {
            sw.u.b.tin[0][lane] = make_uint2(sw.fse[0].delta_nb[llc], (uint32_t)(int)sw.fse[0].delta_find[llc]);
            sw.u.b.tin[1][lane] = make_uint2(sw.fse[1].delta_nb[ofc], (uint32_t)(int)sw.fse[1].delta_find[ofc]);
            sw.u.b.tin[2][lane] = make_uint2(sw.fse[2].delta_nb[mlc], (uint32_t)(int)sw.fse[2].delta_find[mlc]);
        }
        __syncwarp();
        if (lane < 3) {                              // the three chains
            const uint16_t* stt = sw.fse[lane].state_tbl;
            const uint2* ti = sw.u.b.tin[lane]; uint16_t* to = sw.u.b.tout[lane];
            uint32_t j = 0;
            if (first) {
                if (sw.fse[lane].mode == 1) st = 0;
                else {
                    const uint2 d = ti[0];
                    const uint32_t nb_out = (d.x + (1u << 15)) >> 16, value = (nb_out << 16) - d.x;
                    st = stt[(value >> nb_out) + (int)d.y];
                }
                to[0] = 0; j = 1;
            }
#pragma unroll 4
            for (; j < cntT; j++) {
                const uint2 d = ti[j];
                const uint32_t nb_out = (st + d.x) >> 16;
                to[j] = (uint16_t)(((st & ((1u << nb_out) - 1u)) << 4) | nb_out);
                st = stt[(st >> nb_out) + (int)d.y];
            }
        }
        first = false;
        __syncwarp();
        // this lane's sequence: state bits (OF, ML, LL), then extra bits (LL, ML, OF)
        unsigned long long v = 0; uint32_t n1 = 0, v2 = 0, n2 = 0;
        if (act) {
            const uint32_t o = sw.u.b.tout[1][lane], m = sw.u.b.tout[2][lane], l = sw.u.b.tout[0][lane];
            v = o >> 4; n1 = o & 15u;
            v |= (unsigned long long)(m >> 4) << n1; n1 += m & 15u;
            v |= (unsigned long long)(l >> 4) << n1; n1 += l & 15u;
            v |= (unsigned long long)(llv - tb.ll_base[llc]) << n1; n1 += tb.ll_bits[llc];
            v |= (unsigned long long)(mlb + 3u - tb.ml_base[mlc]) << n1; n1 += tb.ml_bits[mlc];
            v2 = ov - (1u << ofc); n2 = ofc;
        }
        uint32_t incl = n1 + n2;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += t; }
        const uint32_t tile_bits = __shfl_sync(0xFFFFFFFFu, incl, 31);
        const uint32_t base_bit = bitpos & 31u;
        if (act) {
            uint32_t pos = base_bit + incl - (n1 + n2);
            if (n1) {
                const uint32_t w = pos >> 5, sh = pos & 31u;
                const unsigned long long lo = v << sh;
                atomicOr(&sw.u.b.stage[w], (uint32_t)lo);
                if (lo >> 32) atomicOr(&sw.u.b.stage[w + 1], (uint32_t)(lo >> 32));
                if (sh) { const uint32_t hi = (uint32_t)(v >> (64u - sh)); if (hi) atomicOr(&sw.u.b.stage[w + 2], hi); }
            }
            pos += n1;
            if (n2) {
                const uint32_t w = pos >> 5, sh = pos & 31u;
                const unsigned long long lo = (unsigned long long)v2 << sh;
                atomicOr(&sw.u.b.stage[w], (uint32_t)lo);
                if (lo >> 32) atomicOr(&sw.u.b.stage[w + 1], (uint32_t)(lo >> 32));
            }
        }
        __syncwarp();
        // flush the full words, keep the partial one as word 0 of the next tile
        const uint32_t nwords = (base_bit + tile_bits) >> 5, word0 = bitpos >> 5;
        if (word0 + nwords > cap_words) ovf = true;
        else for (uint32_t w = lane; w < nwords; w += 32) gw[word0 + w] = sw.u.b.stage[w];
        const uint32_t carry = sw.u.b.stage[nwords];
        __syncwarp();
        for (uint32_t w = lane; w <= nwords + 2; w += 32) sw.u.b.stage[w] = w == 0 ? carry : 0u;
        __syncwarp();
        bitpos += tile_bits;
        hi_i -= cntT;
    }
    // final states (ML, OF, LL), then the end mark
    const uint32_t s_l = __shfl_sync(0xFFFFFFFFu, st, 0), s_o = __shfl_sync(0xFFFFFFFFu, st, 1), s_m = __shfl_sync(0xFFFFFFFFu, st, 2);
    const uint32_t lg_l = (uint32_t)sw.fse[0].log, lg_o = (uint32_t)sw.fse[1].log, lg_m = (uint32_t)sw.fse[2].log;
    unsigned long long fin = s_m & ((1u << lg_m) - 1u); uint32_t nf = lg_m;
    fin |= (unsigned long long)(s_o & ((1u << lg_o) - 1u)) << nf; nf += lg_o;
    fin |= (unsigned long long)(s_l & ((1u << lg_l) - 1u)) << nf; nf += lg_l;
    fin |= 1ull << nf; nf += 1;
    const uint32_t base_bit = bitpos & 31u, word0 = bitpos >> 5;
    const unsigned long long tail = ((unsigned long long)sw.u.b.stage[0]) | (fin << base_bit);      // <= 31 + 25 bits
    const uint32_t total_bits = bitpos + nf;
    const uint32_t sb = (total_bits + 7u) >> 3;
    if (ovf || word0 + 2 > cap_words) return false;
    if (lane == 0) { gw[word0] = (uint32_t)tail; gw[word0 + 1] = (uint32_t)(tail >> 32); }
    *hdr_bytes = hp; *bits_bytes = sb;
    return true;
}

__global__ void __launch_bounds__(32 * ZKC_SW) zk_seq_enc_kernel(ZkEncodeArgs a) {
    ZK_DYN_SMEM(smem);
    ZkcTabs* tb = (ZkcTabs*)smem;
    ZkcSeqWarp* sws = (ZkcSeqWarp*)(smem + ((sizeof(ZkcTabs) + 15) & ~(size_t)15));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, tid = threadIdx.x, nt = 32 * ZKC_SW;
    for (int i = tid; i < 36; i += nt) { tb->ll_base[i] = ZK_LL_BASE[i]; tb->ll_bits[i] = ZK_LL_BITS[i]; }
    for (int i = tid; i < 53; i += nt) { tb->ml_base[i] = ZK_ML_BASE[i]; tb->ml_bits[i] = ZK_ML_BITS[i]; }
    for (int i = tid; i < 64; i += nt) tb->ll_code[i] = ZKC_LL_CODE[i];
    for (int i = tid; i < 128; i += nt) tb->ml_code[i] = ZKC_ML_CODE[i];
    __syncthreads();
    const uint32_t b = blockIdx.x * ZKC_SW + warp;
    if (b >= a.n_blocks) return;
    const uint32_t nseq = a.blocks[b].nseq;
    uint32_t hb = 0, sb = 0;
    if (nseq) {
        const bool ok = zkc_encode_sequences(sws[warp], *tb, a.seq_ll + (size_t)b * ZKC_MAXSEQ, a.seq_ml + (size_t)b * ZKC_MAXSEQ,
                                             a.seq_off + (size_t)b * ZKC_MAXSEQ, nseq, a.seqsec + (size_t)b * ZKC_SEQSEC, &hb, &sb, lane);
        if (!ok) { hb = 0; sb = 0; }
    }
    if (lane == 0) { a.blocks[b].seq_hdr = hb; a.blocks[b].seq_bits = sb; }
}

#define ZKC_LW 4                        // K-C2l warps per CTA, one block each
#define ZKC_LWIN 48u                    // stream packing window in words: the carried partial word + one 128-symbol tile (<= 1408 bits) + 2

// per-warp shared state of K-C2l (4 KiB).  The phases (tree build + code lengths and codes, weight coding, stream packing)
// never overlap, so their scratch shares one union; with four warps per CTA, registers rather than shared memory set the
// warps per SM of this latency-bound kernel.
struct ZkcLitWarp {
    uint32_t hist4[2][256];             // per-stream counts, two 16-bit fields per word (streams 0|1, 2|3); a symbol's count is their sum
    uint16_t hcode[256];                // (length << 11) | code; 0: symbol absent
    union {
        struct { uint16_t node[511]; uint32_t num[33]; uint32_t cls[16]; } t;      // tree (weights -> parents -> depths), lengths, code cursors
        struct { ZkcFse fse; uint8_t symof[64]; uint8_t weights[256]; uint32_t wc[16]; uint16_t cumul[16]; } w;    // FSE coding of the weights
        uint32_t win[ZKC_LWIN];         // stream packing: [0] carries the partial word of the previous tile
    } u;
    uint8_t hdr[128];                   // tree description
};

// Huffman code lengths limited to 11 bits, into sm.hcode (length << 11).  Whole warp: the present symbols are ranked by
// (count, symbol) with a bitonic sort of the keys (count << 8) | symbol, eight per lane in registers; lane 0 runs the
// two-queue tree build in one array (a consumed node's slot takes its parent, then the depths replace the parents in
// place); the warp turns depths into limited lengths.  Returns max code length (0 = fewer than two symbols).
__device__ int zkc_huf_build(ZkcLitWarp& sm, int lane) {
    uint32_t key[8];
    int n = 0;
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const uint32_t s = 32u * r + (uint32_t)lane, a0 = sm.hist4[0][s], a1 = sm.hist4[1][s];
        const uint32_t c = (a0 & 0xFFFFu) + (a0 >> 16) + (a1 & 0xFFFFu) + (a1 >> 16);
        key[r] = (c << 8) | s;
        n += __popc(__ballot_sync(0xFFFFFFFFu, c != 0));
    }
    if (n < 2) return 0;
    // ascending over e = 8 * lane + r: strides of 8 and more are lane shuffles, smaller ones stay in the lane
#pragma unroll
    for (int ks = 1; ks <= 8; ks++) {
#pragma unroll
        for (int js = ks - 1; js >= 0; js--) {
            if (js >= 3) {
                const int lj = 1 << (js - 3);
                const bool upper = (lane & lj) != 0, desc = ((lane >> (ks - 3)) & 1) != 0;
#pragma unroll
                for (int r = 0; r < 8; r++) {
                    const uint32_t o = __shfl_xor_sync(0xFFFFFFFFu, key[r], lj);
                    key[r] = upper != desc ? max(key[r], o) : min(key[r], o);
                }
            } else {
#pragma unroll
                for (int r = 0; r < 8; r++) {
                    if (r & (1 << js)) continue;
                    const int p = r | (1 << js);
                    const bool desc = (((8 * lane + r) >> ks) & 1) != 0;
                    const uint32_t lo = min(key[r], key[p]), hi = max(key[r], key[p]);
                    key[r] = desc ? hi : lo; key[p] = desc ? lo : hi;
                }
            }
        }
    }
    // the present symbols are the top n keys: rank k = e - (256 - n)
    uint16_t* node = sm.u.t.node;                             // leaves 0..n-1 (sorted), internal nodes n..2n-2
    uint32_t* num = sm.u.t.num;
    const int off = 256 - n;
#pragma unroll
    for (int r = 0; r < 8; r++) { const int k = 8 * lane + r - off; if (k >= 0) node[k] = (uint16_t)(key[r] >> 8); }
    for (int i = lane; i <= 32; i += 32) num[i] = 0;
    __syncwarp();
    if (lane == 0) {
        int leaf = 0, inode = n, next = n;
        for (int k = 0; k < n - 1; k++) {       // weights fit 16 bits: they sum to at most ZKC_BLOCK
            int a, b;
            if (leaf < n && (inode >= next || node[leaf] <= node[inode])) a = leaf++; else a = inode++;
            if (leaf < n && (inode >= next || node[leaf] <= node[inode])) b = leaf++; else b = inode++;
            const uint32_t w = (uint32_t)node[a] + node[b];
            node[a] = (uint16_t)next; node[b] = (uint16_t)next; node[next] = (uint16_t)w; next++;
        }
        node[next - 1] = 0;
        for (int i = next - 2; i >= 0; i--) node[i] = (uint16_t)(node[node[i]] + 1);
    }
    __syncwarp();
    // histogram of code lengths, limited to 11 (miniz-style redistribution keeps the code complete)
    const int L = 11;
    for (int i = lane; i < n; i += 32) { const uint32_t d = node[i]; atomicAdd(&num[d < (uint32_t)L ? d : (uint32_t)L], 1u); }
    __syncwarp();
    if (lane == 0) {
        unsigned total = 0;
        for (int i = L; i > 0; i--) total += num[i] << (L - i);
        while (total != (1u << L)) {
            num[L]--;
            for (int i = L - 1; i > 0; i--) if (num[i]) { num[i]--; num[i + 1] += 2; break; }
            total--;
        }
    }
    __syncwarp();
    // most frequent symbols (top ranks) get the shortest codes: rank k from the top takes the length whose class holds it
    int maxlen = L; while (!num[maxlen]) maxlen--;
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const int k = 8 * lane + r - off;
        if (k >= 0) {
            const uint32_t p = (uint32_t)(n - 1 - k);
            uint32_t l = 1, c = num[1];
            while (p >= c) c += num[++l];
            sm.hcode[key[r] & 255u] = (uint16_t)(l << 11);
        }
    }
    __syncwarp();
    return maxlen;
}

// are all n >= 2 literals the same byte?  4-byte words (the buffer is 32 KiB aligned); most blocks settle in the first round
__device__ __forceinline__ bool zkc_lits_rle(const uint8_t* lits, uint32_t n, int lane) {
    const uint32_t c4 = lits[0] * 0x01010101u, n4 = n & ~3u;
    bool rle = n >= 2;
    for (uint32_t i0 = 0; rle && i0 < n4; i0 += 128) {
        const uint32_t i = i0 + 4u * (uint32_t)lane;
        rle = __all_sync(0xFFFFFFFFu, i >= n4 || *(const uint32_t*)(lits + i) == c4);
    }
    return __all_sync(0xFFFFFFFFu, (uint32_t)lane >= n - n4 || lits[n4 + lane] == lits[0]) && rle;
}

// HUF = false (the fast tier): literals are only ever Raw or RLE, decided without a histogram or shared memory.
// NW warps per CTA, one block per warp (64 registers at most with HUF, so that 32 warps fit an SM).
template <bool HUF, int NW>
__global__ void __launch_bounds__(32 * NW, HUF ? 32 / NW : 1) zk_lit_enc_kernel(ZkEncodeArgs a) {
    __shared__ ZkcLitWarp sms[HUF ? NW : 1];
    const int lane = threadIdx.x & 31;
    const uint32_t b = blockIdx.x * NW + (threadIdx.x >> 5);
    if (b >= a.n_blocks) return;
    ZkcLitWarp& sm = sms[HUF ? threadIdx.x >> 5 : 0];
    const ZkcGeo g = a.geo[b];
    const uint32_t len = g.len;
    const uint32_t last_flag = g.last;
    const uint32_t nlit = a.blocks[b].nlit;
    const uint8_t* lits = a.lits + (size_t)b * ZKC_BLOCK;
    uint8_t* out = a.stage + (size_t)b * ZKC_SLOT;
    uint32_t opos = 3;                                   // block header written last
    bool raw_block = len < 32;                           // tiny blocks: not worth entropy coding

    // ------------------------------------------------------------------ literals section (A.3)
    if (!raw_block) {
        int maxlen = 0; uint32_t lit_mode = 0;           // 0 raw, 1 rle, 2 huffman
        if (!HUF) lit_mode = zkc_lits_rle(lits, nlit, lane) ? 1u : 0u;
        else {
            for (int i = lane; i < 256; i += 32) { sm.hist4[0][i] = 0; sm.hist4[1][i] = 0; sm.hcode[i] = 0; }
            __syncwarp();
            {   // four literals per lane and load (the buffer is 32 KiB aligned); the stream a literal belongs to follows from its index
                const uint32_t seg = (nlit + 3) / 4, n4 = nlit & ~3u;
                for (uint32_t i = 4u * (uint32_t)lane; i < n4; i += 128) {
                    const uint32_t w = *(const uint32_t*)(lits + i);
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        const uint32_t idx = i + q, st = (idx >= seg) + (idx >= 2 * seg) + (idx >= 3 * seg);
                        atomicAdd(&sm.hist4[st >> 1][(w >> (8 * q)) & 255u], 1u << ((st & 1u) * 16u));
                    }
                }
                if ((uint32_t)lane < nlit - n4) {
                    const uint32_t idx = n4 + lane, st = (idx >= seg) + (idx >= 2 * seg) + (idx >= 3 * seg);
                    atomicAdd(&sm.hist4[st >> 1][lits[idx]], 1u << ((st & 1u) * 16u));
                }
            }
            __syncwarp();
            // decide: Raw / RLE / Huffman
            uint32_t mx = 0;
            for (int s = lane; s < 256; s += 32) {
                const uint32_t a0 = sm.hist4[0][s], a1 = sm.hist4[1][s];
                mx = max(mx, (a0 & 0xFFFFu) + (a0 >> 16) + (a1 & 0xFFFFu) + (a1 >> 16));
            }
            for (int d = 16; d; d >>= 1) mx = max(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, d));
            if (nlit > 0 && mx == nlit && nlit >= 2) lit_mode = 1;
            else if (nlit >= 64) {
                maxlen = zkc_huf_build(sm, lane);
                if (maxlen) {
                    uint32_t bits = 0;
                    for (int s = lane; s < 256; s += 32) {
                        const uint32_t a0 = sm.hist4[0][s], a1 = sm.hist4[1][s];
                        bits += ((a0 & 0xFFFFu) + (a0 >> 16) + (a1 & 0xFFFFu) + (a1 >> 16)) * (uint32_t)(sm.hcode[s] >> 11);
                    }
                    for (int d = 16; d; d >>= 1) bits += __shfl_xor_sync(0xFFFFFFFFu, bits, d);
                    uint32_t est = (bits + 7) / 8 + 8 + 130;
                    if (est < nlit) lit_mode = 2;
                }
            }
        }

        uint32_t tree_bytes = 0;
        if (HUF && lit_mode == 2) {
            // canonical codes exactly as the decoder lays out its table: weight ascending, symbol ascending (A.4).  A symbol's
            // code is its class's start cell (lane w scans the cells of the classes below w) plus its rank among the class's
            // earlier symbols (a match over each 32 symbols, then the class cursor moves on)
            int last_sym = 0;
            for (int s0 = 224; s0 >= 0; s0 -= 32) {
                const uint32_t m = __ballot_sync(0xFFFFFFFFu, sm.hcode[s0 + lane] != 0);
                if (m) { last_sym = s0 + 31 - __clz((int)m); break; }
            }
            uint32_t* cls = sm.u.t.cls;
            {
                const bool in = lane >= 1 && lane <= maxlen;
                const uint32_t v = in ? sm.u.t.num[maxlen + 1 - lane] << (lane - 1) : 0u;
                uint32_t incl = v;
                for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += t; }
                if (in) cls[lane] = incl - v;
            }
            __syncwarp();
            for (int s0 = 0; s0 <= last_sym; s0 += 32) {
                const uint32_t l = sm.hcode[s0 + lane] >> 11;
                const int w = l ? maxlen + 1 - (int)l : 0;
                const uint32_t m = __match_any_sync(0xFFFFFFFFu, (uint32_t)w), below = m & ((1u << lane) - 1u);
                if (l) sm.hcode[s0 + lane] = (uint16_t)(((cls[w] >> (w - 1)) + (uint32_t)__popc(below)) | (l << 11));
                __syncwarp();
                if (l && !below) cls[w] += (uint32_t)__popc(m) << (w - 1);
                __syncwarp();
            }
            // tree description: weights of symbols 0..last_sym-1 (the last one is implied)
            const int nw = last_sym;
            if (lane < 16) sm.u.w.wc[lane] = 0;
            __syncwarp();
            int maxw = 0;
            for (int s = lane; s < nw; s += 32) {
                const int l = sm.hcode[s] >> 11, wt = l ? maxlen + 1 - l : 0;
                sm.u.w.weights[s] = (uint8_t)wt; atomicAdd(&sm.u.w.wc[wt], 1u); maxw = max(maxw, wt);
            }
            for (int d = 16; d; d >>= 1) maxw = max(maxw, __shfl_xor_sync(0xFFFFFFFFu, maxw, d));
            __syncwarp();
            uint32_t tb = 0;
            if (lane == 0) {
                // FSE-compressed weights (two interleaved states), A.4
                if (nw > 1) {
                    uint32_t distinct = 0; for (int i = 0; i <= maxw; i++) distinct += sm.u.w.wc[i] != 0;
                    if (distinct > 1) {
                        ZkcFse& t = sm.u.w.fse;
                        int lg = 6; while (lg > 5 && (1 << lg) > nw) lg--;        // table log 5..6
                        zkc_fse_normalize(t, sm.u.w.wc, maxw + 1, (uint32_t)nw, lg);
                        t.mode = 2;
                        zkc_fse_build_in(t, sm.u.w.symof, sm.u.w.cumul);
                        uint32_t hb = zkc_fse_write_ncount(t, sm.hdr + 1, 120);
                        if (hb) {
                            ZkcBitW w; w.init(sm.hdr + 1 + hb, 127 - hb);
                            // encode from the last weight to the first, alternating two states
                            uint32_t s1, s2; int n = nw;
                            if (n & 1) { zkc_fse_init_state(t, sm.u.w.weights[n - 1], s1); zkc_fse_init_state(t, sm.u.w.weights[n - 2], s2); n -= 2;
                                         zkc_fse_encode(t, w, sm.u.w.weights[n - 1], s1); n--; }
                            else { zkc_fse_init_state(t, sm.u.w.weights[n - 1], s2); zkc_fse_init_state(t, sm.u.w.weights[n - 2], s1); n -= 2; }
                            while (n >= 2) { zkc_fse_encode(t, w, sm.u.w.weights[n - 1], s2); zkc_fse_encode(t, w, sm.u.w.weights[n - 2], s1); n -= 2; }
                            zkc_fse_flush(t, w, s2); zkc_fse_flush(t, w, s1);
                            uint32_t sb = w.finish();
                            if (sb && hb + sb < 128 && hb + sb < (uint32_t)(nw + 1) / 2) { sm.hdr[0] = (uint8_t)(hb + sb); tb = 1 + hb + sb; }
                        }
                    }
                }
                if (!tb) {
                    if (nw <= 128) {
                        sm.hdr[0] = (uint8_t)(127 + nw);
                        for (int s = 0; s < nw; s += 2) sm.hdr[1 + s / 2] = (uint8_t)((sm.u.w.weights[s] << 4) | (s + 1 < nw ? sm.u.w.weights[s + 1] : 0));
                        tb = 1 + (uint32_t)(nw + 1) / 2;
                    }
                }
            }
            tree_bytes = __shfl_sync(0xFFFFFFFFu, tb, 0);
            if (!tree_bytes) lit_mode = 0;               // cannot describe the tree: raw literals
        }

        if (HUF && lit_mode == 2) {
            // stream sizes first (so the section header, which precedes the streams, can be sized)
            const uint32_t seg = (nlit + 3) / 4;
            uint32_t ssz[4];
            {
                uint32_t b0 = 0, b1 = 0, b2 = 0, b3 = 0;
                for (int sy = lane; sy < 256; sy += 32) {
                    const uint32_t l = sm.hcode[sy] >> 11, a0 = sm.hist4[0][sy], a1 = sm.hist4[1][sy];
                    b0 += (a0 & 0xFFFFu) * l; b1 += (a0 >> 16) * l; b2 += (a1 & 0xFFFFu) * l; b3 += (a1 >> 16) * l;
                }
                for (int d = 16; d; d >>= 1) {
                    b0 += __shfl_xor_sync(0xFFFFFFFFu, b0, d); b1 += __shfl_xor_sync(0xFFFFFFFFu, b1, d);
                    b2 += __shfl_xor_sync(0xFFFFFFFFu, b2, d); b3 += __shfl_xor_sync(0xFFFFFFFFu, b3, d);
                }
                ssz[0] = (b0 + 1 + 7) / 8; ssz[1] = (b1 + 1 + 7) / 8; ssz[2] = (b2 + 1 + 7) / 8; ssz[3] = (b3 + 1 + 7) / 8;   // + end mark
            }
            const uint32_t comp = tree_bytes + 6 + ssz[0] + ssz[1] + ssz[2] + ssz[3];
            if (comp >= nlit || ssz[0] > 0xFFFF || ssz[1] > 0xFFFF || ssz[2] > 0xFFFF) lit_mode = 0;
            else {
                // header: 4 streams, size format by magnitude
                uint32_t hsz;
                if (nlit < 1024 && comp < 1024) { hsz = 3; unsigned long long v = 2u | (1u << 2) | ((unsigned long long)nlit << 4) | ((unsigned long long)comp << 14);
                    if (lane == 0) { out[opos] = (uint8_t)v; out[opos + 1] = (uint8_t)(v >> 8); out[opos + 2] = (uint8_t)(v >> 16); } }
                else if (nlit < 16384 && comp < 16384) { hsz = 4; unsigned long long v = 2u | (2u << 2) | ((unsigned long long)nlit << 4) | ((unsigned long long)comp << 18);
                    if (lane == 0) { out[opos] = (uint8_t)v; out[opos + 1] = (uint8_t)(v >> 8); out[opos + 2] = (uint8_t)(v >> 16); out[opos + 3] = (uint8_t)(v >> 24); } }
                else { hsz = 5; unsigned long long v = 2u | (3u << 2) | ((unsigned long long)nlit << 4) | ((unsigned long long)comp << 22);
                    if (lane == 0) { out[opos] = (uint8_t)v; out[opos + 1] = (uint8_t)(v >> 8); out[opos + 2] = (uint8_t)(v >> 16); out[opos + 3] = (uint8_t)(v >> 24); out[opos + 4] = (uint8_t)(v >> 32); } }
                opos += hsz;
                for (uint32_t i = lane; i < tree_bytes; i += 32) out[opos + i] = sm.hdr[i];
                opos += tree_bytes;
                if (lane == 0) { out[opos] = (uint8_t)ssz[0]; out[opos + 1] = (uint8_t)(ssz[0] >> 8); out[opos + 2] = (uint8_t)ssz[1]; out[opos + 3] = (uint8_t)(ssz[1] >> 8);
                                 out[opos + 4] = (uint8_t)ssz[2]; out[opos + 5] = (uint8_t)(ssz[2] >> 8); }
                opos += 6;
                // encode each stream: symbol i of the stream sits above all later symbols (the decoder reads backward),
                // so its bit position is the sum of the code lengths of the symbols after it -> warp scan over reversed order.
                // Every stream goes through the window as whole words of the staging slot (the slot is 4-byte aligned), flushed
                // after each 128 symbols; its first word starts with the bytes before the stream, read back from the slot.
                // The last word may run up to 3 bytes past the stream: the next stream or K-C2f writes over them.
                __syncwarp();                                         // the tree description has left the union; the bytes above are in the slot
                uint32_t* const win = sm.u.win;
                for (int st = 0; st < 4; st++) {
                    const uint32_t s0 = st * seg, s1 = st < 3 ? s0 + seg : nlit, m = s1 - s0;
                    const uint32_t pre = opos & 3u;
                    uint32_t* const gw = (uint32_t*)(out + (opos - pre));
                    for (uint32_t i = lane; i < ZKC_LWIN; i += 32) win[i] = (i == 0 && pre) ? gw[0] & ((1u << (8u * pre)) - 1u) : 0u;
                    __syncwarp();
                    uint32_t base = 8u * pre;                         // bit position in gw
                    for (uint32_t g = 0; g < m; g += 128) {
                        // four symbols per lane (reversed indices r .. r+3, r lowest in the stream): one scan and at most
                        // three atomics serve 128 symbols
                        const uint32_t r = g + 4u * (uint32_t)lane;
                        unsigned long long v = 0; uint32_t l = 0;
                        if (r + 4 <= m) {
                            // the four symbols are the bytes [s1-4-r, s1-r): one unaligned 4-byte load (two aligned ones)
                            const uint32_t ad = s1 - 4u - r, mis = ad & 3u;
                            const uint32_t* wp = (const uint32_t*)(lits + (ad - mis));
                            const uint32_t w4 = mis ? __funnelshift_r(wp[0], wp[1], mis * 8u) : wp[0];
#pragma unroll
                            for (int q = 0; q < 4; q++) {
                                const uint32_t cl = sm.hcode[(w4 >> (8 * (3 - q))) & 255u]; v |= (unsigned long long)(cl & 2047u) << l; l += cl >> 11;
                            }
                        } else {
#pragma unroll
                            for (int q = 0; q < 4; q++) {
                                if (r + q < m) { const uint32_t cl = sm.hcode[lits[s1 - 1 - r - q]]; v |= (unsigned long long)(cl & 2047u) << l; l += cl >> 11; }
                            }
                        }
                        uint32_t incl = l;
                        for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += t; }
                        const uint32_t org = base & 31u;                  // bit position of the tile inside win
                        const uint32_t bitpos = org + incl - l;
                        if (l) {
                            const uint32_t sh = bitpos & 31u, w = bitpos >> 5;
                            const unsigned long long lo2 = v << sh;
                            atomicOr(&win[w], (uint32_t)lo2);
                            if (lo2 >> 32) atomicOr(&win[w + 1], (uint32_t)(lo2 >> 32));
                            if (sh) { const uint32_t hi2 = (uint32_t)(v >> (64u - sh)); if (hi2) atomicOr(&win[w + 2], hi2); }
                        }
                        const uint32_t tile_bits = __shfl_sync(0xFFFFFFFFu, incl, 31);
                        __syncwarp();
                        const uint32_t nwords = (org + tile_bits) >> 5, word0 = base >> 5;
                        for (uint32_t i = lane; i < nwords; i += 32) gw[word0 + i] = win[i];
                        const uint32_t carry = win[nwords];
                        __syncwarp();
                        for (uint32_t i = lane; i <= nwords + 2; i += 32) win[i] = i == 0 ? carry : 0u;
                        __syncwarp();
                        base += tile_bits;
                    }
                    if (lane == 0) gw[base >> 5] = win[0] | (1u << (base & 31u));   // the partial word and the end mark
                    opos += ssz[st];
                    __syncwarp();
                }
            }
        }
        if (lit_mode == 1) {
            // RLE literals
            uint32_t hsz = nlit < 32 ? 1 : (nlit < 4096 ? 2 : 3);
            if (lane == 0) {
                if (hsz == 1) out[opos] = (uint8_t)(1u | (nlit << 3));
                else if (hsz == 2) { uint32_t v = 1u | (1u << 2) | (nlit << 4); out[opos] = (uint8_t)v; out[opos + 1] = (uint8_t)(v >> 8); }
                else { uint32_t v = 1u | (3u << 2) | (nlit << 4); out[opos] = (uint8_t)v; out[opos + 1] = (uint8_t)(v >> 8); out[opos + 2] = (uint8_t)(v >> 16); }
                out[opos + hsz] = lits[0];
            }
            opos += hsz + 1;
        } else if (lit_mode == 0) {
            uint32_t hsz = nlit < 32 ? 1 : (nlit < 4096 ? 2 : 3);
            if (lane == 0) {
                if (hsz == 1) out[opos] = (uint8_t)(0u | (nlit << 3));
                else if (hsz == 2) { uint32_t v = 0u | (1u << 2) | (nlit << 4); out[opos] = (uint8_t)v; out[opos + 1] = (uint8_t)(v >> 8); }
                else { uint32_t v = 0u | (3u << 2) | (nlit << 4); out[opos] = (uint8_t)v; out[opos + 1] = (uint8_t)(v >> 8); out[opos + 2] = (uint8_t)(v >> 16); }
            }
            opos += hsz;
            if (opos + nlit + 4 >= len + 3) raw_block = true;       // cannot win any more
            else { zkc_warp_copy(out + opos, lits, nlit, lane); opos += nlit; }
        }
    }

    // the sequences section is coded concurrently by K-C2s on another stream; zk_block_finish_kernel joins the two
    if (lane == 0) { a.blocks[b].lit_bytes = raw_block ? 0u : opos; a.blocks[b].last_flag = last_flag; }
}

// K-C2f: join literals + sequences, fall back to a Raw block when that is not smaller, write the block header (A.2)
__global__ void __launch_bounds__(128) zk_block_finish_kernel(ZkEncodeArgs a) {
    const int lane = threadIdx.x & 31;
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= a.n_blocks) return;
    const ZkcBlock bl = a.blocks[b];
    const ZkcGeo g = a.geo[b];
    const size_t lo = g.lo;
    const uint32_t len = g.len;
    uint8_t* out = a.stage + (size_t)b * ZKC_SLOT;
    uint32_t opos = bl.lit_bytes;
    bool raw_block = opos == 0;
    if (!raw_block) {
        if (bl.nseq == 0) { if (lane == 0) out[opos] = 0; opos += 1; }
        else {
            const uint32_t hp = bl.seq_hdr, sb = bl.seq_bits;
            if (!hp || opos + hp + sb >= len + 3) raw_block = true;
            else {
                const uint8_t* sec = a.seqsec + (size_t)b * ZKC_SEQSEC;
                for (uint32_t i = lane; i < hp; i += 32) out[opos + i] = sec[i];
                opos += hp;
                for (uint32_t i = lane; i < sb; i += 32) out[opos + i] = sec[ZKC_SEQHDR + i];
                opos += sb;
            }
        }
    }
    if (!raw_block && opos >= len + 3) raw_block = true;
    if (raw_block) {
        for (uint32_t i = lane; i < len; i += 32) out[3 + i] = a.src[lo + i];
        opos = 3 + len;
    }
    if (lane == 0) {
        uint32_t bh = bl.last_flag | ((raw_block ? 0u : 2u) << 1) | ((raw_block ? len : opos - 3) << 3);
        out[0] = (uint8_t)bh; out[1] = (uint8_t)(bh >> 8); out[2] = (uint8_t)(bh >> 16);
        a.blocks[b].csize = opos;
    }
}

// =============================================================================================
// K-C3: frame layout + gather, over the a.res[0] frames and a.res[1] blocks of the tables
// =============================================================================================
// XXH64 (A.8) of each frame's input, one warp per frame (zk_warp_xxh64: coalesced loads, products off the chain)
__global__ void __launch_bounds__(128) zk_frame_hash_kernel(ZkEncodeArgs a) {
    const int lane = threadIdx.x & 31;
    const uint32_t f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (f >= a.res[0]) return;
    const uint8_t* p = a.src + a.frames[f].start; const uint32_t len = a.frames[f].size;
    const unsigned long long h = zk_warp_xxh64(p, len, lane);
    if (lane == 0) a.frame_hash[f] = (uint32_t)h;
}

// record and staging slot of block b, block k of its frame: those of its variant min(k, V - 1)
__device__ __forceinline__ size_t zkc_variant_slot(const ZkEncodeArgs& a, uint32_t b, uint32_t k) {
    return (size_t)min(k, a.V - 1) * a.n_blocks + b;
}

// one warp per frame: block offsets inside the frame (warp scan over its blocks), frame size
__global__ void __launch_bounds__(128) zk_frame_size_kernel(ZkEncodeArgs a) {
    const int lane = threadIdx.x & 31;
    const uint32_t f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (f >= a.res[0]) return;
    const uint32_t s = a.frames[f].first_block, e = s + a.frames[f].n_blocks;
    uint32_t run = ZKC_FRAME_HDR;
    for (uint32_t j = s; j < e; j += 32) {
        const uint32_t b = j + (uint32_t)lane;
        ZkcBlock* bl = b < e ? a.blocks + zkc_variant_slot(a, b, b - s) : nullptr;
        const uint32_t cs = bl ? bl->csize : 0u;
        uint32_t incl = cs;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += t; }
        if (bl) bl->out_off = run + incl - cs;
        run += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
    if (lane == 0) a.res[ZKC_RES_HDR + f] = run + (a.checksum ? 4u : 0u);
}

// exclusive prefix sum of x(i), i < n, by one CTA of 1024 threads: put(i, x(0) + .. + x(i - 1)); returns the sum of all to every thread
template <class X, class Put>
__device__ __forceinline__ unsigned long long zkc_cta_scan(uint32_t n, X x, Put put) {
    __shared__ unsigned long long part[1024];
    __shared__ unsigned long long carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const unsigned long long v = i < n ? x(i) : 0;
        part[threadIdx.x] = v;
        __syncthreads();
        for (uint32_t d = 1; d < 1024; d <<= 1) {
            const unsigned long long t = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
            __syncthreads();
            part[threadIdx.x] += t;
            __syncthreads();
        }
        if (i < n) put(i, carry + part[threadIdx.x] - v);
        __syncthreads();
        if (threadIdx.x == 1023) carry += part[1023];
        __syncthreads();
    }
    return carry;
}

// frame offsets and the total (one CTA); with a chain (ZkEncodeParams::chain), the frames follow the chain[0] bytes the batches before
// wrote, and chain[1] receives the end of this batch's
__global__ void __launch_bounds__(1024) zk_frame_scan_kernel(ZkEncodeArgs a, unsigned long long* chain) {
    const unsigned long long base = chain ? chain[0] : 0ull;
    const unsigned long long total = zkc_cta_scan(a.res[0], [&](uint32_t f) { return (unsigned long long)a.res[ZKC_RES_HDR + f]; },
                                                  [&](uint32_t f, unsigned long long o) { a.frame_off[f] = base + o; });
    if (threadIdx.x == 0) {
        *(unsigned long long*)(a.res + 4) = total;
        if (base + total > a.dst_cap) a.res[2] = ZKZ_DST_TOO_SMALL;
        if (chain) chain[1] = base + total;
    }
}

// gather: one warp per block copies its staged bytes to the final position and sets Last_Block (a variant was staged with its own
// layout's flag); block 0 of a frame also writes the frame header, the last block the checksum
__global__ void __launch_bounds__(128) zk_frame_gather_kernel(ZkEncodeArgs a) {
    const int lane = threadIdx.x & 31;
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= a.res[1] || a.res[2]) return;
    const ZkcGeo g = a.geo[b];
    const uint32_t f = g.frame;
    const size_t slot = zkc_variant_slot(a, b, g.k);
    const ZkcBlock bl = a.blocks[slot];
    uint8_t* fo = a.dst + a.frame_off[f];
    if (g.k == 0 && lane == 0) {
        const ZkcFrame F = a.frames[f];
        const uint32_t fcs = F.size;
        // the smallest Window_Size = 2^(10 + e) * (1 + m / 8) >= max(wmin, min(fcs + reach, wmax)), where reach is the prefix bytes the
        // frame's offsets may reach: its tail, or all of its prefix up to 2^27 back (a.far == 2, or 1 and a prefix); an empty frame holds
        // no match, so it takes the minimum whatever the prefix
        const bool far = a.far == 2 || (a.far == 1 && F.plen);
        const size_t reach = fcs ? (far ? F.plen : F.tail) : 0, wmax = far ? 1u << 27 : a.wmax;
        size_t want = fcs + reach < wmax ? fcs + reach : wmax;
        if (want < a.wmin) want = a.wmin;
        uint32_t e = 0, m = 0;
        while (((size_t)8 + m) << (7 + e) < want) { if (++m == 8) { m = 0; e++; } }
        fo[0] = 0x28; fo[1] = 0xB5; fo[2] = 0x2F; fo[3] = 0xFD;
        fo[4] = (uint8_t)(0x80 | (a.checksum ? 0x04 : 0));       // FCS 4 bytes, no single segment, no dict
        fo[5] = (uint8_t)((e << 3) | m);
        fo[6] = (uint8_t)fcs; fo[7] = (uint8_t)(fcs >> 8); fo[8] = (uint8_t)(fcs >> 16); fo[9] = (uint8_t)(fcs >> 24);
        if (a.checksum) {
            const uint32_t h = a.frame_hash[f]; uint8_t* c = fo + a.res[ZKC_RES_HDR + f] - 4;
            c[0] = (uint8_t)h; c[1] = (uint8_t)(h >> 8); c[2] = (uint8_t)(h >> 16); c[3] = (uint8_t)(h >> 24);
        }
    }
    const uint8_t* s = a.stage + slot * ZKC_SLOT; uint8_t* d = fo + bl.out_off;
    const uint32_t n = bl.csize;
    // staged slots are 16-byte aligned; destinations are arbitrary -> byte-granular head, 16-byte body when co-aligned
    uint32_t head = (uint32_t)((16 - ((uintptr_t)d & 15)) & 15); if (head > n) head = n;
    if (lane < (int)head) d[lane] = s[lane];
    const uint8_t* s2 = s + head; uint8_t* d2 = d + head; const uint32_t n2 = n - head, nvec = n2 >> 4;
    const uint32_t mis = (uint32_t)((uintptr_t)s2 & 3);
    const uint32_t* sa = (const uint32_t*)(s2 - mis); const uint32_t sh = mis * 8;
    for (uint32_t i = lane; i < nvec; i += 32) {
        const uint32_t* q = sa + 4 * i;
        uint32_t w0 = q[0], w1 = q[1], w2 = q[2], w3 = q[3], w4 = mis ? q[4] : 0;
        ((uint4*)d2)[i] = mis ? make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh), __funnelshift_r(w3, w4, sh))
                              : make_uint4(w0, w1, w2, w3);
    }
    for (uint32_t i = (nvec << 4) + lane; i < n2; i += 32) d2[i] = s2[i];
    __syncwarp();
    if (lane == 0) d[0] = (uint8_t)((s[0] & 0xFEu) | g.last);
}

// =============================================================================================
// K-C3c: FrameSizePolicy::Compressed(target) over one pass of at most 1 GiB (zk_encode_csize).
//
// A block's compressed bytes depend only on its own input, on how many earlier blocks of its frame it may search (its history
// depth: <= 1 below the wide tier, <= ZKC_WIDE_HIST in it) and on whether it opens its frame (prefix tail, repeat offsets
// {1,4,8}).  So K-C1/K-C2 run once per depth d = 0 .. V-1 over the whole pass ("variant d"), and block i of a frame that starts
// at block s is variant min(i - s, V-1) of block i.  Every frame's size is then known for every possible start, and the cut is
// exact: a frame closes after the first block at which header + blocks >= target, or at 1 GiB of input.  The cut writes the
// frame table of the frames it closes; K-C3 assembles them.
// =============================================================================================
#define ZKC_CAP_BLOCKS (0x40000000u / ZKC_BLOCK)     // SEEKABLE_MAX_FRAME_SIZE in blocks
#define ZKC_OPEN 0xFFFFFFFFu                         // next[i]: the frame starting at block i does not close inside this pass

struct ZkCsizeArgs {
    size_t n;                                        // the pass
    uint32_t nb, V, target;
    uint32_t end_closes;                             // the pass ends the input and the caller is done with it: the rest is the last frame
    uint32_t end_lazy;                               // the pass ends the input but more may follow: a frame that ends there stays open
    const ZkcBlock* vblocks;                         // V x nb: variant d of block i at [d * nb + i]
    unsigned long long* psum;                        // nb + 1: prefix sum of variant V-1's sizes
    uint32_t* next;                                  // nb: first block after the frame that starts at block i, or ZKC_OPEN
    uint32_t* starts;                                // nb + 1: first blocks of the frames the walk closes, then the end of the last
    ZkcFrame* frames;                                // their frame table
    uint32_t* res;                                   // the result area of the chosen frames (ZKC_RES_HDR)
    uint32_t pfx, plen;                              // every frame's prefix: the whole buffer of plen bytes (pfx == 0: none)
};

// prefix sum of variant V-1's block sizes (one CTA)
__global__ void __launch_bounds__(1024) zk_csize_psum_kernel(ZkCsizeArgs c) {
    const ZkcBlock* bl = c.vblocks + (size_t)(c.V - 1) * c.nb;
    const unsigned long long total = zkc_cta_scan(c.nb, [&](uint32_t i) { return (unsigned long long)bl[i].csize; },
                                                  [&](uint32_t i, unsigned long long s) { c.psum[i] = s; });
    if (threadIdx.x == 0) c.psum[c.nb] = total;
}

// next[i] for every block i: the first V-1 blocks of the frame from their own variants, the rest by binary search in psum
__global__ void __launch_bounds__(256) zk_csize_next_kernel(ZkCsizeArgs c) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= c.nb) return;
    const uint32_t lim = c.nb - i < ZKC_CAP_BLOCKS ? c.nb : i + ZKC_CAP_BLOCKS;       // exclusive: end of the pass or the 1 GiB cap
    unsigned long long acc = ZKC_FRAME_HDR;
    uint32_t end = 0;                                                              // 0: target not reached before lim
    for (uint32_t t = 0; t + 1 < c.V && i + t < lim; t++) {
        acc += c.vblocks[(size_t)t * c.nb + i + t].csize;
        if (acc >= c.target) { end = i + t + 1; break; }
    }
    if (!end && i + c.V - 1 < lim) {
        // smallest j in [i + V, lim] with acc + psum[j] - psum[i + V - 1] >= target
        const unsigned long long need = c.target - acc + c.psum[i + c.V - 1];
        uint32_t lo = i + c.V, hi = lim + 1;
        while (lo < hi) { const uint32_t mid = lo + (hi - lo) / 2; if (c.psum[mid] >= need) hi = mid; else lo = mid + 1; }
        if (lo <= lim) end = lo;
    }
    bool closed = true;
    if (!end) { end = lim; closed = lim - i == ZKC_CAP_BLOCKS || c.end_closes; }
    if (end == c.nb && c.end_lazy) closed = false;
    c.next[i] = closed ? end : ZKC_OPEN;
}

// the chain of frame starts from block 0 (one CTA; next[] in shared memory: a 1 GiB pass is 128 KiB of it)
__global__ void __launch_bounds__(1024) zk_csize_walk_kernel(ZkCsizeArgs c) {
    ZK_DYN_SMEM(smem);
    uint32_t* nx = (uint32_t*)smem;
    for (uint32_t i = threadIdx.x; i < c.nb; i += blockDim.x) nx[i] = c.next[i];
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t f = 0, p = 0;
        while (p < c.nb && nx[p] != ZKC_OPEN) { c.starts[f++] = p; p = nx[p]; }
        c.starts[f] = p;
        c.res[0] = f; c.res[1] = p;
    }
}

// the frame table of the frames the walk closed and their input sizes, one thread per frame
__global__ void __launch_bounds__(256) zk_geo_starts_kernel(ZkCsizeArgs c) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= c.res[0]) return;
    const uint32_t s = c.starts[f], e = c.starts[f + 1];
    const size_t hi = (size_t)e * ZKC_BLOCK < c.n ? (size_t)e * ZKC_BLOCK : c.n;
    ZkcFrame r;
    r.start = (size_t)s * ZKC_BLOCK; r.size = (uint32_t)(hi - r.start); r.first_block = s; r.n_blocks = e - s;
    zkc_frame_prefix(r, c.pfx, 0, c.plen);
    r.vpre = (unsigned long long)f * r.tail;
    c.frames[f] = r; c.res[ZKC_RES_HDR + c.nb + f] = r.size;
}

// =============================================================================================
// host-side launcher
// =============================================================================================
size_t zk_encode_bound(size_t n, uint32_t frame_size) {
    if (frame_size == 0) frame_size = 1;
    size_t frames = n / frame_size + 1;
    size_t blocks = n / ZKC_BLOCK + frames + 1;
    return n + frames * (ZKC_FRAME_HDR + 4) + blocks * 3 + 64;
}

// blocks of a frame of d bytes
static inline uint32_t zkc_frame_blocks(size_t d) { return d ? (uint32_t)((d + ZKC_BLOCK - 1) / ZKC_BLOCK) : 1u; }

size_t zk_encode_bound_sized(const uint32_t* sizes, uint32_t n_frames) {
    size_t b = 64;
    for (uint32_t f = 0; f < n_frames; f++) b += (size_t)sizes[f] + ZKC_FRAME_HDR + 4 + 3 * (size_t)zkc_frame_blocks(sizes[f]);
    return b;
}

size_t ZkFrames::bound() const { return sizes ? zk_encode_bound_sized(sizes, count) : zk_encode_bound(n, frame_size); }

void zk_encode_ws_free(ZkEncodeWs* ws) {
    if (ws->buf) cudaFree(ws->buf);
    if (ws->cut) cudaFree(ws->cut);
    if (ws->reuse) cudaFree(ws->reuse);
    if (ws->patch) cudaFree(ws->patch);
    if (ws->h_sizes) cudaFreeHost(ws->h_sizes);
    if (ws->side) cudaStreamDestroy(ws->side);
    if (ws->ev_a) cudaEventDestroy(ws->ev_a);
    if (ws->ev_b) cudaEventDestroy(ws->ev_b);
    if (ws->ev_c) cudaEventDestroy(ws->ev_c);
    if (ws->ev_chain) cudaEventDestroy(ws->ev_chain);
    ws->prof.destroy();
    *ws = ZkEncodeWs();
}

static size_t zkc_align(size_t v) { return (v + 255) & ~(size_t)255; }
// the level a caller asks for -> the one the kernels run: 0 is the default (3), levels below ZSTD_minCLevel() clamp to it
static int zkc_level(int level) { return level == 0 ? 3 : (level < ZKC_MIN_LEVEL ? ZKC_MIN_LEVEL : level); }
struct ZkcHcPass;
struct ZkcHcRun;
static int zkc_run_blocks(ZkEncodeWs* ws, cudaStream_t stream, cudaStream_t ss, const ZkEncodeArgs& a, const ZkcHcRun* hc);

// the frame and block tables of a batch and their counts, on `stream`: the uniform layout is generated on the device, the caller's sizes
// are uploaded to d_sizes (and, with per-frame prefixes, the ranges behind them, two words per frame) and scanned there.  pfx: the batch
// has a prefix, the buffer of plen bytes that every frame's prefix lies in (ranges == nullptr: all of it)
static int zkc_build_geometry(ZkEncodeWs* ws, cudaStream_t stream, ZkcGeo* geo, ZkcFrame* fr, uint32_t* count, const ZkFrames& frames,
                              uint32_t n_blocks, uint32_t* d_sizes, uint32_t pfx, uint32_t plen, const uint32_t* ranges) {
    const uint32_t n_frames = frames.count;
    if (frames.sizes) {
        ZK_CUDA_OK(cudaMemcpyAsync(d_sizes, frames.sizes, (size_t)n_frames * 4, cudaMemcpyHostToDevice, stream));
        uint32_t* d_ranges = ranges ? d_sizes + n_frames : nullptr;
        if (ranges) ZK_CUDA_OK(cudaMemcpyAsync(d_ranges, ranges, (size_t)n_frames * 8, cudaMemcpyHostToDevice, stream));
        ZK_LAUNCH(zk_geo_sized_kernel, 1, 1024, 0, stream, fr, count, (const uint32_t*)d_sizes, n_frames, (const uint32_t*)d_ranges, pfx, plen);
    } else ZK_LAUNCH(zk_geo_uniform_kernel, (n_frames + 255) / 256, 256, 0, stream, fr, count, n_frames, frames.n, frames.frame_size, pfx, plen);
    ZK_LAUNCH(zk_geo_block_kernel, (n_blocks + 255) / 256, 256, 0, stream, geo, (const ZkcFrame*)fr, (const uint32_t*)count);
    ws->launches += 2;
    return 0;
}

// the stream K-C2s and the checksum run on: the workspace's side stream, created at its first use
static int zkc_side_stream(ZkEncodeWs* ws, cudaStream_t* ss) {
    if (!ws->side) {
        ZK_CUDA_OK(cudaStreamCreateWithPriority(&ws->side, cudaStreamNonBlocking, ws->prio));
        ZK_CUDA_OK(cudaEventCreateWithFlags(&ws->ev_a, cudaEventDisableTiming));
        ZK_CUDA_OK(cudaEventCreateWithFlags(&ws->ev_b, cudaEventDisableTiming));
        ZK_CUDA_OK(cudaEventCreateWithFlags(&ws->ev_c, cudaEventDisableTiming));
    }
    *ss = ws->side;
    return 0;
}

#include "zk_hc.inc"
#include "zk_cdc.inc"

// The workspace of a batch of n_frames frames over n_blocks blocks, with V variants of every block's record and staged bytes (1 except in
// zk_encode_csize) and, when the frames have prefixes (pfx), their prefix staging slots: a's scratch pointers into it from `base`
// (nullptr: only counts its bytes; the caller's own regions follow), and the fields every batch of tier `lvl` sets alike.  far: the tier
// matches up to 2^27 bytes back, 1 into the prefix of a frame that has one (long-distance matching), 2 also within every frame (long
// mode).  Returns the bytes it takes.
static size_t zkc_carve(ZkEncodeArgs& a, uint8_t* base, uint32_t n_frames, size_t n_blocks, uint32_t V, int lvl, uint32_t far, bool pfx,
                        const ZkEncodeParams& p) {
    size_t off = 0;
    auto at = [&](size_t bytes) { const size_t o = off; off = zkc_align(off + bytes); return (uint8_t*)((uintptr_t)base + o); };
    a.n_frames = n_frames; a.n_blocks = (uint32_t)n_blocks; a.V = V;
    a.geo = (const ZkcGeo*)at(n_blocks * sizeof(ZkcGeo)); a.frames = (const ZkcFrame*)at((size_t)n_frames * sizeof(ZkcFrame));
    a.blocks = (ZkcBlock*)at(V * n_blocks * sizeof(ZkcBlock));
    a.seq_ll = (uint16_t*)at(n_blocks * ZKC_MAXSEQ * 2); a.seq_ml = (uint16_t*)at(n_blocks * ZKC_MAXSEQ * 2);
    a.seq_off = (uint32_t*)at(n_blocks * ZKC_MAXSEQ * 4);
    a.lits = at(n_blocks * ZKC_BLOCK); a.stage = at(V * n_blocks * ZKC_SLOT + 64); a.seqsec = at(n_blocks * ZKC_SEQSEC);
    a.res = (uint32_t*)at((ZKC_RES_HDR + 2 * (size_t)n_frames) * 4);
    a.frame_off = (unsigned long long*)at((size_t)n_frames * 8); a.frame_hash = (uint32_t*)at((size_t)n_frames * 4);
    a.pstage = at(pfx ? (size_t)n_frames * ZKC_PSLOT : 0);
    a.level = lvl; a.checksum = p.checksum ? 1 : 0;
    a.prefix = pfx ? p.prefix : nullptr;
    a.hist_cap = ~(size_t)0; a.hc = nullptr;
    // the window every frame announces (zk_frame_gather_kernel): 128 KiB below the wide tier, whose offsets stay below 64 KiB; the wide
    // tier's offsets reach (ZKC_WIDE_HIST + 1) blocks back, the high-level tier's ZKC_HC_WINDOW bytes within the frame and its prefix tail.
    // Up to 2^27 bytes back (far), the largest window a default libzstd decoder and this one accept (zkc_ldm_window keeps every offset
    // within it), all of the frame's prefix is in reach
    a.wmin = a.wmax = 128u << 10; a.far = far;
    if (lvl >= ZKC_HC_LEVEL) a.wmax = ZKC_HC_WINDOW;
    else if (lvl >= ZKC_WIDE_LEVEL) a.wmin = a.wmax = 256u << 10;
    return off;
}

int zk_encode_enqueue(ZkEncodeWs* ws, cudaStream_t stream, const uint8_t* d_src, const ZkFrames& fr, const ZkEncodeParams& p, uint8_t* d_dst,
                      size_t dst_cap) {
    const size_t n = fr.n; const uint32_t n_frames = fr.count;
    ws->pending_frames = 0;
    if (n_frames == 0) return 0;
    size_t n_blocks = 0;
    if (fr.sizes) {
        for (uint32_t f = 0; f < n_frames; f++) {
            if (fr.sizes[f] > 0x40000000u) return -(int)ZKZ_PARAM_OUT_OF_BOUND;
            n_blocks += zkc_frame_blocks(fr.sizes[f]);
        }
    } else {
        if (fr.frame_size == 0 || fr.frame_size > 0x40000000u) return -(int)ZKZ_PARAM_OUT_OF_BOUND;
        n_blocks = (size_t)(n_frames - 1) * zkc_frame_blocks(fr.frame_size) + zkc_frame_blocks(n - (size_t)(n_frames - 1) * fr.frame_size);
    }
    if (n_blocks > 0x7FFFFFFFull) return -(int)ZKZ_PARAM_OUT_OF_BOUND;
    if (p.ranges && !fr.sizes) return -(int)ZKZ_PARAM_OUT_OF_BOUND;
    // the frames have prefixes: each one's range of the buffer (zk_geo_sized_kernel), its last ZKC_BLOCK bytes staged in front of it
    const bool pfx = p.prefix && p.prefix_len && n;
    // long-distance matching is a part of K-C1h: with it every level runs that tier.  Long mode indexes the input too (positions are u32)
    // and matches the prefix as the long-distance switch does
    if (p.long_mode && n > 0xFFFFFFFFull) return -(int)ZKZ_PARAM_OUT_OF_BOUND;
    const bool ldm = (p.ldm || p.long_mode) && pfx, lin = p.long_mode && n;
    const int lvl = ldm || p.long_mode ? ZKC_HC_LEVEL : zkc_level(p.level);
    const uint32_t far = p.long_mode ? 2u : (ldm ? 1u : 0u);
    ZkcHcRun hc;
    uint32_t hc_span = 0;
    if (lvl >= ZKC_HC_LEVEL) {
        // K-C1h's passes follow the frames' tails; with long-distance matching, every distinct range is indexed once, as a region of
        // its own: its last min(length, ZKC_LDM_REACH) bytes, at virtual positions after those of the regions before it
        std::vector<uint32_t> tails(pfx ? n_frames : 0);
        if (ldm) hc.fregion.assign(n_frames, ZKC_LDM_NOREGION);
        std::map<unsigned long long, uint32_t> seen;
        unsigned long long vtotal = 0;
        for (uint32_t f = 0; pfx && f < n_frames; f++) {
            const uint32_t lo = p.ranges ? p.ranges[2 * f] : 0u, hi = p.ranges ? p.ranges[2 * f + 1] : p.prefix_len;
            tails[f] = hi - lo < ZKC_BLOCK ? hi - lo : ZKC_BLOCK;
            if (!ldm || hi == lo) continue;
            const unsigned long long key = (unsigned long long)lo << 32 | hi;
            auto it = seen.find(key);
            if (it == seen.end()) {
                ZkcLdmRegion r;
                r.reach = hi - lo < ZKC_LDM_REACH ? hi - lo : ZKC_LDM_REACH; r.pbase = hi - r.reach;
                r.vbase = (uint32_t)vtotal; r.run0 = hc.runs;
                vtotal += r.reach; hc.runs += zkc_ldm_runs(r.reach);
                if (vtotal > 0xFFFFFFFFull) return -(int)ZKZ_PARAM_OUT_OF_BOUND;
                it = seen.emplace(key, (uint32_t)hc.regions.size()).first;
                hc.regions.push_back(r);
            }
            hc.fregion[f] = it->second;
        }
        hc_span = zkc_hc_plan(fr, (uint32_t)n_blocks, pfx ? tails.data() : nullptr, hc.plan);
    }
    hc.input = lin;
    const uint32_t n_regions = (uint32_t)hc.regions.size();
    ZkEncodeArgs a;
    size_t off = zkc_carve(a, nullptr, n_frames, n_blocks, 1, lvl, far, pfx, p);
    const size_t o_fsz = off; if (fr.sizes) off = zkc_align(off + (size_t)n_frames * (p.ranges ? 12 : 4));
    const size_t o_hc = off;
    if (lvl >= ZKC_HC_LEVEL) off = zkc_align(off + zkc_hc_layout(hc_span, nullptr, nullptr));
    const size_t o_ldm = off;
    const uint32_t in_slots = lin ? (uint32_t)n_blocks * ZKC_LDM_BSLOTS : 0u;
    if (ldm || lin) off = zkc_align(off + zkc_ldm_layout(hc.runs * ZKC_LDM_PER_RUN, n_regions, n_frames, in_slots, n_blocks, nullptr, nullptr, nullptr, nullptr));
    int rc = zk_grow(&ws->buf, &ws->cap, off, 1);
    if (!rc) rc = zk_grow((void**)&ws->h_sizes, &ws->cap_frames, ZKC_RES_HDR + (size_t)n_frames, 4, true);
    if (rc) return rc;
    uint8_t* base = (uint8_t*)ws->buf;
    zkc_carve(a, base, n_frames, n_blocks, 1, lvl, far, pfx, p);
    a.src = d_src; a.n = n; a.dst = d_dst; a.dst_cap = dst_cap;
    a.hc = base + o_hc;
    if (ldm || lin) hc.ldm = base + o_ldm;
    ZK_CUDA_OK(cudaMemsetAsync(a.res, 0, ZKC_RES_HDR * 4, stream));
    rc = zkc_build_geometry(ws, stream, (ZkcGeo*)a.geo, (ZkcFrame*)a.frames, a.res, fr, (uint32_t)n_blocks, (uint32_t*)(base + o_fsz), pfx,
                            p.prefix_len, p.ranges);
    if (rc) return rc;
    if (pfx) {
        ZK_LAUNCH(zk_prefix_stage_kernel, n_frames, 256, 0, stream, a);
        ws->launches += 1;
    }
    // the content checksum only needs the input: it runs beside the match finder on the side stream (one warp per frame, bound
    // by the latency of its four serial chains, so it leaves the machine to K-C1)
    cudaStream_t ss;
    if ((rc = zkc_side_stream(ws, &ss))) return rc;
    if (p.checksum) {                                       // joined by ev_b in zkc_run_blocks
        ZK_CUDA_OK(cudaEventRecord(ws->ev_c, stream)); ZK_CUDA_OK(cudaStreamWaitEvent(ss, ws->ev_c, 0));     // after whatever produced the input
        ZK_LAUNCH(zk_frame_hash_kernel, (n_frames + 3) / 4, 128, 0, ss, a);
    }
    rc = zkc_run_blocks(ws, stream, ss, a, &hc);
    if (rc) return rc;
    ws->prof.begin(7, stream);
    ZK_LAUNCH(zk_frame_size_kernel, (n_frames + 3) / 4, 128, 0, stream, a);
    if (p.chain_wait) ZK_CUDA_OK(cudaStreamWaitEvent(stream, p.chain_wait, 0));     // the scan of the batch before wrote chain[0]
    ZK_LAUNCH(zk_frame_scan_kernel, 1, 1024, 0, stream, a, p.chain);
    if (p.chain) {
        if (!ws->ev_chain) ZK_CUDA_OK(cudaEventCreateWithFlags(&ws->ev_chain, cudaEventDisableTiming));
        ZK_CUDA_OK(cudaEventRecord(ws->ev_chain, stream));
    }
    ZK_LAUNCH(zk_frame_gather_kernel, (uint32_t)((n_blocks + 3) / 4), 128, 0, stream, a);
    ws->prof.end(7, stream);
    ZK_CUDA_OK(cudaMemcpyAsync(ws->h_sizes, a.res, (ZKC_RES_HDR + (size_t)n_frames) * 4, cudaMemcpyDeviceToHost, stream));
    ws->launches += 7 + (p.checksum ? 1 : 0);
    ws->pending_frames = n_frames;
    return 0;
}

// K-C1 and K-C2 over every block of `a` (match finding, then sequences on `ss` beside literals on `stream`, joined by the finish kernel);
// hc: what the high-level tier needs beside `a` (its levels only)
static int zkc_run_blocks(ZkEncodeWs* ws, cudaStream_t stream, cudaStream_t ss, const ZkEncodeArgs& a, const ZkcHcRun* hc) {
    const size_t n_blocks = a.n_blocks;
    ws->prof.begin(5, stream);
    // six tiers (EncodeOptions::compression_level, encode.rs:176): 1 = 2048-entry table, no history, no lazy step; 2-3 = 4096 entries,
    // previous-block history, one lazy step; 4-6 = double table (8-byte + 5-byte hashes, 4096 entries each), two warps per CTA; 7-9 = double
    // table of 8192 entries each, one warp per CTA; 10-12 = one table of 16384 entries, one warp per CTA; >= 13 = 256 KiB history, 32768 x u32
    // entries in dynamic shared memory.  Ratio on the reference's corpus: 2.12 / 2.24 / 2.28 / 2.38 / 2.40 / 2.50.  Below them the fast tier
    // (level < 0): level 1's table with sparse probing, literals without Huffman coding.  From ZKC_HC_LEVEL on, K-C1h (zk_hc.inc): hash chains
    // over 2 MiB of the frame and a price-based parse
    if (a.level >= ZKC_HC_LEVEL) { const int rc = zkc_run_hc(ws, stream, a, *hc); if (rc) return rc; }
    else if (a.level < 0) ZK_LAUNCH((zk_match_fast_kernel<ZKC_HLOG_FAST, ZKC_C1_WARPS>), (uint32_t)((n_blocks + ZKC_C1_WARPS - 1) / ZKC_C1_WARPS), ZKC_C1_WARPS * 32, 0, stream, a);
    else if (a.level <= 1) ZK_LAUNCH((zk_match_kernel<ZKC_HLOG_FAST, ZKC_C1_WARPS, false>), (uint32_t)((n_blocks + ZKC_C1_WARPS - 1) / ZKC_C1_WARPS), ZKC_C1_WARPS * 32, 0, stream, a);
    else if (a.level <= 3) ZK_LAUNCH((zk_match_kernel<ZKC_HLOG, ZKC_C1_WARPS, false>), (uint32_t)((n_blocks + ZKC_C1_WARPS - 1) / ZKC_C1_WARPS), ZKC_C1_WARPS * 32, 0, stream, a);
    else if (a.level <= 6) ZK_LAUNCH((zk_match_kernel<ZKC_HLOG, 2, true>), (uint32_t)((n_blocks + 1) / 2), 64, 0, stream, a);
    else if (a.level <= 9) ZK_LAUNCH((zk_match_kernel<13, 1, true>), (uint32_t)n_blocks, 32, 0, stream, a);
    else if (a.level < ZKC_WIDE_LEVEL) ZK_LAUNCH((zk_match_kernel<14, 1, false>), (uint32_t)n_blocks, 32, 0, stream, a);
    else {
        const int wide_smem = (int)sizeof(uint32_t) << ZKC_WIDE_HLOG;
        if (!ws->attr_set_wide) { ZK_CUDA_OK(cudaFuncSetAttribute(zk_match_wide_kernel<ZKC_WIDE_HLOG>, cudaFuncAttributeMaxDynamicSharedMemorySize, wide_smem)); ws->attr_set_wide = true; }
        ZK_LAUNCH((zk_match_wide_kernel<ZKC_WIDE_HLOG>), (uint32_t)n_blocks, 32, wide_smem, stream, a);
    }
    ws->prof.end(5, stream);
    const size_t seq_smem = ((sizeof(ZkcTabs) + 15) & ~(size_t)15) + sizeof(ZkcSeqWarp) * ZKC_SW;
    if (!ws->attr_set) { ZK_CUDA_OK(cudaFuncSetAttribute(zk_seq_enc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)seq_smem)); ws->attr_set = true; }
    // the two entropy kernels are independent and both latency-bound: run them side by side, join in zk_block_finish_kernel
    ws->prof.begin(6, stream);
    ZK_CUDA_OK(cudaEventRecord(ws->ev_a, stream)); ZK_CUDA_OK(cudaStreamWaitEvent(ss, ws->ev_a, 0));
    ZK_LAUNCH(zk_seq_enc_kernel, (uint32_t)((n_blocks + ZKC_SW - 1) / ZKC_SW), 32 * ZKC_SW, seq_smem, ss, a);
    ZK_CUDA_OK(cudaEventRecord(ws->ev_b, ss));
    if (a.level < 0) ZK_LAUNCH((zk_lit_enc_kernel<false, 1>), (uint32_t)n_blocks, 32, 0, stream, a);
    else ZK_LAUNCH((zk_lit_enc_kernel<true, ZKC_LW>), (uint32_t)((n_blocks + ZKC_LW - 1) / ZKC_LW), 32 * ZKC_LW, 0, stream, a);
    ZK_CUDA_OK(cudaStreamWaitEvent(stream, ws->ev_b, 0));
    ZK_LAUNCH(zk_block_finish_kernel, (uint32_t)((n_blocks + 3) / 4), 128, 0, stream, a);
    ws->prof.end(6, stream);
    return 0;
}

int zk_encode_collect(ZkEncodeWs* ws, cudaStream_t stream, uint32_t* c_sizes, size_t* dst_len) {
    const uint32_t nf = ws->pending_frames;
    if (nf == 0) { if (dst_len) *dst_len = 0; return 0; }
    if (const int rc = zk_sync_check(stream)) return rc;
    ws->pending_frames = 0;
    ws->prof.harvest();
    const uint32_t* h = ws->h_sizes;
    if (h[2]) return -(int)h[2];
    unsigned long long total; memcpy(&total, h + 4, 8);
    if (c_sizes) memcpy(c_sizes, h + ZKC_RES_HDR, (size_t)nf * 4);
    if (dst_len) *dst_len = (size_t)total;
    return 0;
}

// FrameSizePolicy::Compressed(target) over one pass of n <= 1 GiB bytes: V variant passes of K-C1/K-C2 (shared sequence, literal
// and section scratch; a ZkcBlock[] and a staging area each), the cut (K-C3c), then K-C3 over the frames it chose.
// One D2H copy of the counts and sizes, then one synchronisation.
int zk_encode_csize(ZkEncodeWs* ws, cudaStream_t stream, const uint8_t* d_src, size_t n, uint32_t target, const ZkEncodeParams& p, int final_,
                    int at_end, uint8_t* d_dst, size_t dst_cap, ZkCsizeOut* out) {
    *out = ZkCsizeOut();
    if (n == 0) return 0;
    if (n > 0x40000000u) return -(int)ZKZ_PARAM_OUT_OF_BOUND;
    // the exact cut needs a bounded history per block (the V variants); the high-level tier's frame-wide chains have none, so its levels
    // run the wide tier here
    const int lvl = zkc_level(p.level) >= ZKC_HC_LEVEL ? ZKC_WIDE_LEVEL : zkc_level(p.level);
    const uint32_t nb = (uint32_t)((n + ZKC_BLOCK - 1) / ZKC_BLOCK);
    const uint32_t V = lvl >= ZKC_WIDE_LEVEL ? ZKC_WIDE_HIST + 1 : 2;
    const bool pfx = p.prefix && p.prefix_len;
    // the batch of the chosen frames (nb at most; the cut writes their tables and result area), the cut's arrays, and the two layouts
    // of the variants with their counts: frames of one block (d = 0), one frame over the pass (d >= 1)
    ZkEncodeArgs a;
    size_t off = zkc_carve(a, nullptr, nb, nb, V, lvl, 0, pfx, p);
    const size_t o_psum = off; off = zkc_align(off + ((size_t)nb + 1) * 8);
    const size_t o_next = off; off = zkc_align(off + (size_t)nb * 4);
    const size_t o_starts = off; off = zkc_align(off + ((size_t)nb + 1) * 4);
    const size_t o_geo0 = off; off = zkc_align(off + (size_t)nb * sizeof(ZkcGeo));
    const size_t o_fr0 = off; off = zkc_align(off + (size_t)nb * sizeof(ZkcFrame));
    const size_t o_geo1 = off; off = zkc_align(off + (size_t)nb * sizeof(ZkcGeo));
    const size_t o_fr1 = off; off = zkc_align(off + sizeof(ZkcFrame));
    const size_t o_cnt = off; off = zkc_align(off + 16);
    int rc = zk_grow(&ws->buf, &ws->cap, off, 1);
    if (!rc) rc = zk_grow((void**)&ws->h_sizes, &ws->cap_frames, ZKC_RES_HDR + 2 * (size_t)nb, 4, true);
    if (rc) return rc;
    uint8_t* base = (uint8_t*)ws->buf;
    zkc_carve(a, base, nb, nb, V, lvl, 0, pfx, p);
    a.src = d_src; a.n = n; a.dst = d_dst; a.dst_cap = dst_cap;
    ZkCsizeArgs c;
    c.n = n; c.nb = nb; c.V = V; c.target = target ? target : 1;
    c.end_closes = at_end && final_; c.end_lazy = at_end && !final_;
    c.vblocks = a.blocks; c.psum = (unsigned long long*)(base + o_psum); c.next = (uint32_t*)(base + o_next);
    c.starts = (uint32_t*)(base + o_starts); c.frames = (ZkcFrame*)a.frames; c.res = a.res;
    c.pfx = pfx; c.plen = p.prefix_len;
    ZK_CUDA_OK(cudaMemsetAsync(a.res, 0, ZKC_RES_HDR * 4, stream));
    cudaStream_t ss;
    if ((rc = zkc_side_stream(ws, &ss))) return rc;
    uint32_t* vcount = (uint32_t*)(base + o_cnt);
    rc = zkc_build_geometry(ws, stream, (ZkcGeo*)(base + o_geo0), (ZkcFrame*)(base + o_fr0), vcount, {nullptr, n, ZKC_BLOCK, nb}, nb, nullptr, pfx,
                            p.prefix_len, nullptr);
    if (!rc) rc = zkc_build_geometry(ws, stream, (ZkcGeo*)(base + o_geo1), (ZkcFrame*)(base + o_fr1), vcount + 2, {nullptr, n, (uint32_t)n, 1}, nb,
                                     nullptr, 0, 0, nullptr);
    if (rc) return rc;
    // variant passes.  d = 0: frames of one block, so every block opens its frame (prefix staging included); d >= 1: one frame
    // over the pass, with the wide tier's history capped at d blocks below V - 1
    for (uint32_t d = 0; d < V; d++) {
        ZkEncodeArgs v = a;
        v.geo = (const ZkcGeo*)(base + (d == 0 ? o_geo0 : o_geo1)); v.frames = (const ZkcFrame*)(base + (d == 0 ? o_fr0 : o_fr1));
        v.n_frames = d == 0 ? nb : 1;
        v.hist_cap = d >= 1 && d + 1 < V ? (size_t)d * ZKC_BLOCK : ~(size_t)0;
        v.blocks = a.blocks + (size_t)d * nb; v.stage = a.stage + (size_t)d * nb * ZKC_SLOT;
        if (d >= 1) v.prefix = nullptr;
        else if (pfx) {
            ZK_LAUNCH(zk_prefix_stage_kernel, nb, 256, 0, stream, v);
            ws->launches += 1;
        }
        rc = zkc_run_blocks(ws, stream, ss, v, nullptr);
        if (rc) return rc;
        ws->launches += 4;
    }
    ws->prof.begin(7, stream);
    const uint32_t walk_smem = nb * 4;
    if (!ws->attr_set_walk) {
        ZK_CUDA_OK(cudaFuncSetAttribute(zk_csize_walk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(ZKC_CAP_BLOCKS * 4)));
        ws->attr_set_walk = true;
    }
    ZK_LAUNCH(zk_csize_psum_kernel, 1, 1024, 0, stream, c);
    ZK_LAUNCH(zk_csize_next_kernel, (nb + 255) / 256, 256, 0, stream, c);
    ZK_LAUNCH(zk_csize_walk_kernel, 1, 1024, walk_smem, stream, c);
    ZK_LAUNCH(zk_geo_starts_kernel, (nb + 255) / 256, 256, 0, stream, c);
    ZK_LAUNCH(zk_geo_block_kernel, (nb + 255) / 256, 256, 0, stream, (ZkcGeo*)a.geo, a.frames, (const uint32_t*)a.res);
    if (p.checksum) ZK_LAUNCH(zk_frame_hash_kernel, (nb + 3) / 4, 128, 0, stream, a);
    ZK_LAUNCH(zk_frame_size_kernel, (nb + 3) / 4, 128, 0, stream, a);
    ZK_LAUNCH(zk_frame_scan_kernel, 1, 1024, 0, stream, a, (unsigned long long*)nullptr);
    ZK_LAUNCH(zk_frame_gather_kernel, (nb + 3) / 4, 128, 0, stream, a);
    ws->prof.end(7, stream);
    ws->launches += 8 + (p.checksum ? 1 : 0);
    ZK_CUDA_OK(cudaMemcpyAsync(ws->h_sizes, a.res, (ZKC_RES_HDR + 2 * (size_t)nb) * 4, cudaMemcpyDeviceToHost, stream));
    if ((rc = zk_sync_check(stream))) return rc;
    ws->prof.harvest();
    const uint32_t* h = ws->h_sizes;
    if (h[2]) return -(int)h[2];
    out->n_frames = h[0];
    out->consumed = (size_t)h[1] * ZKC_BLOCK < n ? (size_t)h[1] * ZKC_BLOCK : n;
    unsigned long long total; memcpy(&total, h + 4, 8);
    out->total = (size_t)total;
    out->c_sizes = h + ZKC_RES_HDR;
    out->d_sizes = h + ZKC_RES_HDR + nb;
    return 0;
}

ZkCdcRule zk_cdc_rule(uint32_t size) {
    const uint32_t s = size < 4096u ? 4096u : (size > 0x40000000u ? 0x40000000u : size);
    ZkCdcRule r;
    r.mn = s / 4;
    r.mx = (uint32_t)((uint64_t)s * 4 < 0x40000000ull ? (uint64_t)s * 4 : 0x40000000ull);
    r.thr = 0ull - ~0ull / (s - r.mn);
    return r;
}

// FrameSizePolicy::ContentDefined(size) over one pass of n <= 1 GiB bytes at d_src, which starts a frame: the cut of zk_cdc.inc, then one
// D2H copy of the counts and sizes and one synchronisation.  cap: candidates kept (0: n / 64 + 1).
int zk_encode_cdc(ZkEncodeWs* ws, cudaStream_t stream, const uint8_t* d_src, size_t n, uint32_t size, int final_, int at_end, uint32_t cap,
                  ZkCdcOut* out) {
    *out = ZkCdcOut();
    if (n == 0) return 0;
    if (n > 0x40000000u) return -(int)ZKZ_PARAM_OUT_OF_BOUND;
    const ZkCdcRule rule = zk_cdc_rule(size);
    ZkCdcArgs a;
    a.src = d_src; a.n = (uint32_t)n; a.mn = rule.mn; a.mx = rule.mx; a.thr = rule.thr;
    a.runs = (uint32_t)((n + ZKC_CDC_RUN - 1) / ZKC_CDC_RUN);
    a.cap = cap ? cap : (uint32_t)(n / 64 + 1);
    a.end_closes = at_end && final_; a.end_lazy = at_end && !final_;
    const size_t nc = (size_t)a.runs + 1, nchunks = (nc + ZKC_HC_SCAN - 1) / ZKC_HC_SCAN;
    const size_t res_words = ZKC_CDC_RES_HDR + n / rule.mn + 2;       // every frame but the last has at least mn bytes
    size_t off = 0;
    const size_t o_cnt = off; off = zkc_align(off + nc * 4);
    const size_t o_sum = off; off = zkc_align(off + (nchunks + 1) * 4);
    const size_t o_cand = off; off = zkc_align(off + (size_t)a.cap * 4);
    const size_t o_nxt = off; off = zkc_align(off + (size_t)a.cap * 8);
    const size_t o_res = off; off = zkc_align(off + res_words * 4);
    int rc = zk_grow(&ws->cut, &ws->cut_cap, off, 1);
    if (!rc) rc = zk_grow((void**)&ws->h_sizes, &ws->cap_frames, res_words, 4, true);
    if (rc) return rc;
    uint8_t* base = (uint8_t*)ws->cut;
    a.counts = (uint32_t*)(base + o_cnt); a.cand = (uint32_t*)(base + o_cand); a.nxt = (uint2*)(base + o_nxt); a.res = (uint32_t*)(base + o_res);
    uint32_t* sums = (uint32_t*)(base + o_sum);
    if (!ws->attr_set_cdc) {
        ZK_CUDA_OK(cudaFuncSetAttribute(zk_cdc_walk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(ZKC_CDC_STAGE * 8)));
        ws->attr_set_cdc = true;
    }
    const uint32_t grid = (a.runs + 255) / 256;
    ws->prof.begin(0, stream);
    ZK_LAUNCH(zk_cdc_count_kernel, grid, 256, 0, stream, a);
    ZK_LAUNCH(zk_hc_scan_kernel, (uint32_t)nchunks, 1024, 0, stream, a.counts, nc, sums);
    ZK_LAUNCH(zk_hc_scan_top_kernel, 1, 1024, 0, stream, sums, (uint32_t)nchunks);
    ZK_LAUNCH(zk_hc_scan_add_kernel, (uint32_t)((nc + 255) / 256), 256, 0, stream, a.counts, nc, (const uint32_t*)sums);
    ZK_LAUNCH(zk_cdc_emit_kernel, grid, 256, 0, stream, a);
    ZK_LAUNCH(zk_cdc_next_kernel, (a.cap + 255) / 256, 256, 0, stream, a);
    ZK_LAUNCH(zk_cdc_walk_kernel, 1, 1024, (a.cap < ZKC_CDC_STAGE ? a.cap : ZKC_CDC_STAGE) * 8, stream, a);
    ws->prof.end(0, stream);
    ws->launches += 7;
    ZK_CUDA_OK(cudaMemcpyAsync(ws->h_sizes, a.res, res_words * 4, cudaMemcpyDeviceToHost, stream));
    if ((rc = zk_sync_check(stream))) return rc;
    ws->prof.harvest();
    out->n_frames = ws->h_sizes[0];
    out->consumed = ws->h_sizes[1];
    out->sizes = ws->h_sizes + ZKC_CDC_RES_HDR;
    return 0;
}

#include "zk_reuse.inc"
#include "zk_patch.inc"
