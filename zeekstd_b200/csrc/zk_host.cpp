// zk_host.cpp -- API-mirror half of the C ABI (include/zeekstd_b200.h): the host layer that owns framing,
// seek-table build/parse and I/O, re-stating the reference's Rust types one function per method:
//
//   SeekTable / Parser / Serializer   lib/src/seek_table.rs
//   EncodeOptions / RawEncoder / Encoder   lib/src/encode.rs
//   Seekable / BytesWrapper           lib/src/seekable.rs
//   DecodeOptions / Decoder (+ Seek)  lib/src/decode.rs
//   Error kinds                       lib/src/error.rs
//
// All codec arithmetic goes through zk_compress_frames / zk_decompress_frames (zk_api.cu) -- i.e. the CUDA
// kernels.  Nothing in this file compresses or decompresses on the CPU.
#include "../../include/zeekstd_b200.h"
#include <string.h>
#include <stdlib.h>
#include <algorithm>
#include <vector>
#include <new>

namespace {

const uint32_t kSkippableMagic = 0x184D2A5Eu;          // ZSTD_MAGIC_SKIPPABLE_START | 0xE, seek_table.rs:89
const size_t kSizePerFrame = 8;                        // seek_table.rs:87
const uint32_t kMaxFrameSize = ZK_SEEKABLE_MAX_FRAME_SIZE;

inline uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

}  // namespace

// ================================================================================================ SeekTable
struct zk_seek_table {
    // cumulative offsets, always N + 1 entries starting with (0, 0) -- seek_table.rs:97-131, 314-321
    std::vector<uint64_t> c, d;
    zk_seek_table() : c(1, 0), d(1, 0) {}
    uint32_t num_frames() const { return (uint32_t)(c.size() - 1); }
    // seek_table.rs:916-934 (binary search; offsets past the end map to the last frame)
    uint32_t index_at(uint64_t off, const std::vector<uint64_t>& a) const {
        uint32_t n = num_frames();
        if (n == 0) return 0;              // (the reference underflows here, seek_table.rs:917-918; callers never index an empty table)
        if (off >= a[n]) return n - 1;
        uint32_t low = 0, high = n;
        while (low + 1 < high) { uint32_t mid = low + (high - low) / 2; if (a[mid] <= off) low = mid; else high = mid; }
        return low;
    }
};

extern "C" zk_seek_table* zk_seek_table_new(void) { return new (std::nothrow) zk_seek_table(); }
extern "C" void zk_seek_table_free(zk_seek_table* st) { delete st; }
extern "C" zk_seek_table* zk_seek_table_clone(const zk_seek_table* st) { return st ? new (std::nothrow) zk_seek_table(*st) : nullptr; }

extern "C" int32_t zk_seek_table_log_frame(zk_seek_table* st, uint32_t c_size, uint32_t d_size) {   // seek_table.rs:513-525
    if (st->num_frames() >= ZK_SEEKABLE_MAX_FRAMES) return ZK_ERR_FRAME_INDEX_TOO_LARGE;
    st->c.push_back(st->c.back() + c_size);
    st->d.push_back(st->d.back() + d_size);
    return 0;
}
extern "C" uint32_t zk_seek_table_num_frames(const zk_seek_table* st) { return st->num_frames(); }
extern "C" uint32_t zk_seek_table_frame_index_comp(const zk_seek_table* st, uint64_t off) { return st->index_at(off, st->c); }
extern "C" uint32_t zk_seek_table_frame_index_decomp(const zk_seek_table* st, uint64_t off) { return st->index_at(off, st->d); }

#define ZK_ST_GETTER(name, expr)                                                                   \
    extern "C" int32_t name(const zk_seek_table* st, uint32_t index, uint64_t* out) {              \
        if (index >= st->num_frames()) return ZK_ERR_FRAME_INDEX_TOO_LARGE;                        \
        *out = (expr);                                                                             \
        return 0;                                                                                  \
    }
ZK_ST_GETTER(zk_seek_table_frame_start_comp, st->c[index])                                         // :598
ZK_ST_GETTER(zk_seek_table_frame_start_decomp, st->d[index])                                       // :626
ZK_ST_GETTER(zk_seek_table_frame_end_comp, st->c[index + 1])                                       // :654
ZK_ST_GETTER(zk_seek_table_frame_end_decomp, st->d[index + 1])                                     // :682
ZK_ST_GETTER(zk_seek_table_frame_size_comp, st->c[index + 1] - st->c[index])                       // :710
ZK_ST_GETTER(zk_seek_table_frame_size_decomp, st->d[index + 1] - st->d[index])                     // :739

extern "C" uint64_t zk_seek_table_max_frame_size_comp(const zk_seek_table* st) {                   // :764-774
    uint64_t m = 0; for (uint32_t i = 0; i < st->num_frames(); i++) m = std::max(m, st->c[i + 1] - st->c[i]); return m;
}
extern "C" uint64_t zk_seek_table_max_frame_size_decomp(const zk_seek_table* st) {                 // :793-803
    uint64_t m = 0; for (uint32_t i = 0; i < st->num_frames(); i++) m = std::max(m, st->d[i + 1] - st->d[i]); return m;
}
extern "C" uint64_t zk_seek_table_size_comp(const zk_seek_table* st) { return st->c.back(); }      // :824
extern "C" uint64_t zk_seek_table_size_decomp(const zk_seek_table* st) { return st->d.back(); }    // :851
extern "C" uint32_t zk_seek_table_offsets(const zk_seek_table* st, uint64_t* c_off, uint64_t* d_off, uint32_t cap) {
    uint32_t n = (uint32_t)st->c.size();
    uint32_t k = std::min(n, cap);
    if (c_off) memcpy(c_off, st->c.data(), (size_t)k * 8);
    if (d_off) memcpy(d_off, st->d.data(), (size_t)k * 8);
    return n;
}

// ---- generic source (trait Seekable, seekable.rs:16-39) --------------------------------------------------
namespace {
struct Source {
    bool is_bytes = false;
    const uint8_t* bytes = nullptr; size_t len = 0, pos = 0;       // BytesWrapper, seekable.rs:43-97
    zk_seekable cb{};
    // -> new position or error
    int32_t set_offset(int whence, int64_t off, uint64_t* newpos = nullptr) {
        if (is_bytes) {
            int64_t p;
            if (whence == 0) { if (off < 0) return ZK_ERR_OFFSET_OUT_OF_RANGE; p = off; }
            else p = (int64_t)len + off;
            if (p < 0 || (uint64_t)p > len) return ZK_ERR_OFFSET_OUT_OF_RANGE;          // seekable.rs:66-69
            pos = (size_t)p; if (newpos) *newpos = (uint64_t)p;
            return 0;
        }
        int64_t r = cb.set_offset(cb.user, whence, off);
        if (r < 0) return ZK_ERR_IO;
        if (newpos) *newpos = (uint64_t)r;
        return 0;
    }
    // -> bytes read (>= 0) or error (< 0)
    int64_t read(uint8_t* buf, size_t n) {
        if (is_bytes) { size_t k = std::min(n, len - pos); memcpy(buf, bytes + pos, k); pos += k; return (int64_t)k; }   // seekable.rs:74-80
        int64_t r = cb.read(cb.user, buf, n);
        return r < 0 ? (int64_t)ZK_ERR_IO : r;
    }
    int32_t read_exact(uint8_t* buf, size_t n) {
        size_t got = 0;
        while (got < n) { int64_t r = read(buf + got, n - got); if (r < 0) return (int32_t)r; if (r == 0) return ZK_ERR_IO; got += (size_t)r; }
        return 0;
    }
    // seek_table_integrity(format), seekable.rs:83-96 / 124-137
    int32_t integrity(zk_format format, uint8_t out[9]) {
        if (is_bytes) {
            size_t off;
            if (format == ZK_FORMAT_HEAD) { if (len < ZK_SKIPPABLE_HEADER_SIZE + ZK_SEEK_TABLE_INTEGRITY_SIZE) return ZK_ERR_OFFSET_OUT_OF_RANGE; off = ZK_SKIPPABLE_HEADER_SIZE; }
            else { if (len < ZK_SEEK_TABLE_INTEGRITY_SIZE) return ZK_ERR_OFFSET_OUT_OF_RANGE; off = len - ZK_SEEK_TABLE_INTEGRITY_SIZE; }
            memcpy(out, bytes + off, 9);
            return 0;
        }
        int32_t rc = format == ZK_FORMAT_HEAD ? set_offset(0, ZK_SKIPPABLE_HEADER_SIZE) : set_offset(1, -(int64_t)ZK_SEEK_TABLE_INTEGRITY_SIZE);
        if (rc) return rc;
        return read_exact(out, 9);
    }
};

// SeekTable::from_seekable_format, seek_table.rs:379-436 (+ Parser :144-225)
int32_t seek_table_from_source(Source& src, zk_format format, zk_seek_table** out) {
    uint8_t integ[9];
    int32_t rc = src.integrity(format, integ);
    if (rc) return rc;
    if (rd32(integ + 5) != ZK_SEEKABLE_MAGIC_NUMBER) return ZK_ERR_ZSTD(10);          // prefix_unknown, :145-147
    if ((integ[4] >> 2) & 0x1f) return ZK_ERR_ZSTD(20);                               // reserved bits, :150-152
    const bool with_checksum = (integ[4] & 0x80) != 0;
    const uint32_t num_frames = rd32(integ);
    if (num_frames > ZK_SEEKABLE_MAX_FRAMES) return ZK_ERR_FRAME_INDEX_TOO_LARGE;
    const size_t per = with_checksum ? 12 : 8;
    const size_t table_size = (size_t)num_frames * per + ZK_SKIPPABLE_HEADER_SIZE + ZK_SEEK_TABLE_INTEGRITY_SIZE;
    rc = format == ZK_FORMAT_HEAD ? src.set_offset(0, 0) : src.set_offset(1, -(int64_t)table_size);
    if (rc) return rc;
    std::vector<uint8_t> buf(std::min<size_t>(8192, table_size));
    size_t have = 0;
    while (have < ZK_SKIPPABLE_HEADER_SIZE) {
        int64_t r = src.read(buf.data() + have, buf.size() - have);
        if (r < 0) return (int32_t)r;
        if (r == 0) return ZK_ERR_ZSTD(20);                                          // EOF, :393-396
        have += (size_t)r;
    }
    if (rd32(buf.data()) != kSkippableMagic) return ZK_ERR_ZSTD(10);                 // :175-181
    if ((size_t)rd32(buf.data() + 4) + ZK_SKIPPABLE_HEADER_SIZE != table_size) return ZK_ERR_ZSTD(20);
    zk_seek_table* st = new (std::nothrow) zk_seek_table();
    if (!st) return ZK_ERR_ZSTD(64);
    st->c.reserve((size_t)num_frames + 1); st->d.reserve((size_t)num_frames + 1);
    size_t start = ZK_SKIPPABLE_HEADER_SIZE + (format == ZK_FORMAT_HEAD ? ZK_SEEK_TABLE_INTEGRITY_SIZE : 0);
    // in Head format the integrity field may not be fully buffered yet
    while (have < start) {
        int64_t r = src.read(buf.data() + have, buf.size() - have);
        if (r <= 0) { delete st; return r < 0 ? (int32_t)r : ZK_ERR_ZSTD(20); }
        have += (size_t)r;
    }
    uint32_t parsed = 0;
    size_t pos = start;
    while (parsed < num_frames) {
        while (parsed < num_frames && pos + per <= have) {                           // parse_entries, :186-209
            st->c.push_back(st->c.back() + rd32(buf.data() + pos));
            st->d.push_back(st->d.back() + rd32(buf.data() + pos + 4));
            pos += per; parsed++;
        }
        if (parsed == num_frames) break;
        memmove(buf.data(), buf.data() + pos, have - pos);                           // keep the partial entry, :419-421
        have -= pos; pos = 0;
        int64_t r = src.read(buf.data() + have, buf.size() - have);
        if (r < 0) { delete st; return (int32_t)r; }
        if (r == 0) { delete st; return ZK_ERR_ZSTD(20); }                           // EOF with data remaining, :425-428
        have += (size_t)r;
    }
    *out = st;
    return 0;
}
}  // namespace

extern "C" int32_t zk_seek_table_from_bytes(const uint8_t* buf, size_t len, zk_format format, zk_seek_table** out) {
    if (!out || (!buf && len)) return ZK_ERR_INVALID_ARG;
    Source s; s.is_bytes = true; s.bytes = buf; s.len = len;
    return seek_table_from_source(s, format, out);
}

// ---- Serializer (seek_table.rs:955-1051): byte-resumable ----------------------------------------------------
struct zk_serializer {
    std::vector<uint32_t> cs, ds;        // per-frame sizes (Entries::into_frames, :113-121)
    zk_format format;
    size_t write_pos = 0;
    size_t encoded_len() const { return ZK_SKIPPABLE_HEADER_SIZE + ZK_SEEK_TABLE_INTEGRITY_SIZE + cs.size() * kSizePerFrame; }
    uint8_t byte_at(size_t p) const {
        const size_t n = cs.size();
        auto le = [](uint32_t v, size_t i) { return (uint8_t)(v >> (8 * i)); };
        if (p < 4) return le(kSkippableMagic, p);
        if (p < 8) return le((uint32_t)(encoded_len() - ZK_SKIPPABLE_HEADER_SIZE), p - 4);
        size_t q = p - 8;
        const size_t frames_bytes = n * kSizePerFrame;
        size_t integ_at = format == ZK_FORMAT_HEAD ? 0 : frames_bytes, frames_at = format == ZK_FORMAT_HEAD ? ZK_SEEK_TABLE_INTEGRITY_SIZE : 0;
        if (q >= integ_at && q < integ_at + ZK_SEEK_TABLE_INTEGRITY_SIZE) {
            size_t k = q - integ_at;
            if (k < 4) return le((uint32_t)n, k);
            if (k == 4) return 0;                                                    // seek table descriptor, always 0 (:71-76)
            return le(ZK_SEEKABLE_MAGIC_NUMBER, k - 5);
        }
        size_t k = q - frames_at, f = k / 8, r = k % 8;
        return r < 4 ? le(cs[f], r) : le(ds[f], r - 4);
    }
};

extern "C" zk_serializer* zk_seek_table_into_serializer(const zk_seek_table* st, zk_format format) {
    zk_serializer* s = new (std::nothrow) zk_serializer();
    if (!s) return nullptr;
    s->format = format;
    uint32_t n = st->num_frames();
    s->cs.resize(n); s->ds.resize(n);
    for (uint32_t i = 0; i < n; i++) { s->cs[i] = (uint32_t)(st->c[i + 1] - st->c[i]); s->ds[i] = (uint32_t)(st->d[i + 1] - st->d[i]); }
    return s;
}
extern "C" void zk_serializer_free(zk_serializer* s) { delete s; }
extern "C" size_t zk_serializer_write_into(zk_serializer* s, uint8_t* buf, size_t len) {           // :967-1005
    size_t total = s->encoded_len(), n = 0;
    while (n < len && s->write_pos < total) buf[n++] = s->byte_at(s->write_pos++);
    return n;
}
extern "C" void zk_serializer_reset(zk_serializer* s) { s->write_pos = 0; }                        // :1021
extern "C" size_t zk_serializer_encoded_len(const zk_serializer* s) { return s->encoded_len(); }    // :1038

// ================================================================================================ encode
struct zk_encode_options {                 // encode.rs:110-207
    zk_ctx* ctx; zk_frame_size_policy kind = ZK_POLICY_UNCOMPRESSED; uint32_t size = ZK_DEFAULT_FRAME_SIZE;
    int32_t checksum = 0; int32_t level = 0;           // CompressionLevel::default() == 0 -> codec default
    int32_t ldm = 0;                                   // long-distance matching against the prefix of compress_with_prefix
    int32_t lmode = 0;                                 // long mode: frames also match their own bytes up to 2^27 back (zk_compress_frames_long)
};
extern "C" zk_encode_options* zk_encode_options_new(zk_ctx* ctx) {
    if (!ctx) return nullptr;
    zk_encode_options* o = new (std::nothrow) zk_encode_options(); if (o) o->ctx = ctx; return o;
}
extern "C" void zk_encode_options_free(zk_encode_options* o) { delete o; }
extern "C" void zk_encode_options_frame_size_policy(zk_encode_options* o, zk_frame_size_policy kind, uint32_t size) { o->kind = kind; o->size = size; }
extern "C" void zk_encode_options_checksum_flag(zk_encode_options* o, int32_t flag) { o->checksum = flag ? 1 : 0; }
extern "C" void zk_encode_options_compression_level(zk_encode_options* o, int32_t level) { o->level = level; }
extern "C" void zk_encode_options_long_distance_matching(zk_encode_options* o, int32_t flag) { o->ldm = flag ? 1 : 0; }
extern "C" void zk_encode_options_long_mode(zk_encode_options* o, int32_t flag) { o->lmode = flag ? 1 : 0; }

struct zk_raw_encoder {                    // encode.rs:266-545
    zk_ctx* ctx; zk_frame_size_policy kind; uint32_t size; int32_t checksum, level, ldm = 0, lmode = 0;
    uint32_t frame_c_size = 0, frame_d_size = 0;
    zk_seek_table seek_table;
    std::vector<uint8_t> in_buf;           // uncompressed bytes of the frame being built (whole frames go to the GPU)
    std::vector<uint8_t> out_buf;          // the frame's compressed bytes once produced
    size_t out_pos = 0; bool compressed = false;
    uint64_t next_trial = 0;               // Compressed(n) policy: input size at which the next trial compression runs
    const uint8_t* prefix = nullptr; size_t prefix_len = 0;   // raw-content prefix of the frame being built (encode.rs:332-338: taken at the frame's first compress call)

    uint32_t uncompressed_limit() const { return kind == ZK_POLICY_UNCOMPRESSED ? std::min(kMaxFrameSize, size) : kMaxFrameSize; }
    size_t remaining_frame_size() const { return uncompressed_limit() - frame_d_size; }             // :528-535
    bool is_frame_complete() const {                                                                 // :537-544
        if (kind == ZK_POLICY_COMPRESSED) return size <= frame_c_size_estimate() || kMaxFrameSize <= frame_d_size;
        return std::min(kMaxFrameSize, size) <= frame_d_size;
    }
    // For FrameSizePolicy::Compressed the reference watches the bytes libzstd has emitted so far.  A batch codec
    // emits nothing before the frame is closed, so progress is estimated by trial-compressing the buffered input.
    uint32_t est_c = 0;
    uint32_t frame_c_size_estimate() const { return compressed ? (uint32_t)out_buf.size() : est_c; }

    int32_t run_codec() {                  // in_buf -> out_buf, one frame
        size_t cap = zk_compress_bound(in_buf.size(), (uint32_t)std::max<size_t>(in_buf.size(), 1));
        out_buf.resize(cap);
        uint32_t cs = 0, ds = 0, nf = 0; size_t len = 0;
        static const uint8_t dummy = 0;
        int32_t rc = (lmode ? zk_compress_frames_long : ldm ? zk_compress_frames_ldm : zk_compress_frames_prefix)(ctx, in_buf.empty() ? &dummy : in_buf.data(), in_buf.size(),
                                               (uint32_t)std::max<size_t>(in_buf.size(), 1), level, checksum, prefix, prefix_len, out_buf.data(), cap, &cs, &ds, 1, &nf, &len);
        if (rc) return rc;
        out_buf.resize(len);
        return 0;
    }
    void reset_frame() { frame_c_size = 0; frame_d_size = 0; in_buf.clear(); out_buf.clear(); out_pos = 0; compressed = false; est_c = 0; next_trial = 0; prefix = nullptr; prefix_len = 0; }
};

extern "C" int32_t zk_encode_options_into_raw_encoder(zk_encode_options* o, zk_raw_encoder** out) {
    if (!o || !out) return ZK_ERR_INVALID_ARG;
    // content-defined frames end where a hash of later bytes says so, and there is no CPU path to hash on: a RawEncoder could not report
    // its progress before the end is known
    if (o->kind == ZK_POLICY_CONTENT) return ZK_ERR_INVALID_ARG;
    zk_raw_encoder* e = new (std::nothrow) zk_raw_encoder();
    if (!e) return ZK_ERR_ZSTD(64);
    e->ctx = o->ctx; e->kind = o->kind; e->size = o->size; e->checksum = o->checksum; e->level = o->level; e->ldm = o->ldm; e->lmode = o->lmode;
    delete o;
    *out = e;
    return 0;
}
extern "C" void zk_raw_encoder_free(zk_raw_encoder* e) { delete e; }

extern "C" int32_t zk_raw_encoder_end_frame(zk_raw_encoder* e, uint8_t* output, size_t out_len, zk_epilogue_progress* prog) {   // :438-472
    if (!e->compressed) {
        int32_t rc = e->run_codec();
        if (rc) return rc;
        e->compressed = true; e->out_pos = 0;
    }
    size_t left = e->out_buf.size() - e->out_pos;
    size_t n = std::min(left, out_len);
    if (n) memcpy(output, e->out_buf.data() + e->out_pos, n);
    e->out_pos += n; e->frame_c_size += (uint32_t)n;
    left -= n;
    if (left > 0) { if (prog) { prog->out_progress = n; prog->data_left = left; } return 0; }       // more buffer space required
    int32_t rc = zk_seek_table_log_frame(&e->seek_table, e->frame_c_size, e->frame_d_size);          // :466
    if (rc) return rc;
    e->reset_frame();
    if (prog) { prog->out_progress = n; prog->data_left = 0; }
    return 0;
}

extern "C" int32_t zk_raw_encoder_compress(zk_raw_encoder* e, const uint8_t* input, size_t in_len, uint8_t* output, size_t out_len,
                                           zk_compression_progress* prog) {                          // :398
    return zk_raw_encoder_compress_with_prefix(e, input, in_len, output, out_len, nullptr, 0, prog);
}

extern "C" int32_t zk_raw_encoder_compress_with_prefix(zk_raw_encoder* e, const uint8_t* input, size_t in_len, uint8_t* output, size_t out_len,
                                                       const uint8_t* prefix, size_t prefix_len, zk_compression_progress* prog) {   // :311-354
    if (e->is_frame_complete()) {                                                                    // :317-327
        size_t out_progress = 0;
        while (out_progress < out_len) {
            zk_epilogue_progress ep{};
            int32_t rc = zk_raw_encoder_end_frame(e, output + out_progress, out_len - out_progress, &ep);
            if (rc) return rc;
            out_progress += ep.out_progress;
            if (ep.data_left == 0) break;
        }
        if (prog) { prog->in_progress = 0; prog->out_progress = out_progress; }
        return 0;
    }
    size_t limit = std::min(in_len, e->remaining_frame_size());                                      // :329
    if (prefix && e->frame_d_size == 0) { e->prefix = prefix; e->prefix_len = prefix_len; }         // :332-338: referenced at the beginning of a frame
    e->in_buf.insert(e->in_buf.end(), input, input + limit);
    e->frame_d_size += (uint32_t)limit;
    if (e->kind == ZK_POLICY_COMPRESSED && e->frame_d_size >= e->size && e->frame_d_size >= e->next_trial) {
        int32_t rc = e->run_codec();
        if (rc) return rc;
        e->est_c = (uint32_t)e->out_buf.size();
        if (e->est_c >= e->size) { e->compressed = true; e->out_pos = 0; }                           // closes on the next call
        else {   // predict where the compressed size reaches the target
            uint64_t d = e->frame_d_size, c = std::max<uint32_t>(e->est_c, 1);
            e->next_trial = std::max<uint64_t>(d + 1, d * e->size / c);
            e->out_buf.clear();
        }
    }
    if (prog) { prog->in_progress = limit; prog->out_progress = 0; }
    return 0;
}

extern "C" const zk_seek_table* zk_raw_encoder_seek_table(const zk_raw_encoder* e) { return &e->seek_table; }
extern "C" zk_seek_table* zk_raw_encoder_into_seek_table(zk_raw_encoder* e) {
    zk_seek_table* st = new (std::nothrow) zk_seek_table(e->seek_table);
    delete e;
    return st;
}
extern "C" void zk_raw_encoder_reset_frame(zk_raw_encoder* e) { e->reset_frame(); }
extern "C" void zk_raw_encoder_reset_seek_table(zk_raw_encoder* e) { e->seek_table = zk_seek_table(); }

// ---- Encoder<W: Write> (encode.rs:568-800) -----------------------------------------------------------------
// Input is buffered and handed to the GPU in batches (the sink is owned by the encoder, so delaying writes is invisible to
// the caller).  Uncompressed(n) batches whole frames; Compressed(n) and ContentDefined(n) hand the buffer to zk_compress_frames_csize /
// zk_compress_frames_cdc, which close frames by the rule of that entry point and leave the open frame in the buffer.
struct zk_encoder {
    zk_raw_encoder raw;
    zk_write_fn write; zk_flush_fn flush; void* user;
    uint64_t written_compressed = 0;
    std::vector<uint8_t> batch;            // complete + partial frames not yet compressed (Uncompressed policy)
    std::vector<uint8_t> stage;
    size_t batch_frames = 8192;            // a GPU call takes the buffered complete frames once there are this many ...
    size_t batch_bytes = (size_t)128 << 20; // ... or this many bytes of them (64 frames of 2 MiB; thousands of small ones: one launch sequence serves them all)
    const uint8_t* prefix = nullptr; size_t prefix_len = 0;   // prefix of the frames in `batch` (compress_with_prefix)
    size_t csize_at = (size_t)128 << 20;   // Compressed(n), ContentDefined(n): buffered bytes at which the next cut runs (doubles while a cut closes no frame)

    int32_t sink(const uint8_t* p, size_t n) {
        if (!n) return 0;
        if (write(user, p, n) != 0) return ZK_ERR_IO;
        written_compressed += n;
        return 0;
    }
    uint32_t frame_limit() const { return std::min(kMaxFrameSize, raw.size); }
    // compress `count` bytes from the front of `batch` (all complete frames, or the final partial one)
    int32_t flush_batch(size_t count, size_t* written, bool allow_empty) {
        if (count == 0 && !allow_empty) { if (written) *written = 0; return 0; }
        const uint32_t fs = frame_limit();
        size_t cap = zk_compress_bound(count, fs);
        stage.resize(cap);
        uint32_t nfmax = (uint32_t)(count / fs + 2);
        std::vector<uint32_t> cs(nfmax), ds(nfmax);
        uint32_t nf = 0; size_t len = 0;
        static const uint8_t dummy = 0;
        int32_t rc = (raw.lmode ? zk_compress_frames_long : raw.ldm ? zk_compress_frames_ldm : zk_compress_frames_prefix)(raw.ctx, count ? batch.data() : &dummy, count, fs, raw.level, raw.checksum,
                                               prefix, prefix_len, stage.data(), cap, cs.data(), ds.data(), nfmax, &nf, &len);
        if (rc) return rc;
        for (uint32_t i = 0; i < nf; i++) { rc = zk_seek_table_log_frame(&raw.seek_table, cs[i], ds[i]); if (rc) return rc; }
        rc = sink(stage.data(), len);
        if (rc) return rc;
        batch.erase(batch.begin(), batch.begin() + (ptrdiff_t)count);
        if (written) *written = len;
        return 0;
    }
    bool cuts_on_gpu() const { return raw.kind == ZK_POLICY_COMPRESSED || raw.kind == ZK_POLICY_CONTENT; }
    // Compressed(n), ContentDefined(n): every frame of `batch` that closes (all of them with final_), in one batch call.  Every frame but
    // the last has at least min_frame bytes.
    int32_t flush_csize(int32_t final_, size_t* written) {
        const bool cdc = raw.kind == ZK_POLICY_CONTENT;
        const size_t count = batch.size(), min_frame = cdc ? 1024 : 32768;
        size_t cap = zk_compress_bound(count, (uint32_t)min_frame);
        stage.resize(cap);
        uint32_t nfmax = (uint32_t)(count / min_frame + 2);
        std::vector<uint32_t> cs(nfmax), ds(nfmax);
        uint32_t nf = 0; size_t len = 0, used = 0;
        static const uint8_t dummy = 0;
        int32_t rc = (cdc ? zk_compress_frames_cdc : zk_compress_frames_csize)(raw.ctx, count ? batch.data() : &dummy, count, raw.size, raw.level, raw.checksum, prefix, prefix_len, final_,
                                              stage.data(), cap, cs.data(), ds.data(), nfmax, &nf, &len, &used);
        if (rc) return rc;
        for (uint32_t i = 0; i < nf; i++) { rc = zk_seek_table_log_frame(&raw.seek_table, cs[i], ds[i]); if (rc) return rc; }
        rc = sink(stage.data(), len);
        if (rc) return rc;
        batch.erase(batch.begin(), batch.begin() + (ptrdiff_t)used);
        csize_at = nf || final_ ? batch_bytes : 2 * count;
        if (written) *written = len;
        return 0;
    }
};

extern "C" int32_t zk_encode_options_into_encoder(zk_encode_options* o, zk_write_fn write, zk_flush_fn flush, void* user, zk_encoder** out) {
    if (!o || !out || !write) return ZK_ERR_INVALID_ARG;
    // the exact cut of Compressed(n) needs a bounded history per block, which the tier that matches over long distances does not have;
    // content-defined frames are meant to stand alone
    if ((o->kind == ZK_POLICY_COMPRESSED || o->kind == ZK_POLICY_CONTENT) && (o->ldm || o->lmode)) return ZK_ERR_INVALID_ARG;
    zk_encoder* e = new (std::nothrow) zk_encoder();
    if (!e) return ZK_ERR_ZSTD(64);
    e->raw.ctx = o->ctx; e->raw.kind = o->kind; e->raw.size = o->size; e->raw.checksum = o->checksum; e->raw.level = o->level; e->raw.ldm = o->ldm; e->raw.lmode = o->lmode;
    e->write = write; e->flush = flush; e->user = user;
    const char* bf = getenv("ZK_ENCODER_BATCH_FRAMES");
    if (bf && atoi(bf) > 0) e->batch_frames = (size_t)atoi(bf);
    delete o;
    *out = e;
    return 0;
}
extern "C" void zk_encoder_free(zk_encoder* e) { delete e; }
extern "C" uint64_t zk_encoder_written_compressed(const zk_encoder* e) { return e->written_compressed; }
extern "C" const zk_seek_table* zk_encoder_seek_table(const zk_encoder* e) { return &e->raw.seek_table; }

extern "C" int32_t zk_encoder_compress(zk_encoder* e, const uint8_t* buf, size_t len, size_t* consumed) {     // :692
    return zk_encoder_compress_with_prefix(e, buf, len, nullptr, 0, consumed);
}

extern "C" int32_t zk_encoder_compress_with_prefix(zk_encoder* e, const uint8_t* buf, size_t len, const uint8_t* prefix, size_t prefix_len,
                                                   size_t* consumed) {                                         // :641-665
    if (prefix != e->prefix || prefix_len != e->prefix_len) {
        // the batch buffer holds frames of ONE prefix: close what was buffered under the previous one first (whole frames only;
        // a partial frame keeps the prefix it started with, as in the reference)
        if (!e->cuts_on_gpu() && !e->batch.empty()) {
            const uint32_t fs0 = e->frame_limit();
            const size_t whole = fs0 ? (e->batch.size() / fs0) * fs0 : 0;
            if (whole && whole == e->batch.size()) { int32_t rc = e->flush_batch(whole, nullptr, false); if (rc) return rc; }
        }
        if (e->batch.empty()) { e->prefix = prefix; e->prefix_len = prefix_len; }
    }
    if (e->cuts_on_gpu()) {
        e->batch.insert(e->batch.end(), buf, buf + len);
        if (e->batch.size() >= e->csize_at) { int32_t rc = e->flush_csize(0, nullptr); if (rc) return rc; }
        if (consumed) *consumed = len;
        return 0;
    }
    const uint32_t fs = e->frame_limit();
    if (fs == 0) { if (consumed) *consumed = 0; return 0; }
    e->batch.insert(e->batch.end(), buf, buf + len);
    // A frame that filled exactly is only closed lazily at the next compress()/finish() (encode.rs:317-327): keep the
    // last complete frame in the buffer unless more input follows it.
    size_t complete = e->batch.size() / fs;
    if (complete && e->batch.size() % fs == 0) complete--;
    if (complete >= e->batch_frames || (complete && complete * (size_t)fs >= e->batch_bytes)) { int32_t rc = e->flush_batch(complete * fs, nullptr, false); if (rc) return rc; }
    if (consumed) *consumed = len;
    return 0;
}

extern "C" int32_t zk_encoder_end_frame(zk_encoder* e, size_t* written) {                                      // :704-717
    if (e->cuts_on_gpu()) return e->flush_csize(1, written);
    // everything buffered becomes frames; the last one may be short (or empty: end_frame on a fresh frame emits an
    // empty frame, exactly what the reference's finish() does on an empty stream)
    return e->flush_batch(e->batch.size(), written, true);
}

extern "C" int32_t zk_encoder_flush(zk_encoder* e) { return e->flush ? (e->flush(e->user) == 0 ? 0 : ZK_ERR_IO) : 0; }   // impl Write::flush

extern "C" int32_t zk_encoder_finish_format(zk_encoder* e, zk_format format, uint64_t* total) {                // :755-775
    size_t w = 0;
    int32_t rc = zk_encoder_end_frame(e, &w);
    if (!rc) {
        zk_serializer* ser = zk_seek_table_into_serializer(&e->raw.seek_table, format);
        if (!ser) rc = ZK_ERR_ZSTD(64);
        else {
            uint8_t tmp[4096];
            for (;;) { size_t n = zk_serializer_write_into(ser, tmp, sizeof tmp); if (!n) break; rc = e->sink(tmp, n); if (rc) break; }
            zk_serializer_free(ser);
        }
    }
    if (!rc) rc = zk_encoder_flush(e);
    if (total) *total = e->written_compressed;
    delete e;
    return rc;
}
extern "C" int32_t zk_encoder_finish(zk_encoder* e, uint64_t* total) { return zk_encoder_finish_format(e, ZK_FORMAT_FOOT, total); }   // :743

// ================================================================================================ decode
struct zk_decode_options {                 // decode.rs:13-114
    zk_ctx* ctx; Source src;
    zk_seek_table* seek_table = nullptr;
    bool has_lower = false, has_upper = false, has_offset = false, has_limit = false;
    uint32_t lower = 0, upper = 0; uint64_t offset = 0, limit = 0;
    ~zk_decode_options() { delete seek_table; }
};
extern "C" zk_decode_options* zk_decode_options_new_bytes(zk_ctx* ctx, const uint8_t* src, size_t len) {
    if (!ctx) return nullptr;
    zk_decode_options* o = new (std::nothrow) zk_decode_options(); if (!o) return nullptr;
    o->ctx = ctx; o->src.is_bytes = true; o->src.bytes = src; o->src.len = len;
    return o;
}
extern "C" zk_decode_options* zk_decode_options_new_seekable(zk_ctx* ctx, zk_seekable src) {
    if (!ctx || !src.read || !src.set_offset) return nullptr;
    zk_decode_options* o = new (std::nothrow) zk_decode_options(); if (!o) return nullptr;
    o->ctx = ctx; o->src.cb = src;
    return o;
}
extern "C" void zk_decode_options_free(zk_decode_options* o) { delete o; }
extern "C" void zk_decode_options_seek_table(zk_decode_options* o, const zk_seek_table* st) { delete o->seek_table; o->seek_table = new zk_seek_table(*st); }
extern "C" void zk_decode_options_lower_frame(zk_decode_options* o, uint32_t i) { o->has_lower = true; o->lower = i; }
extern "C" void zk_decode_options_upper_frame(zk_decode_options* o, uint32_t i) { o->has_upper = true; o->upper = i; }
extern "C" void zk_decode_options_offset(zk_decode_options* o, uint64_t v) { o->has_offset = true; o->offset = v; }
extern "C" void zk_decode_options_offset_limit(zk_decode_options* o, uint64_t v) { o->has_limit = true; o->limit = v; }

struct zk_decoder {                        // decode.rs:121-466
    zk_ctx* ctx; Source src; zk_seek_table seek_table;
    uint64_t offset = 0, offset_limit = 0, read_compressed = 0;
    // decoded window: frames [win_lo, win_hi) live in `window` (whole frames; forward seeks inside it cost nothing,
    // mirroring "no reset when seeking forward in the same frame", decode.rs:407-410)
    uint32_t win_lo = 0, win_hi = 0; std::vector<uint8_t> window; std::vector<uint8_t> comp;
    uint64_t win_valid_end = 0;            // the window is decoded up to this decompressed offset (< d[win_hi] after a range read)
    size_t max_window_bytes = (size_t)256 << 20;
    const uint8_t* prefix = nullptr; size_t prefix_len = 0;   // the prefix the window was decoded with (decompress_with_prefix)
    const uint64_t* ranges = nullptr;                          // and every entry's range of it (nullptr: the whole prefix)
    bool archive = false;                                      // the prefix is OLD of this reference chain instead (a copy of its
    std::vector<zk_reference_archive> chain;                   // descriptors, root first)

    void reset_dctx() { read_compressed = 0; win_lo = win_hi = 0; win_valid_end = 0; window.clear(); }                           // :352-357
    int32_t check_offset(uint64_t off) const { return off > seek_table.d.back() ? ZK_ERR_OFFSET_OUT_OF_RANGE : 0; }   // :439-445

    // make frames [f0, f1) resident; need_end < d[f1]: the last frame only as far as need_end (a range read stops at
    // offset_limit, decode.rs:228-266 -- the codec then stops at the next block boundary)
    int32_t load(uint32_t f0, uint32_t f1, uint64_t need_end) {
        const uint64_t c0 = seek_table.c[f0], c1 = seek_table.c[f1], d0 = seek_table.d[f0], d1 = seek_table.d[f1];
        comp.resize((size_t)(c1 - c0) + 64);
        int32_t rc = src.set_offset(0, (int64_t)c0);
        if (rc) return rc;
        size_t got = 0, want = (size_t)(c1 - c0);
        while (got < want) {
            int64_t r = src.read(comp.data() + got, want - got);
            if (r < 0) return (int32_t)r;
            if (r == 0) return ZK_ERR_ZSTD(72);                    // srcSize_wrong: archive shorter than its seek table says
            got += (size_t)r;
        }
        read_compressed += want;
        window.resize((size_t)(d1 - d0) + 64);
        const uint32_t n = f1 - f0;
        std::vector<uint64_t> co(n + 1), dof(n + 1);
        for (uint32_t i = 0; i <= n; i++) { co[i] = seek_table.c[f0 + i] - c0; dof[i] = seek_table.d[f0 + i] - d0; }
        std::vector<uint32_t> need;
        if (need_end < d1 && need_end > seek_table.d[f1 - 1]) {
            need.assign(n, 0xFFFFFFFFu);
            need[n - 1] = (uint32_t)(need_end - seek_table.d[f1 - 1]);
        } else need_end = d1;
        const uint32_t* np = need.empty() ? nullptr : need.data();
        const uint64_t* rg = ranges ? ranges + 2 * (size_t)f0 : nullptr;
        rc = archive ? zk_decompress_frames_prefixes_chain(ctx, comp.data(), co.data(), dof.data(), n, window.data(), np, 1, nullptr, chain.data(),
                                                           (uint32_t)chain.size(), rg)
                     : zk_decompress_frames_prefixes(ctx, comp.data(), co.data(), dof.data(), n, window.data(), np, 1, nullptr, prefix, prefix_len, rg);
        if (rc) { win_lo = win_hi = 0; win_valid_end = 0; return rc; }
        win_lo = f0; win_hi = f1; win_valid_end = need_end;
        return 0;
    }
};

extern "C" int32_t zk_decode_options_into_decoder(zk_decode_options* o, zk_decoder** out) {                    // :111, 152-187
    if (!o || !out) return ZK_ERR_INVALID_ARG;
    zk_decoder* d = new (std::nothrow) zk_decoder();
    if (!d) { delete o; return ZK_ERR_ZSTD(64); }
    d->ctx = o->ctx; d->src = o->src;
    int32_t rc = 0;
    if (o->seek_table) d->seek_table = *o->seek_table;
    else { zk_seek_table* st = nullptr; rc = seek_table_from_source(d->src, ZK_FORMAT_FOOT, &st); if (!rc) { d->seek_table = *st; delete st; } }
    uint64_t offset = 0, limit = 0;
    if (!rc) {
        if (o->has_lower) rc = zk_seek_table_frame_start_decomp(&d->seek_table, o->lower, &offset);
        else offset = o->has_offset ? o->offset : 0;
    }
    if (!rc) rc = d->check_offset(offset);
    if (!rc) {
        if (o->has_upper) rc = zk_seek_table_frame_end_decomp(&d->seek_table, o->upper, &limit);
        else limit = o->has_limit ? o->limit : d->seek_table.d.back();
    }
    if (!rc) rc = d->check_offset(limit);
    delete o;
    if (rc) { delete d; return rc; }
    d->offset = offset; d->offset_limit = limit;
    const char* mw = getenv("ZK_DECODER_WINDOW_BYTES");
    if (mw && atoll(mw) > 0) d->max_window_bytes = (size_t)atoll(mw);
    *out = d;
    return 0;
}
extern "C" void zk_decoder_free(zk_decoder* d) { delete d; }

extern "C" int32_t zk_decoder_decompress(zk_decoder* d, uint8_t* buf, size_t len, size_t* produced) {           // :314
    return zk_decoder_decompress_with_prefix(d, buf, len, nullptr, 0, produced);
}

extern "C" int32_t zk_decoder_decompress_with_prefix(zk_decoder* d, uint8_t* buf, size_t len, const uint8_t* prefix, size_t prefix_len,
                                                     size_t* produced) {                                        // :201-270
    return zk_decoder_decompress_with_prefix_ranges(d, buf, len, prefix, prefix_len, nullptr, produced);
}

static int32_t zk_decoder_run(zk_decoder* d, uint8_t* buf, size_t len, size_t* produced);

extern "C" int32_t zk_decoder_decompress_with_prefix_ranges(zk_decoder* d, uint8_t* buf, size_t len, const uint8_t* prefix, size_t prefix_len,
                                                            const uint64_t* ranges, size_t* produced) {
    if (d->archive || prefix != d->prefix || prefix_len != d->prefix_len || ranges != d->ranges) {   // frames decoded under another prefix are not reusable
        d->win_lo = d->win_hi = 0; d->win_valid_end = 0;
        d->prefix = prefix; d->prefix_len = prefix_len; d->ranges = ranges; d->archive = false;
    }
    return zk_decoder_run(d, buf, len, produced);
}

extern "C" int32_t zk_decoder_decompress_with_reference_archive(zk_decoder* d, uint8_t* buf, size_t len, const uint8_t* ref_comp, size_t ref_len,
                                                                const uint64_t* ref_c_off, const uint64_t* ref_d_off, uint32_t ref_n,
                                                                const uint64_t* ranges, size_t* produced) {
    const zk_reference_archive r = {ref_comp, ref_len, ref_c_off, ref_d_off, ref_n};
    return zk_decoder_decompress_with_reference_chain(d, buf, len, &r, 1, ranges, produced);
}

// the window stays valid while the ranges and every level's descriptor are the ones it was decoded with
extern "C" int32_t zk_decoder_decompress_with_reference_chain(zk_decoder* d, uint8_t* buf, size_t len, const zk_reference_archive* chain, uint32_t depth,
                                                              const uint64_t* ranges, size_t* produced) {
    if (!chain || depth == 0 || depth > ZK_CHAIN_MAX_DEPTH) return ZK_ERR_INVALID_ARG;
    bool same = d->archive && ranges == d->ranges && depth == d->chain.size();
    for (uint32_t i = 0; same && i < depth; i++) {
        const zk_reference_archive &a = chain[i], &b = d->chain[i];
        same = a.comp == b.comp && a.len == b.len && a.c_off == b.c_off && a.d_off == b.d_off && a.n == b.n;
    }
    if (!same) {
        d->win_lo = d->win_hi = 0; d->win_valid_end = 0;
        d->prefix = nullptr; d->prefix_len = 0; d->ranges = ranges; d->archive = true;
        d->chain.assign(chain, chain + depth);
    }
    return zk_decoder_run(d, buf, len, produced);
}

// decode.rs:201-270 with the prefix the decoder holds
static int32_t zk_decoder_run(zk_decoder* d, uint8_t* buf, size_t len, size_t* produced) {
    size_t progress = 0;
    const uint32_t nframes = d->seek_table.num_frames();
    while (d->offset < d->offset_limit && progress < len && nframes) {
        const uint32_t f = d->seek_table.index_at(d->offset, d->seek_table.d);
        if (!(f >= d->win_lo && f < d->win_hi) || d->offset >= d->win_valid_end) {
            // decode the frames covering the rest of this request in one batch (bounded)
            const uint64_t want_end = std::min<uint64_t>(d->offset_limit, d->offset + (len - progress));
            uint32_t f1 = d->seek_table.index_at(want_end ? want_end - 1 : 0, d->seek_table.d) + 1;
            if (f1 <= f) f1 = f + 1;
            while (f1 > f + 1 && d->seek_table.d[f1] - d->seek_table.d[f] > d->max_window_bytes) f1--;
            int32_t rc = d->load(f, f1, d->offset_limit);
            if (rc) { if (produced) *produced = progress; return rc; }
        }
        const uint64_t w0 = d->seek_table.d[d->win_lo], w1 = d->seek_table.d[d->win_hi];
        const uint64_t end = std::min<uint64_t>(std::min<uint64_t>(d->offset_limit, std::min<uint64_t>(w1, d->win_valid_end)), d->offset + (len - progress));
        if (end <= d->offset) break;                                   // empty frames only
        const size_t n = (size_t)(end - d->offset);
        memcpy(buf + progress, d->window.data() + (size_t)(d->offset - w0), n);
        d->offset += n; progress += n;
    }
    if (produced) *produced = progress;
    return 0;
}

extern "C" void zk_decoder_reset(zk_decoder* d) { d->reset_dctx(); d->offset = 0; d->offset_limit = d->seek_table.d.back(); }   // :346-350

extern "C" int32_t zk_decoder_set_offset(zk_decoder* d, uint64_t offset) {                                       // :402-414
    int32_t rc = d->check_offset(offset);
    if (rc) return rc;
    const uint32_t cur = d->seek_table.index_at(d->offset, d->seek_table.d), tgt = d->seek_table.index_at(offset, d->seek_table.d);
    if (cur != tgt || offset < d->offset) d->reset_dctx();
    d->offset = offset;
    return 0;
}
extern "C" int32_t zk_decoder_set_offset_limit(zk_decoder* d, uint64_t limit) {                                  // :432-437
    int32_t rc = d->check_offset(limit);
    if (rc) return rc;
    d->offset_limit = limit;
    return 0;
}
extern "C" int32_t zk_decoder_set_lower_frame(zk_decoder* d, uint32_t index, uint64_t* offset) {                 // :367-371
    uint64_t off; int32_t rc = zk_seek_table_frame_start_decomp(&d->seek_table, index, &off);
    if (rc) return rc;
    rc = zk_decoder_set_offset(d, off);
    if (!rc && offset) *offset = off;
    return rc;
}
extern "C" int32_t zk_decoder_set_upper_frame(zk_decoder* d, uint32_t index, uint64_t* offset) {                 // :383-387
    uint64_t off; int32_t rc = zk_seek_table_frame_end_decomp(&d->seek_table, index, &off);
    if (rc) return rc;
    rc = zk_decoder_set_offset_limit(d, off);
    if (!rc && offset) *offset = off;
    return rc;
}
extern "C" uint64_t zk_decoder_read_compressed(const zk_decoder* d) { return d->read_compressed; }
extern "C" uint64_t zk_decoder_offset(const zk_decoder* d) { return d->offset; }
extern "C" uint64_t zk_decoder_offset_limit(const zk_decoder* d) { return d->offset_limit; }
extern "C" const zk_seek_table* zk_decoder_seek_table(const zk_decoder* d) { return &d->seek_table; }

extern "C" int32_t zk_decoder_seek(zk_decoder* d, int32_t whence, int64_t n, uint64_t* new_offset) {             // decode.rs:545-579
    uint64_t off;
    if (whence == 0) { if (n < 0) return ZK_ERR_OFFSET_OUT_OF_RANGE; off = (uint64_t)n; }
    else if (whence == 1) {
        if (n > 0) return ZK_ERR_OFFSET_OUT_OF_RANGE;
        uint64_t size = d->seek_table.d.back(), back = (uint64_t)(-n);
        if (back > size) return ZK_ERR_OFFSET_OUT_OF_RANGE;
        off = size - back;
    } else if (whence == 2) {
        if (n < 0) { uint64_t back = (uint64_t)(-n); if (back > d->offset) return ZK_ERR_OFFSET_OUT_OF_RANGE; off = d->offset - back; }
        else { off = d->offset + (uint64_t)n; if (off < d->offset) return ZK_ERR_OFFSET_OUT_OF_RANGE; }
    } else return ZK_ERR_INVALID_ARG;
    int32_t rc = zk_decoder_set_offset(d, off);
    if (!rc && new_offset) *new_offset = off;
    return rc;
}
