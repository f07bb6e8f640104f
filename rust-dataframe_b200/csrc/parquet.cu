// parquet.cu -- the host half of the Parquet reader: files and directories, the Thrift compact-protocol footer, the column types,
// and the page-header walk of every on-path column chunk; bdf_parquet_open / _describe / _column / _temporal_column / _check /
// _stats / _close, and the read plan runtime.cu's bdf_parquet_read uploads and decodes (k_parquet.cu).  No GPU is needed here.
// At the end, the writer's half: the page headers and the footer bdf_parquet_write (runtime.cu) serialises.
// The rules are in include/b200df.h ("Parquet files straight to the device").
#include <algorithm>
#include <cerrno>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <dirent.h>
#include <fcntl.h>
#include <new>
#include <string>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <vector>

#include "../../include/b200df.h"
#define PQ_HOST_PLAN
#include "parquet_decode.cuh"
#define PQ_HOST_WRITE
#include "parquet_encode.cuh"

#include "ipc_schema.cuh"

namespace bdf { int set_error(int status, const char* msg); }

namespace {

int pq_fail(int status, const char* fmt, ...) {
    char buf[768];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    return bdf::set_error(status, buf);
}

const char* codec_name(int c) {
    static const char* n[] = {"UNCOMPRESSED", "SNAPPY", "GZIP", "LZO", "BROTLI", "LZ4", "ZSTD", "LZ4_RAW"};
    return c >= 0 && c < 8 ? n[c] : "an unknown codec";
}
const char* encoding_name(int e) {
    static const char* n[] = {"PLAIN", "GROUP_VAR_INT", "PLAIN_DICTIONARY", "RLE", "BIT_PACKED", "DELTA_BINARY_PACKED",
                              "DELTA_LENGTH_BYTE_ARRAY", "DELTA_BYTE_ARRAY", "RLE_DICTIONARY", "BYTE_STREAM_SPLIT"};
    return e >= 0 && e < 10 ? n[e] : "an unknown encoding";
}

// ---- Thrift compact protocol (bounds-checked; a malformed byte sequence sets ok = false and every later read returns 0) ----------
enum { TC_STOP = 0, TC_TRUE = 1, TC_FALSE = 2, TC_BYTE = 3, TC_I16 = 4, TC_I32 = 5, TC_I64 = 6, TC_DOUBLE = 7, TC_BINARY = 8, TC_LIST = 9,
       TC_SET = 10, TC_MAP = 11, TC_STRUCT = 12 };
constexpr int kMaxDepth = 32;

struct Thrift {
    const uint8_t* p;
    size_t n, pos = 0;
    bool ok = true;
    int depth = 0;
    uint64_t varint() {
        uint64_t v = 0;
        for (int s = 0; s < 64; s += 7) {
            if (pos >= n) { ok = false; return 0; }
            const uint8_t b = p[pos++];
            v |= (uint64_t)(b & 0x7f) << s;
            if (!(b & 0x80)) return v;
        }
        ok = false;
        return 0;
    }
    int64_t zz() { const uint64_t v = varint(); return (int64_t)(v >> 1) ^ -(int64_t)(v & 1); }
    uint8_t byte() { if (pos >= n) { ok = false; return 0; } return p[pos++]; }
    std::string binary() {
        const uint64_t len = varint();
        if (!ok || len > n - pos) { ok = false; return std::string(); }
        std::string s((const char*)p + pos, (size_t)len);
        pos += (size_t)len;
        return s;
    }
    // A field header: false at STOP (or on error).  bool fields carry their value in the type.
    bool field(int16_t* id, int* type, int16_t* last) {
        const uint8_t b = byte();
        if (!ok || b == 0) return false;
        *type = b & 0x0f;
        const int delta = b >> 4;
        *id = delta ? (int16_t)(*last + delta) : (int16_t)zz();
        *last = *id;
        return ok;
    }
    void list(int* elem, uint32_t* count) {
        const uint8_t b = byte();
        *elem = b & 0x0f;
        uint64_t c = b >> 4;
        if (c == 15) c = varint();
        if (c > n) ok = false;   // every element takes at least one byte ... except bools in a list: still one byte each
        *count = (uint32_t)c;
    }
    void skip(int type) {
        if (!ok) return;
        switch (type) {
            case TC_TRUE: case TC_FALSE: break;
            case TC_BYTE: byte(); break;
            case TC_I16: case TC_I32: case TC_I64: varint(); break;
            case TC_DOUBLE: if (n - pos < 8) ok = false; else pos += 8; break;
            case TC_BINARY: binary(); break;
            case TC_LIST: case TC_SET: {
                int et; uint32_t c;
                list(&et, &c);
                if (++depth > kMaxDepth) { ok = false; return; }
                for (uint32_t i = 0; i < c && ok; i++) skip(et == TC_TRUE || et == TC_FALSE ? TC_BYTE : et);
                depth--;
                break;
            }
            case TC_MAP: {
                const uint64_t c = varint();
                if (c > n) { ok = false; return; }
                if (!c) break;
                const uint8_t kv = byte();
                if (++depth > kMaxDepth) { ok = false; return; }
                for (uint64_t i = 0; i < c && ok; i++) { skip(kv >> 4); skip(kv & 0x0f); }
                depth--;
                break;
            }
            case TC_STRUCT: {
                if (++depth > kMaxDepth) { ok = false; return; }
                int16_t id, last = 0; int t;
                while (field(&id, &t, &last)) skip(t);
                depth--;
                break;
            }
            default: ok = false;
        }
    }
    // Walk a struct: fn(id, type) consumes the fields it knows and returns false for the others, which are skipped.
    template <class F> void walk(F fn) {
        if (++depth > kMaxDepth) { ok = false; return; }
        int16_t id, last = 0; int t;
        while (field(&id, &t, &last))
            if (!fn(id, t)) skip(t);
        depth--;
    }
    int32_t i32() { return (int32_t)zz(); }
};

// ---- the footer ---------------------------------------------------------------------------------------------------------------------
struct SchemaEl {
    int type = -1, type_length = 0, repetition = 0, num_children = 0, converted = -1;
    std::string name;
    int logical = 0;                 // LogicalType union member (0: none)
    int int_bits = 0, int_signed = 1;
    int time_unit = 0;               // 1 MILLIS, 2 MICROS, 3 NANOS
    bool utc = false;
};

void parse_time_unit(Thrift& t, int* unit) {
    t.walk([&](int16_t id, int) { *unit = id; t.skip(TC_STRUCT); return true; });
}

void parse_logical(Thrift& t, SchemaEl* s) {
    t.walk([&](int16_t id, int type) {
        if (type != TC_STRUCT) return false;
        s->logical = id;
        if (id == 10) {   // IntType
            t.walk([&](int16_t f, int ft) {
                if (f == 1 && ft == TC_BYTE) { s->int_bits = (int8_t)t.byte(); return true; }
                if (f == 2 && (ft == TC_TRUE || ft == TC_FALSE)) { s->int_signed = ft == TC_TRUE; return true; }
                return false;
            });
            return true;
        }
        if (id == 7 || id == 8) {   // TimeType / TimestampType
            t.walk([&](int16_t f, int ft) {
                if (f == 1 && (ft == TC_TRUE || ft == TC_FALSE)) { s->utc = ft == TC_TRUE; return true; }
                if (f == 2 && ft == TC_STRUCT) { parse_time_unit(t, &s->time_unit); return true; }
                return false;
            });
            return true;
        }
        return false;
    });
}

struct ChunkMeta {
    std::string file_path;
    bool has_file_path = false;
    int type = -1, codec = 0;
    int64_t num_values = 0, total_compressed = 0, data_page_offset = 0, dict_page_offset = -1;
};

struct Footer {
    std::vector<SchemaEl> schema;
    int64_t num_rows = 0;
    std::vector<int64_t> rg_rows;
    std::vector<std::vector<ChunkMeta>> rg_cols;
    std::string arrow_schema;
    bool has_arrow_schema = false;
};

bool parse_footer(const uint8_t* p, size_t n, Footer* F) {
    Thrift t{p, n};
    t.walk([&](int16_t id, int type) {
        if (id == 2 && type == TC_LIST) {
            int et; uint32_t c;
            t.list(&et, &c);
            if (et != TC_STRUCT) { t.ok = false; return true; }
            for (uint32_t i = 0; i < c && t.ok; i++) {
                SchemaEl s;
                t.walk([&](int16_t f, int ft) {
                    switch (f) {
                        case 1: if (ft != TC_I32) return false; s.type = t.i32(); return true;
                        case 2: if (ft != TC_I32) return false; s.type_length = t.i32(); return true;
                        case 3: if (ft != TC_I32) return false; s.repetition = t.i32(); return true;
                        case 4: if (ft != TC_BINARY) return false; s.name = t.binary(); return true;
                        case 5: if (ft != TC_I32) return false; s.num_children = t.i32(); return true;
                        case 6: if (ft != TC_I32) return false; s.converted = t.i32(); return true;
                        case 10: if (ft != TC_STRUCT) return false; parse_logical(t, &s); return true;
                        default: return false;
                    }
                });
                F->schema.push_back(std::move(s));
            }
            return true;
        }
        if (id == 3 && type == TC_I64) { F->num_rows = t.zz(); return true; }
        if (id == 4 && type == TC_LIST) {
            int et; uint32_t c;
            t.list(&et, &c);
            if (et != TC_STRUCT) { t.ok = false; return true; }
            for (uint32_t i = 0; i < c && t.ok; i++) {
                int64_t rows = 0;
                std::vector<ChunkMeta> cols;
                t.walk([&](int16_t f, int ft) {
                    if (f == 3 && ft == TC_I64) { rows = t.zz(); return true; }
                    if (f != 1 || ft != TC_LIST) return false;
                    int cet; uint32_t cc;
                    t.list(&cet, &cc);
                    if (cet != TC_STRUCT) { t.ok = false; return true; }
                    for (uint32_t k = 0; k < cc && t.ok; k++) {
                        ChunkMeta m;
                        t.walk([&](int16_t g, int gt) {
                            if (g == 1 && gt == TC_BINARY) { m.file_path = t.binary(); m.has_file_path = true; return true; }
                            if (g != 3 || gt != TC_STRUCT) return false;
                            t.walk([&](int16_t h, int ht) {
                                switch (h) {
                                    case 1: if (ht != TC_I32) return false; m.type = t.i32(); return true;
                                    case 4: if (ht != TC_I32) return false; m.codec = t.i32(); return true;
                                    case 5: if (ht != TC_I64) return false; m.num_values = t.zz(); return true;
                                    case 7: if (ht != TC_I64) return false; m.total_compressed = t.zz(); return true;
                                    case 9: if (ht != TC_I64) return false; m.data_page_offset = t.zz(); return true;
                                    case 11: if (ht != TC_I64) return false; m.dict_page_offset = t.zz(); return true;
                                    default: return false;
                                }
                            });
                            return true;
                        });
                        cols.push_back(std::move(m));
                    }
                    return true;
                });
                F->rg_rows.push_back(rows);
                F->rg_cols.push_back(std::move(cols));
            }
            return true;
        }
        if (id == 5 && type == TC_LIST) {
            int et; uint32_t c;
            t.list(&et, &c);
            if (et != TC_STRUCT) { t.ok = false; return true; }
            for (uint32_t i = 0; i < c && t.ok; i++) {
                std::string k, v;
                bool has_v = false;
                t.walk([&](int16_t f, int ft) {
                    if (ft != TC_BINARY || (f != 1 && f != 2)) return false;
                    if (f == 1) k = t.binary(); else { v = t.binary(); has_v = true; }
                    return true;
                });
                if (k == "ARROW:schema" && has_v) { F->arrow_schema = v; F->has_arrow_schema = true; }
            }
            return true;
        }
        return false;
    });
    return t.ok;
}

struct PageHdr {
    int type = -1, raw = -1, comp = -1;
    int num_values = -1, encoding = -1, def_encoding = -1, num_nulls = 0, num_rows = -1, def_len = 0, rep_len = 0;
    bool is_compressed = true;
    size_t hdr_len = 0;
};

bool parse_page_header(const uint8_t* p, size_t n, PageHdr* h) {
    Thrift t{p, n};
    t.walk([&](int16_t id, int type) {
        switch (id) {
            case 1: if (type != TC_I32) return false; h->type = t.i32(); return true;
            case 2: if (type != TC_I32) return false; h->raw = t.i32(); return true;
            case 3: if (type != TC_I32) return false; h->comp = t.i32(); return true;
            case 5: case 7: case 8:
                if (type != TC_STRUCT) return false;
                t.walk([&](int16_t f, int ft) {
                    if (ft == TC_TRUE || ft == TC_FALSE) {
                        if (id == 8 && f == 7) { h->is_compressed = ft == TC_TRUE; return true; }
                        return false;
                    }
                    if (ft != TC_I32) return false;
                    const int v = t.i32();
                    if (f == 1) h->num_values = v;
                    else if (id == 5 && f == 2) h->encoding = v;
                    else if (id == 5 && f == 3) h->def_encoding = v;
                    else if (id == 7 && f == 2) h->encoding = v;
                    else if (id == 8 && f == 2) h->num_nulls = v;
                    else if (id == 8 && f == 3) h->num_rows = v;
                    else if (id == 8 && f == 4) h->encoding = v;
                    else if (id == 8 && f == 5) h->def_len = v;
                    else if (id == 8 && f == 6) h->rep_len = v;
                    return true;
                });
                return true;
            default: return false;
        }
    });
    h->hdr_len = t.pos;
    return t.ok;
}

bool base64_decode(const std::string& s, std::string* out) {
    auto val = [](char c) -> int {
        if (c >= 'A' && c <= 'Z') return c - 'A';
        if (c >= 'a' && c <= 'z') return c - 'a' + 26;
        if (c >= '0' && c <= '9') return c - '0' + 52;
        if (c == '+') return 62;
        if (c == '/') return 63;
        return -1;
    };
    uint32_t acc = 0;
    int bits = 0;
    for (char c : s) {
        if (c == '=') break;
        const int v = val(c);
        if (v < 0) return false;
        acc = (acc << 6) | (uint32_t)v;
        bits += 6;
        if (bits >= 8) { bits -= 8; out->push_back((char)((acc >> bits) & 0xff)); }
    }
    return true;
}

}  // namespace

// ---- the open file --------------------------------------------------------------------------------------------------------------------
struct PqPageH { int64_t data; pq::Page pg; };   // data: file offset of the page's bytes after its header
struct PqChunkH {
    int64_t start = 0, len = 0;
    int status = BDF_OK;
    std::string msg;                  // the message of a host-detected problem (status != BDF_OK)
    std::vector<PqPageH> pages;
};
struct PqColH { std::string name; int dtype = -1, nullable = 0, phys = -1, max_def = 0, leaf = -1; bdf_temporal_type tt{0, 0, nullptr}; bool has_tz = false; std::string tz; };
struct PqFileH {
    std::string path;
    int fd = -1;
    const uint8_t* map = nullptr;
    size_t size = 0;
    int64_t rows = 0;
    std::vector<int64_t> rg_rows;
    std::vector<PqColH> cols;
    std::vector<std::vector<PqChunkH>> chunks;   // [row group][column]; empty for a column off the path
};

struct bdf_parquet {
    std::vector<PqFileH> files;
    std::vector<PqColH> cols;    // the schema of the first file, nullable OR-ed over the files
    int64_t batch = 1024, n_rows = 0, n_batches = 0;
    mutable int64_t n_pages = 0, uploaded = 0;
    mutable double upload_ms = 0;
};

namespace {

std::string where(const PqFileH& f, int rg, int col, int page) {
    std::string s = "Parquet error in " + f.path;
    char b[96];
    if (rg >= 0) { snprintf(b, sizeof b, ", row group %d", rg); s += b; }
    if (col >= 0) { snprintf(b, sizeof b, ", column %d", col); s += b; }
    if (page >= 0) { snprintf(b, sizeof b, ", page %d", page); s += b; }
    return s;
}

// The column type of a top-level primitive leaf (b200df.h's table), or -1.
void column_type(const SchemaEl& s, PqColH* c) {
    c->dtype = -1;
    c->phys = s.type;
    const int lg = s.logical, cv = s.converted;
    auto intty = [&](int bits, bool sg) {
        const int k = bits == 8 ? 0 : bits == 16 ? 1 : bits == 32 ? 2 : bits == 64 ? 3 : -1;
        if (k < 0) return -1;
        if ((s.type == pq::PHYS_INT32) != (k < 3)) return -1;
        return sg ? BDF_I8 + k : BDF_U8 + k;
    };
    if (s.type == pq::PHYS_BOOLEAN) { if (!lg && cv < 0) c->dtype = BDF_BOOL; return; }
    if (s.type == pq::PHYS_FLOAT) { if (!lg && cv < 0) c->dtype = BDF_F32; return; }
    if (s.type == pq::PHYS_DOUBLE) { if (!lg && cv < 0) c->dtype = BDF_F64; return; }
    if (s.type != pq::PHYS_INT32 && s.type != pq::PHYS_INT64) return;
    const bool i32 = s.type == pq::PHYS_INT32;
    const int base = i32 ? BDF_I32 : BDF_I64;
    if (lg) {
        switch (lg) {
            case 10: c->dtype = intty(s.int_bits, s.int_signed != 0); return;
            case 6: if (i32) { c->dtype = BDF_I32; c->tt = {BDF_DATE32, 0, nullptr}; } return;
            case 7:
                if (i32 && s.time_unit == 1) { c->dtype = BDF_I32; c->tt = {BDF_TIME32, BDF_MILLISECOND, nullptr}; }
                if (!i32 && (s.time_unit == 2 || s.time_unit == 3)) { c->dtype = BDF_I64; c->tt = {BDF_TIME64, s.time_unit == 2 ? BDF_MICROSECOND : BDF_NANOSECOND, nullptr}; }
                return;
            case 8:
                if (!i32 && s.time_unit >= 1 && s.time_unit <= 3) {
                    c->dtype = BDF_I64;
                    c->tt = {BDF_TIMESTAMP, s.time_unit, nullptr};   // MILLIS 1 .. NANOS 3 = bdf_time_unit
                    if (s.utc) { c->has_tz = true; c->tz = "UTC"; }
                }
                return;
            default: return;
        }
    }
    switch (cv) {
        case -1: c->dtype = base; return;
        case 6: if (i32) { c->dtype = BDF_I32; c->tt = {BDF_DATE32, 0, nullptr}; } return;
        case 7: if (i32) { c->dtype = BDF_I32; c->tt = {BDF_TIME32, BDF_MILLISECOND, nullptr}; } return;
        case 8: if (!i32) { c->dtype = BDF_I64; c->tt = {BDF_TIME64, BDF_MICROSECOND, nullptr}; } return;
        case 9: case 10:   // TIMESTAMP_MILLIS / _MICROS stand for TIMESTAMP(unit, isAdjustedToUTC = true)
            if (!i32) { c->dtype = BDF_I64; c->tt = {BDF_TIMESTAMP, cv == 9 ? BDF_MILLISECOND : BDF_MICROSECOND, nullptr}; c->has_tz = true; c->tz = "UTC"; }
            return;
        case 11: case 12: case 13: c->dtype = intty(8 << (cv - 11), false); return;
        case 14: c->dtype = intty(64, false); return;
        case 15: case 16: case 17: c->dtype = intty(8 << (cv - 15), true); return;
        case 18: c->dtype = intty(64, true); return;
        default: return;
    }
}

int phys_width(int phys) { return phys == pq::PHYS_INT32 || phys == pq::PHYS_FLOAT ? 4 : phys == pq::PHYS_BOOLEAN ? 0 : 8; }

// Walk the page headers of one column chunk; a problem is kept in the chunk (the status a read of the column gives).
void walk_chunk(const PqFileH& f, int rg, int col, const ChunkMeta& m, int64_t rg_rows, PqChunkH* ch) {
    const PqColH& c = f.cols[(size_t)col];
    auto bad = [&](int page, int status, const char* fmt, ...) {
        char b[384];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(b, sizeof b, fmt, ap);
        va_end(ap);
        ch->status = status;
        ch->msg = where(f, rg, col, page) + ": " + b;
    };
    if (m.codec != 0 && m.codec != 1) return bad(-1, BDF_UNSUPPORTED, "codec %s is not supported (UNCOMPRESSED and SNAPPY are)", codec_name(m.codec));
    if (m.type != c.phys) return bad(-1, BDF_INVALID, "the chunk's physical type %d differs from the schema's %d", m.type, c.phys);
    const int64_t start = m.dict_page_offset > 0 && m.dict_page_offset < m.data_page_offset ? m.dict_page_offset : m.data_page_offset;
    const int64_t limit = (int64_t)f.size - 8;
    if (start < 4 || m.total_compressed < 0 || start > limit || m.total_compressed > limit - start)
        return bad(-1, BDF_INVALID, "the column chunk [%lld, +%lld) lies outside the file", (long long)start, (long long)m.total_compressed);
    ch->start = start;
    ch->len = m.total_compressed;
    const int64_t end = start + m.total_compressed;
    int64_t pos = start, values = 0;
    int page = 0, dict = -1;
    for (; pos < end; page++) {
        PageHdr h;
        if (!parse_page_header(f.map + pos, (size_t)(end - pos), &h)) return bad(page, BDF_INVALID, "the page header runs past its column chunk or is malformed");
        const int64_t data = pos + (int64_t)h.hdr_len;
        if (h.comp < 0 || h.raw < 0 || h.comp > end - data) return bad(page, BDF_INVALID, "the page (%d bytes) runs past its column chunk", h.comp);
        pos = data + h.comp;
        if (h.type == 1) continue;   // INDEX_PAGE
        pq::Page pg{};
        pg.comp = h.comp;
        pg.raw = h.raw;
        pg.phys = c.phys;
        pg.width = phys_width(c.phys);
        pg.out_width = c.dtype == BDF_BOOL ? 0 : (c.dtype == BDF_I8 || c.dtype == BDF_U8 ? 1 : c.dtype == BDF_I16 || c.dtype == BDF_U16 ? 2 : c.dtype == BDF_I32 || c.dtype == BDF_U32 || c.dtype == BDF_F32 ? 4 : 8);
        pg.max_def = c.max_def;
        pg.snappy = m.codec == 1;
        pg.dict = -1;
        if (h.type == 2) {
            if (dict >= 0) return bad(page, BDF_INVALID, "more than one dictionary page");
            if (!ch->pages.empty()) return bad(page, BDF_INVALID, "a dictionary page after a data page");
            if (h.num_values < 0) return bad(page, BDF_INVALID, "a dictionary page without num_values");
            if (h.encoding != pq::ENC_PLAIN && h.encoding != pq::ENC_PLAIN_DICTIONARY)
                return bad(page, BDF_UNSUPPORTED, "dictionary page encoding %s is not supported", encoding_name(h.encoding));
            if (c.phys == pq::PHYS_BOOLEAN) return bad(page, BDF_UNSUPPORTED, "a Boolean dictionary is not supported");
            if ((int64_t)h.num_values * pg.width > (int64_t)h.raw) return bad(page, BDF_INVALID, "%d dictionary values do not fit in %d bytes", h.num_values, h.raw);
            pg.kind = pq::KIND_DICT;
            pg.num_values = h.num_values;
            pg.encoding = pq::ENC_PLAIN;
            dict = (int)ch->pages.size();
            ch->pages.push_back(PqPageH{data, pg});
            continue;
        }
        if (h.type != 0 && h.type != 3) return bad(page, BDF_INVALID, "unknown page type %d", h.type);
        if (h.num_values < 0) return bad(page, BDF_INVALID, "a data page without num_values");
        pg.kind = h.type == 0 ? pq::KIND_V1 : pq::KIND_V2;
        pg.num_values = h.num_values;
        pg.encoding = h.encoding;
        const int e = h.encoding;
        const bool dict_enc = e == pq::ENC_PLAIN_DICTIONARY || e == pq::ENC_RLE_DICTIONARY;
        const bool ok = e == pq::ENC_PLAIN || dict_enc || (e == pq::ENC_RLE && c.phys == pq::PHYS_BOOLEAN) ||
                        (e == pq::ENC_BYTE_STREAM_SPLIT && c.phys != pq::PHYS_BOOLEAN);
        if (!ok) return bad(page, BDF_UNSUPPORTED, "encoding %s is not supported for this column", encoding_name(e));
        if (dict_enc && dict < 0) return bad(page, BDF_INVALID, "a dictionary-encoded page without a dictionary page");
        pg.dict = dict_enc ? dict : -1;
        if (pg.kind == pq::KIND_V1) {
            if (c.max_def > 0 && h.def_encoding != pq::ENC_RLE)
                return bad(page, BDF_UNSUPPORTED, "definition-level encoding %s is not supported", encoding_name(h.def_encoding));
        } else {
            if (h.def_len < 0 || h.rep_len < 0 || (int64_t)h.def_len + h.rep_len > h.comp) return bad(page, BDF_INVALID, "level sections outside the page");
            if (h.rep_len != 0) return bad(page, BDF_INVALID, "repetition levels in a top-level column");
            if (c.max_def == 0 && h.def_len != 0) return bad(page, BDF_INVALID, "definition levels in a required column");
            pg.def_len = h.def_len;
            pg.rep_len = h.rep_len;
            if (!h.is_compressed) pg.snappy = 0;
            if (pg.snappy) pg.raw = h.raw - h.def_len - h.rep_len;   // the codec covers the values section only
            if (pg.raw < 0) return bad(page, BDF_INVALID, "uncompressed size below the level sections");
        }
        values += h.num_values;
        ch->pages.push_back(PqPageH{data, pg});
    }
    if (values != rg_rows) return bad(-1, BDF_INVALID, "data-page num_values add up to %lld, the row group has %lld rows", (long long)values, (long long)rg_rows);
}

void file_close(PqFileH& f) {
    if (f.map) munmap((void*)f.map, f.size);
    if (f.fd >= 0) close(f.fd);
    f.map = nullptr; f.fd = -1;
}

// Map and parse one file.  *empty: it has no row groups.
int open_file(const std::string& path, PqFileH* f) {
    f->path = path;
    f->fd = open(path.c_str(), O_RDONLY | O_CLOEXEC);
    struct stat st;
    if (f->fd < 0 || fstat(f->fd, &st) != 0) return pq_fail(BDF_INVALID, "cannot open %s: %s", path.c_str(), strerror(errno));
    f->size = (size_t)st.st_size;
    if (f->size < 12) return pq_fail(BDF_INVALID, "%s: the file is too short to be a Parquet file", where(*f, -1, -1, -1).c_str());
    void* m = mmap(nullptr, f->size, PROT_READ, MAP_PRIVATE, f->fd, 0);
    if (m == MAP_FAILED) return pq_fail(BDF_INVALID, "cannot map %s: %s", path.c_str(), strerror(errno));
    f->map = (const uint8_t*)m;
    const uint8_t* tail = f->map + f->size - 4;
    if (memcmp(tail, "PARE", 4) == 0) return pq_fail(BDF_UNSUPPORTED, "%s: encrypted files are not supported", where(*f, -1, -1, -1).c_str());
    if (memcmp(f->map, "PAR1", 4) != 0 || memcmp(tail, "PAR1", 4) != 0) return pq_fail(BDF_INVALID, "%s: bad magic (PAR1 missing)", where(*f, -1, -1, -1).c_str());
    uint32_t flen;
    memcpy(&flen, f->map + f->size - 8, 4);
    if ((uint64_t)flen > f->size - 12) return pq_fail(BDF_INVALID, "%s: the footer (%u bytes) lies outside the file", where(*f, -1, -1, -1).c_str(), flen);
    Footer F;
    if (!parse_footer(f->map + f->size - 8 - flen, flen, &F)) return pq_fail(BDF_INVALID, "%s: malformed footer", where(*f, -1, -1, -1).c_str());
    if (F.schema.empty() || F.schema[0].num_children < 0) return pq_fail(BDF_INVALID, "%s: the footer has no schema", where(*f, -1, -1, -1).c_str());
    // top-level fields: a leaf is a column; a group is one column off the path, its leaves skipped
    size_t i = 1;
    int leaf = 0;
    for (int k = 0; k < F.schema[0].num_children; k++) {
        if (i >= F.schema.size()) return pq_fail(BDF_INVALID, "%s: the schema has fewer elements than its root's children", where(*f, -1, -1, -1).c_str());
        const SchemaEl& s = F.schema[i];
        PqColH c;
        c.name = s.name;
        c.nullable = s.repetition != 0;
        if (s.num_children > 0) {   // a group: skip its subtree
            int64_t pending = s.num_children;
            i++;
            while (pending > 0) {
                if (i >= F.schema.size()) return pq_fail(BDF_INVALID, "%s: the schema ends inside a group", where(*f, -1, -1, -1).c_str());
                if (F.schema[i].num_children > 0) pending += F.schema[i].num_children; else leaf++;
                pending--;
                i++;
            }
        } else {
            c.leaf = leaf++;
            i++;
            if (s.repetition == 0 || s.repetition == 1) {
                column_type(s, &c);
                c.max_def = s.repetition == 1 ? 1 : 0;
            }
            if (c.dtype < 0) c.tt = {0, 0, nullptr}, c.has_tz = false, c.tz.clear();
        }
        f->cols.push_back(std::move(c));
    }
    // an Arrow schema stored by the writer gives a Timestamp its tz (same position, name and unit)
    std::string raw;
    std::vector<bdf::ArrowField> af;
    if (F.has_arrow_schema && base64_decode(F.arrow_schema, &raw) && bdf::arrow_schema_fields((const uint8_t*)raw.data(), raw.size(), &af))
        for (size_t k = 0; k < f->cols.size() && k < af.size(); k++) {
            PqColH& c = f->cols[k];
            if (c.tt.kind == BDF_TIMESTAMP && af[k].name == c.name && af[k].kind == BDF_TIMESTAMP && af[k].unit == c.tt.unit) {
                c.has_tz = af[k].has_tz;
                c.tz = af[k].tz;
            }
        }
    f->rg_rows = F.rg_rows;
    for (size_t g = 0; g < F.rg_cols.size(); g++) {
        if (F.rg_rows[g] < 0 || F.rg_cols[g].size() != (size_t)leaf)
            return pq_fail(BDF_INVALID, "%s: %zu column chunks for %d leaf columns (or negative rows)", where(*f, (int)g, -1, -1).c_str(), F.rg_cols[g].size(), leaf);
        for (const ChunkMeta& m : F.rg_cols[g])
            if (m.has_file_path) return pq_fail(BDF_UNSUPPORTED, "%s: a column chunk in another file (%s) is not supported", where(*f, (int)g, -1, -1).c_str(), m.file_path.c_str());
        f->rows += F.rg_rows[g];
    }
    f->chunks.assign(F.rg_cols.size(), std::vector<PqChunkH>(f->cols.size()));
    for (size_t g = 0; g < F.rg_cols.size(); g++)
        for (size_t k = 0; k < f->cols.size(); k++)
            if (f->cols[k].dtype >= 0) walk_chunk(*f, (int)g, (int)k, F.rg_cols[g][(size_t)f->cols[k].leaf], F.rg_rows[g], &f->chunks[g][k]);
    return BDF_OK;
}

void parquet_free(bdf_parquet* p) {
    if (!p) return;
    for (auto& f : p->files) file_close(f);
    delete p;
}

int check_col(const bdf_parquet* f, int col) {
    if (col < 0 || col >= (int)f->cols.size()) return pq_fail(BDF_INVALID, "column %d out of range (the files have %zu)", col, f->cols.size());
    if (f->cols[(size_t)col].dtype < 0)
        return pq_fail(BDF_UNSUPPORTED, "column %d (%s) is not on the device path (a string, nested, repeated or unsupported type)", col, f->cols[(size_t)col].name.c_str());
    for (const auto& file : f->files)
        for (const auto& rg : file.chunks) {
            const PqChunkH& ch = rg[(size_t)col];
            if (ch.status != BDF_OK) return pq_fail(ch.status, "%s", ch.msg.c_str());
        }
    return BDF_OK;
}

const char* error_text(int code) {
    switch (code) {
        case pq::E_SNAPPY: return "corrupt snappy stream";
        case pq::E_SNAPPY_SIZE: return "the decompressed size does not match the page header";
        case pq::E_LEVELS: return "the definition-level stream is malformed or ends early";
        case pq::E_INDEX: return "the dictionary-index (or Boolean RLE) stream is malformed or ends early";
        case pq::E_DICT_RANGE: return "a dictionary index lies outside the dictionary";
        case pq::E_VALUES: return "the value stream ends early";
        case pq::E_LAYOUT: return "the level section lies outside the page";
        case pq::E_BIT_WIDTH: return "bit width above 32";
        case pq::E_LEVEL_VALUE: return "a definition level above the column's maximum";
        case pq::E_RUNS: return "more runs than values";
        default: return "unknown device error";
    }
}

}  // namespace

namespace pq {

int plan(const bdf_parquet* f, int n, const int32_t* cols, Plan* P) {
    for (int i = 0; i < n; i++) {
        const int st = check_col(f, cols[i]);
        if (st != BDF_OK) return st;
    }
    P->batch = f->batch;
    std::vector<long long> file_chunk0;
    for (const auto& file : f->files) {
        file_chunk0.push_back((long long)P->chunk_lens.size());
        for (int64_t r = 0; r < file.rows; r += f->batch) P->chunk_lens.push_back(std::min<int64_t>(f->batch, file.rows - r));
    }
    const long long n_chunks = (long long)P->chunk_lens.size();
    for (int i = 0; i < n; i++)
        for (size_t fi = 0; fi < f->files.size(); fi++) {
            const PqFileH& file = f->files[fi];
            int64_t row0 = 0;
            for (size_t g = 0; g < file.chunks.size(); g++) {
                const PqChunkH& ch = file.chunks[g][(size_t)cols[i]];
                const long long seg = P->upload_bytes;
                P->segs.push_back(Plan::Seg{file.map + ch.start, ch.len, seg});
                P->upload_bytes += (ch.len + 15) / 16 * 16;
                const int first = (int)P->pages.size();
                int64_t r = row0;
                for (size_t k = 0; k < ch.pages.size(); k++) {
                    Page pg = ch.pages[k].pg;
                    pg.src = seg + (ch.pages[k].data - ch.start);
                    pg.dst = -1;
                    if (pg.snappy) { pg.dst = P->scratch_bytes; P->scratch_bytes += ((long long)pg.raw + 15) / 16 * 16; }
                    if (pg.dict >= 0) pg.dict += first;
                    pg.out0 = (int)(i * n_chunks + file_chunk0[fi]);
                    if (pg.kind != KIND_DICT) {
                        pg.row0 = r;
                        r += pg.num_values;
                        // bytes that can hold each stream: V2 levels have their own length; the rest lies in the (decompressed) page
                        const long long page_n = pg.snappy ? pg.raw : pg.comp - (pg.kind == KIND_V2 ? pg.def_len + pg.rep_len : 0);
                        const long long def_n = pg.kind == KIND_V2 ? pg.def_len : page_n;
                        pg.cap_def = pg.max_def ? (int)std::min<long long>(pg.num_values, def_n) + 1 : 0;
                        pg.cap_idx = uses_index(pg.encoding) ? (int)std::min<long long>(pg.num_values, page_n) + 1 : 0;
                        pg.runs = P->run_entries;
                        P->run_entries += (long long)pg.cap_def + pg.cap_idx;
                        pg.tile0 = (long long)P->tiles.size();
                        pg.n_tiles = (pg.num_values + kTileRows - 1) / kTileRows;
                        for (int t = 0; t < pg.n_tiles; t++) P->tiles.push_back(Tile{(int)P->pages.size(), t * kTileRows});
                    }
                    P->pages.push_back(pg);
                    P->label.insert(P->label.end(), {(int)fi, (int)g, cols[i], (int)k});
                }
                row0 += file.rg_rows[g];
            }
        }
    if (P->tiles.size() > (size_t)0x7fffffff || P->pages.size() > (size_t)0x3fffffff)
        return pq_fail(BDF_UNSUPPORTED, "the read has more pages or tiles than one launch covers");
    return BDF_OK;
}

int page_error(const bdf_parquet* f, const Plan& P, int page, int code) {
    const int* l = &P.label[(size_t)page * 4];
    return pq_fail(BDF_INVALID, "%s: %s", where(f->files[(size_t)l[0]], l[1], l[2], l[3]).c_str(), error_text(code));
}

}  // namespace pq

// ---- C ABI ------------------------------------------------------------------------------------------------------------------------------
#pragma GCC visibility push(default)
extern "C" {

int bdf_parquet_open(const char* path, const bdf_parquet_options* o, bdf_parquet** out) {
    if (!path || !out) return pq_fail(BDF_INVALID, "null argument");
    *out = nullptr;
    const int64_t batch = o ? o->batch_size : 1024;
    if (batch < 1) return pq_fail(BDF_INVALID, "batch_size must be at least 1");
    struct stat st;
    if (stat(path, &st) != 0) return pq_fail(BDF_INVALID, "cannot open %s: %s", path, strerror(errno));
    std::vector<std::string> paths;
    if (S_ISDIR(st.st_mode)) {
        DIR* d = opendir(path);
        if (!d) return pq_fail(BDF_INVALID, "cannot read directory %s: %s", path, strerror(errno));
        while (dirent* e = readdir(d)) {
            if (e->d_name[0] == '.' || e->d_name[0] == '_') continue;   // hidden files and markers such as _SUCCESS
            const std::string p = std::string(path) + "/" + e->d_name;
            struct stat fs;
            if (stat(p.c_str(), &fs) == 0 && S_ISREG(fs.st_mode)) paths.push_back(e->d_name);
        }
        closedir(d);
        std::sort(paths.begin(), paths.end());   // byte order of the names
        for (auto& p : paths) p = std::string(path) + "/" + p;
    } else {
        paths.push_back(path);
    }
    bdf_parquet* f = new (std::nothrow) bdf_parquet();
    if (!f) return pq_fail(BDF_OOM, "host allocation failed");
    struct Guard { bdf_parquet* f; ~Guard() { parquet_free(f); } } guard{f};
    f->batch = batch;
    for (const std::string& p : paths) {
        PqFileH file;
        const int s = open_file(p, &file);
        if (s != BDF_OK) { file_close(file); return s; }
        if (file.chunks.empty()) { file_close(file); continue; }   // no row groups
        f->files.push_back(std::move(file));
    }
    if (f->files.empty()) return pq_fail(BDF_WOULD_PANIC, "no Parquet file with row groups in %s: the reference's schema.unwrap() panics", path);
    f->cols = f->files[0].cols;
    for (size_t k = 1; k < f->files.size(); k++) {
        const PqFileH& g = f->files[k];
        if (g.cols.size() != f->cols.size())
            return pq_fail(BDF_INVALID, "%s: %zu columns, %s has %zu", where(g, -1, -1, -1).c_str(), g.cols.size(), f->files[0].path.c_str(), f->cols.size());
        for (size_t c = 0; c < g.cols.size(); c++) {
            const PqColH &a = f->cols[c], &b = g.cols[c];
            if (a.name != b.name || a.dtype != b.dtype || a.tt.kind != b.tt.kind || a.tt.unit != b.tt.unit || a.has_tz != b.has_tz || a.tz != b.tz)
                return pq_fail(BDF_INVALID, "%s: column %s differs from %s's (name, type or time zone)", where(g, -1, (int)c, -1).c_str(), b.name.c_str(),
                               f->files[0].path.c_str());
            f->cols[c].nullable |= b.nullable;
        }
    }
    for (const auto& file : f->files) {
        f->n_rows += file.rows;
        f->n_batches += (file.rows + batch - 1) / batch;
    }
    for (auto& c : f->cols) c.tt.tz = c.has_tz ? c.tz.c_str() : nullptr;
    guard.f = nullptr;
    *out = f;
    return BDF_OK;
}

int bdf_parquet_describe(const bdf_parquet* f, int32_t* n_columns, int64_t* n_batches, int64_t* n_rows) {
    if (!f) return pq_fail(BDF_INVALID, "null file");
    if (n_columns) *n_columns = (int32_t)f->cols.size();
    if (n_batches) *n_batches = f->n_batches;
    if (n_rows) *n_rows = f->n_rows;
    return BDF_OK;
}

int bdf_parquet_column(const bdf_parquet* f, int32_t col, const char** name, int32_t* dtype, int32_t* nullable) {
    if (!f) return pq_fail(BDF_INVALID, "null file");
    if (col < 0 || col >= (int32_t)f->cols.size()) return pq_fail(BDF_INVALID, "column %d out of range", col);
    if (name) *name = f->cols[(size_t)col].name.c_str();
    if (dtype) *dtype = f->cols[(size_t)col].dtype;
    if (nullable) *nullable = f->cols[(size_t)col].nullable;
    return BDF_OK;
}

int bdf_parquet_temporal_column(const bdf_parquet* f, int32_t col, bdf_temporal_type* out) {
    if (!f || !out) return pq_fail(BDF_INVALID, "null argument");
    if (col < 0 || col >= (int32_t)f->cols.size()) return pq_fail(BDF_INVALID, "column %d out of range", col);
    *out = f->cols[(size_t)col].tt;
    return BDF_OK;
}

int bdf_parquet_check(const bdf_parquet* f, int32_t col) {
    if (!f) return pq_fail(BDF_INVALID, "null file");
    return check_col(f, col);
}

int bdf_parquet_stats(const bdf_parquet* f, int64_t* n_pages, int64_t* uploaded_bytes, double* upload_ms) {
    if (!f) return pq_fail(BDF_INVALID, "null file");
    if (n_pages) *n_pages = f->n_pages;
    if (uploaded_bytes) *uploaded_bytes = f->uploaded;
    if (upload_ms) *upload_ms = f->upload_ms;
    return BDF_OK;
}

void bdf_parquet_close(bdf_parquet* f) { parquet_free(f); }

}  // extern "C"
#pragma GCC visibility pop

// The last read's figures (runtime.cu's bdf_parquet_read).
namespace pq {
void set_stats(const bdf_parquet* f, long long n_pages, long long uploaded, double upload_ms) {
    f->n_pages = n_pages;
    f->uploaded = uploaded;
    f->upload_ms = upload_ms;
}
}  // namespace pq

// ---- the writer's footer and page headers (Thrift compact protocol; runtime.cu's bdf_parquet_write) ------------------------------------
namespace {

struct ThriftOut {
    std::string b;
    std::vector<int16_t> stack;
    int16_t last = 0;
    void varint(uint64_t v) {
        while (v >= 0x80) { b.push_back((char)(v | 0x80)); v >>= 7; }
        b.push_back((char)v);
    }
    static uint64_t zz(int64_t v) { return ((uint64_t)v << 1) ^ (uint64_t)(v >> 63); }
    void field(int16_t id, int type) {
        const int d = id - last;
        if (d > 0 && d <= 15) b.push_back((char)((d << 4) | type));
        else { b.push_back((char)type); varint(zz(id)); }
        last = id;
    }
    void i32(int16_t id, int32_t v) { field(id, TC_I32); varint(zz(v)); }
    void i64(int16_t id, int64_t v) { field(id, TC_I64); varint(zz(v)); }
    void binary(int16_t id, const std::string& s) { field(id, TC_BINARY); varint(s.size()); b += s; }
    void boolean(int16_t id, bool v) { field(id, v ? TC_TRUE : TC_FALSE); }
    void byte(int16_t id, int8_t v) { field(id, TC_BYTE); b.push_back((char)v); }
    void begin(int16_t id) { field(id, TC_STRUCT); elem(); }
    void elem() { stack.push_back(last); last = 0; }   // a struct that is a list element
    void end() { b.push_back(0); last = stack.back(); stack.pop_back(); }
    void list(int16_t id, int type, uint32_t n) {
        field(id, TC_LIST);
        if (n < 15) b.push_back((char)((n << 4) | type));
        else { b.push_back((char)(0xf0 | type)); varint(n); }
    }
};

}  // namespace

namespace pq {

std::string page_header(int kind, int raw_len, int comp_len, int num_values, int encoding) {
    ThriftOut t;
    t.elem();
    t.i32(1, kind == KIND_DICT ? 2 : 0);
    t.i32(2, raw_len);
    t.i32(3, comp_len);
    if (kind == KIND_DICT) {
        t.begin(7);
        t.i32(1, num_values);
        t.i32(2, encoding);
        t.end();
    } else {
        t.begin(5);
        t.i32(1, num_values);
        t.i32(2, encoding);
        t.i32(3, ENC_RLE);
        t.i32(4, ENC_RLE);
        t.end();
    }
    t.end();
    return t.b;
}

std::string file_metadata(const std::vector<WColumn>& cols, const std::vector<long long>& rg_rows, const std::vector<std::vector<WChunkMeta>>& chunks,
                          const std::string& arrow_schema_b64) {
    ThriftOut t;
    t.elem();
    t.i32(1, 1);
    t.list(2, TC_STRUCT, (uint32_t)cols.size() + 1);
    t.elem();
    t.binary(4, "schema");
    t.i32(5, (int32_t)cols.size());
    t.end();
    for (const WColumn& c : cols) {
        t.elem();
        t.i32(1, c.phys);
        t.i32(3, 1);   // OPTIONAL
        t.binary(4, c.name);
        if (c.converted >= 0) t.i32(6, c.converted);
        if (c.logical) {
            t.begin(10);
            t.begin((int16_t)c.logical);
            if (c.logical == 10) { t.byte(1, (int8_t)c.int_bits); t.boolean(2, c.int_signed != 0); }
            if (c.logical == 7 || c.logical == 8) {
                t.boolean(1, c.utc);
                t.begin(2);
                t.begin((int16_t)c.time_unit);
                t.end();
                t.end();
            }
            t.end();
            t.end();
        }
        t.end();
    }
    long long rows = 0;
    for (long long r : rg_rows) rows += r;
    t.i64(3, rows);
    t.list(4, TC_STRUCT, (uint32_t)rg_rows.size());
    for (size_t g = 0; g < rg_rows.size(); g++) {
        t.elem();
        t.list(1, TC_STRUCT, (uint32_t)cols.size());
        long long bytes = 0;
        for (size_t k = 0; k < cols.size(); k++) {
            const WChunkMeta& m = chunks[g][k];
            bytes += m.total_uncompressed;
            t.elem();
            t.i64(2, m.dict_page_offset >= 0 ? m.dict_page_offset : m.data_page_offset);
            t.begin(3);
            t.i32(1, m.phys);
            t.list(2, TC_I32, (uint32_t)m.encodings.size());
            for (int e : m.encodings) t.varint(ThriftOut::zz(e));
            t.list(3, TC_BINARY, 1);
            t.varint(cols[k].name.size());
            t.b += cols[k].name;
            t.i32(4, m.codec);
            t.i64(5, m.num_values);
            t.i64(6, m.total_uncompressed);
            t.i64(7, m.total_compressed);
            t.i64(9, m.data_page_offset);
            if (m.dict_page_offset >= 0) t.i64(11, m.dict_page_offset);
            if (m.has_stats) {
                t.begin(12);
                t.i64(3, m.null_count);
                if (m.has_minmax) { t.binary(5, m.max_value); t.binary(6, m.min_value); }
                t.end();
            }
            t.end();
            t.end();
        }
        t.i64(2, bytes);
        t.i64(3, rg_rows[g]);
        t.end();
    }
    t.list(5, TC_STRUCT, 1);
    t.elem();
    t.binary(1, "ARROW:schema");
    t.binary(2, arrow_schema_b64);
    t.end();
    t.binary(6, "b200df parquet writer");
    t.list(7, TC_STRUCT, (uint32_t)cols.size());
    for (size_t k = 0; k < cols.size(); k++) {
        t.elem();
        t.begin(1);   // TYPE_ORDER: TypeDefinedOrder
        t.end();
        t.end();
    }
    t.end();
    return t.b;
}

std::string base64(const std::string& s) {
    static const char* a = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    std::string o;
    size_t i = 0;
    for (; i + 2 < s.size(); i += 3) {
        const uint32_t v = (uint8_t)s[i] << 16 | (uint8_t)s[i + 1] << 8 | (uint8_t)s[i + 2];
        o += a[v >> 18]; o += a[(v >> 12) & 63]; o += a[(v >> 6) & 63]; o += a[v & 63];
    }
    if (i + 1 == s.size()) {
        const uint32_t v = (uint8_t)s[i] << 16;
        o += a[v >> 18]; o += a[(v >> 12) & 63]; o += "==";
    } else if (i + 2 == s.size()) {
        const uint32_t v = (uint8_t)s[i] << 16 | (uint8_t)s[i + 1] << 8;
        o += a[v >> 18]; o += a[(v >> 12) & 63]; o += a[(v >> 6) & 63]; o += '=';
    }
    return o;
}

}  // namespace pq
