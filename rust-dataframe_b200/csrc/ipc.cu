// ipc.cu -- SURVEY 8(f) N4: Arrow IPC *files* either side of the path (host code only; no kernels here).
//
// DataFrame::from_arrow (src/dataframe.rs:391-407) reads every RecordBatch of an IPC file through
// arrow::ipc::reader::FileReader into host arrays, and to_arrow (:515-525) writes them back with FileWriter.  The body
// buffers of an IPC file ARE the device layout of this library (values buffer + LSB-first validity bitmap per
// primitive column per batch), so the file is mapped, its footer/schema/RecordBatch metadata (flatbuffers, parsed by
// hand below: there is no flatbuffers or arrow dependency) is decoded into (offset, length) pairs, and bdf_ipc_read
// hands views INTO THE MAPPING to bdf_upload_many: page cache -> pinned staging -> HBM, one chunk per RecordBatch, no
// intermediate host arrays.  Columns whose type is outside the path (strings, lists, dictionaries, dates ...) are
// skipped by their buffer count and reported with dtype -1.
//
// Format restated from the Arrow columnar specification (format/File.fbs, Schema.fbs, Message.fbs; metadata V4 and V5,
// with or without the 0xFFFFFFFF continuation marker).  Checked against pyarrow in tests/test_ipc.py (both directions).
// Everything here goes through the public C ABI of the library (bdf_upload_many, bdf_download ...).
#include "../../include/b200df.h"
#include "ipc_schema.cuh"

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cerrno>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace bdf { int set_error(int status, const char* msg); }

namespace {

int ipc_fail(int status, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    return bdf::set_error(status, buf);
}

// ---- flatbuffers, read side (bounds-checked; every accessor returns false on a malformed buffer) ----------------
struct FbBuf {
    const uint8_t* p;
    size_t n;
    template <typename T> bool rd(size_t at, T* v) const {
        if (at > n || n - at < sizeof(T)) return false;
        memcpy(v, p + at, sizeof(T));
        return true;
    }
};
struct FbTable {
    const FbBuf* b = nullptr;
    size_t pos = 0, vt = 0;
    uint16_t vt_len = 0;
    bool init(const FbBuf* buf, size_t table_pos) {
        b = buf; pos = table_pos;
        int32_t so;
        if (!b->rd(pos, &so)) return false;
        const int64_t v = (int64_t)pos - so;
        if (v < 0 || (size_t)v + 4 > b->n) return false;
        vt = (size_t)v;
        return b->rd(vt, &vt_len) && vt_len >= 4 && vt + vt_len <= b->n;
    }
    size_t field(int id) const {   // absolute position of the field's inline data, 0 if absent
        const size_t e = 4 + 2 * (size_t)id;
        uint16_t off = 0;
        if (e + 2 > vt_len || !b->rd(vt + e, &off) || off == 0) return 0;
        return pos + off;
    }
    template <typename T> T scalar(int id, T dflt) const {
        const size_t f = field(id);
        T v = dflt;
        if (f && !b->rd(f, &v)) v = dflt;
        return v;
    }
    size_t ref(int id) const {     // target of an offset field (table, string or vector), 0 if absent/bad
        const size_t f = field(id);
        uint32_t o;
        if (!f || !b->rd(f, &o) || o == 0 || f + o >= b->n) return 0;
        return f + o;
    }
    bool table(int id, FbTable* t) const { const size_t r = ref(id); return r && t->init(b, r); }
    bool vec(int id, size_t* first, uint32_t* count, size_t elem) const {   // absent vector = empty
        *first = 0; *count = 0;
        const size_t r = ref(id);
        if (!r) return field(id) == 0;
        if (!b->rd(r, count)) return false;
        *first = r + 4;
        return (uint64_t)*count * elem <= b->n - *first;
    }
    bool str(int id, std::string* s) const {
        size_t first; uint32_t cnt;
        if (!vec(id, &first, &cnt, 1)) return false;
        s->assign((const char*)b->p + first, cnt);
        return true;
    }
};

// Schema.fbs Type union tags
enum { T_NONE = 0, T_Null, T_Int, T_FloatingPoint, T_Binary, T_Utf8, T_Bool, T_Decimal, T_Date, T_Time, T_Timestamp, T_Interval, T_List,
       T_Struct, T_Union, T_FixedSizeBinary, T_FixedSizeList, T_Map, T_Duration, T_LargeBinary, T_LargeUtf8, T_LargeList };

struct IpcField {
    std::string name;
    int dtype = -1;       // bdf_dtype, BDF_BOOL, or -1: a type outside the path
    int list_child = -1;  // a List<T> of one numeric T (dtype stays -1: bdf_ipc_list_column / bdf_ipc_read_list): T
    // a Date / Time / Timestamp field that forms a valid bdf_temporal_type (dtype stays -1: bdf_ipc_temporal_column /
    // bdf_ipc_read_temporal): its kind, unit, tz and physical dtype
    int temporal_kind = 0, temporal_unit = 0, temporal_dtype = -1;
    bool has_tz = false;
    std::string tz;
    bool nullable = false;
    int64_t n_nodes = 0, n_buffers = 0;   // what the field (with its children) occupies in every RecordBatch
};

// Field table -> IpcField; recursion only to count the nodes/buffers of nested children.
// `budget` bounds the TOTAL number of field tables visited while decoding a schema: child offsets of a crafted file may
// all point at the same table, so depth alone does not bound the work (k children per level -> k^depth visits).
bool parse_field(const FbTable& f, IpcField* out, int depth, int64_t* budget, std::string* why) {
    if (depth > 32) { *why = "schema nested too deeply"; return false; }
    if (--*budget < 0) { *why = "schema describes more fields than the footer can hold"; return false; }
    if (!f.str(0, &out->name)) { *why = "bad field name"; return false; }
    out->nullable = f.scalar<uint8_t>(1, 0) != 0;
    const int tt = f.scalar<uint8_t>(2, 0);
    const bool dict = f.field(4) != 0;
    out->n_nodes = 1;
    out->dtype = -1;
    if (dict) { out->n_buffers = 2; return true; }   // stored as its index column; the dictionary lives in its own batches
    FbTable ty;
    const bool has_ty = f.table(3, &ty);
    int own = 0;
    bool nested = false;
    switch (tt) {
        case T_Null: own = 0; break;
        case T_Int: {
            own = 2;
            if (has_ty) {
                const int bw = ty.scalar<int32_t>(0, 0);
                const bool sg = ty.scalar<uint8_t>(1, 0) != 0;
                const int k = bw == 8 ? 0 : bw == 16 ? 1 : bw == 32 ? 2 : bw == 64 ? 3 : -1;
                if (k >= 0) out->dtype = sg ? (BDF_I8 + k) : (BDF_U8 + k);
            }
            break;
        }
        case T_FloatingPoint: {
            own = 2;
            const int prec = has_ty ? ty.scalar<int16_t>(0, 0) : 0;   // HALF, SINGLE, DOUBLE
            if (prec == 1) out->dtype = BDF_F32;
            if (prec == 2) out->dtype = BDF_F64;
            break;
        }
        case T_Bool: own = 2; out->dtype = BDF_BOOL; break;
        case T_Date: {   // Schema.fbs: Date { unit: DateUnit = MILLISECOND }, DAY = 0
            own = 2;
            const int unit = has_ty ? ty.scalar<int16_t>(0, 1) : 1;
            if (unit == 0) { out->temporal_kind = BDF_DATE32; out->temporal_dtype = BDF_I32; }
            if (unit == 1) { out->temporal_kind = BDF_DATE64; out->temporal_unit = BDF_MILLISECOND; out->temporal_dtype = BDF_I64; }
            break;
        }
        case T_Time: {   // Time { unit: TimeUnit = MILLISECOND; bitWidth: int = 32 }
            own = 2;
            const int unit = has_ty ? ty.scalar<int16_t>(0, 1) : 1;
            const int bw = has_ty ? ty.scalar<int32_t>(1, 32) : 32;
            if (bw == 32 && (unit == BDF_SECOND || unit == BDF_MILLISECOND)) { out->temporal_kind = BDF_TIME32; out->temporal_dtype = BDF_I32; }
            if (bw == 64 && (unit == BDF_MICROSECOND || unit == BDF_NANOSECOND)) { out->temporal_kind = BDF_TIME64; out->temporal_dtype = BDF_I64; }
            out->temporal_unit = out->temporal_kind ? unit : 0;
            break;
        }
        case T_Timestamp: {   // Timestamp { unit: TimeUnit; timezone: string }
            own = 2;
            const int unit = has_ty ? ty.scalar<int16_t>(0, 0) : 0;
            // a timezone string that does not decode leaves the field stepped over (kind 0): the file still opens, as it did before
            // temporal columns were read
            const bool tz_ok = !(has_ty && ty.field(1)) || ty.str(1, &out->tz);
            if (unit >= BDF_SECOND && unit <= BDF_NANOSECOND && tz_ok) {
                out->temporal_kind = BDF_TIMESTAMP; out->temporal_unit = unit; out->temporal_dtype = BDF_I64;
                out->has_tz = has_ty && ty.field(1) != 0;
            }
            break;
        }
        case T_Decimal: case T_Interval: case T_FixedSizeBinary: case T_Duration: own = 2; break;
        case T_Binary: case T_Utf8: case T_LargeBinary: case T_LargeUtf8: own = 3; break;
        case T_List: case T_LargeList: case T_Map: own = 2; nested = true; break;
        case T_Struct: case T_FixedSizeList: own = 1; nested = true; break;
        default: *why = "column '" + out->name + "' has a type this reader cannot skip (union / view / run-end encoded)"; return false;
    }
    out->n_buffers = own;
    if (nested) {
        size_t first; uint32_t cnt;
        if (!f.vec(5, &first, &cnt, 4)) { *why = "bad children vector"; return false; }
        for (uint32_t i = 0; i < cnt; i++) {
            uint32_t o;
            FbTable ch;
            if (!f.b->rd(first + 4 * i, &o) || !ch.init(f.b, first + 4 * i + o)) { *why = "bad child field"; return false; }
            IpcField c;
            if (!parse_field(ch, &c, depth + 1, budget, why)) return false;
            out->n_nodes += c.n_nodes;
            out->n_buffers += c.n_buffers;
            // List<T> of one numeric child T: the list path (bdf_ipc_read_list); every other nested type stays outside
            if (tt == T_List && cnt == 1 && c.dtype >= BDF_I8 && c.dtype <= BDF_F64) out->list_child = c.dtype;
        }
    }
    return true;
}

struct IpcBuf { int64_t off = 0, len = 0; };
struct IpcColChunk {
    int64_t len = 0, null_count = 0;
    IpcBuf validity, values;            // a List<T> column: values = its Int32 offsets
    int64_t child_len = 0, child_nulls = 0;
    IpcBuf child_validity, child_values;
    bool list_ok = true;                // a List column: its buffers fit the batch (checked by bdf_ipc_read_list)
};
struct IpcBatch {
    int64_t rows = 0;
    size_t body = 0;          // file offset of the body
    int64_t body_len = 0;
    std::vector<IpcColChunk> cols;   // top-level columns; entries of skipped columns stay zero
};

int dtype_bytes(int dtype, int64_t len, int64_t* out) {
    static const int w[10] = {1, 2, 4, 8, 1, 2, 4, 8, 4, 8};
    if (dtype == BDF_BOOL) { *out = (len + 7) / 8; return 0; }
    if (dtype < 0 || dtype > 9) return -1;
    *out = len * w[dtype];
    return 0;
}

}  // namespace

namespace bdf {
bool arrow_schema_fields(const uint8_t* p, size_t n, std::vector<ArrowField>* out) {
    if (n < 8) return false;
    size_t at = 0;
    int32_t word;
    memcpy(&word, p, 4);
    if (word == -1) { at = 4; memcpy(&word, p + 4, 4); }
    at += 4;
    if (word <= 0 || (size_t)word > n - at) return false;
    const FbBuf mb{p + at, (size_t)word};
    uint32_t root;
    FbTable msg, schema;
    if (!mb.rd(0, &root) || !msg.init(&mb, root) || msg.scalar<uint8_t>(1, 0) != 1 || !msg.table(2, &schema)) return false;
    size_t first; uint32_t cnt;
    if (!schema.vec(1, &first, &cnt, 4)) return false;
    int64_t budget = (int64_t)word / 8 + 16;
    for (uint32_t i = 0; i < cnt; i++) {
        uint32_t o;
        FbTable ft;
        if (!mb.rd(first + 4 * i, &o) || !ft.init(&mb, first + 4 * i + o)) return false;
        IpcField fld;
        std::string why;
        if (!parse_field(ft, &fld, 0, &budget, &why)) return false;
        out->push_back(ArrowField{fld.name, fld.temporal_kind, fld.temporal_unit, fld.has_tz, fld.tz});
    }
    return true;
}
}  // namespace bdf

struct bdf_ipc {
    int fd = -1;
    const uint8_t* map = nullptr;
    size_t size = 0;
    std::vector<IpcField> fields;
    std::vector<IpcBatch> batches;
    int64_t rows = 0;
};

#pragma GCC visibility push(default)
extern "C" {

void bdf_ipc_close(bdf_ipc* f) {
    if (!f) return;
    if (f->map) munmap((void*)f->map, f->size);
    if (f->fd >= 0) close(f->fd);
    delete f;
}

int bdf_ipc_open(const char* path, bdf_ipc** out) {
    if (!path || !out) return ipc_fail(BDF_INVALID, "null argument");
    *out = nullptr;
    bdf_ipc* f = new (std::nothrow) bdf_ipc();
    if (!f) return ipc_fail(BDF_OOM, "host allocation failed");
    struct Guard { bdf_ipc* f; ~Guard() { if (f) bdf_ipc_close(f); } } guard{f};
    f->fd = open(path, O_RDONLY | O_CLOEXEC);
    if (f->fd < 0) return ipc_fail(BDF_INVALID, "cannot open %s: %s", path, strerror(errno));
    struct stat st;
    if (fstat(f->fd, &st) != 0) return ipc_fail(BDF_INVALID, "cannot stat %s: %s", path, strerror(errno));
    f->size = (size_t)st.st_size;
    if (f->size < 8 + 4 + 6) return ipc_fail(BDF_INVALID, "%s is too short to be an Arrow IPC file", path);
    void* m = mmap(nullptr, f->size, PROT_READ, MAP_PRIVATE, f->fd, 0);
    if (m == MAP_FAILED) return ipc_fail(BDF_INVALID, "cannot map %s: %s", path, strerror(errno));
    f->map = (const uint8_t*)m;
    madvise(m, f->size, MADV_SEQUENTIAL);
    if (memcmp(f->map, "ARROW1", 6) != 0 || memcmp(f->map + f->size - 6, "ARROW1", 6) != 0)
        return ipc_fail(BDF_INVALID, "%s is not an Arrow IPC file (magic ARROW1 missing; the stream format has no footer)", path);
    int32_t flen;
    memcpy(&flen, f->map + f->size - 10, 4);
    if (flen <= 0 || (size_t)flen > f->size - 18) return ipc_fail(BDF_INVALID, "bad footer length %d", flen);
    const FbBuf fb{f->map + f->size - 10 - (size_t)flen, (size_t)flen};
    uint32_t root;
    FbTable footer, schema;
    if (!fb.rd(0, &root) || !footer.init(&fb, root)) return ipc_fail(BDF_INVALID, "malformed footer");
    if (!footer.table(1, &schema)) return ipc_fail(BDF_INVALID, "footer without schema");
    if (schema.scalar<int16_t>(0, 0) != 0) return ipc_fail(BDF_UNSUPPORTED, "big-endian IPC file");
    size_t first; uint32_t cnt;
    if (!schema.vec(1, &first, &cnt, 4)) return ipc_fail(BDF_INVALID, "malformed schema");
    int64_t nodes_per_batch = 0, buffers_per_batch = 0;
    int64_t field_budget = (int64_t)flen / 8 + 16;   // a Field table cannot be smaller than its vtable + offset
    for (uint32_t i = 0; i < cnt; i++) {
        uint32_t o;
        FbTable ft;
        if (!fb.rd(first + 4 * i, &o) || !ft.init(&fb, first + 4 * i + o)) return ipc_fail(BDF_INVALID, "malformed field %u", i);
        IpcField fld;
        std::string why;
        if (!parse_field(ft, &fld, 0, &field_budget, &why)) return ipc_fail(BDF_UNSUPPORTED, "%s", why.c_str());
        nodes_per_batch += fld.n_nodes;
        buffers_per_batch += fld.n_buffers;
        f->fields.push_back(std::move(fld));
    }
    // record batch blocks: struct Block { offset: long; metaDataLength: int; bodyLength: long } (24 bytes)
    size_t bfirst; uint32_t bcnt;
    if (!footer.vec(3, &bfirst, &bcnt, 24)) return ipc_fail(BDF_INVALID, "malformed record batch index");
    for (uint32_t k = 0; k < bcnt; k++) {
        int64_t off, body_len; int32_t meta_len;
        fb.rd(bfirst + 24 * (size_t)k, &off); fb.rd(bfirst + 24 * (size_t)k + 8, &meta_len); fb.rd(bfirst + 24 * (size_t)k + 16, &body_len);
        // overflow-free: every term is compared with what is left of the file, nothing is added up first
        if (off < 8 || meta_len < 8 || body_len < 0 || (uint64_t)off > f->size || (uint64_t)meta_len > f->size - (uint64_t)off ||
            (uint64_t)body_len > f->size - (uint64_t)off - (uint64_t)meta_len)
            return ipc_fail(BDF_INVALID, "record batch %u lies outside the file", k);
        // encapsulated message: [0xFFFFFFFF] <int32 metadata size> <flatbuffer> <padding> <body>
        size_t p = (size_t)off;
        int32_t word;
        memcpy(&word, f->map + p, 4);
        if (word == -1) { p += 4; memcpy(&word, f->map + p, 4); }
        p += 4;
        if (word <= 0 || p + (size_t)word > (size_t)off + (size_t)meta_len) return ipc_fail(BDF_INVALID, "record batch %u: bad metadata size", k);
        const FbBuf mb{f->map + p, (size_t)word};
        FbTable msg, rb;
        if (!mb.rd(0, &root) || !msg.init(&mb, root)) return ipc_fail(BDF_INVALID, "record batch %u: malformed message", k);
        if (msg.scalar<uint8_t>(1, 0) != 3 || !msg.table(2, &rb)) return ipc_fail(BDF_INVALID, "block %u is not a RecordBatch message", k);
        if (rb.field(3)) return ipc_fail(BDF_UNSUPPORTED, "compressed IPC bodies are not supported (write the file uncompressed)");
        IpcBatch b;
        b.rows = rb.scalar<int64_t>(0, 0);
        if (b.rows < 0 || b.rows > (int64_t)f->size * 8) return ipc_fail(BDF_INVALID, "record batch %u: impossible row count %lld", k, (long long)b.rows);
        b.body = (size_t)off + (size_t)meta_len;
        b.body_len = body_len;
        size_t nfirst, bufirst; uint32_t ncnt, bucnt;
        if (!rb.vec(1, &nfirst, &ncnt, 16) || !rb.vec(2, &bufirst, &bucnt, 16)) return ipc_fail(BDF_INVALID, "record batch %u: malformed nodes/buffers", k);
        if ((int64_t)ncnt != nodes_per_batch || (int64_t)bucnt != buffers_per_batch)
            return ipc_fail(BDF_INVALID, "record batch %u: %u nodes / %u buffers, the schema needs %lld / %lld", k, ncnt, bucnt, (long long)nodes_per_batch, (long long)buffers_per_batch);
        b.cols.resize(f->fields.size());
        size_t ni = 0, bi = 0;
        for (size_t c = 0; c < f->fields.size(); c++) {
            const IpcField& fld = f->fields[c];
            if (fld.dtype >= 0 || fld.list_child >= 0 || fld.temporal_kind) {
                IpcColChunk& cc = b.cols[c];
                mb.rd(nfirst + 16 * ni, &cc.len); mb.rd(nfirst + 16 * ni + 8, &cc.null_count);
                mb.rd(bufirst + 16 * bi, &cc.validity.off); mb.rd(bufirst + 16 * bi + 8, &cc.validity.len);
                mb.rd(bufirst + 16 * (bi + 1), &cc.values.off); mb.rd(bufirst + 16 * (bi + 1) + 8, &cc.values.len);
                int64_t need = cc.len > 0 ? (cc.len + 1) * 4 : 0;   // a list's offsets (a list array without lists may have none)
                if (fld.dtype >= 0) dtype_bytes(fld.dtype, cc.len, &need);
                if (fld.temporal_kind) dtype_bytes(fld.temporal_dtype, cc.len, &need);
                const bool has_v = cc.null_count > 0;
                // offsets and lengths come from the file: compare each with what is left of the body (off + len may wrap)
                auto fits = [body_len](const IpcBuf& bf, int64_t min_len) {
                    return bf.off >= 0 && bf.len >= min_len && bf.off <= body_len && bf.len <= body_len - bf.off;
                };
                const bool ok = cc.len == b.rows && cc.null_count >= 0 && cc.null_count <= cc.len && fits(cc.values, need) &&
                                (!has_v || fits(cc.validity, (cc.len + 7) / 8));
                // a List or temporal column is only checked when it is read: a file whose such column that reader cannot use still opens
                if (!ok && fld.dtype >= 0)
                    return ipc_fail(BDF_INVALID, "record batch %u, column '%s': buffers do not fit the batch", k, fld.name.c_str());
                cc.list_ok = ok;
                if (fld.list_child >= 0 && ok) {   // the child's node and buffers follow the list's
                    mb.rd(nfirst + 16 * (ni + 1), &cc.child_len); mb.rd(nfirst + 16 * (ni + 1) + 8, &cc.child_nulls);
                    mb.rd(bufirst + 16 * (bi + 2), &cc.child_validity.off); mb.rd(bufirst + 16 * (bi + 2) + 8, &cc.child_validity.len);
                    mb.rd(bufirst + 16 * (bi + 3), &cc.child_values.off); mb.rd(bufirst + 16 * (bi + 3) + 8, &cc.child_values.len);
                    int64_t cneed = 0;
                    dtype_bytes(fld.list_child, cc.child_len, &cneed);
                    cc.list_ok = cc.child_len >= 0 && cc.child_nulls >= 0 && cc.child_nulls <= cc.child_len && fits(cc.child_values, cneed) &&
                                 (cc.child_nulls == 0 || fits(cc.child_validity, (cc.child_len + 7) / 8));
                }
            }
            ni += fld.n_nodes;
            bi += fld.n_buffers;
        }
        f->rows += b.rows;
        f->batches.push_back(std::move(b));
    }
    guard.f = nullptr;
    *out = f;
    return BDF_OK;
}

int bdf_ipc_describe(const bdf_ipc* f, int32_t* n_columns, int64_t* n_batches, int64_t* n_rows) {
    if (!f) return ipc_fail(BDF_INVALID, "null argument");
    if (n_columns) *n_columns = (int32_t)f->fields.size();
    if (n_batches) *n_batches = (int64_t)f->batches.size();
    if (n_rows) *n_rows = f->rows;
    return BDF_OK;
}

int bdf_ipc_column(const bdf_ipc* f, int32_t col, const char** name, int32_t* dtype, int32_t* nullable) {
    if (!f || col < 0 || (size_t)col >= f->fields.size()) return ipc_fail(BDF_INVALID, "column index out of range");
    if (name) *name = f->fields[col].name.c_str();
    if (dtype) *dtype = f->fields[col].dtype;
    if (nullable) *nullable = f->fields[col].nullable;
    return BDF_OK;
}

int bdf_ipc_batch_rows(const bdf_ipc* f, int64_t batch, int64_t* rows) {
    if (!f || !rows || batch < 0 || (size_t)batch >= f->batches.size()) return ipc_fail(BDF_INVALID, "batch index out of range");
    *rows = f->batches[batch].rows;
    return BDF_OK;
}

int bdf_ipc_view(const bdf_ipc* f, int64_t batch, int32_t col, bdf_view* out) {
    if (!f || !out || batch < 0 || (size_t)batch >= f->batches.size() || col < 0 || (size_t)col >= f->fields.size())
        return ipc_fail(BDF_INVALID, "batch/column index out of range");
    if (f->fields[col].dtype < 0) return ipc_fail(BDF_UNSUPPORTED, "column '%s' has a type outside the numeric path", f->fields[col].name.c_str());
    const IpcBatch& b = f->batches[batch];
    const IpcColChunk& c = b.cols[col];
    out->values = f->map + b.body + c.values.off;
    out->validity = c.null_count > 0 ? f->map + b.body + c.validity.off : nullptr;
    out->len = c.len;
    out->offset = 0;
    out->null_count = c.null_count;
    return BDF_OK;
}

int bdf_ipc_read_batches(bdf_ctx* ctx, const bdf_ipc* f, int32_t n_cols, const int32_t* cols, int64_t n_batches, const int64_t* batches, int flags,
                         bdf_col** out) {
    if (!ctx || !f || !cols || !out || n_cols <= 0 || n_batches < 0 || (n_batches && !batches)) return ipc_fail(BDF_INVALID, "null argument");
    std::vector<std::vector<bdf_view>> views((size_t)n_cols);
    std::vector<const bdf_view*> vp((size_t)n_cols);
    std::vector<int32_t> dtypes((size_t)n_cols);
    std::vector<int64_t> nch((size_t)n_cols, n_batches);
    for (int32_t i = 0; i < n_cols; i++) {
        if (cols[i] < 0 || (size_t)cols[i] >= f->fields.size()) return ipc_fail(BDF_INVALID, "column index out of range");
        dtypes[i] = f->fields[cols[i]].dtype;
        views[i].resize((size_t)std::max<int64_t>(n_batches, 1));
        for (int64_t b = 0; b < n_batches; b++) {
            const int st = bdf_ipc_view(f, batches[b], cols[i], &views[i][b]);
            if (st != BDF_OK) return st;
        }
        vp[i] = views[i].data();
    }
    return bdf_upload_many(ctx, n_cols, dtypes.data(), nch.data(), vp.data(), flags, out);
}

int bdf_ipc_read_list(bdf_ctx* ctx, const bdf_ipc* f, int32_t col, int flags, bdf_list** out) {
    if (!ctx || !f || !out) return ipc_fail(BDF_INVALID, "null argument");
    if (col < 0 || (size_t)col >= f->fields.size()) return ipc_fail(BDF_INVALID, "column index out of range");
    const int dt = f->fields[col].list_child;
    if (dt < 0) return ipc_fail(BDF_UNSUPPORTED, "column '%s' is not a List of a numeric type", f->fields[col].name.c_str());
    std::vector<bdf_list_view> views(std::max<size_t>(f->batches.size(), 1));
    for (size_t b = 0; b < f->batches.size(); b++) {
        const IpcBatch& bt = f->batches[b];
        const IpcColChunk& c = bt.cols[col];
        if (!c.list_ok) return ipc_fail(BDF_INVALID, "record batch %zu, column '%s': list buffers do not fit the batch", b, f->fields[col].name.c_str());
        const uint8_t* body = f->map + bt.body;
        views[b].offsets = c.len > 0 ? (const int32_t*)(body + c.values.off) : nullptr;
        views[b].validity = c.null_count > 0 ? body + c.validity.off : nullptr;
        views[b].len = c.len;
        views[b].offset = 0;
        views[b].null_count = c.null_count;
        views[b].values = bdf_view{body + c.child_values.off, c.child_nulls > 0 ? body + c.child_validity.off : nullptr, c.child_len, 0, c.child_nulls};
    }
    return bdf_list_upload(ctx, dt, (int64_t)f->batches.size(), views.data(), flags, out);
}

int bdf_ipc_list_column(const bdf_ipc* f, int32_t col, int32_t* dtype) {
    if (!f || !dtype || col < 0 || (size_t)col >= f->fields.size()) return ipc_fail(BDF_INVALID, "column index out of range");
    *dtype = f->fields[col].list_child < 0 ? -1 : BDF_LIST_BASE + f->fields[col].list_child;
    return BDF_OK;
}

int bdf_ipc_temporal_column(const bdf_ipc* f, int32_t col, bdf_temporal_type* out) {
    if (!f || !out || col < 0 || (size_t)col >= f->fields.size()) return ipc_fail(BDF_INVALID, "column index out of range");
    const IpcField& fld = f->fields[col];
    *out = bdf_temporal_type{fld.temporal_kind, fld.temporal_unit, fld.has_tz ? fld.tz.c_str() : nullptr};
    return BDF_OK;
}

int bdf_ipc_read_temporal(bdf_ctx* ctx, const bdf_ipc* f, int32_t col, int flags, bdf_col** out) {
    if (!ctx || !f || !out) return ipc_fail(BDF_INVALID, "null argument");
    if (col < 0 || (size_t)col >= f->fields.size()) return ipc_fail(BDF_INVALID, "column index out of range");
    const IpcField& fld = f->fields[col];
    if (!fld.temporal_kind) return ipc_fail(BDF_UNSUPPORTED, "column '%s' is not a Date, Time or Timestamp column", fld.name.c_str());
    std::vector<bdf_view> views(std::max<size_t>(f->batches.size(), 1));
    for (size_t b = 0; b < f->batches.size(); b++) {
        const IpcBatch& bt = f->batches[b];
        const IpcColChunk& c = bt.cols[col];
        if (!c.list_ok) return ipc_fail(BDF_INVALID, "record batch %zu, column '%s': buffers do not fit the batch", b, fld.name.c_str());
        views[b] = bdf_view{f->map + bt.body + c.values.off, c.null_count > 0 ? f->map + bt.body + c.validity.off : nullptr, c.len, 0, c.null_count};
    }
    const int32_t dt = fld.temporal_dtype;
    const int64_t nch = (int64_t)f->batches.size();
    const bdf_view* vp = views.data();
    return bdf_upload_many(ctx, 1, &dt, &nch, &vp, flags, out);
}

int bdf_ipc_read(bdf_ctx* ctx, const bdf_ipc* f, int32_t n_cols, const int32_t* cols, int flags, bdf_col** out) {
    if (!f) return ipc_fail(BDF_INVALID, "null argument");
    std::vector<int64_t> all(f->batches.size());
    for (size_t b = 0; b < all.size(); b++) all[b] = (int64_t)b;
    return bdf_ipc_read_batches(ctx, f, n_cols, cols, (int64_t)all.size(), all.data(), flags, out);
}

}  // extern "C"
#pragma GCC visibility pop

// ---- write side ------------------------------------------------------------------------------------------------
namespace {

// Minimal flatbuffers writer, front to back: a table is laid out before the objects it refers to, reference fields
// are patched once the target exists (uoffsets point forward, the vtable sits right before its table).
struct FbOut {
    std::vector<uint8_t> b;
    template <typename T> void put(T v) { const uint8_t* p = (const uint8_t*)&v; b.insert(b.end(), p, p + sizeof v); }
    template <typename T> void set(size_t at, T v) { memcpy(&b[at], &v, sizeof v); }
    void pad_to(size_t a) { while (b.size() % a) b.push_back(0); }
    void link(size_t ref_pos, size_t target) { set<uint32_t>(ref_pos, (uint32_t)(target - ref_pos)); }
};
struct FbF { int id; int size; uint64_t bits; };   // size 0 = reference (4 bytes, patched later)

// Returns the table position; ref_pos receives the absolute position of every reference field, in `fields` order.
size_t fb_table(FbOut& o, const std::vector<FbF>& fields, std::vector<size_t>* ref_pos) {
    int max_id = -1;
    for (const FbF& f : fields) max_id = f.id > max_id ? f.id : max_id;
    const size_t vt_len = 4 + 2 * (size_t)(max_id + 1);
    std::vector<uint16_t> offs((size_t)(max_id + 1), 0);
    size_t off = 4;
    std::vector<size_t> at(fields.size());
    for (size_t i = 0; i < fields.size(); i++) {
        const size_t sz = fields[i].size ? (size_t)fields[i].size : 4;
        off = (off + sz - 1) / sz * sz;
        at[i] = off; offs[fields[i].id] = (uint16_t)off;
        off += sz;
    }
    const size_t tsize = (off + 3) / 4 * 4;
    o.pad_to(2);
    while ((o.b.size() + vt_len) % 8) o.b.push_back(0);
    const size_t vt = o.b.size();
    o.put<uint16_t>((uint16_t)vt_len); o.put<uint16_t>((uint16_t)tsize);
    for (uint16_t x : offs) o.put<uint16_t>(x);
    const size_t t = o.b.size();
    o.b.resize(t + tsize, 0);
    o.set<int32_t>(t, (int32_t)(t - vt));
    if (ref_pos) ref_pos->clear();
    for (size_t i = 0; i < fields.size(); i++) {
        if (fields[i].size == 0) { if (ref_pos) ref_pos->push_back(t + at[i]); }
        else memcpy(&o.b[t + at[i]], &fields[i].bits, (size_t)fields[i].size);
    }
    return t;
}
size_t fb_string(FbOut& o, const std::string& s) {
    o.pad_to(4);
    const size_t p = o.b.size();
    o.put<uint32_t>((uint32_t)s.size());
    o.b.insert(o.b.end(), s.begin(), s.end());
    o.b.push_back(0);
    return p;
}
size_t fb_struct_vec(FbOut& o, const void* data, uint32_t count, size_t elem) {   // 8-byte aligned elements
    o.pad_to(4);
    while ((o.b.size() + 4) % 8) o.b.push_back(0);
    const size_t p = o.b.size();
    o.put<uint32_t>(count);
    const uint8_t* d = (const uint8_t*)data;
    o.b.insert(o.b.end(), d, d + (size_t)count * elem);
    return p;
}

size_t fb_field(FbOut& o, const char* name, int dt, const bdf_temporal_type* type);

// Schema table (fields of primitive, boolean, temporal or List<numeric> type) at the current end of `o`; returns its position.
size_t fb_schema(FbOut& o, int n_cols, const char* const* names, const int32_t* dtypes, const bdf_temporal_type* types) {
    std::vector<size_t> refs;
    const size_t schema = fb_table(o, {{1, 0, 0}}, &refs);
    o.pad_to(4);
    const size_t vec = o.b.size();
    o.link(refs[0], vec);
    o.put<uint32_t>((uint32_t)n_cols);
    const size_t slots = o.b.size();
    o.b.resize(slots + 4 * (size_t)n_cols, 0);
    for (int c = 0; c < n_cols; c++) {
        const size_t field = fb_field(o, names[c], dtypes[c], types ? &types[c] : nullptr);
        o.link(slots + 4 * (size_t)c, field);
    }
    return schema;
}

// One nullable Field; a List<T> (dtype BDF_LIST_BASE + T) has one child field, pyarrow's "item" of type T.
size_t fb_field(FbOut& o, const char* name, int dt, const bdf_temporal_type* type) {
    const int kind = type ? type->kind : 0;
    const bool list = dt >= BDF_LIST_BASE;
    uint8_t tt = list ? T_List : dt == BDF_BOOL ? T_Bool : (dt == BDF_F32 || dt == BDF_F64) ? T_FloatingPoint : T_Int;
    if (kind == BDF_DATE32 || kind == BDF_DATE64) tt = T_Date;
    if (kind == BDF_TIME32 || kind == BDF_TIME64) tt = T_Time;
    if (kind == BDF_TIMESTAMP) tt = T_Timestamp;
    std::vector<size_t> fr;
    // Field: name(0) nullable(1) type_type(2) type(3) children(5)
    const size_t field = fb_table(o, {{0, 0, 0}, {1, 1, 1}, {2, 1, tt}, {3, 0, 0}, {5, 0, 0}}, &fr);
    o.link(fr[0], fb_string(o, name));
    size_t ty;
    if (tt == T_Bool) ty = fb_table(o, {}, nullptr);
    else if (tt == T_Date) ty = fb_table(o, {{0, 2, (uint64_t)(kind == BDF_DATE32 ? 0 : 1)}}, nullptr);
    else if (tt == T_Time) ty = fb_table(o, {{0, 2, (uint64_t)type->unit}, {1, 4, (uint64_t)(kind == BDF_TIME32 ? 32 : 64)}}, nullptr);
    else if (tt == T_Timestamp) {
        std::vector<size_t> tr;
        if (type->tz) {
            ty = fb_table(o, {{0, 2, (uint64_t)type->unit}, {1, 0, 0}}, &tr);
            o.link(tr[0], fb_string(o, type->tz));
        } else ty = fb_table(o, {{0, 2, (uint64_t)type->unit}}, nullptr);
    }
    else if (tt == T_FloatingPoint) ty = fb_table(o, {{0, 2, (uint64_t)(dt == BDF_F32 ? 1 : 2)}}, nullptr);
    else if (tt == T_List) ty = fb_table(o, {}, nullptr);
    else {
        static const int bw[8] = {8, 16, 32, 64, 8, 16, 32, 64};
        ty = fb_table(o, {{0, 4, (uint64_t)bw[dt]}, {1, 1, (uint64_t)(dt <= BDF_I64 ? 1 : 0)}}, nullptr);
    }
    o.link(fr[1], ty);
    o.pad_to(4);
    o.link(fr[2], o.b.size());
    o.put<uint32_t>(list ? 1 : 0);   // children
    if (list) {
        const size_t slot = o.b.size();
        o.put<uint32_t>(0);
        o.link(slot, fb_field(o, "item", dt - BDF_LIST_BASE, nullptr));
    }
    return field;
}

struct Block { int64_t offset; int32_t meta_len; int32_t pad; int64_t body_len; };

// Bits [bit0, bit0+n) of src, re-based to bit 0 of dst (dst zero padded to whole bytes).
void copy_bits(const uint8_t* src, int64_t bit0, int64_t n, uint8_t* dst) {
    const int64_t nbytes = (n + 7) / 8;
    if (nbytes == 0) return;
    const int sh = (int)(bit0 & 7);
    const uint8_t* s = src + (bit0 >> 3);
    if (sh == 0) memcpy(dst, s, (size_t)nbytes);
    else {
        const int64_t last_src = (bit0 + n - 1) >> 3;   // index of the last source byte that holds a wanted bit
        for (int64_t i = 0; i < nbytes; i++) {
            const uint8_t lo = s[i];
            const uint8_t hi = ((bit0 >> 3) + i + 1 <= last_src) ? s[i + 1] : 0;
            dst[i] = (uint8_t)((lo >> sh) | (hi << (8 - sh)));
        }
    }
    if (n & 7) dst[nbytes - 1] &= (uint8_t)((1u << (n & 7)) - 1u);
}

// What one column contributes to one RecordBatch, and where its buffers land in the file.
struct ChunkSpec {
    int64_t rows = 0, nulls = 0;
    bool has_validity = false;            // a validity buffer is written (always when nulls > 0)
    int64_t validity_pos = 0, values_pos = 0;   // absolute file offsets (filled by plan_file)
    int64_t validity_len = 0, values_len = 0;
    // a List<T> column: the offsets, then the child's node and buffers
    int64_t offsets_pos = 0, offsets_len = 0;
    int64_t child_rows = 0, child_nulls = 0;
    bool child_has_validity = false;
    int64_t child_validity_pos = 0, child_values_pos = 0, child_validity_len = 0, child_values_len = 0;
};

// The whole file is laid out before a byte of data moves: metadata is small and known up front, so the file can be
// sized, mapped, and the body buffers produced IN PLACE (memcpy from host views, or device->host copies that land
// directly in the page cache).  Bodies start on 64-byte file offsets; padding stays zero (ftruncate).
struct FilePlan {
    struct Piece { int64_t pos; std::vector<uint8_t> bytes; };
    std::vector<Piece> meta;   // magic, framed messages, EOS, footer, trailer
    int64_t size = 0;
};

void frame_message(FilePlan* plan, int64_t* pos, const FbOut& fb, int32_t* meta_len) {
    // continuation marker, metadata size, flatbuffer, zero padding up to the next 64-byte file offset
    const int64_t after = (*pos + 8 + (int64_t)fb.b.size() + 63) / 64 * 64;
    const int32_t mlen = (int32_t)(after - *pos - 8);
    FilePlan::Piece pc{*pos, {}};
    const int32_t marker = -1;
    pc.bytes.insert(pc.bytes.end(), (const uint8_t*)&marker, (const uint8_t*)&marker + 4);
    pc.bytes.insert(pc.bytes.end(), (const uint8_t*)&mlen, (const uint8_t*)&mlen + 4);
    pc.bytes.insert(pc.bytes.end(), fb.b.begin(), fb.b.end());
    plan->meta.push_back(std::move(pc));
    *meta_len = mlen + 8;
    *pos = after;
}

// The Schema message flatbuffer (before framing).
FbOut schema_message(int n_cols, const char* const* names, const int32_t* dtypes, const bdf_temporal_type* types) {
    FbOut fb;
    fb.put<uint32_t>(0);
    std::vector<size_t> refs;
    const size_t msg = fb_table(fb, {{0, 2, 4 /* MetadataVersion::V5 */}, {1, 1, 1 /* Schema */}, {2, 0, 0}, {3, 8, 0}}, &refs);
    fb.link(0, msg);
    fb.link(refs[0], fb_schema(fb, n_cols, names, dtypes, types));
    fb.pad_to(8);
    return fb;
}

void plan_file(int n_cols, const char* const* names, const int32_t* dtypes, const bdf_temporal_type* types, int64_t n_batches,
               std::vector<std::vector<ChunkSpec>>& spec, FilePlan* plan) {
    int64_t pos = 0;
    plan->meta.push_back({0, {'A', 'R', 'R', 'O', 'W', '1', 0, 0}});
    pos = 8;
    {   // schema message
        int32_t ml;
        frame_message(plan, &pos, schema_message(n_cols, names, dtypes, types), &ml);
    }
    std::vector<Block> blocks;
    for (int64_t b = 0; b < n_batches; b++) {
        const int64_t rows = spec[0][b].rows;
        struct Node { int64_t len, nulls; };
        struct Buf { int64_t off, len; };
        std::vector<Node> nodes;
        std::vector<Buf> bufs;
        int64_t body = 0;
        auto buffer = [&](int64_t len, int64_t* pos) {   // positions are relative for now
            bufs.push_back({body, len});
            *pos = body;
            body += (len + 63) / 64 * 64;
        };
        for (int c = 0; c < n_cols; c++) {
            ChunkSpec& cs = spec[c][b];
            const bool list = dtypes[c] >= BDF_LIST_BASE;
            nodes.push_back({rows, cs.nulls});
            cs.validity_len = cs.has_validity ? (rows + 7) / 8 : 0;
            buffer(cs.validity_len, &cs.validity_pos);
            if (list) {   // List<T>: validity, offsets; then the child node with its validity and values
                cs.offsets_len = 4 * (rows + 1);
                buffer(cs.offsets_len, &cs.offsets_pos);
                nodes.push_back({cs.child_rows, cs.child_nulls});
                cs.child_validity_len = cs.child_has_validity ? (cs.child_rows + 7) / 8 : 0;
                buffer(cs.child_validity_len, &cs.child_validity_pos);
                dtype_bytes(dtypes[c] - BDF_LIST_BASE, cs.child_rows, &cs.child_values_len);
                buffer(cs.child_values_len, &cs.child_values_pos);
            } else {
                dtype_bytes(dtypes[c], rows, &cs.values_len);
                buffer(cs.values_len, &cs.values_pos);
            }
        }
        FbOut fb;
        fb.put<uint32_t>(0);
        std::vector<size_t> mr, rr;
        const size_t msg = fb_table(fb, {{0, 2, 4}, {1, 1, 3 /* RecordBatch */}, {2, 0, 0}, {3, 8, (uint64_t)body}}, &mr);
        fb.link(0, msg);
        const size_t rb = fb_table(fb, {{0, 8, (uint64_t)rows}, {1, 0, 0}, {2, 0, 0}}, &rr);
        fb.link(mr[0], rb);
        fb.link(rr[0], fb_struct_vec(fb, nodes.data(), (uint32_t)nodes.size(), 16));
        fb.link(rr[1], fb_struct_vec(fb, bufs.data(), (uint32_t)bufs.size(), 16));
        fb.pad_to(8);
        Block blk{pos, 0, 0, body};
        frame_message(plan, &pos, fb, &blk.meta_len);
        for (int c = 0; c < n_cols; c++)
            for (int64_t* p : {&spec[c][b].validity_pos, &spec[c][b].values_pos, &spec[c][b].offsets_pos, &spec[c][b].child_validity_pos,
                               &spec[c][b].child_values_pos})
                *p += pos;
        pos += body;
        blocks.push_back(blk);
    }
    // end-of-stream marker, footer, footer size, magic
    FbOut fb;
    fb.put<uint32_t>(0);
    std::vector<size_t> fr;
    const size_t footer = fb_table(fb, {{0, 2, 4}, {1, 0, 0}, {2, 0, 0}, {3, 0, 0}}, &fr);   // version, schema, dictionaries, recordBatches
    fb.link(0, footer);
    fb.link(fr[0], fb_schema(fb, n_cols, names, dtypes, types));
    fb.link(fr[1], fb_struct_vec(fb, nullptr, 0, 24));
    fb.link(fr[2], fb_struct_vec(fb, blocks.data(), (uint32_t)blocks.size(), 24));
    fb.pad_to(8);
    FilePlan::Piece tail{pos, {}};
    const int32_t eos[2] = {-1, 0};
    const int32_t flen = (int32_t)fb.b.size();
    tail.bytes.insert(tail.bytes.end(), (const uint8_t*)eos, (const uint8_t*)eos + 8);
    tail.bytes.insert(tail.bytes.end(), fb.b.begin(), fb.b.end());
    tail.bytes.insert(tail.bytes.end(), (const uint8_t*)&flen, (const uint8_t*)&flen + 4);
    tail.bytes.insert(tail.bytes.end(), {'A', 'R', 'R', 'O', 'W', '1'});
    plan->size = pos + (int64_t)tail.bytes.size();
    plan->meta.push_back(std::move(tail));
}

// A new file of the planned size, mapped read/write, metadata already in place.  The data goes to `<path>.tmp.<pid>`
// whose blocks are RESERVED up front (posix_fallocate: a full disk is an error return here, not a SIGBUS on the first
// store through the mapping); commit() renames it over `path`, any failure before that unlinks it, so `path` either
// keeps its old contents or holds a complete file.
struct OutFile {
    int fd = -1;
    uint8_t* map = nullptr;
    size_t size = 0;
    std::string tmp;
    int open_planned(const char* path, const FilePlan& plan) {
        tmp = std::string(path) + ".tmp." + std::to_string((long long)getpid());
        fd = open(tmp.c_str(), O_RDWR | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
        if (fd < 0) { const int e = errno; tmp.clear(); return ipc_fail(BDF_INVALID, "cannot create %s: %s", path, strerror(e)); }
        size = (size_t)plan.size;
        const int fe = posix_fallocate(fd, 0, (off_t)size);
        if (fe != 0) return ipc_fail(fe == ENOSPC || fe == EDQUOT ? BDF_OOM : BDF_INVALID, "cannot reserve %zu bytes for %s: %s", size, path, strerror(fe));
        void* m = mmap(nullptr, size, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
        if (m == MAP_FAILED) return ipc_fail(BDF_INVALID, "cannot map %s: %s", path, strerror(errno));
        map = (uint8_t*)m;
        for (const FilePlan::Piece& pc : plan.meta) memcpy(map + pc.pos, pc.bytes.data(), pc.bytes.size());
        return BDF_OK;
    }
    // status: what the caller has seen so far; the file is published only when everything succeeded
    int commit(const char* path, int status) {
        int st = status;
        if (map && munmap(map, size) != 0 && st == BDF_OK) st = ipc_fail(BDF_INVALID, "unmapping %s failed: %s", path, strerror(errno));
        map = nullptr;
        if (fd >= 0 && close(fd) != 0 && st == BDF_OK) st = ipc_fail(BDF_INVALID, "closing %s failed: %s", path, strerror(errno));
        fd = -1;
        if (st == BDF_OK && rename(tmp.c_str(), path) != 0) st = ipc_fail(BDF_INVALID, "cannot move the finished file to %s: %s", path, strerror(errno));
        if (st != BDF_OK && !tmp.empty()) unlink(tmp.c_str());
        tmp.clear();
        return st;
    }
    ~OutFile() {
        if (map) munmap(map, size);
        if (fd >= 0) close(fd);
        if (!tmp.empty()) unlink(tmp.c_str());   // abandoned before commit
    }
};

}  // namespace

namespace bdf {
std::string arrow_schema_message(int n_cols, const char* const* names, const int32_t* dtypes, const bdf_temporal_type* types) {
    FilePlan plan;
    int64_t pos = 0;
    int32_t ml;
    frame_message(&plan, &pos, schema_message(n_cols, names, dtypes, types), &ml);
    const std::vector<uint8_t>& b = plan.meta[0].bytes;
    std::string s(b.begin(), b.end());
    s.resize((size_t)pos, '\0');   // the framing pads the message to a multiple of 64 bytes
    return s;
}
}  // namespace bdf

#pragma GCC visibility push(default)
extern "C" {

int bdf_ipc_write_host(const char* path, int32_t n_cols, const char* const* names, const int32_t* dtypes, int64_t n_batches,
                       const bdf_view* const* cols) {
    if (!path || !names || !dtypes || n_cols <= 0 || n_batches < 0 || (n_batches && !cols)) return ipc_fail(BDF_INVALID, "null argument");
    std::vector<std::vector<ChunkSpec>> spec((size_t)n_cols, std::vector<ChunkSpec>((size_t)n_batches));
    for (int c = 0; c < n_cols; c++) {
        if (!names[c] || !((dtypes[c] >= 0 && dtypes[c] <= 9) || dtypes[c] == BDF_BOOL)) return ipc_fail(BDF_INVALID, "column %d: bad name or dtype", c);
        for (int64_t b = 0; b < n_batches; b++) {
            const bdf_view& v = cols[c][b];
            if (v.len != cols[0][b].len || v.len < 0 || v.offset < 0)
                return ipc_fail(BDF_LENGTH_MISMATCH, "batch %lld: column '%s' has %lld rows, column '%s' has %lld", (long long)b, names[c],
                                (long long)v.len, names[0], (long long)cols[0][b].len);
            int64_t nulls = v.validity ? v.null_count : 0;
            if (v.validity && nulls < 0) {
                nulls = 0;
                for (int64_t i = 0; i < v.len; i++) nulls += !((v.validity[(v.offset + i) >> 3] >> ((v.offset + i) & 7)) & 1);
            }
            spec[c][b].rows = v.len; spec[c][b].nulls = nulls; spec[c][b].has_validity = nulls > 0;
        }
    }
    FilePlan plan;
    plan_file(n_cols, names, dtypes, nullptr, n_batches, spec, &plan);
    OutFile of;
    const int st = of.open_planned(path, plan);
    if (st != BDF_OK) return st;
    static const int w[10] = {1, 2, 4, 8, 1, 2, 4, 8, 4, 8};
    for (int c = 0; c < n_cols; c++)
        for (int64_t b = 0; b < n_batches; b++) {
            const bdf_view& v = cols[c][b];
            const ChunkSpec& cs = spec[c][b];
            if (cs.validity_len) copy_bits(v.validity, v.offset, cs.rows, of.map + cs.validity_pos);
            if (!cs.values_len) continue;
            if (dtypes[c] == BDF_BOOL) copy_bits((const uint8_t*)v.values, v.offset, cs.rows, of.map + cs.values_pos);
            else memcpy(of.map + cs.values_pos, (const uint8_t*)v.values + v.offset * w[dtypes[c]], (size_t)cs.values_len);
        }
    return of.commit(path, BDF_OK);
}

int bdf_ipc_write(bdf_ctx* ctx, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols) {
    return bdf_ipc_write_typed(ctx, path, n_cols, names, cols, nullptr);
}

int bdf_ipc_write_typed(bdf_ctx* ctx, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols,
                        const bdf_temporal_type* types) {
    if (!cols) return ipc_fail(BDF_INVALID, "null argument");
    return bdf_ipc_write_lists(ctx, path, n_cols, names, cols, types, nullptr);
}

int bdf_ipc_write_lists(bdf_ctx* ctx, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols,
                        const bdf_temporal_type* types, const bdf_list* const* lists) {
    if (!ctx || !path || !names || !cols || n_cols <= 0) return ipc_fail(BDF_INVALID, "null argument");
    std::vector<int32_t> dtypes((size_t)n_cols);
    std::vector<std::vector<ChunkSpec>> spec((size_t)n_cols);
    int64_t n_batches = -1;
    for (int c = 0; c < n_cols; c++) {
        int64_t nch = 0, total = 0;
        const bdf_list* l = lists ? lists[c] : nullptr;
        if (!(l ? !cols[c] : cols[c] != nullptr) || !names[c]) return ipc_fail(BDF_INVALID, "column %d: null column or name, or both a column and a list", c);
        if (l && types && types[c].kind) return ipc_fail(BDF_INVALID, "list column '%s' cannot carry a temporal type", names[c]);
        int st = l ? bdf_list_describe(l, &dtypes[c], &nch, &total) : bdf_col_describe(cols[c], &dtypes[c], &nch, &total);
        if (st != BDF_OK) return st;
        if (l) dtypes[c] += BDF_LIST_BASE;
        if (types && types[c].kind) {   // the same validation as the temporal functions' (bdf_temporal_result)
            int32_t rd = 0;
            st = bdf_temporal_result(BDF_TEMPORAL_UNIX_TIMESTAMP, &types[c], 0, &rd, nullptr);
            if (st == BDF_UNSUPPORTED) st = bdf_temporal_result(BDF_TEMPORAL_HOUR, &types[c], 0, &rd, nullptr);   // time kinds
            if (st != BDF_OK) return st;
            const int phys = (types[c].kind == BDF_DATE32 || types[c].kind == BDF_TIME32) ? BDF_I32 : BDF_I64;
            if (dtypes[c] != phys) return ipc_fail(BDF_INVALID, "column '%s' of dtype %d does not hold temporal kind %d", names[c], dtypes[c], types[c].kind);
        }
        if (n_batches < 0) n_batches = nch;
        if (nch != n_batches) return ipc_fail(BDF_LENGTH_MISMATCH, "columns have different numbers of chunks (%lld, %lld)", (long long)nch, (long long)n_batches);
        spec[c].resize((size_t)nch);
        for (int64_t b = 0; b < nch; b++) {
            int64_t len = 0, nulls = 0; int32_t hv = 0;
            ChunkSpec& cs = spec[c][b];
            if (l) {
                int64_t ne = 0, cl = 0, cn = 0; int32_t chv = 0;
                st = bdf_list_chunk_info(ctx, l, b, &len, &nulls, &ne);
                if (st == BDF_OK) st = bdf_col_chunk_info(ctx, bdf_list_values(l), b, &cl, &cn, &chv);
                if (st != BDF_OK) return st;
                hv = nulls > 0;
                cs.child_rows = cl; cs.child_nulls = chv ? cn : 0; cs.child_has_validity = chv != 0;
            } else {
                st = bdf_col_chunk_info(ctx, cols[c], b, &len, &nulls, &hv);
                if (st != BDF_OK) return st;
            }
            if (len != spec[0][b].rows && c > 0)
                return ipc_fail(BDF_LENGTH_MISMATCH, "chunk %lld: column '%s' has %lld rows, column '%s' has %lld", (long long)b, names[c], (long long)len,
                                names[0], (long long)spec[0][b].rows);
            cs.rows = len; cs.nulls = hv ? nulls : 0; cs.has_validity = hv != 0;
        }
    }
    FilePlan plan;
    plan_file(n_cols, names, dtypes.data(), types, n_batches, spec, &plan);
    OutFile of;
    int st = of.open_planned(path, plan);
    if (st != BDF_OK) return st;
    // device -> host copies land in the mapping: every column's chunks go to their final place in the file
    std::vector<std::vector<bdf_out>> outs((size_t)n_cols);
    std::vector<std::vector<bdf_list_out>> louts((size_t)n_cols);
    std::vector<std::vector<uint8_t>> unused_bits;   // the bitmap of a list chunk without a null list is downloaded, not written
    for (int c = 0; c < n_cols; c++) {
        const size_t nb = (size_t)std::max<int64_t>(n_batches, 1);
        if (lists && lists[c]) louts[c].resize(nb);
        else outs[c].resize(nb);
        for (int64_t b = 0; b < n_batches; b++) {
            const ChunkSpec& cs = spec[c][b];
            if (lists && lists[c]) {
                uint8_t* lv = of.map + cs.validity_pos;
                if (!cs.has_validity) {
                    unused_bits.emplace_back((size_t)(cs.rows + 7) / 8 + 8);
                    lv = unused_bits.back().data();
                }
                louts[c][b] = bdf_list_out{(int32_t*)(of.map + cs.offsets_pos), lv, of.map + cs.child_values_pos,
                                           cs.child_has_validity ? of.map + cs.child_validity_pos : nullptr, 0, 0, 0, 0};
            } else {
                outs[c][b] = bdf_out{of.map + cs.values_pos, cs.has_validity ? of.map + cs.validity_pos : nullptr, cs.rows, 0, 0};
            }
        }
    }
    int begun = 0;
    for (; begun < n_cols && st == BDF_OK; begun++)
        if (!(lists && lists[begun])) st = bdf_download_begin(ctx, cols[begun], outs[begun].data());
    if (st != BDF_OK) begun--;   // the failing column never started
    for (int c = 0; c < begun; c++) {
        const int s2 = lists && lists[c] ? bdf_list_download(ctx, lists[c], louts[c].data()) : bdf_download_end(ctx, cols[c], outs[c].data());
        if (st == BDF_OK) st = s2;
    }
    return of.commit(path, st);
}

}  // extern "C"
#pragma GCC visibility pop
