// oracle/compaction.cc — TEST INFRASTRUCTURE (CPU oracle). Not part of the product path.
//
// CPU restatement of Cassandra's compaction hot path for big-format `oa` SSTables, driven by the same manifest struct as
// the product's C ABI (include/b200c.h) so that tests can hand both sides identical inputs and compare outputs byte for byte.
// One call = one CompactionTask.runMayThrow hot loop (S/db/compaction/CompactionTask.java:184-236), single threaded as the
// reference is. S/ = src/java/org/apache/cassandra/ of the reference. Each block cites the file:line it follows.
//
// Scope restated: simple regular and static columns, multi-cell and counter regular columns, tombstoneOption NONE, no 2i
// (rowProcessingNeeded() == false), forward order. Anything else returns B200C_EUNSUPPORTED — same envelope as the GPU engine.
#include "codec.h"
#include "../include/b200c.h"
#include "parallel.h"
#include <cstring>
#include <vector>
#include <string>
#include <algorithm>
#include <chrono>
#include <climits>
#include <memory>
#include <map>
#include <cmath>

namespace oracle {

static const int64_t NO_TS = INT64_MIN;          // LivenessInfo.NO_TIMESTAMP
static const int64_t NO_DEL = INT64_MAX;         // Cell.NO_DELETION_TIME / LivenessInfo.NO_EXPIRATION_TIME
static const int32_t EXPIRED_TTL = INT32_MAX;    // LivenessInfo.EXPIRED_LIVENESS_TTL

// ---- DeletionTime: S/db/DeletionTime.java:46 (LIVE), :158-176 (supersedes/deletes) -------------------------------
struct DT {
    int64_t mfda = INT64_MIN; int64_t ldt = INT64_MAX;
    bool live() const { return mfda == INT64_MIN && ldt == INT64_MAX; }
    bool supersedes(const DT& o) const { return mfda > o.mfda || (mfda == o.mfda && ldt > o.ldt); }
    bool deletes(int64_t ts) const { return ts <= mfda; }
    bool operator==(const DT& o) const { return mfda == o.mfda && ldt == o.ldt; }
};
// ---- LivenessInfo: S/db/LivenessInfo.java:40-340 ----------------------------------------------------------------------
struct Live {
    int64_t ts = NO_TS; int32_t ttl = 0; int64_t ldt = NO_DEL;
    bool empty() const { return ts == NO_TS; }
    bool expiring() const { return ttl != 0; }
    bool expired() const { return ttl == EXPIRED_TTL; }
    bool is_live(int64_t now) const { if (empty()) return false; if (expired()) return false; if (expiring()) return now < ldt; return true; }
    // :216-225
    bool supersedes(const Live& o) const {
        if (ts != o.ts) return ts > o.ts;
        if (expired() != o.expired()) return expired();
        if (expiring() == o.expiring()) return ldt > o.ldt;
        return expiring();
    }
};
struct Val { const uint8_t* p = nullptr; int32_t len = 0; bool null = false; };
struct Clust { uint8_t kind = 4; int n = 0; Val v[B200C_MAX_CLUSTERING]; };
struct CellV {
    int col; int64_t ts; int32_t ttl; int64_t ldt; const uint8_t* val; int32_t vlen;
    const uint8_t* path = nullptr; int32_t plen = 0;                   // cell path: cells of multi-cell columns only (Cell.path())
    bool tombstone() const { return ldt != NO_DEL && ttl == 0; }       // AbstractCell.java:58-61
    bool expiring() const { return ttl != 0; }
    bool is_live(int64_t now) const { return ldt == NO_DEL || (ttl != 0 && now < ldt); }   // :53-56
};
struct Unf {
    bool is_row = true;
    Clust c;
    // row
    Live info; DT del; std::vector<CellV> cells;        // cells in (column, path) order
    std::vector<std::pair<int, DT>> cdel;             // multi-cell columns of this row that carry a complex deletion (non-live), by column
    bool has_column(int col) const { for (const CellV& c : cells) if (c.col == col) return true; for (auto& d : cdel) if (d.first == col) return true; return false; }
    DT complex_deletion(int col) const { for (auto& d : cdel) if (d.first == col) return d.second; return DT(); }
    bool has_data() const { return !cells.empty() || !cdel.empty(); }
    // marker: bound -> dt_open or dt_close by kind; boundary -> both
    DT m_close, m_open;
    std::vector<std::shared_ptr<std::vector<uint8_t>>> owned;      // merged counter contexts this row's cells point into (they have no place in an input stream)
};

// ClusteringPrefix.Kind: S/db/ClusteringPrefix.java:65-82
enum { K_EXCL_END = 0, K_INCL_START = 1, K_EXCL_END_INCL_START = 2, K_STATIC = 3, K_CLUSTERING = 4, K_INCL_END_EXCL_START = 5, K_INCL_END = 6, K_EXCL_START = 7 };
static inline int kind_comparison(int k) { static const int c[8] = {0, 0, 0, 1, 2, 3, 3, 3}; return c[k]; }
static inline int kind_vs_clustering(int k) { static const int c[8] = {-1, -1, -1, -1, 0, 1, 1, 1}; return c[k]; }
static inline bool kind_is_boundary(int k) { return k == K_EXCL_END_INCL_START || k == K_INCL_END_EXCL_START; }
static inline bool kind_is_start(int k) { return k == K_INCL_START || k == K_EXCL_START; }

struct Schema {
    int nclust; b200c_column clust[B200C_MAX_CLUSTERING];
    int ncols; b200c_column cols[B200C_MAX_COLUMNS];
    int nstat; b200c_column stat[B200C_MAX_STATIC_COLUMNS];      // static columns (SerializationHeader.columns(true))
    int ncomplex = 0;                                             // multi-cell columns among cols[] (they follow the simple ones)
};

// multi-cell columns (include/b200c.h B200C_COLUMN_COMPLEX / _FIXED): class and fixed length of the cell values / of the cell paths
static inline bool col_complex(const b200c_column& t) { return ((t.type >> 8) & 0xFF) != 0; }
static inline b200c_column col_value_type(const b200c_column& t) { return b200c_column{t.type & 0xFF, t.fixed_len & 0xFFFF}; }
static inline b200c_column col_path_type(const b200c_column& t) { return b200c_column{((t.type >> 8) & 0xFF) - 1, (int32_t)((uint32_t)t.fixed_len >> 16)}; }
// AbstractType.compare for the supported comparison classes (S/db/marshal/AbstractType.java:212-215; LongType.compareLongs:
// empty < non-empty, first byte signed then unsigned bytes; BytesType/UTF8Type: unsigned lexicographic)
static int compare_value(const b200c_column& t, const Val& a, const Val& b) {
    if (t.type == B200C_TYPE_TIMEUUID) {              // AbstractTimeUUIDType.compareCustom S/db/marshal/AbstractTimeUUIDType.java:58-87,126-144
        const bool pa = a.len == 16, pb = b.len == 16;
        if (!(pa && pb)) return pa ? 1 : (pb ? -1 : 0);
        auto be64 = [](const uint8_t* p) { uint64_t v = 0; for (int i = 0; i < 8; i++) v = (v << 8) | p[i]; return v; };
        auto reorder = [](uint64_t x) { return (int64_t)((x << 48) | ((x << 16) & 0xFFFF00000000ull) | (x >> 32)); };
        const int64_t m1 = reorder(be64(a.p)), m2 = reorder(be64(b.p));
        if (m1 != m2) return m1 < m2 ? -1 : 1;
        const int64_t l1 = (int64_t)(be64(a.p + 8) ^ 0x0080808080808080ull), l2 = (int64_t)(be64(b.p + 8) ^ 0x0080808080808080ull);
        return l1 == l2 ? 0 : (l1 < l2 ? -1 : 1);
    }
    if (t.type == B200C_TYPE_FIXED_SIGNED || t.type == B200C_TYPE_VAR_SIGNED) {
        if (a.len == 0 || b.len == 0) return a.len == 0 ? (b.len == 0 ? 0 : -1) : 1;
        int d = (int)(int8_t)a.p[0] - (int)(int8_t)b.p[0];
        if (d) return d < 0 ? -1 : 1;
        int n = std::min(a.len, b.len);
        int c = memcmp(a.p + 1, b.p + 1, n - 1);
        if (c) return c < 0 ? -1 : 1;
        return a.len == b.len ? 0 : (a.len < b.len ? -1 : 1);
    }
    int n = std::min(a.len, b.len);
    int c = n ? memcmp(a.p, b.p, n) : 0;
    if (c) return c < 0 ? -1 : 1;
    return a.len == b.len ? 0 : (a.len < b.len ? -1 : 1);
}
// ClusteringComparator.compare: S/db/ClusteringComparator.java:140-157,184-192
static int compare_clust(const Schema& s, const Clust& a, const Clust& b) {
    int m = std::min(a.n, b.n);
    for (int i = 0; i < m; i++) {
        const Val& x = a.v[i]; const Val& y = b.v[i];
        if (x.null) { if (!y.null) return -1; continue; }
        if (y.null) return 1;
        int c = compare_value(s.clust[i], x, y);
        if (c) return c;
    }
    if (a.n == b.n) { int d = kind_comparison(a.kind) - kind_comparison(b.kind); return d < 0 ? -1 : (d > 0 ? 1 : 0); }
    return a.n < b.n ? kind_vs_clustering(a.kind) : -kind_vs_clustering(b.kind);
}

// ---- input side ---------------------------------------------------------------------------------------------------------
struct Source {
    int idx;
    const b200c_input* in;
    // uncompressed Data stream: allocated uninitialised and decompressed chunk by chunk on first touch (CompressedChunkReader reads
    // chunks on demand too, S/io/util/CompressedChunkReader.java:103-173), so a token sub-range only pays for the chunks it crosses
    // A token sub-range allocates only the span of the stream it can touch (span0 .. span0 + span bytes, chunk aligned): thousands of range
    // tasks each mapping a whole-file buffer would serialise on the kernel's address-space lock.
    // The buffer comes from a per-thread pool that only grows (one slot per input): the range tasks of the parallel driver (parallel.cc) would
    // otherwise mmap / munmap a few MiB per input and task, and on a 128-thread host those address-space operations serialise all the threads.
    uint8_t* buf = nullptr; uint64_t dlen = 0, span0 = 0, span1 = 0;
    std::vector<bool> have_chunk;
    const uint8_t* dptr() const { return buf - span0; }       // biased: dptr() + stream offset, valid for offsets in [span0, span1)
    uint8_t* wptr() { return buf - span0; }
    uint64_t dsize() const { return dlen; }
    void need(uint64_t lo, uint64_t hi);      // make bytes [lo, hi) of the stream available
    uint64_t pos = 0;               // cursor: start of the current partition
    // Index.db cursor (BigTableScanner walks Index.db: S/io/sstable/format/big/BigTableScanner.java:135-184)
    uint64_t ipos = 0;
    // current partition
    bool has = false;
    const uint8_t* key = nullptr; int keylen = 0; int64_t token = 0;
    bool has_prev = false; int64_t prev_token = 0; const uint8_t* prev_key = nullptr; int prev_klen = 0;
    DT pdel; uint64_t upos = 0;     // cursor inside the partition (next unfiltered)
    Unf stat; bool has_stat = false;     // the partition's static row (non-empty)
    const struct Schema* schema = nullptr;
    uint64_t part_start = 0, part_end = 0;
    uint64_t range_bytes = 0;       // uncompressed bytes of the partitions inside the token range (scanner accounting)
};

struct Reader {
    const uint8_t* p; const uint8_t* end; int input;
    uint8_t u8() { need(1); return *p++; }
    uint16_t u16() { need(2); uint16_t v = (uint16_t)((p[0] << 8) | p[1]); p += 2; return v; }
    uint64_t vint() { uint64_t v; int n = vint_read(p, end, &v); if (n < 0) throw Corrupt{input, 4, 0, 0, "truncated vint"}; p += n; return v; }
    // readUnsignedVInt32 = checkedCast(readUnsignedVInt): S/utils/vint/VIntCoding.java:269-272
    int32_t vint32() { uint64_t v = vint(); int32_t r = (int32_t)v; if ((int64_t)r != (int64_t)v) throw Corrupt{input, 4, 0, 0, "vint32 out of range"}; return r; }
    void need(size_t n) { if ((size_t)(end - p) < n) throw Corrupt{input, 4, 0, 0, "truncated data"}; }
    const uint8_t* bytes(size_t n) { need(n); const uint8_t* r = p; p += n; return r; }
};

// ClusteringPrefix.Serializer.deserializeValuesWithoutSize: S/db/ClusteringPrefix.java:502-522 (header :548-562)
static void read_clust_values(Reader& r, const Schema& s, int n, Clust& c) {
    c.n = n;
    int off = 0;
    while (off < n) {
        int limit = std::min(n, off + 32);
        uint64_t header = r.vint();
        for (; off < limit; off++) {
            Val& v = c.v[off];
            int bit = (off % 32) * 2;          // shifts are modulo 64 in the reference (:555-559)
            if ((header >> (bit + 1)) & 1) { v = Val{nullptr, 0, true}; continue; }
            if ((header >> bit) & 1) { v = Val{r.p, 0, false}; continue; }
            const b200c_column& t = s.clust[off];
            int len = t.fixed_len > 0 ? t.fixed_len : (int)r.vint32();
            if (len < 0) throw Corrupt{r.input, 4, 0, 0, "negative value length"};
            v.p = r.bytes(len); v.len = len; v.null = false;
        }
    }
}

// header.readDeletionTime: S/db/SerializationHeader.java:186-206, then DeletionTime.build (S/db/DeletionTime.java:54-58): a negative local
// deletion time (the writer's (int) cast wrapped a delta of 2^31 or more) or one above Cell.MAX_DELETION_TIME reads as InvalidDeletionTime,
// whose ldt is INVALID_DELETION_TIME. Row deletions, range tombstone markers and complex deletions all come through here; the complex
// deletion's own "negative ldt" repair (UnfilteredSerializer.java:670-676) cannot fire on a value built this way.
static DT read_delta_dt(Reader& r, const b200c_encoding_stats& hs) {
    DT d; d.mfda = (int64_t)(r.vint() + (uint64_t)hs.min_timestamp); d.ldt = (int64_t)r.vint32() + hs.min_local_deletion_time;
    if (d.ldt < 0 || d.ldt > (int64_t)UINT32_MAX - 2) d.ldt = (int64_t)UINT32_MAX - 1;
    return d;
}

// DeletionTime.Serializer.deserialize (oa): S/db/DeletionTime.java:222-243
static DT read_partition_dt(Reader& r) {
    uint8_t flags = r.u8();
    if (flags & 0x80) { if (flags != 0x80) throw Corrupt{r.input, 4, 0, 0, "bad DeletionTime flags"}; return DT(); }
    const uint8_t* b = r.bytes(11);
    DT d; uint64_t m = flags; for (int i = 0; i < 7; i++) m = (m << 8) | b[i];
    d.mfda = (int64_t)m; d.ldt = (int64_t)(((uint32_t)b[7] << 24) | ((uint32_t)b[8] << 16) | ((uint32_t)b[9] << 8) | b[10]);
    return d;
}

// Cell.decodeLocalDeletionTime: S/db/rows/Cell.java:221-239 (messaging version >= 5.0 for oa)
static int64_t decode_ldt(int64_t ldt, int32_t ttl) {
    if (ldt >= ttl) return ldt;
    if (ldt < 0) return (int64_t)(uint32_t)(int32_t)ldt;
    if (ttl == EXPIRED_TTL) return ldt;
    return (int64_t)UINT32_MAX - 1;    // INVALID_DELETION_TIME
}

// UnfilteredSerializer.deserialize: S/db/rows/UnfilteredSerializer.java:433-645. Returns false at end of partition.
// UnfilteredSerializer.deserializeRowBody :574-650 (sizes, liveness, deletion, columns subset, cells) for the regular or the static column set
static void read_row_body(Reader& r, Source& src, uint8_t flags, int ncols_in, const int32_t* colmap, const b200c_column* types, Unf& u) {
    const b200c_encoding_stats& hs = src.in->header_stats;
    r.vint(); r.vint();                                   // row size, previous unfiltered size
    u.info = Live(); u.del = DT();
    if (flags & 0x04) u.info.ts = (int64_t)(r.vint() + (uint64_t)hs.min_timestamp);
    if (flags & 0x08) {                                   // the liveness ldt is decoded as a cell's is (:596-598)
        u.info.ttl = r.vint32() + hs.min_ttl; u.info.ldt = decode_ldt((int64_t)r.vint32() + hs.min_local_deletion_time, u.info.ttl);
    }
    if (flags & 0x10) u.del = read_delta_dt(r, hs);
    uint64_t missing = 0;
    if (!(flags & 0x20)) {                                // Columns.deserializeSubset: S/db/Columns.java:533-560
        if (ncols_in >= 64) throw Unsupported{">= 64 columns"};
        missing = r.vint();
    }
    u.cells.clear(); u.cdel.clear();
    auto read_cell = [&](int oc, const b200c_column& t, bool complex) {      // Cell.Serializer.deserialize: S/db/rows/Cell.java:307-349
        const b200c_column vt = col_value_type(t);
        uint8_t cf = r.u8();
        bool has_value = !(cf & 0x04), deleted = cf & 0x01, expiring = cf & 0x02, use_ts = cf & 0x08, use_ttl = cf & 0x10;
        CellV c; c.col = oc;
        c.ts = use_ts ? u.info.ts : (int64_t)(r.vint() + (uint64_t)hs.min_timestamp);
        c.ldt = use_ttl ? u.info.ldt : ((deleted || expiring) ? (int64_t)r.vint32() + hs.min_local_deletion_time : NO_DEL);
        c.ttl = use_ttl ? u.info.ttl : (expiring ? r.vint32() + hs.min_ttl : 0);
        if (complex) {                                   // :330-332 column.cellPathSerializer().deserialize: CollectionPathSerializer = vint length + bytes (fixed-length types: bare)
            const b200c_column pt = col_path_type(t);
            int plen = pt.fixed_len > 0 ? pt.fixed_len : (int)r.vint32();
            if (plen < 0) throw Corrupt{src.idx, 4, 0, 0, "negative path length"};
            c.path = r.bytes(plen); c.plen = plen;
        }
        c.val = r.p; c.vlen = 0;
        if (has_value) {
            int len = vt.fixed_len > 0 ? vt.fixed_len : (int)r.vint32();
            if (len < 0) throw Corrupt{src.idx, 4, 0, 0, "negative value length"};
            c.val = r.bytes(len); c.vlen = len;
        }
        if (c.ttl < 0) throw Corrupt{src.idx, 4, 0, 0, "Invalid TTL"};
        if (c.ldt != NO_DEL) c.ldt = decode_ldt(c.ldt, c.ttl);
        u.cells.push_back(c);
    };
    for (int i = 0; i < ncols_in; i++) {
        if ((missing >> i) & 1) continue;
        int oc = colmap[i];
        const b200c_column& t = types[oc];
        if (!col_complex(t)) { read_cell(oc, t, false); continue; }
        // UnfilteredSerializer.readComplexColumn :652-672: [complex deletion when the row says HAS_COMPLEX_DELETION] vint count, cells.
        // ComplexColumnData.Builder.build :350-356: a column with a live deletion and no cell does not exist.
        DT cd;
        if (flags & 0x40) cd = read_delta_dt(r, hs);
        int64_t count = (int64_t)r.vint32();
        if (count < 0) throw Corrupt{src.idx, 4, 0, 0, "negative cell count"};
        for (int64_t k = 0; k < count; k++) read_cell(oc, t, true);
        // BTreeRow.Builder's CellResolver (S/db/rows/BTreeRow.java:770-778) keeps a complex deletion only if its timestamp is above Long.MIN_VALUE:
        // LIVE, written by a row that has a complex deletion in another column, reads back as (MIN_VALUE, InvalidDeletionTime) and is dropped there
        if (cd.mfda != INT64_MIN) u.cdel.push_back({oc, cd});
    }
    std::stable_sort(u.cells.begin(), u.cells.end(), [](const CellV& a, const CellV& b) { return a.col < b.col; });
    std::sort(u.cdel.begin(), u.cdel.end(), [](const std::pair<int, DT>& a, const std::pair<int, DT>& b) { return a.first < b.first; });
}
static bool read_unfiltered_one(Source& src, const Schema& s, Unf& u);
static bool read_unfiltered(Source& src, const Schema& s, Unf& u) {
    // UnfilteredSerializer.deserialize :433-447: empty rows (e.g. all columns dropped) are skipped at read time
    for (;;) {
        if (!read_unfiltered_one(src, s, u)) return false;
        if (u.is_row && u.info.empty() && u.del.live() && !u.has_data()) continue;
        return true;
    }
}
static bool read_unfiltered_one(Source& src, const Schema& s, Unf& u) {
    const b200c_input& in = *src.in;
    Reader r{src.dptr() + src.upos, src.dptr() + src.part_end, src.idx};
    uint8_t flags = r.u8();
    if (flags & 0x01) { src.upos = r.p - src.dptr(); return false; }
    const b200c_encoding_stats& hs = in.header_stats;
    if (flags & 0x02) {
        u.is_row = false; u.cells.clear();
        u.c.kind = r.u8();
        if (u.c.kind > 7 || u.c.kind == K_STATIC || u.c.kind == K_CLUSTERING) throw Corrupt{src.idx, 4, 0, 0, "bad bound kind"};
        int n = r.u16();
        if (n > s.nclust) throw Corrupt{src.idx, 4, 0, 0, "bound size"};
        read_clust_values(r, s, n, u.c);
        r.vint(); r.vint();                                   // body size, previous unfiltered size
        if (kind_is_boundary(u.c.kind)) { u.m_close = read_delta_dt(r, hs); u.m_open = read_delta_dt(r, hs); }
        else if (kind_is_start(u.c.kind)) { u.m_open = read_delta_dt(r, hs); u.m_close = DT(); }
        else { u.m_close = read_delta_dt(r, hs); u.m_open = DT(); }
    } else {
        u.is_row = true;
        uint8_t ext = (flags & 0x80) ? r.u8() : 0;
        if (ext & 0x01) throw Corrupt{src.idx, 4, 0, 0, "static flag on a clustered row"};      // UnfilteredSerializer.deserialize :477-479
        if (ext & 0x02) throw Unsupported{"shadowable deletion"};
        if ((flags & 0x40) && !s.ncomplex) throw Unsupported{"complex deletion"};       // (a table without multi-cell columns has none)
        u.c.kind = K_CLUSTERING;
        read_clust_values(r, s, s.nclust, u.c);
        read_row_body(r, src, flags, in.ncolumns, in.column_map, s.cols, u);
    }
    src.upos = r.p - src.dptr();
    return true;
}

// CompressedChunkReader.readChunk: S/io/util/CompressedChunkReader.java:103-173
static void load_chunk(Source& src, uint64_t i) {
    const b200c_input& in = *src.in;
    const uint64_t nch = in.nchunks;
    uint64_t off = in.chunk_offsets[i];
    uint64_t next = (i + 1 < nch) ? in.chunk_offsets[i + 1] : in.data_len;
    if (off + 4 > next || next > in.data_len) throw Corrupt{src.idx, 2, i, off, "chunk bounds"};
    uint32_t clen = (uint32_t)(next - off - 4);
    const uint8_t* c = in.data + off;
    uint32_t stored = ((uint32_t)c[clen] << 24) | ((uint32_t)c[clen + 1] << 16) | ((uint32_t)c[clen + 2] << 8) | c[clen + 3];
    if (crc32_ieee(0, c, clen) != stored) throw Corrupt{src.idx, 1, i, off, "chunk CRC mismatch"};
    uint64_t ustart = i * (uint64_t)in.chunk_len;
    int ulen = (int)std::min<uint64_t>(in.chunk_len, in.data_length - ustart);
    if ((int64_t)clen >= (int64_t)in.max_compressed_len) {              // raw chunk (:116,219)
        if ((int)clen < ulen) throw Corrupt{src.idx, 2, i, off, "short raw chunk"};
        memcpy(src.wptr() + ustart, c, ulen);
    } else {
        int got = chunk_decompress(in.compressor, c, (int)clen, src.wptr() + ustart, ulen);
        if (got != ulen) throw Corrupt{src.idx, 2, i, off, "malformed compressed chunk"};
    }
    src.have_chunk[i] = true;
}
void Source::need(uint64_t lo, uint64_t hi) {
    if (hi > dlen) hi = dlen;
    if (lo >= hi) return;
    const uint64_t L = (uint64_t)in->chunk_len;
    if (lo < span0 || hi > span1) throw Corrupt{idx, 3, 0, lo, "Index.db position outside the range the Summary.db samples bracket"};
    for (uint64_t i = lo / L; i <= (hi - 1) / L; i++) if (!have_chunk[i]) load_chunk(*this, i);
}
static int64_t order_token(const uint8_t* key, int kl);
// data position stored in the Index.db entry at `off` (u16 keyLen | key | vint position | ...)
static uint64_t entry_position(const b200c_input& in, uint64_t off, int idx) {
    Reader r{in.index + off, in.index + in.index_len, idx};
    int kl = r.u16(); r.bytes(kl); return r.vint();
}
// Opens the stream for (tok_lo, tok_hi]. Ranged scanner: the Index.db walk starts at the last Summary.db sample whose token is <= tok_lo
// instead of at the file start and cannot pass the first sample whose token is > tok_hi (BigTableScanner seeks with the index summary too,
// S/io/sstable/format/big/BigTableScanner.java:105-132); the stream buffer covers exactly the chunks between those two samples.
static void open_source(Source& src, int64_t tok_lo, int64_t tok_hi) {
    const b200c_input& in = *src.in;
    uint64_t nch = in.nchunks; const uint64_t L = (uint64_t)in.chunk_len;
    if (nch != (in.data_length + in.chunk_len - 1) / L) throw Corrupt{src.idx, 2, 0, 0, "chunk count"};
    src.dlen = in.data_length; src.have_chunk.assign(nch, false);
    uint64_t lo = 0, hi = in.data_length;
    const bool whole = tok_lo == INT64_MIN && tok_hi == INT64_MAX;
    if (!whole && in.summary_positions && in.nsummary && in.index_len) {
        auto tok_at = [&](uint64_t k) { uint64_t off = in.summary_positions[k]; if (off + 2 > in.index_len) throw Corrupt{src.idx, 3, 0, off, "summary position"};
                                        int kl = (in.index[off] << 8) | in.index[off + 1]; if (off + 2 + kl > in.index_len) throw Corrupt{src.idx, 3, 0, off, "summary position"};
                                        return order_token(in.index + off + 2, kl); };
        uint64_t a = 0, b = in.nsummary;                                   // first sample with token > tok_lo
        if (tok_lo != INT64_MIN) while (a < b) { uint64_t mid = (a + b) / 2; if (tok_at(mid) <= tok_lo) a = mid + 1; else b = mid; }
        const uint64_t first = a ? a - 1 : 0;
        a = first; b = in.nsummary;                                        // first sample with token > tok_hi
        while (a < b) { uint64_t mid = (a + b) / 2; if (tok_at(mid) <= tok_hi) a = mid + 1; else b = mid; }
        src.ipos = in.summary_positions[first];
        lo = entry_position(in, in.summary_positions[first], src.idx);
        if (a < in.nsummary) hi = entry_position(in, in.summary_positions[a], src.idx);
        if (lo > hi || hi > in.data_length) throw Corrupt{src.idx, 3, 0, src.ipos, "Index.db positions"};
    }
    src.span0 = lo / L * L; src.span1 = std::min<uint64_t>(in.data_length, (hi + L - 1) / L * L);
    if (src.span1 < src.span0) src.span1 = src.span0;
    {
        struct Slot { std::unique_ptr<uint8_t[]> p; uint64_t cap = 0; };
        static thread_local std::vector<Slot> pool;
        if (pool.size() <= (size_t)src.idx) pool.resize((size_t)src.idx + 1);
        Slot& sl = pool[src.idx]; const uint64_t need = src.span1 - src.span0 + 64;
        if (sl.cap < need) { sl.p.reset(); sl.cap = need + need / 4; sl.p.reset(new uint8_t[sl.cap]); }      // uninitialised on purpose: nothing is read before its chunk was decoded
        src.buf = sl.p.get();
    }
    memset(src.buf + (src.span1 - src.span0), 0, 64);
    if (whole) src.need(0, in.data_length);                               // a whole-ring compaction reads (and checksums) every chunk, as the reference does
}

// the order-defining token: Murmur3Partitioner.getToken (S/dht/Murmur3Partitioner.java:256-296), or for ByteOrderedPartitioner
// (S/dht/ByteOrderedPartitioner.java: the token is the key) the sign-flipped big-endian 8-byte key prefix — an order-preserving stand-in
// whose ties compare_key() resolves on the full key bytes, i.e. exactly unsigned lexicographic key order
static thread_local int g_partitioner = B200C_PARTITIONER_MURMUR3;
static int64_t order_token(const uint8_t* key, int kl) {
    if (g_partitioner == B200C_PARTITIONER_MURMUR3) return murmur3_token(key, kl);
    uint64_t pre = 0; for (int q = 0; q < 8; q++) pre = (pre << 8) | (q < kl ? key[q] : 0);
    return (int64_t)(pre ^ 0x8000000000000000ull);
}
static void next_partition(Source& src, int64_t tok_lo, int64_t tok_hi) {
    const b200c_input& in = *src.in;
    for (;;) {
        if (src.ipos >= in.index_len) { src.has = false; return; }
        Reader ir{in.index + src.ipos, in.index + in.index_len, src.idx};
        try {
            int kl = ir.u16(); const uint8_t* key = ir.bytes(kl);
            uint64_t pos = ir.vint(); int32_t psize = ir.vint32();
            if (psize < 0) throw Corrupt{src.idx, 3, 0, src.ipos, "promoted index size"};
            ir.bytes(psize);
            src.ipos = ir.p - in.index;
            int64_t tok = order_token(key, kl);
            if (src.has_prev) {                        // SortedTableWriter.verifyPartition :165-178: keys strictly increase in (token, key bytes) order
                bool bad = tok < src.prev_token;
                if (!bad && tok == src.prev_token) { int n = std::min(kl, src.prev_klen); int c = n ? memcmp(src.prev_key, key, n) : 0; bad = c > 0 || (c == 0 && src.prev_klen >= kl); }
                if (bad) throw Corrupt{src.idx, 3, 0, src.ipos, "Index.db is not in partitioner order"};
            }
            src.has_prev = true; src.prev_token = tok; src.prev_key = key; src.prev_klen = kl;
            if (tok > tok_hi) { src.has = false; src.ipos = in.index_len; return; }     // sorted input: nothing further can be in range
            if (!(tok_lo == INT64_MIN || tok > tok_lo)) continue;
            // the partition ends where the next Index.db entry says the next one starts (or at the end of the stream)
            uint64_t end = src.dsize();
            if (src.ipos < in.index_len) {
                Reader nr{in.index + src.ipos, in.index + in.index_len, src.idx};
                int nkl = nr.u16(); nr.bytes(nkl); end = nr.vint();
            }
            if (end > src.dsize() || end <= pos || pos + 2 + kl > end) throw Corrupt{src.idx, 3, 0, src.ipos, "Index.db positions"};
            src.need(pos, end);
            const uint8_t* d = src.dptr();
            if (((d[pos] << 8) | d[pos + 1]) != kl || memcmp(d + pos + 2, key, kl) != 0)
                throw Corrupt{src.idx, 3, 0, src.ipos, "Index.db entry does not match Data.db"};
            Reader r{d + pos + 2 + kl, d + end, src.idx};
            src.pdel = read_partition_dt(r);                               // SSTableIdentityIterator.create :62-78
            src.has_stat = false;
            if (in.nstatic_columns > 0) {                                  // SSTableSimpleIterator.readStaticRow -> UnfilteredSerializer.deserializeStaticRow :538-552
                uint8_t flags = r.u8();
                if ((flags & 0x01) || (flags & 0x02) || !(flags & 0x80)) throw Corrupt{src.idx, 4, 0, 0, "static row flags"};
                uint8_t ext = r.u8();
                if (!(ext & 0x01)) throw Corrupt{src.idx, 4, 0, 0, "static row flags"};
                if ((ext & 0x02) || (flags & 0x40)) throw Unsupported{"shadowable / complex deletion"};
                src.stat.is_row = true; src.stat.c = Clust(); src.stat.c.kind = K_STATIC;
                read_row_body(r, src, flags, in.nstatic_columns, in.static_column_map, src.schema->stat, src.stat);
                src.has_stat = !(src.stat.info.empty() && src.stat.del.live() && src.stat.cells.empty());
            }
            src.key = d + pos + 2; src.keylen = kl; src.token = tok; src.part_start = pos; src.part_end = end;
            src.range_bytes += end - pos;
            src.upos = r.p - d;
            src.has = true;
            return;
        } catch (Corrupt& c) { if (c.kind == 4) { c.kind = 3; c.offset = src.ipos; } throw; }
    }
}

// DecoratedKey.compareTo: S/db/DecoratedKey.java:79-91
static int compare_key(const Source& a, const Source& b) {
    if (a.token != b.token) return a.token < b.token ? -1 : 1;
    int n = std::min(a.keylen, b.keylen);
    int c = n ? memcmp(a.key, b.key, n) : 0;
    if (c) return c < 0 ? -1 : 1;
    return a.keylen == b.keylen ? 0 : (a.keylen < b.keylen ? -1 : 1);
}

// ---- purge: PurgeFunction S/db/partitions/PurgeFunction.java:36-145 -------------------------------------------------------
struct Purger {
    int64_t now, gc_before, max_ts;
    // :39-42 with onlyPurgeRepairedTombstones = false; evaluator = ts < min timestamp of overlapping sstables (CompactionController.java:247-286)
    bool should_purge(int64_t ts, int64_t ldt) const { return ldt < gc_before && (max_ts == INT64_MAX || ts < max_ts); }
    bool should_purge(const DT& d) const { return !d.live() && should_purge(d.mfda, d.ldt); }       // DeletionPurger.java:28-31
    bool should_purge(const Live& l) const { return !l.is_live(now) && should_purge(l.ts, l.ldt); } // :33-36
};

// AbstractCell.purge: S/db/rows/AbstractCell.java:78-99. Returns false if the cell is dropped.
static bool purge_cell(CellV& c, const Purger& pg) {
    if (!c.is_live(pg.now)) {
        if (pg.should_purge(c.ts, c.ldt)) return false;
        if (c.expiring()) {                       // expired TTL cell -> tombstone with ldt - ttl, value dropped, then purged again
            c.ldt = c.ldt - c.ttl; c.ttl = 0; c.vlen = 0;
            if (!c.is_live(pg.now) && pg.should_purge(c.ts, c.ldt)) return false;
        }
    }
    return true;
}
// BTreeRow.purge: S/db/rows/BTreeRow.java:457-470,488-499. Returns false if the row disappears.
static bool purge_row(Unf& r, const Purger& pg) {
    if (pg.should_purge(r.info)) r.info = Live();
    if (pg.should_purge(r.del)) r.del = DT();
    size_t w = 0;
    for (size_t i = 0; i < r.cells.size(); i++) if (purge_cell(r.cells[i], pg)) r.cells[w++] = r.cells[i];
    r.cells.resize(w);
    // ComplexColumnData.purge S/db/rows/ComplexColumnData.java:212-216 (+ update :229-238): a purgeable complex deletion becomes LIVE; the column goes when nothing is left
    w = 0;
    for (size_t i = 0; i < r.cdel.size(); i++) if (!pg.should_purge(r.cdel[i].second)) r.cdel[w++] = r.cdel[i];
    r.cdel.resize(w);
    return !(r.info.empty() && r.del.live() && !r.has_data());
}
// PurgeFunction.applyToMarker :116-143. Returns false if the marker disappears.
static bool purge_marker(Unf& m, const Purger& pg) {
    if (kind_is_boundary(m.c.kind)) {
        bool pc = pg.should_purge(m.m_close), po = pg.should_purge(m.m_open);
        if (pc) {
            if (po) return false;
            m.c.kind = (m.c.kind == K_EXCL_END_INCL_START) ? K_INCL_START : K_EXCL_START;   // createCorrespondingOpenMarker
            m.m_close = DT();
            return true;
        }
        if (po) { m.c.kind = (m.c.kind == K_EXCL_END_INCL_START) ? K_EXCL_END : K_INCL_END; m.m_open = DT(); }   // ...CloseMarker
        return true;
    }
    const DT& d = kind_is_start(m.c.kind) ? m.m_open : m.m_close;
    return !pg.should_purge(d);
}

// ---- counter contexts: S/db/context/CounterContext.java ---------------------------------------------------------------
// context = [i16 n = number of header elements][n x i16 element][shards: 16-byte counter id, i64 clock, i64 count] (:40-58); element e >= 0: the shard
// with index e is LOCAL, e < 0: the shard with index e - Short.MIN_VALUE is GLOBAL; shards without an element are REMOTE. Shards are in id order.
namespace ctr {
enum { STEP = 32 };
static inline int be16s(const uint8_t* p) { return (int16_t)(((uint16_t)p[0] << 8) | p[1]); }
static inline int64_t be64s(const uint8_t* p) { uint64_t v = 0; for (int i = 0; i < 8; i++) v = (v << 8) | p[i]; return (int64_t)v; }
static inline int header_length(const uint8_t* c) { int n = be16s(c); return 2 + (n < 0 ? -n : n) * 2; }      // headerLength :173-176
struct State {                                                                // ContextState :757-914
    const uint8_t* c; int len, hlen, hoff, boff; bool global = false, local = false;
    State(const uint8_t* ctx, int n) : c(ctx), len(n) { hlen = boff = header_length(ctx); hoff = 2; upd(); }
    int index() const { return (boff - hlen) / STEP; }
    void upd() {                                                              // updateIsGlobalOrLocal :810-822
        if (hoff >= hlen) { global = local = false; return; }
        const int e = be16s(c + hoff);
        global = e == index() + INT16_MIN; local = e == index();
    }
    bool has() const { return boff < len; }
    void next() { boff += STEP; if (global || local) hoff += 2; upd(); }
    void reset() { hoff = 2; boff = hlen; upd(); }
    int64_t clock() const { return be64s(c + boff + 16); }
    int64_t count() const { return be64s(c + boff + 24); }
    int cmp_id(const State& o) const { return memcmp(c + boff, o.c + o.boff, 16); }      // compareId :178-181 (ByteBufferUtil.compareSubArrays, unsigned)
};
enum Rel { EQUAL, GREATER, LESS, DISJOINT };
static Rel compare(const State& l, const State& r) {                          // :443-529
    const int64_t lc = l.clock(), ln = l.count(), rc = r.clock(), rn = r.count();
    if (l.global || r.global) {
        if (l.global && r.global) { if (lc == rc) return ln > rn ? GREATER : (ln == rn ? EQUAL : LESS); return lc > rc ? GREATER : LESS; }
        return l.global ? GREATER : LESS;
    }
    if (l.local || r.local) { if (l.local && r.local) return DISJOINT; return l.local ? GREATER : LESS; }
    if (lc == rc) return ln > rn ? GREATER : (ln == rn ? EQUAL : LESS);
    return lc > rc ? GREATER : LESS;
}
struct Out {                                                                   // ContextState.allocate :784-793 + writeElement :891-903
    std::vector<uint8_t>& b; int hlen, hoff = 2, boff;
    Out(std::vector<uint8_t>& buf, int g, int l, int rm) : b(buf) { hlen = 2 + (g + l) * 2; b.assign(hlen + (g + l + rm) * STEP, 0); b[0] = (uint8_t)((g + l) >> 8); b[1] = (uint8_t)(g + l); boff = hlen; }
    void write(const uint8_t* id, int64_t clock, int64_t count, bool global, bool local) {
        memcpy(&b[boff], id, 16);
        for (int i = 0; i < 8; i++) { b[boff + 16 + i] = (uint8_t)((uint64_t)clock >> (56 - 8 * i)); b[boff + 24 + i] = (uint8_t)((uint64_t)count >> (56 - 8 * i)); }
        if (global || local) { const int e = (boff - hlen) / STEP + (global ? INT16_MIN : 0); b[hoff] = (uint8_t)((uint16_t)(int16_t)e >> 8); b[hoff + 1] = (uint8_t)e; hoff += 2; }
        boff += STEP;
    }
    void copy(const State& s) { write(s.c + s.boff, s.clock(), s.count(), s.global, s.local); }
};
// CounterContext.merge :296-447. Returns 0 = the left context is the result, 1 = the right one, 2 = `out` holds a new context.
static int merge(const uint8_t* lp, int ll, const uint8_t* rp, int rl, std::vector<uint8_t>& out) {
    bool lsup = true, rsup = true; int g = 0, lo = 0, rm = 0;
    State l(lp, ll), r(rp, rl);
    auto tally = [&](bool isg, bool isl) { if (isg) g++; else if (isl) lo++; else rm++; };
    while (l.has() && r.has()) {
        const int cmp = l.cmp_id(r);
        if (cmp == 0) {
            const Rel rel = compare(l, r);
            if (rel == GREATER) rsup = false; else if (rel == LESS) lsup = false; else if (rel == DISJOINT) lsup = rsup = false;
            tally(l.global || r.global, l.local || r.local);
            l.next(); r.next();
        } else if (cmp > 0) { lsup = false; tally(r.global, r.local); r.next(); }
        else { rsup = false; tally(l.global, l.local); l.next(); }
    }
    if (l.has()) rsup = false; else if (r.has()) lsup = false;
    if (lsup) return 0;
    if (rsup) return 1;
    while (l.has()) { tally(l.global, l.local); l.next(); }
    while (r.has()) { tally(r.global, r.local); r.next(); }
    l.reset(); r.reset();
    Out o(out, g, lo, rm);
    while (l.has() && r.has()) {
        const int cmp = l.cmp_id(r);
        if (cmp == 0) {
            const Rel rel = compare(l, r);
            if (rel == DISJOINT) o.write(l.c + l.boff, (int64_t)((uint64_t)l.clock() + (uint64_t)r.clock()), (int64_t)((uint64_t)l.count() + (uint64_t)r.count()), false, true);
            else if (rel == GREATER) o.copy(l); else o.copy(r);
            r.next(); l.next();
        } else if (cmp > 0) { o.copy(r); r.next(); } else { o.copy(l); l.next(); }
    }
    while (l.has()) { o.copy(l); l.next(); }
    while (r.has()) { o.copy(r); r.next(); }
    return 2;
}
// hasLegacyShards :595-608
static bool has_legacy_shards(const uint8_t* c, int len) {
    const int total = (len - header_length(c)) / STEP; int n = be16s(c); if (n < 0) n = -n;
    if (n < total) return true;
    for (int i = 0; i < n; i++) if (be16s(c + 2 + 2 * i) >= 0) return true;
    return false;
}
// what the walk of ContextState needs from stored bytes: a whole header, whole shards (anything else throws in the reference's ByteBuffer reads)
static bool well_formed(const uint8_t* c, int len) { return len >= 2 && header_length(c) <= len && (len - header_length(c)) % STEP == 0; }
}  // namespace ctr

// ---- Cells.reconcile: S/db/rows/Cells.java:68-121 ---------------------------------------------------------------------
static const CellV& reconcile(const CellV& l, const CellV& r) {
    if (l.ts != r.ts) return l.ts > r.ts ? l : r;
    bool le = l.ldt != NO_DEL, re = r.ldt != NO_DEL;
    if (le | re) {
        if (le != re) return le ? l : r;
        bool lt = !l.expiring(), rt = !r.expiring();
        if (lt != rt) return lt ? l : r;
        if (l.ldt != r.ldt) return l.ldt > r.ldt ? l : r;
    }
    int n = std::min(l.vlen, r.vlen);
    int c = n ? memcmp(l.val, r.val, n) : 0;
    if (c == 0) c = l.vlen - r.vlen;
    return c >= 0 ? l : r;
}

// Cells.reconcile for a counter column :73-74 -> resolveCounter :121-162 (isCounterCell = the column is a counter and the cell is no tombstone,
// S/db/rows/AbstractCell.java:46-49). `out` owns the merged context when a new one is built.
static CellV reconcile_counter(const CellV& l, const CellV& r, Unf& out) {
    const bool lt = l.tombstone(), rt = r.tombstone();
    if (lt && rt) return reconcile(l, r);                                     // neither is a counter cell: resolveRegular
    if (lt | rt) return lt ? l : r;                                           // a tombstone always wins (CASSANDRA-7346)
    const bool le = l.vlen == 0, re = r.vlen == 0;
    if (le || re) { if (le != re) return le ? l : r; return l.ts > r.ts ? l : r; }      // :142-149
    if (!ctr::well_formed(l.val, l.vlen) || !ctr::well_formed(r.val, r.vlen)) throw Corrupt{0, 4, 0, 0, "malformed counter context"};
    auto buf = std::make_shared<std::vector<uint8_t>>();
    const int which = ctr::merge(l.val, l.vlen, r.val, r.vlen, *buf);
    const int64_t ts = std::max(l.ts, r.ts);
    if (which == 0 && ts == l.ts) return l;
    if (which == 1 && ts == r.ts) return r;
    CellV m = l; m.ts = ts; m.ttl = 0; m.ldt = NO_DEL;                        // new BufferCell(left.column(), timestamp, NO_TTL, NO_DELETION_TIME, merged, left.path())
    if (which == 0) { m.val = l.val; m.vlen = l.vlen; } else if (which == 1) { m.val = r.val; m.vlen = r.vlen; }
    else { out.owned.push_back(buf); m.val = buf->data(); m.vlen = (int32_t)buf->size(); }
    return m;
}

// Row.Merger.merge: S/db/rows/Row.java:730-781; ColumnDataReducer.getReduced :838-883 (simple cell / multi-cell column). Returns false for null.
static bool merge_rows(std::vector<Unf*>& versions, DT active, Unf& out, const Schema* sc = nullptr, bool stat = false) {
    if (versions.size() == 1 && active.live()) { out = *versions[0]; return true; }
    Live info; DT del;
    for (Unf* v : versions) {
        if (v->info.supersedes(info)) info = v->info;
        if (v->del.supersedes(del)) del = v->del;
    }
    if (del.supersedes(active)) active = del; else del = DT();
    if (active.deletes(info.ts)) info = Live();          // deletes(LivenessInfo) = deletes(timestamp); EMPTY ts = MIN is always "deleted" but stays EMPTY
    out.is_row = true; out.c = versions[0]->c; out.info = info; out.del = del; out.cells.clear(); out.cdel.clear(); out.owned.clear();
    size_t cur[B200C_MAX_INPUTS] = {0};
    uint64_t cols_present = 0;                             // columns any version has data for (a multi-cell column may consist of its deletion only)
    for (Unf* v : versions) { for (const CellV& c : v->cells) cols_present |= 1ull << c.col; for (auto& d : v->cdel) cols_present |= 1ull << d.first; }
    for (int col = 0; col < 64; col++) {
        if (!((cols_present >> col) & 1)) continue;
        const bool complex = sc && !stat && col_complex(sc->cols[col]);
        if (!complex && sc && (stat ? sc->stat[col] : sc->cols[col]).type == B200C_TYPE_COUNTER) {
            bool have = false; CellV merged{};
            for (size_t i = 0; i < versions.size(); i++) {
                if (cur[i] < versions[i]->cells.size() && versions[i]->cells[cur[i]].col == col) {
                    const CellV& c = versions[i]->cells[cur[i]++];
                    if (active.deletes(c.ts)) continue;
                    if (have) merged = reconcile_counter(merged, c, out); else { merged = c; have = true; }
                }
            }
            if (have) out.cells.push_back(merged);
            continue;
        }
        if (!complex) {
            const CellV* merged = nullptr;
            for (size_t i = 0; i < versions.size(); i++) {
                if (cur[i] < versions[i]->cells.size() && versions[i]->cells[cur[i]].col == col) {
                    const CellV& c = versions[i]->cells[cur[i]++];
                    if (!active.deletes(c.ts)) merged = merged ? &reconcile(*merged, c) : &c;
                }
            }
            if (merged) out.cells.push_back(*merged);
            continue;
        }
        // multi-cell column :851-883: the strongest complex deletion; kept (and it shadows the cells) only if it supersedes the active deletion
        DT cd;
        for (Unf* v : versions) { DT d = v->complex_deletion(col); if (d.supersedes(cd)) cd = d; }
        DT cell_del = active;
        if (cd.supersedes(active)) cell_del = cd; else cd = DT();
        if (!cd.live()) out.cdel.push_back({col, cd});
        // MergeIterator over the versions' cells in cell-path order (Cell.comparator = column.cellPathComparator())
        const b200c_column pt = col_path_type(sc->cols[col]);
        for (;;) {
            const CellV* head = nullptr;
            for (size_t i = 0; i < versions.size(); i++) {
                if (cur[i] >= versions[i]->cells.size() || versions[i]->cells[cur[i]].col != col) continue;
                const CellV& c = versions[i]->cells[cur[i]];
                if (!head || compare_value(pt, Val{c.path, c.plen, false}, Val{head->path, head->plen, false}) < 0) head = &c;
            }
            if (!head) break;
            const Val hp{head->path, head->plen, false};
            const CellV* merged = nullptr;
            for (size_t i = 0; i < versions.size(); i++) {                 // CellReducer :900-918, in source order
                if (cur[i] >= versions[i]->cells.size() || versions[i]->cells[cur[i]].col != col) continue;
                const CellV& c = versions[i]->cells[cur[i]];
                if (compare_value(pt, Val{c.path, c.plen, false}, hp) != 0) continue;
                cur[i]++;
                if (!cell_del.deletes(c.ts)) merged = merged ? &reconcile(*merged, c) : &c;
            }
            if (merged) out.cells.push_back(*merged);
        }
    }
    return !(out.info.empty() && out.del.live() && !out.has_data());
}

// RangeTombstoneMarker.Merger: S/db/rows/RangeTombstoneMarker.java:72-199 (forward order)
struct MarkerMerger {
    DT partition_del; std::vector<DT> open; std::vector<bool> has_open; int biggest = -1;
    void init(size_t n, DT pd) { partition_del = pd; open.assign(n, DT()); has_open.assign(n, false); biggest = -1; }
    DT current_open() const {            // :160-168
        if (biggest < 0) return DT();
        return !open[biggest].supersedes(partition_del) ? DT() : open[biggest];
    }
    DT active() const { DT o = current_open(); return o.live() ? partition_del : o; }   // :191-197
    // versions: (source slot, marker). Returns false when nothing is emitted.
    bool merge(const std::vector<std::pair<int, Unf*>>& versions, Unf& out) {
        DT prev = current_open();
        for (auto& pr : versions) {      // updateOpenMarkers :170-189
            Unf* m = pr.second; bool is_open = kind_is_boundary(m->c.kind) || kind_is_start(m->c.kind);
            if (is_open) { open[pr.first] = m->m_open; has_open[pr.first] = true; } else has_open[pr.first] = false;
        }
        biggest = -1;
        for (size_t i = 0; i < open.size(); i++) if (has_open[i] && (biggest < 0 || open[i].supersedes(open[biggest]))) biggest = (int)i;
        DT now = current_open();
        if (prev == now) return false;
        const Clust& bound = versions.back().second->c;     // `bound` = clustering of the last marker added (:99-103)
        bool before = kind_vs_clustering(bound.kind) < 0;
        out.is_row = false; out.cells.clear(); out.c = bound; out.m_close = DT(); out.m_open = DT();
        if (prev.live()) { out.c.kind = before ? K_INCL_START : K_EXCL_START; out.m_open = now; }
        else if (now.live()) { out.c.kind = before ? K_EXCL_END : K_INCL_END; out.m_close = prev; }
        else { out.c.kind = before ? K_EXCL_END_INCL_START : K_INCL_END_EXCL_START; out.m_close = prev; out.m_open = now; }
        return true;
    }
};

// ---- output side ----------------------------------------------------------------------------------------------------------
struct OutBuf { std::vector<uint8_t> b; void u8(uint8_t v) { b.push_back(v); } void put(const void* p, size_t n) { const uint8_t* q = (const uint8_t*)p; b.insert(b.end(), q, q + n); }
    void vint(uint64_t v) { uint8_t t[9]; int n = vint_write(t, v); put(t, n); }
    void be16(uint16_t v) { u8(v >> 8); u8(v & 0xff); } void be32(uint32_t v) { u8(v >> 24); u8(v >> 16); u8(v >> 8); u8(v); }
    void be64(uint64_t v) { be32((uint32_t)(v >> 32)); be32((uint32_t)v); } size_t size() const { return b.size(); } };

// DeletionTime.Serializer.serialize (oa): S/db/DeletionTime.java:205-220
static void write_partition_dt(OutBuf& o, const DT& d) { if (d.live()) o.u8(0x80); else { o.be64((uint64_t)d.mfda); o.be32((uint32_t)d.ldt); } }
static int partition_dt_size(const DT& d) { return d.live() ? 1 : 12; }


// ---- the rest of the sstable (SURVEY §8 f1): what MetadataCollector, the bloom filter and the index summary builder gather while the
// writer appends (S/io/sstable/format/SortedTableWriter.java:183-258). One Meta per output file. ---------------------------------------------
static std::vector<int64_t> histogram_offsets(int size) {                 // EstimatedHistogram.newOffsets(size, false) S/utils/EstimatedHistogram.java:91-109
    std::vector<int64_t> r(size); int64_t last = 1; r[0] = 1;
    for (int i = 1; i < size; i++) { int64_t next = (int64_t)std::llround((double)last * 1.2); if (next == last) next++; r[i] = next; last = next; }
    return r;
}
static int histogram_index(const std::vector<int64_t>& offs, int64_t n) {     // findIndex: first offset >= n, else the overflow bucket
    return (int)(std::lower_bound(offs.begin(), offs.end(), n) - offs.begin());
}
struct Meta {
    bool ts_set = false, ldt_set = false, ttl_set = false;
    int64_t min_ts = 0, max_ts = 0, min_ldt = 0, max_ldt = 0; int32_t min_ttl = 0, max_ttl = 0;
    uint64_t total_rows = 0, total_columns_set = 0, total_cells = 0, total_tombstones = 0, cur_cells = 0;
    bool has_partition_deletions = false;
    std::vector<uint64_t> psize, cells;
    std::map<int64_t, uint64_t> tdrop;
    std::vector<uint8_t> hll;
    std::vector<uint8_t> bloom; int bloom_k = 0;
    std::vector<uint32_t> sum_offsets; std::vector<uint8_t> sum_entries; uint64_t keys_written = 0; int interval = 128;
    std::string first, last;
    int64_t now = 0;
    void init(const b200c_manifest* m) {
        psize.assign(B200C_PSIZE_BUCKETS, 0); cells.assign(B200C_CELLS_BUCKETS, 0); hll.assign(1 << B200C_HLL_P, 0);
        bloom.assign(m->bloom_words * 8, 0); bloom_k = m->bloom_hash_count; interval = m->min_index_interval > 0 ? m->min_index_interval : 128; now = m->now_in_sec;
    }
    // MetadataCollector.MinMax*Tracker :402-447
    void ts(int64_t v) { if (!ts_set) { min_ts = max_ts = v; ts_set = true; } else { min_ts = std::min(min_ts, v); max_ts = std::max(max_ts, v); } }
    void ttl(int32_t v) { if (!ttl_set) { min_ttl = max_ttl = v; ttl_set = true; } else { min_ttl = std::min(min_ttl, v); max_ttl = std::max(max_ttl, v); } }
    void ldt(int64_t v) {                                                  // updateLocalDeletionTime :263-268
        if (!ldt_set) { min_ldt = max_ldt = v; ldt_set = true; } else { min_ldt = std::min(min_ldt, v); max_ldt = std::max(max_ldt, v); }
        if (v != NO_DEL) { int64_t d = v % 60; tdrop[d == 0 ? v : v + (60 - d)]++; }      // StreamingTombstoneHistogramBuilder.ceilKey, TOMBSTONE_HISTOGRAM_TTL_ROUND_SECONDS = 60
    }
    void update(const Live& l) { if (l.empty()) return; ts(l.ts); ttl(l.ttl); ldt(l.ldt); if (!l.is_live(now)) total_tombstones++; }     // :208-218
    void update(const DT& d) { if (d.live()) return; ts(d.mfda); ldt(d.ldt); total_tombstones++; }                                        // :237-245
    void update(const CellV& c) { cur_cells++; total_cells++; ts(c.ts); ttl(c.ttl); ldt(c.ldt); if (!c.is_live(now)) total_tombstones++; } // :220-228
    void partition_deletion(const DT& d) { if (!d.live()) has_partition_deletions = true; update(d); }                                    // :230-235
    bool has_legacy_counter_shards = false;
    void row(const Unf& u, const b200c_column* types = nullptr) {           // Rows.collectStats S/db/rows/Rows.java:102-113 (types: of the row's columns, regular or static)
        update(u.info); update(u.del);
        if (types) for (const CellV& c : u.cells)                             // Cells.collectStats S/db/rows/Cells.java:44-50
            if (types[c.col].type == B200C_TYPE_COUNTER && !c.tombstone() && c.vlen >= 2 && ctr::has_legacy_shards(c.val, c.vlen)) has_legacy_counter_shards = true;
        for (auto& d : u.cdel) update(d.second);                              // StatsAccumulation.accumulateOnColumnData S/db/rows/Rows.java:66-82
        int cols_with_cells = 0, last = -1;
        for (const CellV& c : u.cells) { update(c); if (c.col != last) { cols_with_cells++; last = c.col; } }
        total_columns_set += cols_with_cells; total_rows++;
    }
    void marker(const Unf& u) {                                             // SortedTableWriter.addRangeTomstoneMarker :222-238
        if (kind_is_boundary(u.c.kind)) { update(u.m_close); update(u.m_open); }
        else update(kind_is_start(u.c.kind) ? u.m_open : u.m_close);
    }
    void end_partition(const uint8_t* key, int kl, uint64_t size, uint64_t index_start) {      // endPartition :240-258 + IndexWriter.append
        static const std::vector<int64_t> po = histogram_offsets(B200C_PSIZE_BUCKETS - 1), co = histogram_offsets(B200C_CELLS_BUCKETS - 1);
        psize[histogram_index(po, (int64_t)size)]++;
        cells[histogram_index(co, (int64_t)cur_cells)]++; cur_cells = 0;
        {   // addKey :160-166 -> HyperLogLogPlus.offerHashed (dense form): register[h >>> (64 - p)] = max(rho of the remaining bits)
            uint64_t h = murmur2_64(key, kl, 0); uint32_t idx = (uint32_t)(h >> (64 - B200C_HLL_P));
            uint64_t w = (h << B200C_HLL_P) | (1ull << (B200C_HLL_P - 1)); uint8_t rho = (uint8_t)(__builtin_clzll(w) + 1);
            if (rho > hll[idx]) hll[idx] = rho;
        }
        if (!bloom.empty()) {                                               // BloomFilter.add S/utils/BloomFilter.java:104-122
            uint64_t hh[2]; murmur3_x64_128(key, kl, 0, hh);
            int64_t base = (int64_t)hh[1], inc = (int64_t)hh[0]; const int64_t cap = (int64_t)bloom.size() * 8;
            for (int i = 0; i < bloom_k; i++) { int64_t r = base % cap; uint64_t idx = (uint64_t)(r < 0 ? -r : r); bloom[idx >> 3] |= (uint8_t)(1u << (idx & 7)); base = (int64_t)((uint64_t)base + (uint64_t)inc); }
        }
        if (keys_written % (uint64_t)interval == 0) {                       // IndexSummaryBuilder.maybeAddEntry :200-228 at full sampling
            sum_offsets.push_back((uint32_t)sum_entries.size());
            sum_entries.insert(sum_entries.end(), key, key + kl);
            for (int b = 0; b < 8; b++) sum_entries.push_back((uint8_t)(index_start >> (8 * b)));     // native (little-endian) long
        }
        if (keys_written == 0) first.assign((const char*)key, kl);
        last.assign((const char*)key, kl);
        keys_written++;
    }
    std::vector<uint8_t> filter_image() const {                             // BloomFilterSerializer.serialize :50-55 + OffHeapBitSet.serialize :115-119
        std::vector<uint8_t> f; if (bloom.empty()) return f;
        uint32_t words = (uint32_t)(bloom.size() / 8);
        for (int b = 3; b >= 0; b--) f.push_back((uint8_t)(bloom_k >> (8 * b)));
        for (int b = 3; b >= 0; b--) f.push_back((uint8_t)(words >> (8 * b)));
        f.insert(f.end(), bloom.begin(), bloom.end());
        return f;
    }
    std::vector<uint8_t> summary_image() const {                            // IndexSummarySerializer.serialize :401-423, then first / last key (int length + bytes)
        std::vector<uint8_t> o; if (!keys_written) return o;
        auto be32 = [&](uint32_t v) { for (int b = 3; b >= 0; b--) o.push_back((uint8_t)(v >> (8 * b))); };
        auto be64 = [&](uint64_t v) { for (int b = 7; b >= 0; b--) o.push_back((uint8_t)(v >> (8 * b))); };
        uint32_t n = (uint32_t)sum_offsets.size();
        be32((uint32_t)interval); be32(n); be64((uint64_t)n * 4 + sum_entries.size()); be32(128); be32((uint32_t)((keys_written + interval - 1) / interval));
        for (uint32_t off : sum_offsets) { uint32_t v = off + n * 4; for (int b = 0; b < 4; b++) o.push_back((uint8_t)(v >> (8 * b))); }
        o.insert(o.end(), sum_entries.begin(), sum_entries.end());
        be32((uint32_t)first.size()); o.insert(o.end(), first.begin(), first.end());
        be32((uint32_t)last.size()); o.insert(o.end(), last.begin(), last.end());
        return o;
    }
    void fill(b200c_sstable_stats* st) const {
        memset(st, 0, sizeof(*st));
        st->min_timestamp = ts_set ? min_ts : INT64_MIN; st->max_timestamp = ts_set ? max_ts : INT64_MAX;            // MinMaxLongTracker defaults
        st->min_local_deletion_time = ldt_set ? min_ldt : NO_DEL; st->max_local_deletion_time = ldt_set ? max_ldt : NO_DEL;
        st->min_ttl = ttl_set ? min_ttl : 0; st->max_ttl = ttl_set ? max_ttl : 0;
        st->total_rows = total_rows; st->total_columns_set = total_columns_set; st->total_cells = total_cells; st->total_tombstones = total_tombstones;
        st->has_partition_level_deletions = has_partition_deletions ? 1 : 0;
        for (int i = 0; i < B200C_PSIZE_BUCKETS; i++) st->partition_size_hist[i] = psize[i];
        for (int i = 0; i < B200C_CELLS_BUCKETS; i++) st->cells_per_partition_hist[i] = cells[i];
        uint32_t k = 0;
        for (auto& kv : tdrop) { if (k >= B200C_TDROP_CAP) { st->tdrop_overflow = 1; break; } st->tdrop_point[k] = kv.first; st->tdrop_count[k] = kv.second; k++; }      // the CAP smallest points
        st->ntdrop = k; st->has_legacy_counter_shards = has_legacy_counter_shards ? 1 : 0;
        memcpy(st->hll_registers, hll.data(), hll.size());
    }
};

struct Writer {
    const b200c_manifest* m; Schema sc;
    // one output sstable
    struct Sst { std::vector<uint8_t> data; std::vector<uint8_t> index; std::vector<uint64_t> offs; uint64_t ulen = 0; uint32_t digest = 0; uint64_t parts = 0, rows = 0; Meta meta; };
    std::vector<Sst> outs;
    std::vector<uint8_t> chunk;         // CompressedSequentialWriter buffer (S/io/compress/CompressedSequentialWriter.java:140-206)
    std::vector<uint8_t> comp;
    uint64_t position = 0;              // uncompressed position in the current output
    uint64_t chunk_offset = 0;          // on-disk bytes flushed (getEstimatedOnDiskBytesWritten :128-131)
    // partition state (SortedTablePartitionWriter / BigFormatPartitionWriter)
    uint64_t part_start = 0, header_len = 0, prev_row_start = 0, block_start = 0;
    bool have_first = false; Clust first_c, last_c; DT open_marker, start_open_marker;
    std::vector<std::vector<uint8_t>> index_infos;
    OutBuf body, tmp;

    bool raw = false;                   // parallel driver (parallel.cc): keep the uncompressed stream, compression happens after stitching
    void start_output() { outs.emplace_back(); outs.back().meta.init(m); position = 0; chunk_offset = 0; chunk.clear(); }
    void flush_chunk() {                // flushData :140-206
        if (chunk.empty()) return;
        Sst& o = outs.back();
        if (raw) { o.data.insert(o.data.end(), chunk.begin(), chunk.end()); o.ulen += chunk.size(); chunk.clear(); return; }
        comp.resize(chunk_max_compressed(m->out_compressor, m->out_chunk_len) + 64);
        int clen = chunk_compress(m->out_compressor, chunk.data(), (int)chunk.size(), comp.data());
        const uint8_t* w = comp.data(); int wlen = clen;
        std::vector<uint8_t> raw;
        if ((int64_t)clen >= (int64_t)m->out_max_compressed_len) {
            raw = chunk;
            if ((int64_t)raw.size() < (int64_t)m->out_max_compressed_len) raw.resize(m->out_max_compressed_len, 0);
            w = raw.data(); wlen = (int)raw.size();
        }
        o.offs.push_back(chunk_offset);
        o.data.insert(o.data.end(), w, w + wlen);
        uint32_t crc = crc32_ieee(0, w, wlen);           // ChecksumWriter.appendDirect :62-89
        uint8_t cb[4] = {(uint8_t)(crc >> 24), (uint8_t)(crc >> 16), (uint8_t)(crc >> 8), (uint8_t)crc};
        o.data.insert(o.data.end(), cb, cb + 4);
        chunk_offset += wlen + 4;
        o.ulen += chunk.size();
        chunk.clear();
    }
    void write(const uint8_t* p, size_t n) {             // BufferedDataOutputStreamPlus fill-then-flush :87-139
        while (n) {                                      // lazy: a full buffer is flushed only when the next byte needs room (doFlush(count))
            if (chunk.size() == (size_t)m->out_chunk_len) flush_chunk();
            size_t room = (size_t)m->out_chunk_len - chunk.size();
            size_t k = std::min(room, n);
            chunk.insert(chunk.end(), p, p + k); p += k; n -= k; position += k;
        }
    }
    void finish_output() { flush_chunk(); Sst& o = outs.back(); o.digest = crc32_ieee(0, o.data.data(), o.data.size()); }

    // ClusteringPrefix.Serializer.serializeValuesWithoutSize: S/db/ClusteringPrefix.java:455-477
    void write_clust_values(OutBuf& o, const Clust& c) {
        int off = 0;
        while (off < c.n) {
            int limit = std::min(c.n, off + 32);
            uint64_t header = 0;
            for (int i = off; i < limit; i++) { if (c.v[i].null) header |= 1ull << (((i % 32) * 2) + 1); else if (c.v[i].len == 0) header |= 1ull << ((i % 32) * 2); }
            o.vint(header);
            for (; off < limit; off++) {
                const Val& v = c.v[off];
                if (v.null || v.len == 0) continue;
                if (sc.clust[off].fixed_len <= 0) o.vint((uint64_t)v.len);     // AbstractType.writeValue :535-552
                o.put(v.p, v.len);
            }
        }
    }
    // ClusteringPrefix.Serializer.serialize (IndexInfo names): :408-421; ClusteringBoundOrBoundary.Serializer :101-108
    void write_clust_prefix(OutBuf& o, const Clust& c) {
        o.u8(c.kind);
        if (c.kind != K_CLUSTERING) o.be16((uint16_t)c.n);
        write_clust_values(o, c);
    }
    void write_delta_dt(OutBuf& o, const DT& d) {        // SerializationHeader.writeDeletionTime :181-184
        o.vint((uint64_t)d.mfda - (uint64_t)m->out_stats.min_timestamp);
        o.vint((uint64_t)(int64_t)(int32_t)(d.ldt - m->out_stats.min_local_deletion_time));
    }

    static int row_flags(const Unf& u, int ncols) {          // UnfilteredSerializer.serialize(Row) :151-186
        int flags = 0;
        if (!u.info.empty()) flags |= 0x04;
        if (u.info.expiring()) flags |= 0x08;
        if (!u.del.live()) flags |= 0x10;
        int present = 0, last = -1;
        for (const CellV& c : u.cells) if (c.col != last) { present++; last = c.col; }
        for (auto& d : u.cdel) { bool has_cell = false; for (const CellV& c : u.cells) if (c.col == d.first) has_cell = true; if (!has_cell) present++; }
        if (present == ncols) flags |= 0x20;                  // row.columnCount() == headerColumns.size() :170-171
        if (!u.cdel.empty()) flags |= 0x40;                   // row.hasComplexDeletion() :166-167, BTreeRow.java:400-405
        return flags;
    }
    void write_row_body(OutBuf& body, const Unf& u, int flags, int ncols, const b200c_column* types) {      // serializeRowBody :213-269
        if (flags & 0x04) body.vint((uint64_t)u.info.ts - (uint64_t)m->out_stats.min_timestamp);
        if (flags & 0x08) { body.vint((uint64_t)(int64_t)(u.info.ttl - m->out_stats.min_ttl));
                            body.vint((uint64_t)(int64_t)(int32_t)(u.info.ldt - m->out_stats.min_local_deletion_time)); }
        if (flags & 0x10) write_delta_dt(body, u.del);
        if (!(flags & 0x20)) {                            // Columns.serializeSubset :503-531, encodeBitmap :586-608
            if (ncols >= 64) throw Unsupported{">= 64 columns"};
            uint64_t missing = (1ull << ncols) - 1;
            for (const CellV& c : u.cells) missing &= ~(1ull << c.col);
            for (auto& d : u.cdel) missing &= ~(1ull << d.first);
            body.vint(missing);
        }
        // multi-cell columns (writeComplexColumn :271-280): [complex deletion when the row has any] vint cell count, then the cells. A column that
        // consists of its deletion only has no cell to hang the header on: written when the walk passes its position.
        size_t next_cd = 0; int open_col = -1;
        auto complex_head = [&](int col) {
            if (flags & 0x40) write_delta_dt(body, u.complex_deletion(col));
            uint64_t cnt = 0; for (const CellV& c : u.cells) if (c.col == col) cnt++;
            body.vint(cnt);
        };
        auto flush_deletion_only = [&](int upto) {             // complex columns < upto that have a deletion but no cell
            for (; next_cd < u.cdel.size() && u.cdel[next_cd].first < upto; next_cd++) {
                bool has_cell = false; for (const CellV& c : u.cells) if (c.col == u.cdel[next_cd].first) has_cell = true;
                if (!has_cell) complex_head(u.cdel[next_cd].first);
            }
        };
        for (size_t ci = 0; ci <= u.cells.size(); ci++) {
            if (ci == u.cells.size()) { flush_deletion_only(INT_MAX); break; }
            const CellV& c = u.cells[ci];
            const bool complex = col_complex(types[c.col]);
            if (complex && c.col != open_col) { flush_deletion_only(c.col); complex_head(c.col); open_col = c.col; }
            else if (!complex) flush_deletion_only(c.col);
            write_cell(body, u, c, types);
        }
    }
    void write_cell(OutBuf& body, const Unf& u, const CellV& c, const b200c_column* types) {      // Cell.Serializer.serialize: S/db/rows/Cell.java:268-305
        {
            bool has_value = c.vlen > 0, deleted = c.tombstone(), expiring = c.expiring();
            bool use_ts = !u.info.empty() && c.ts == u.info.ts;
            bool use_ttl = expiring && u.info.expiring() && c.ttl == u.info.ttl && c.ldt == u.info.ldt;
            int cf = 0;
            if (!has_value) cf |= 0x04;
            if (deleted) cf |= 0x01; else if (expiring) cf |= 0x02;
            if (use_ts) cf |= 0x08;
            if (use_ttl) cf |= 0x10;
            body.u8((uint8_t)cf);
            if (!use_ts) body.vint((uint64_t)c.ts - (uint64_t)m->out_stats.min_timestamp);
            if ((deleted || expiring) && !use_ttl) body.vint((uint64_t)(int64_t)(int32_t)(c.ldt - m->out_stats.min_local_deletion_time));
            if (expiring && !use_ttl) body.vint((uint64_t)(int64_t)(c.ttl - m->out_stats.min_ttl));
            if (col_complex(types[c.col])) { if (col_path_type(types[c.col]).fixed_len <= 0) body.vint((uint64_t)c.plen); body.put(c.path, c.plen); }      // :300-301 cellPathSerializer
            if (has_value) { if (col_value_type(types[c.col]).fixed_len <= 0) body.vint((uint64_t)c.vlen); body.put(c.val, c.vlen); }
        }
    }

    // stat: the merged, purged static row, or nullptr when it is empty. Tables with static columns always carry one per partition
    // (SortedTableWriter.append :144-146, SortedTablePartitionWriter.addStaticRow :117-126, UnfilteredSerializer.serializeStaticRow :144-149)
    void start_partition(const uint8_t* key, int keylen, const DT& pdel, const Unf* stat = nullptr) {     // SortedTablePartitionWriter.start :97-115
        part_start = position;
        tmp.b.clear(); tmp.be16((uint16_t)keylen); tmp.put(key, keylen); write_partition_dt(tmp, pdel);
        write(tmp.b.data(), tmp.b.size());
        if (sc.nstat > 0) {
            static const Unf empty_static;
            const Unf& u = stat ? *stat : empty_static;
            tmp.b.clear(); body.b.clear();
            int flags = row_flags(u, sc.nstat) | 0x80;                         // hasExtendedFlags(row) = row.isStatic() || shadowable :755-758
            tmp.u8((uint8_t)flags); tmp.u8(0x01);                             // extended flags: IS_STATIC
            write_row_body(body, u, flags, sc.nstat, sc.stat);
            tmp.vint(body.size() + vint_size(0)); tmp.vint(0);
            write(tmp.b.data(), tmp.b.size()); write(body.b.data(), body.b.size());
            if (stat) outs.back().meta.row(u, sc.stat);                       // SortedTableWriter.addStaticRow :188-197: collectStats unless empty
        }
        header_len = position - part_start;
        prev_row_start = 0; have_first = false; open_marker = DT(); index_infos.clear(); block_start = 0;
        outs.back().meta.partition_deletion(pdel);                          // startPartition :183-189
    }
    uint64_t cur_pos() const { return position - part_start; }

    void add_index_block() {                              // BigFormatPartitionWriter.addIndexBlock :128-190, IndexInfo.Serializer :107-117
        OutBuf o;
        write_clust_prefix(o, first_c); write_clust_prefix(o, last_c);
        o.vint(block_start);
        o.vint(zigzag_enc((int64_t)(cur_pos() - block_start) - 65536));
        o.u8(open_marker.live() ? 0 : 1);
        if (!open_marker.live()) write_partition_dt(o, open_marker);
        index_infos.push_back(std::move(o.b));
        have_first = false;
    }

    void add_unfiltered(const Unf& u) {                   // SortedTablePartitionWriter.addUnfiltered :128-154 + UnfilteredSerializer.serialize :131-305
        uint64_t pos = cur_pos();
        if (!have_first) { first_c = u.c; start_open_marker = open_marker; block_start = pos; have_first = true; }
        uint64_t prev_size = pos - prev_row_start;
        tmp.b.clear(); body.b.clear();
        if (!u.is_row) {
            tmp.u8(0x02); tmp.u8(u.c.kind); tmp.be16((uint16_t)u.c.n); write_clust_values(tmp, u.c);
            if (kind_is_boundary(u.c.kind)) { write_delta_dt(body, u.m_close); write_delta_dt(body, u.m_open); }
            else write_delta_dt(body, kind_is_start(u.c.kind) ? u.m_open : u.m_close);
            tmp.vint(body.size() + vint_size(prev_size)); tmp.vint(prev_size);
        } else {
            int flags = row_flags(u, sc.ncols);
            tmp.u8((uint8_t)flags);
            write_clust_values(tmp, u.c);
            write_row_body(body, u, flags, sc.ncols, sc.cols);
            tmp.vint(body.size() + vint_size(prev_size)); tmp.vint(prev_size);
        }
        write(tmp.b.data(), tmp.b.size());
        write(body.b.data(), body.b.size());
        last_c = u.c; prev_row_start = pos;
        if (u.is_row) outs.back().meta.row(u, sc.cols); else outs.back().meta.marker(u);
        if (!u.is_row) open_marker = (kind_is_boundary(u.c.kind) || kind_is_start(u.c.kind)) ? u.m_open : DT();
        outs.back().rows++;
        if (cur_pos() - block_start >= (uint64_t)m->column_index_size) add_index_block();     // BigFormatPartitionWriter.addUnfiltered :208-215
    }

    void end_partition(const uint8_t* key, int keylen, const DT& pdel, uint64_t written) {   // finish :217-243 + RowIndexEntry / IndexWriter.append
        uint8_t eop = 0x01; write(&eop, 1);
        if (written && have_first) add_index_block();
        Sst& o = outs.back();
        OutBuf e; e.be16((uint16_t)keylen); e.put(key, keylen);
        e.vint(part_start);
        if (index_infos.size() > 1) {                     // RowIndexEntry.create :217-243; IndexedEntry.serialize :625-642
            uint64_t infos = 0; for (auto& ii : index_infos) infos += ii.size();
            uint64_t size = vint_size(header_len) + partition_dt_size(pdel) + vint_size(index_infos.size()) + infos + 4 * index_infos.size();
            e.vint(size); e.vint(header_len); write_partition_dt(e, pdel); e.vint(index_infos.size());
            for (auto& ii : index_infos) e.put(ii.data(), ii.size());
            uint32_t off = 0; for (auto& ii : index_infos) { e.be32(off); off += (uint32_t)ii.size(); }
        } else e.vint(0);
        o.meta.end_partition(key, keylen, position - part_start, o.index.size());
        o.index.insert(o.index.end(), e.b.begin(), e.b.end());
        o.parts++;
    }
};

// ro != nullptr: raw mode for the parallel driver — the uncompressed stream and the (range-relative) Index.db of output 0 are moved
// into *ro instead of being compressed and copied into the caller's buffers
int compact_impl(const b200c_manifest* m, b200c_result* res, RangeOut* ro) {
    auto t0 = std::chrono::steady_clock::now();
    if (m->abi_version != B200C_ABI_VERSION || m->ninputs <= 0 || m->ninputs > B200C_MAX_INPUTS) return B200C_EINVAL;
    if (m->tombstone_option != 0 || m->enforce_strict_liveness) return B200C_EUNSUPPORTED;
    if (m->nclustering > B200C_MAX_CLUSTERING || m->ncolumns > B200C_MAX_COLUMNS || m->ncolumns >= 64) return B200C_EUNSUPPORTED;
    if (m->nstatic_columns < 0 || m->nstatic_columns > B200C_MAX_STATIC_COLUMNS) return B200C_EUNSUPPORTED;
    for (int i = 0; i < m->ninputs; i++) {
        const b200c_input& in = m->inputs[i];
        if (in.nstatic_columns < 0 || in.nstatic_columns > m->nstatic_columns) return B200C_EINVAL;
        for (int k = 0; k < in.nstatic_columns; k++) if (in.static_column_map[k] < 0 || in.static_column_map[k] >= m->nstatic_columns) return B200C_EINVAL;
    }
    Schema sc; sc.nclust = m->nclustering; sc.ncols = m->ncolumns; sc.nstat = m->nstatic_columns;
    memcpy(sc.clust, m->clustering, sizeof(sc.clust)); memcpy(sc.cols, m->columns, sizeof(sc.cols)); memcpy(sc.stat, m->static_columns, sizeof(sc.stat));
    for (int k = 0; k < m->ncolumns; k++) {                                // multi-cell columns follow the simple ones (ColumnMetadata.comparisonOrder)
        if (col_complex(sc.cols[k])) sc.ncomplex++; else if (sc.ncomplex) return B200C_EINVAL;
        const int pt = col_path_type(sc.cols[k]).type;
        if (col_complex(sc.cols[k]) && (pt < 0 || pt > B200C_TYPE_TIMEUUID)) return B200C_EINVAL;
    }
    if (sc.ncomplex > B200C_MAX_COMPLEX_COLUMNS) return B200C_EUNSUPPORTED;
    for (int k = 0; k < m->nstatic_columns; k++) if (col_complex(sc.stat[k])) return B200C_EUNSUPPORTED;
    for (int k = 0; k < m->ncolumns; k++) if (col_complex(sc.cols[k]) && col_value_type(sc.cols[k]).type == B200C_TYPE_COUNTER) return B200C_EINVAL;      // (no collections of counters)
    g_partitioner = m->partitioner;
    std::vector<Source> srcs(m->ninputs);
    uint64_t bytes_read = 0;
    for (int i = 0; i < m->ninputs; i++) { srcs[i].idx = i; srcs[i].in = &m->inputs[i]; srcs[i].schema = &sc; open_source(srcs[i], m->token_lo, m->token_hi); bytes_read += srcs[i].dsize(); next_partition(srcs[i], m->token_lo, m->token_hi); }
    if (m->partitioner != B200C_PARTITIONER_MURMUR3 && m->partitioner != B200C_PARTITIONER_BYTE_ORDERED) return B200C_EUNSUPPORTED;
    if (m->partitioner == B200C_PARTITIONER_BYTE_ORDERED && (m->token_lo != INT64_MIN || m->token_hi != INT64_MAX || m->npurge_ranges)) return B200C_EUNSUPPORTED;
    Purger pg{m->now_in_sec, m->gc_before, m->purge_max_timestamp};
    Writer w; w.m = m; w.sc = sc; w.raw = ro != nullptr; w.start_output();
    if (ro) {                                              // a range task: one allocation for the piece of the stream it can produce, none while it grows
        uint64_t span = 0, ispan = 0;
        for (auto& sr : srcs) { span += sr.span1 - sr.span0; ispan += sr.in->index_len ? (uint64_t)((double)sr.in->index_len * (double)(sr.span1 - sr.span0) / (double)std::max<uint64_t>(1, sr.in->data_length)) : 0; }
        w.outs.back().data.reserve(span + (span >> 3) + 4096); w.outs.back().index.reserve(ispan + (ispan >> 2) + 4096);
    }
    if (ro && m->max_sstable_bytes) return B200C_EUNSUPPORTED;
    memset(res->merged_row_counts, 0, sizeof(res->merged_row_counts));
    uint64_t total_source_rows = 0, input_partitions = 0;
    std::vector<Unf> heads(m->ninputs);
    std::vector<bool> head_ok(m->ninputs);
    for (;;) {
        // MergeIterator over partitions (S/utils/MergeIterator.java:154-219): equal keys reduce together, source order
        int best = -1;
        for (int i = 0; i < m->ninputs; i++) if (srcs[i].has && (best < 0 || compare_key(srcs[i], srcs[best]) < 0)) best = i;
        if (best < 0) break;
        std::vector<int> group;
        for (int i = 0; i < m->ninputs; i++) if (srcs[i].has && compare_key(srcs[i], srcs[best]) == 0) group.push_back(i);
        res->merged_row_counts[group.size() - 1]++;       // CompactionIterator.updateCounterFor :220-232
        total_source_rows++;                               // Purger.applyToStatic -> updateProgress(): BaseRows applies it to every partition's static row, the empty one included
                                                           // (S/db/transform/BaseRows.java:106-110, S/db/partitions/PurgeFunction.java:101-106, CompactionIterator.java:365-371)
        input_partitions += group.size();
        // LCS: CompactionAwareWriter.maybeSwitchWriter / MaxSSTableSizeWriter.shouldSwitchWriterInCurrentLocation :76-79 (before each partition)
        if (m->max_sstable_bytes && w.chunk_offset > m->max_sstable_bytes) { w.finish_output(); w.start_output(); }
        // partition deletion: collectPartitionLevelDeletion S/db/rows/UnfilteredRowIterators.java:465-482
        DT pdel;
        for (int i : group) if (!pdel.supersedes(srcs[i].pdel)) pdel = srcs[i].pdel;
        // purge evaluator of this key (CompactionController.getPurgeEvaluator :247-286), bucketed by token in the manifest
        pg.max_ts = m->purge_max_timestamp;
        for (int k = 0; k < m->npurge_ranges; k++) if (m->purge_range_hi[k] >= srcs[best].token) { pg.max_ts = m->purge_range_max_ts[k]; break; }
        DT out_pdel = pg.should_purge(pdel) ? DT() : pdel;     // PurgeFunction.applyToDeletion :95-99
        std::string keycopy((const char*)srcs[group[0]].key, srcs[group[0]].keylen);
        bool started = false; uint64_t written = 0;
        // static row: UnfilteredRowMergeIterator's constructor merges them eagerly, whatever the fan-in, with the partition deletion as the
        // active deletion (mergeStaticRows S/db/rows/UnfilteredRowIterators.java:484-505); then PurgeFunction.applyToStatic :101-106
        Unf stat_out; bool have_static = false;
        if (sc.nstat > 0) {
            std::vector<Unf*> vs; for (int i : group) if (srcs[i].has_stat) vs.push_back(&srcs[i].stat);
            if (!vs.empty()) have_static = merge_rows(vs, pdel, stat_out, &sc, true) && purge_row(stat_out, pg);
        }
        auto emit = [&](Unf& u) {
            total_source_rows++;                               // Purger.updateProgress :366-371
            bool keep = u.is_row ? purge_row(u, pg) : purge_marker(u, pg);
            if (!keep) return;
            if (!started) { w.start_partition((const uint8_t*)keycopy.data(), (int)keycopy.size(), out_pdel, have_static ? &stat_out : nullptr); started = true; }
            w.add_unfiltered(u); written++;
        };
        if (group.size() == 1) {
            // single source: MergeIterator.get -> TrivialOneToOne (trivialReduceIsTrivial() == true without a listener,
            // UnfilteredRowIterators.java:552-556): unfiltereds pass through untouched, then purge
            Source& s = srcs[group[0]]; Unf u;
            while (read_unfiltered(s, sc, u)) emit(u);
        } else {
            MarkerMerger mm; mm.init(group.size(), pdel);
            for (size_t g = 0; g < group.size(); g++) head_ok[g] = read_unfiltered(srcs[group[g]], sc, heads[g]);
            for (;;) {
                int b = -1;
                for (size_t g = 0; g < group.size(); g++) if (head_ok[g] && (b < 0 || compare_clust(sc, heads[g].c, heads[b].c) < 0)) b = (int)g;
                if (b < 0) break;
                std::vector<size_t> eq;
                for (size_t g = 0; g < group.size(); g++) if (head_ok[g] && compare_clust(sc, heads[g].c, heads[b].c) == 0) eq.push_back(g);
                Unf out; bool have;
                if (heads[b].is_row) {                         // MergeReducer.getReduced :575-591
                    std::vector<Unf*> vs; for (size_t g : eq) vs.push_back(&heads[g]);
                    have = merge_rows(vs, mm.active(), out, &sc);
                } else {
                    std::vector<std::pair<int, Unf*>> vs; for (size_t g : eq) vs.push_back({(int)g, &heads[g]});
                    have = mm.merge(vs, out);
                }
                if (have) emit(out);
                for (size_t g : eq) head_ok[g] = read_unfiltered(srcs[group[g]], sc, heads[g]);
            }
        }
        // partition.isEmpty(): S/db/rows/UnfilteredRowIterator.java:63-68; SortedTableWriter.append :134
        if (!started && (!out_pdel.live() || have_static)) { w.start_partition((const uint8_t*)keycopy.data(), (int)keycopy.size(), out_pdel, have_static ? &stat_out : nullptr); started = true; }
        if (started) w.end_partition((const uint8_t*)keycopy.data(), (int)keycopy.size(), out_pdel, written);
        for (int i : group) next_partition(srcs[i], m->token_lo, m->token_hi);
    }
    w.finish_output();
    if (w.outs.size() > 1 && w.outs.back().parts == 0) w.outs.pop_back();
    res->noutputs = (int)w.outs.size();
    res->bytes_read = bytes_read; res->total_source_rows = total_source_rows; res->input_partitions = input_partitions;
    res->bytes_in_range = 0; for (auto& sr : srcs) res->bytes_in_range += sr.range_bytes;
    if (ro) {
        ro->ustream = std::move(w.outs[0].data); ro->index = std::move(w.outs[0].index); ro->partitions = w.outs[0].parts; ro->rows = w.outs[0].rows;
        res->bytes_written = ro->ustream.size(); res->noutputs = 1;
        return B200C_OK;
    }
    uint64_t bw = 0; int rc = B200C_OK;
    res->required_data_cap = res->required_index_cap = res->required_chunk_cap = 0;
    for (size_t i = 0; i < w.outs.size(); i++) {
        auto& o = w.outs[i]; bw += o.ulen;
        res->required_data_cap = std::max<uint64_t>(res->required_data_cap, o.data.size());
        res->required_index_cap = std::max<uint64_t>(res->required_index_cap, o.index.size());
        res->required_chunk_cap = std::max<uint64_t>(res->required_chunk_cap, o.offs.size());
        if ((int)i >= res->noutputs_cap) { rc = B200C_ETOOSMALL; continue; }
        b200c_output& out = res->outputs[i];
        if (o.data.size() > out.data_cap || o.index.size() > out.index_cap || o.offs.size() > out.chunk_cap) { rc = B200C_ETOOSMALL; continue; }
        memcpy(out.data, o.data.data(), o.data.size()); out.data_len = o.data.size();
        memcpy(out.index, o.index.data(), o.index.size()); out.index_len = o.index.size();
        memcpy(out.chunk_offsets, o.offs.data(), o.offs.size() * 8); out.nchunks = o.offs.size();
        out.data_length = o.ulen; out.digest = o.digest; out.partitions = o.parts; out.rows = o.rows;
        // optional components (b200c_output: NULL pointer = skip)
        out.first_key_len = (uint32_t)o.meta.first.size(); out.last_key_len = (uint32_t)o.meta.last.size();
        if (out.key_buf) { if (out.key_cap < o.meta.first.size() + o.meta.last.size()) rc = B200C_ETOOSMALL; else { memcpy(out.key_buf, o.meta.first.data(), o.meta.first.size()); memcpy(out.key_buf + o.meta.first.size(), o.meta.last.data(), o.meta.last.size()); } }
        if (out.filter) { auto f = o.meta.filter_image(); out.filter_len = f.size(); if (f.size() > out.filter_cap) rc = B200C_ETOOSMALL; else if (!f.empty()) memcpy(out.filter, f.data(), f.size()); }
        if (out.summary) { auto sm = o.meta.summary_image(); out.summary_len = sm.size(); if (sm.size() > out.summary_cap) rc = B200C_ETOOSMALL; else if (!sm.empty()) memcpy(out.summary, sm.data(), sm.size()); }
        if (out.stats) o.meta.fill(out.stats);
    }
    res->bytes_written = bw;
    res->kernel_ms = 0; res->kernel_launches = 0; res->index_slow_path_inputs = 0;
    res->total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return rc;
}

} // namespace oracle

extern "C" int orc_compact(const b200c_manifest* m, b200c_result* res, char* errbuf, int errcap) {
    try { return oracle::compact_impl(m, res, nullptr); }
    catch (oracle::Unsupported& u) { if (errbuf) snprintf(errbuf, errcap, "unsupported: %s", u.what.c_str()); return B200C_EUNSUPPORTED; }
    catch (oracle::Corrupt& c) {
        res->corruption.input = c.input; res->corruption.kind = c.kind; res->corruption.chunk = c.chunk; res->corruption.offset = c.offset;
        if (errbuf) snprintf(errbuf, errcap, "corrupt: %s", c.what.c_str());
        return B200C_ECORRUPT;
    }
}

// test hook: CounterContext.merge on two contexts. Returns the merged length (bytes in out), or -1 when a context is malformed / out too small.
extern "C" int orc_counter_merge(const uint8_t* l, int ll, const uint8_t* r, int rl, uint8_t* out, int cap, int* which) {
    if (!oracle::ctr::well_formed(l, ll) || !oracle::ctr::well_formed(r, rl)) return -1;
    std::vector<uint8_t> buf;
    const int w = oracle::ctr::merge(l, ll, r, rl, buf);
    if (which) *which = w;
    const uint8_t* p = w == 0 ? l : (w == 1 ? r : buf.data()); const int n = w == 0 ? ll : (w == 1 ? rl : (int)buf.size());
    if (n > cap) return -1;
    memcpy(out, p, n);
    return n;
}
extern "C" int orc_counter_has_legacy_shards(const uint8_t* c, int n) { return oracle::ctr::well_formed(c, n) ? (oracle::ctr::has_legacy_shards(c, n) ? 1 : 0) : -1; }
