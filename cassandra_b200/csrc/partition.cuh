// partition.cuh — per-partition row merge, tombstone/timestamp reconciliation, purge and big-format serialisation.
//
// One thread owns one OUTPUT partition (the group of same-key input partitions found by the tournament merge) and runs
// the same code twice: a size pass (counting sinks) and an emit pass (byte sinks) — "size -> exclusive scan -> emit".
// Replaces, for that partition, the reference's lazy iterator stack:
//   UnfilteredRowIterators.UnfilteredRowMergeIterator   S/db/rows/UnfilteredRowIterators.java:398-601
//   Row.Merger.merge / ColumnDataReducer                S/db/rows/Row.java:730-849
//   Cells.reconcile / resolveRegular                    S/db/rows/Cells.java:68-121
//   RangeTombstoneMarker.Merger                         S/db/rows/RangeTombstoneMarker.java:72-199
//   PurgeFunction + BTreeRow.purge + AbstractCell.purge S/db/partitions/PurgeFunction.java:36-145, S/db/rows/BTreeRow.java:457-499,
//                                                       S/db/rows/AbstractCell.java:78-99
//   SortedTablePartitionWriter / UnfilteredSerializer   S/io/sstable/format/SortedTablePartitionWriter.java:97-166,
//                                                       S/db/rows/UnfilteredSerializer.java:151-305, S/db/rows/Cell.java:268-305
//   BigFormatPartitionWriter / IndexInfo / RowIndexEntry S/io/sstable/format/big/BigFormatPartitionWriter.java:128-251,
//                                                       S/io/sstable/IndexInfo.java:107-117, .../big/RowIndexEntry.java:625-642
// Envelope: simple regular columns (< 64), simple static columns (<= 16), <= 8 clustering columns, no complex columns / counters.
#pragma once
#include "common.cuh"

namespace b200c {

enum { MAXK = 64, MAXCOLS = 64, MAXCLUST = 8, MAXSTAT = 16, MAXCX = 8 };
enum { TYPE_BYTES = 0, TYPE_FIXED_SIGNED = 1, TYPE_FIXED_BYTES = 2, TYPE_VAR_SIGNED = 3, TYPE_TIMEUUID = 4 };
enum { K_EXCL_END = 0, K_INCL_START = 1, K_EXCL_END_INCL_START = 2, K_STATIC = 3, K_CLUSTERING = 4, K_INCL_END_EXCL_START = 5, K_INCL_END = 6, K_EXCL_START = 7 };
enum { PERR_NONE = 0, PERR_CORRUPT = 1, PERR_UNSUPPORTED = 2 };

#define I64_MIN ((int64_t)0x8000000000000000LL)
#define I64_MAX ((int64_t)0x7FFFFFFFFFFFFFFFLL)

struct InDesc {
    uint64_t ubase, ulen;          // this input's uncompressed stream inside U
    uint64_t ibase, ilen;          // this input's Index.db (or the slice of it a token sub-range needs) inside IDX
    uint64_t uend;                 // end of the last partition the Index.db slice describes, as an offset in this input's stream (= ulen for the whole file)
    int64_t min_ts, min_ldt; int32_t min_ttl; int32_t ncols;
    int32_t colmap[MAXCOLS];
    int32_t nstat, _pad; int32_t smap[MAXSTAT];      // static columns of this input's header -> output static columns
};
struct CParams {
    const uint8_t* U;              // all inputs' uncompressed Data streams, back to back (16-byte aligned bases)
    int32_t ninputs, nclust, ncols, column_index_size;
    int32_t ctype[MAXCLUST], cfix[MAXCLUST], vfix[MAXCOLS];
    int64_t o_min_ts, o_min_ldt; int32_t o_min_ttl;
    int32_t nstat, sfix[MAXSTAT];  // static columns of the output header (0: the table has none, no static rows anywhere)
    int32_t mcols;                 // max(ncols, nstat): cells of scratch a merged row needs
    // multi-cell (complex) columns: the LAST ncx regular columns (ColumnMetadata.comparisonOrder puts them behind the simple ones); vfix[] of
    // those is the fixed length of their cell VALUES, ptype / pfix class and fixed length of their cell PATHS
    int32_t ncx, cx_first;
    int32_t ptype[MAXCX], pfix[MAXCX];
    uint64_t ctr_mask;             // bit c: regular simple column c is a counter column (cells merged shard by shard; tables with any use the CX kernels)
    uint64_t sctr_mask;            // the same for the static columns
    int32_t partitioner;           // 0 Murmur3Partitioner, 1 ByteOrderedPartitioner (tok[] then holds the sign-flipped 8-byte key prefix)
    int64_t now, gc_before, purge_max_ts;
    // optional purge table (b200c_manifest.purge_range_*): ascending token bounds and the threshold that applies up to each of them
    const int64_t* purge_hi; const int64_t* purge_ts; int64_t npurge;
    const InDesc* in;              // ninputs descriptors (device memory; the header above is small enough to be copied into shared memory)
};

struct DT { int64_t mfda, ldt; };
__device__ __forceinline__ DT dt_live() { DT d; d.mfda = I64_MIN; d.ldt = I64_MAX; return d; }
__device__ __forceinline__ bool dt_is_live(const DT& d) { return d.mfda == I64_MIN && d.ldt == I64_MAX; }
__device__ __forceinline__ bool dt_supersedes(const DT& a, const DT& b) { return a.mfda > b.mfda || (a.mfda == b.mfda && a.ldt > b.ldt); }
__device__ __forceinline__ bool dt_deletes(const DT& d, int64_t ts) { return ts <= d.mfda; }
__device__ __forceinline__ bool dt_eq(const DT& a, const DT& b) { return a.mfda == b.mfda && a.ldt == b.ldt; }

struct Live { int64_t ts, ldt; int32_t ttl; };
__device__ __forceinline__ Live live_empty() { Live l; l.ts = I64_MIN; l.ldt = I64_MAX; l.ttl = 0; return l; }
__device__ __forceinline__ bool live_is_empty(const Live& l) { return l.ts == I64_MIN; }
__device__ __forceinline__ bool live_is_live(const Live& l, int64_t now) {
    if (l.ts == I64_MIN) return false; if (l.ttl == 0x7FFFFFFF) return false; if (l.ttl != 0) return now < l.ldt; return true; }
__device__ __forceinline__ bool live_supersedes(const Live& a, const Live& b) {      // LivenessInfo.supersedes :216-225
    if (a.ts != b.ts) return a.ts > b.ts;
    bool ae = a.ttl == 0x7FFFFFFF, be = b.ttl == 0x7FFFFFFF;
    if (ae != be) return ae;
    if ((a.ttl != 0) == (b.ttl != 0)) return a.ldt > b.ldt;
    return a.ttl != 0;
}

struct MCell { int64_t ts, ldt; uint64_t voff; int32_t ttl, vlen; bool present; };

__device__ __forceinline__ int kind_comparison(int k) { return (0x33321000 >> (4 * k)) & 0xF; }          // {0,0,0,1,2,3,3,3}
__device__ __forceinline__ int kind_vs_clustering(int k) { return k < 4 ? -1 : (k == 4 ? 0 : 1); }
__device__ __forceinline__ bool kind_is_boundary(int k) { return k == K_EXCL_END_INCL_START || k == K_INCL_END_EXCL_START; }
__device__ __forceinline__ bool kind_is_start(int k) { return k == K_INCL_START || k == K_EXCL_START; }

// vint decode / encode as free functions with by-value arguments and results: member functions that are not inlined would take
// `this`, which forces the reader / sink / writer objects out of registers and into local memory.
__device__ __noinline__ void vint_store(uint8_t* dst, uint64_t v, int size) {
    if (size == 1) { dst[0] = (uint8_t)v; return; }
    if (size < 9) {
        uint64_t reg = (v << ((8 - size) << 3)) | ((uint64_t)(uint8_t)(~(0xffu >> (size - 1))) << 56);
#pragma unroll 1
        for (int i = 0; i < size; i++) dst[i] = (uint8_t)(reg >> (56 - 8 * i));
        return;
    }
    dst[0] = 0xFF; for (int i = 0; i < 8; i++) dst[1 + i] = (uint8_t)(v >> (56 - 8 * i));
}
__device__ __noinline__ void bytes_copy(uint8_t* dst, const uint8_t* src, uint32_t n) {
    for (uint32_t i = 0; i < n; i += 8) {                // one wide (unaligned) load per 8 bytes, byte stores
        uint64_t x = load_be64(src + i);
        uint32_t k = n - i < 8 ? n - i : 8;
#pragma unroll 1
        for (uint32_t b = 0; b < k; b++) dst[i + b] = (uint8_t)(x >> (56 - 8 * b));
    }
}

// ---- bounded reader over U ------------------------------------------------------------------------------------------------
// vint decode as a free noinline function with by-value result (one copy in the instruction cache, nothing forced to local
// memory); the bytes of a multi-byte vint come from one unaligned 8-byte fetch instead of a byte loop.
struct VintR { uint64_t v; uint32_t n; };
__device__ __noinline__ VintR vint_decode(const uint8_t* p, uint32_t avail) {      // avail = bytes readable at p (capped at 9)
    VintR r; r.v = 0; r.n = 0;
    if (!avail) return r;
    uint32_t first = p[0];
    if (first < 0x80) { r.v = first; r.n = 1; return r; }
    uint32_t extra = __clz((int)(~(first << 24)));                                 // leading one bits = extra bytes (8 for 0xFF)
    if (1 + extra > avail) return r;
    if (extra == 8) { r.v = load_be64(p + 1); r.n = 9; return r; }
    uint64_t x = load_be64(p);                                                     // p[0..7], big-endian
    uint32_t nbits = 8 * (extra + 1) - extra;                                      // value bits of the (extra + 1)-byte field
    r.v = (x >> (8 * (7 - extra))) & ((1ull << nbits) - 1ull); r.n = 1 + extra;
    return r;
}
// value and position behind it; np == ~0: the vint runs past `end` (every buffer the reader walks has >= 16 bytes of slack behind it: one unaligned 8-byte fetch)
struct VintP { uint64_t v, np; };
__device__ __noinline__ VintP rd_vint_fn(const uint8_t* U, uint64_t p, uint64_t end) {
    VintP r; r.v = 0; r.np = ~0ull;
    if (p >= end) return r;
    const uint64_t x = load_be64(U + p);
    const uint32_t first = (uint32_t)(x >> 56);
    if (first < 0x80) { r.v = first; r.np = p + 1; return r; }
    const uint32_t extra = __clz((int)(~(first << 24)));                       // leading one bits = extra bytes (8 for 0xFF)
    if (end - p < 1 + (uint64_t)extra) return r;
    if (extra == 8) r.v = (x << 8) | U[p + 8];
    else r.v = (x >> (8 * (7 - extra))) & ((1ull << (8 + 7 * extra)) - 1ull);
    r.np = p + 1 + extra;
    return r;
}
struct Rd {
    const uint8_t* U; uint64_t p, end; int err;
    __device__ __forceinline__ uint32_t u8() { if (p >= end) { err = PERR_CORRUPT; return 1; } return U[p++]; }
    __device__ __forceinline__ uint32_t be16() { uint32_t a = u8(); return (a << 8) | u8(); }
    // VIntCoding.readUnsignedVInt (S/utils/vint/VIntCoding.java:66-98). ONE out-of-line copy (rd_vint_fn): this reader is used at ~40 places of
    // the per-partition code; inlined, its copies alone were a quarter of the instructions the hot loop touches, the kernel's hot code
    // did not fit the instruction cache, and "no instruction" was the top stall reason.
    __device__ __forceinline__ uint64_t vint() {
        const VintP r = rd_vint_fn(U, p, end);
        if (r.np == ~0ull) { err = PERR_CORRUPT; p = end; return 0; }
        p = r.np; return r.v;
    }
    __device__ __forceinline__ int32_t vint32() { uint64_t v = vint(); int32_t r = (int32_t)v; if ((int64_t)r != (int64_t)v) err = PERR_CORRUPT; return r; }
    __device__ __forceinline__ void skip(uint64_t n) { if (end - p < n) { err = PERR_CORRUPT; p = end; } else p += n; }
};

// ---- sinks ----------------------------------------------------------------------------------------------------------------
template <bool EMIT> struct Sink {
    uint8_t* base; uint64_t pos; bool on;      // on: this lane performs the stores (tile mode: lane 0 only; every lane tracks pos)
    uint64_t cap;                              // bytes available at base: stores beyond it are dropped (the caller sees pos > cap)
    __device__ __forceinline__ void u8(uint32_t v) { if (EMIT && on && pos < cap) base[pos] = (uint8_t)v; pos++; }
    __device__ __forceinline__ void be16(uint32_t v) { u8(v >> 8); u8(v); }
    __device__ __forceinline__ void be32(uint32_t v) { u8(v >> 24); u8(v >> 16); u8(v >> 8); u8(v); }
    __device__ __forceinline__ void be64(uint64_t v) { be32((uint32_t)(v >> 32)); be32((uint32_t)v); }
    __device__ __forceinline__ void vint(uint64_t v) {
        int size = vint_size(v);
        if (EMIT && on && pos + size <= cap) vint_store(base + pos, v, size);
        pos += size;
    }
    __device__ __forceinline__ void copy(const uint8_t* src, uint32_t n) { if (EMIT && on && pos + n <= cap) bytes_copy(base + pos, src, n); pos += n; }
};

struct CkRef { uint64_t off; uint32_t len; uint8_t kind, n; };      // serialised clustering values (header vint + values) in U

// cursor of one contributing input partition; it lives in shared memory, so its size decides how many partitions an SM can hold.
// OFF: type of the stream positions (offsets from P.U), REL: type of the offsets inside one unfiltered header.
//   Cur   = CurT<uint64_t, uint32_t> (48 bytes): P.U is the whole decompressed input in global memory
//   CurS  = CurT<uint32_t, uint16_t> (32 bytes): P.U is a tile of < 64 KiB staged in shared memory (k_partition_staged)
template <int PAD> struct CurPad { uint8_t pad_[PAD]; };
template <> struct CurPad<0> {};
template <typename OFF, typename REL, int PAD = 0> struct CurT : CurPad<PAD> {
    uint64_t k0;                   // order-preserving 64-bit prefix of the first clustering component (see cur_load)
    OFF pos, next, end;            // current unfiltered, the one after it, end of the partition
    REL ckend_rel, body_rel;       // offsets from pos: end of the clustering values, start of the body
    uint8_t ck_rel;                // offset from pos of the clustering values (1..4)
    uint8_t flags, ext, kind, n, src; bool done;
    uint8_t fast;                  // 0: no prefix key; 1: k0 orders unequal prefixes, ties need cmp_clust; 2: k0 is the whole clustering
    typedef REL rel_t;
    __host__ __device__ static constexpr uint64_t rel_max() { return (uint64_t)(REL)~(REL)0; }
};
typedef CurT<uint64_t, uint32_t> Cur;
// The same cursor in 32 bytes, for the thread-per-partition kernels whose residency is set by shared memory (16 cursors per thread): stream
// offsets in 40 bits (the engine refuses inputs whose decompressed streams add up to 2^40 bytes), header-relative offsets in 20 bits (a
// clustering prefix is at most 8 values of < 64 KiB each), the small fields in what is left. Bit-fields keep the field syntax, so the
// code above and below is the same for every cursor type; the extra shifts and masks ride in issue slots this latency-bound kernel leaves idle.
struct Cur32 {
    uint64_t k0;
    uint64_t pos : 40, ckend_rel : 20, n : 4;
    uint64_t next : 40, body_rel : 20, kind : 3, done : 1;
    uint64_t end : 40, flags : 8, src : 6, ck_rel : 3, ext : 2, fast : 2;
    typedef uint32_t rel_t;
    __host__ __device__ static constexpr uint64_t rel_max() { return (1ull << 20) - 1; }
};
static_assert(sizeof(Cur32) == 32, "packed cursor layout");
// 40-byte stride: 32-byte cursors of different threads would all start in one of four bank groups (8-way conflicts on every field)
typedef CurT<uint32_t, uint16_t, 8> CurS;
static_assert(sizeof(Cur) == 48 && sizeof(CurS) == 40, "cursor layouts");

// parses the unfiltered header at c.pos (skipping empty rows: UnfilteredSerializer.deserialize :433-447)
template <class CUR> __device__ __noinline__ int cur_load_impl(const CParams& P, CUR& c) {
    int err = 0;
    for (;;) {
        Rd r{P.U, c.pos, c.end, 0};
        uint32_t flags = r.u8();
        if (r.err) { c.done = true; return PERR_CORRUPT; }
        if (flags & 0x01) { c.done = true; c.next = r.p; return 0; }
        c.flags = (uint8_t)flags; c.ext = 0;
        if (flags & 0x02) {
            const uint32_t kind = r.u8(), nv = r.be16();           // (checked before they go into the cursor: its fields may be narrower)
            if (kind > 7 || kind == K_STATIC || kind == K_CLUSTERING || nv > (uint32_t)P.nclust) { c.done = true; return PERR_CORRUPT; }
            c.kind = (uint8_t)kind; c.n = (uint8_t)nv;
        } else {
            if (flags & 0x80) c.ext = (uint8_t)(r.u8() & 0x03);
            if (c.ext & 0x01) { c.done = true; return PERR_CORRUPT; }       // a static row among the clustered ones (UnfilteredSerializer.deserialize :477-479)
            if ((c.ext & 0x02) || ((flags & 0x40) && !P.ncx)) { c.done = true; return PERR_UNSUPPORTED; }      // shadowable deletion; HAS_COMPLEX_DELETION without multi-cell columns
            c.kind = K_CLUSTERING; c.n = (uint8_t)P.nclust;
        }
        c.ck_rel = (uint8_t)(r.p - c.pos);
        c.fast = 0; c.k0 = 0;
        if (c.n) {
            uint64_t header = r.vint();
            for (int i = 0; i < c.n; i++) {
                if ((header >> (2 * i)) & 3) continue;
                uint64_t len = P.cfix[i] > 0 ? (uint64_t)P.cfix[i] : r.vint();
                if (i == 0 && !r.err && r.end - r.p >= len) {
                    // first component, non-null and non-empty: big-endian prefix, sign bit flipped for the signed classes
                    int t = P.ctype[0]; int take = len < 8 ? (int)len : 8;
                    uint64_t k = load_be64(P.U + r.p);
                    if (take < 8) k &= ~0ull << (8 * (8 - take));
                    if (t == TYPE_FIXED_SIGNED || t == TYPE_VAR_SIGNED) k ^= 0x8000000000000000ull;
                    c.k0 = k;
                    bool whole = (t == TYPE_FIXED_SIGNED || t == TYPE_FIXED_BYTES) && len <= 8;      // equal prefix <=> equal value
                    c.fast = (whole && P.nclust == 1 && c.n == 1) ? 2 : ((t == TYPE_VAR_SIGNED && len > 8) ? 0 : 1);
                }
                r.skip(len);
            }
        }
        c.ckend_rel = (typename CUR::rel_t)(r.p - c.pos);
        uint64_t sz = r.vint();
        uint64_t after = r.p;
        r.vint();                                   // previous unfiltered size
        c.body_rel = (typename CUR::rel_t)(r.p - c.pos);
        const uint64_t nx = after + sz;                  // (64-bit: a damaged size must not wrap a narrow cursor)
        if (r.err || nx > c.end || nx < r.p || r.p - c.pos > CUR::rel_max()) { c.done = true; return PERR_CORRUPT; }
        c.next = (decltype(c.next))nx;
        if (!(flags & 0x02) && !(flags & 0x14)) {   // maybe an empty row: no liveness, no deletion — any cells?
            int ncin = P.in[c.src].ncols; bool any;
            if (flags & 0x20) any = ncin > 0;
            else { Rd b{P.U, c.pos + c.body_rel, c.next, 0}; uint64_t missing = b.vint(); uint64_t mask = ncin >= 64 ? ~0ull : ((1ull << ncin) - 1); any = ((~missing) & mask) != 0; }
            if (!any) { c.pos = c.next; continue; }
        }
        return err;
    }
}
template <class CUR> __device__ __forceinline__ void cur_load(const CParams& P, CUR& c, int& err) { int e = cur_load_impl(P, c); if (e) err = e; }

// The static row at c.pos, right after the partition deletion (SSTableSimpleIterator.readStaticRow -> UnfilteredSerializer.deserializeStaticRow
// :538-552): parsed INTO the cursor (flags, body_rel, next) so that row_header / fold_cells read it like any other row. *nonempty: it
// has liveness, a deletion or at least one cell.
template <class CUR> __device__ __noinline__ int static_load(const CParams& P, CUR& c, bool* nonempty) {
    Rd r{P.U, c.pos, c.end, 0};
    uint32_t flags = r.u8(), ext = r.u8();
    if (r.err || (flags & 0x03) || !(flags & 0x80) || !(ext & 0x01)) return PERR_CORRUPT;
    if ((ext & 0x02) || (flags & 0x40)) return PERR_UNSUPPORTED;
    c.flags = (uint8_t)flags; c.ext = (uint8_t)(ext & 0x03); c.kind = K_STATIC; c.n = 0; c.ck_rel = 2; c.ckend_rel = 2; c.fast = 0;
    uint64_t sz = r.vint();
    uint64_t after = r.p;
    r.vint();                                       // previous unfiltered size (0)
    c.body_rel = (typename CUR::rel_t)(r.p - c.pos);
    const uint64_t nx = after + sz;
    if (r.err || nx > c.end || nx < r.p) return PERR_CORRUPT;
    c.next = (decltype(c.next))nx;
    *nonempty = true;
    if (!(flags & 0x14)) {
        int ncin = P.in[c.src].nstat;
        if (flags & 0x20) *nonempty = ncin > 0;
        else { Rd b{P.U, c.pos + c.body_rel, c.next, 0}; uint64_t missing = b.vint(); *nonempty = ((~missing) & ((1ull << ncin) - 1)) != 0; }
    }
    return 0;
}

__device__ __forceinline__ int cmp_bytes(const uint8_t* a, int la, const uint8_t* b, int lb) {
    int n = la < lb ? la : lb;
    for (int i = 0; i < n; i += 8) {                     // unsigned lexicographic order == big-endian integer order
        uint64_t x = load_be64(a + i), y = load_be64(b + i);
        int k = n - i;
        if (k < 8) { uint64_t mk = ~0ull << (8 * (8 - k)); x &= mk; y &= mk; }
        if (x != y) return x < y ? -1 : 1;
    }
    return la == lb ? 0 : (la < lb ? -1 : 1);
}
__device__ __forceinline__ int cmp_value(int type, const uint8_t* a, int la, const uint8_t* b, int lb) {
    if (type == TYPE_FIXED_SIGNED || type == TYPE_VAR_SIGNED) {
        if (la == 0 || lb == 0) return la == 0 ? (lb == 0 ? 0 : -1) : 1;
        int d = (int)(int8_t)a[0] - (int)(int8_t)b[0];
        if (d) return d < 0 ? -1 : 1;
        return cmp_bytes(a + 1, la - 1, b + 1, lb - 1);
    }
    return cmp_bytes(a, la, b, lb);
}

// ClusteringComparator.compare: S/db/ClusteringComparator.java:140-157
template <class CUR> __device__ __noinline__ int cmp_clust(const CParams& P, const CUR& a, const CUR& b) {
    const uint8_t* pa = P.U + a.pos + a.ck_rel; const uint8_t* pb = P.U + b.pos + b.ck_rel;
    const uint8_t* ea = P.U + a.pos + a.ckend_rel; const uint8_t* eb = P.U + b.pos + b.ckend_rel;
    int m = a.n < b.n ? a.n : b.n;
    uint64_t ha = 0, hb = 0;
    if (a.n) pa += vint_read(pa, ea, &ha);
    if (b.n) pb += vint_read(pb, eb, &hb);
    for (int i = 0; i < m; i++) {
        bool na = (ha >> (2 * i + 1)) & 1, nb = (hb >> (2 * i + 1)) & 1;
        bool xa = (ha >> (2 * i)) & 1, xb = (hb >> (2 * i)) & 1;
        int la = 0, lb = 0;
        if (!na && !xa) { if (P.cfix[i] > 0) la = P.cfix[i]; else { uint64_t v = 0; pa += vint_read(pa, ea, &v); la = (int)v; } }
        if (!nb && !xb) { if (P.cfix[i] > 0) lb = P.cfix[i]; else { uint64_t v = 0; pb += vint_read(pb, eb, &v); lb = (int)v; } }
        if (na || nb) { if (na != nb) return na ? -1 : 1; }
        else { int c = cmp_value(P.ctype[i], pa, la, pb, lb); if (c) return c; }
        pa += la; pb += lb;
    }
    if (a.n == b.n) { int d = kind_comparison(a.kind) - kind_comparison(b.kind); return d < 0 ? -1 : (d > 0 ? 1 : 0); }
    return a.n < b.n ? kind_vs_clustering(a.kind) : -kind_vs_clustering(b.kind);
}

// cmp_clust with the cached prefix keys in front: unequal prefixes decide, equal "whole" keys only need the kind comparison
template <class CUR> __device__ __forceinline__ int cmp_heads(const CParams& P, const CUR& a, const CUR& b) {
    if (a.fast && b.fast) {
        if (a.k0 != b.k0) return a.k0 < b.k0 ? -1 : 1;
        if (a.fast == 2 && b.fast == 2) { int d = kind_comparison(a.kind) - kind_comparison(b.kind); return d < 0 ? -1 : (d > 0 ? 1 : 0); }
    }
    return cmp_clust(P, a, b);
}

// header.readDeletionTime + DeletionTime.build (S/db/DeletionTime.java:54-58): an ldt below 0 (a wrapped delta) or above MAX_DELETION_TIME reads
// as InvalidDeletionTime (ldt 2^32 - 2). Row deletions, markers and complex deletions all read through here. One unsigned compare and a select.
__device__ __forceinline__ DT read_delta_dt(Rd& r, const InDesc& in) {
    DT d; d.mfda = (int64_t)(r.vint() + (uint64_t)in.min_ts); d.ldt = (int64_t)r.vint32() + in.min_ldt;
    d.ldt = (uint64_t)d.ldt > 0xFFFFFFFDull ? (int64_t)0xFFFFFFFEu : d.ldt;
    return d;
}
__device__ __forceinline__ int64_t decode_ldt(int64_t ldt, int32_t ttl) {          // Cell.decodeLocalDeletionTime :221-239
    if (ldt >= ttl) return ldt;
    if (ldt < 0) return (int64_t)(uint32_t)(int32_t)ldt;
    if (ttl == 0x7FFFFFFF) return ldt;
    return (int64_t)0xFFFFFFFEu;
}
// the row liveness's ldt is decoded as a cell's (UnfilteredSerializer.java:596-598). Out of line: row_header is inlined into every K4 kernel, and
// rows with a TTL are rare enough that a call costs less than the registers an inlined copy takes in the emitting kernels.
__device__ __noinline__ int64_t decode_liveness_ldt(int64_t ldt, int32_t ttl) { return decode_ldt(ldt, ttl); }
// DeletionTime.Serializer.deserialize (oa): S/db/DeletionTime.java:222-243
__device__ __forceinline__ DT read_partition_dt(Rd& r) {
    uint32_t f = r.u8();
    if (f & 0x80) { if (f != 0x80) r.err = PERR_CORRUPT; return dt_live(); }
    uint64_t m = f; for (int i = 0; i < 7; i++) m = (m << 8) | r.u8();
    uint64_t l = 0; for (int i = 0; i < 4; i++) l = (l << 8) | r.u8();
    DT d; d.mfda = (int64_t)m; d.ldt = (int64_t)l; return d;
}

struct Purger {
    int64_t now, gc_before, max_ts;
    __device__ __forceinline__ bool ts_ldt(int64_t ts, int64_t ldt) const { return ldt < gc_before && (max_ts == I64_MAX || ts < max_ts); }
    __device__ __forceinline__ bool dt(const DT& d) const { return !dt_is_live(d) && ts_ldt(d.mfda, d.ldt); }
    __device__ __forceinline__ bool live(const Live& l) const { return !live_is_live(l, now) && ts_ldt(l.ts, l.ldt); }
};

// Cells.resolveRegular: S/db/rows/Cells.java:83-121. true => keep `l`, false => take `r`
__device__ bool reconcile_keep_left(const CParams& P, const MCell& l, const MCell& r) {
    if (l.ts != r.ts) return l.ts > r.ts;
    bool le = l.ldt != I64_MAX, re = r.ldt != I64_MAX;
    if (le | re) {
        if (le != re) return le;
        bool lt = l.ttl == 0, rt = r.ttl == 0;
        if (lt != rt) return lt;
        if (l.ldt != r.ldt) return l.ldt > r.ldt;
    }
    return cmp_bytes(P.U + l.voff, l.vlen, P.U + r.voff, r.vlen) >= 0;
}

// promoted-index slot of the scratch pass: [partition deletion (mfda, ldt), headerLength: 3 x int64][i32 offsets x nb_max][IndexInfo bytes, IXS_PER_BLOCK budget per block]
enum { IXS_HEAD = 24, IXS_PER_BLOCK = 204, IXS_BLOCK_STRIDE = 4 + IXS_PER_BLOCK };

// ---- MetadataCollector's reductions, gathered where the rows are written (S/io/sstable/metadata/MetadataCollector.java:208-270; called from
// SortedTableWriter.startPartition / addRow / addRangeTomstoneMarker S/io/sstable/format/SortedTableWriter.java:183-238 and Rows.collectStats
// S/db/rows/Rows.java:102-113). One accumulator per thread, in registers; the kernels fold them into a StatGlobal at the end of the block.
enum { TDROP_SLOTS = 65536 };             // distinct 60 s-rounded drop times the table can hold (45 days of minutes); beyond: overflow flag
struct TdropTable { unsigned long long key[TDROP_SLOTS]; unsigned long long cnt[TDROP_SLOTS]; unsigned int overflow; unsigned int _pad; };   // rounded drop time -> count
struct StatAcc {
    int64_t min_ts, max_ts, min_ldt, max_ldt; int32_t min_ttl, max_ttl; uint32_t seen;     // seen: bit0 ts, bit1 ldt, bit2 ttl
    unsigned long long rows, cols, cells, tombs; uint32_t pdel, part_cells;
    int64_t now; TdropTable* td;
    __device__ __forceinline__ void init(int64_t now_, TdropTable* td_) { min_ts = max_ts = min_ldt = max_ldt = 0; min_ttl = max_ttl = 0; seen = 0; rows = cols = cells = tombs = 0; pdel = part_cells = 0; now = now_; td = td_; }
    __device__ __forceinline__ void ts(int64_t v) { if (!(seen & 1)) { min_ts = max_ts = v; seen |= 1; } else { min_ts = v < min_ts ? v : min_ts; max_ts = v > max_ts ? v : max_ts; } }
    __device__ __forceinline__ void ttl(int32_t v) { if (!(seen & 4)) { min_ttl = max_ttl = v; seen |= 4; } else { min_ttl = v < min_ttl ? v : min_ttl; max_ttl = v > max_ttl ? v : max_ttl; } }
    __device__ __noinline__ void tdrop(int64_t v) {                        // StreamingTombstoneHistogramBuilder.ceilKey with roundSeconds = 60, exact counts
#ifdef __CUDA_ARCH__
        if (!td) return;
        const int64_t d = v % 60; const unsigned long long pt = (unsigned long long)(d == 0 ? v : v + (60 - d));
        uint32_t h = (uint32_t)(((pt / 60) * 2654435761ull) >> 8) & (TDROP_SLOTS - 1);
        for (int probe = 0; probe < 1024; probe++, h = (h + 1) & (TDROP_SLOTS - 1)) {
            unsigned long long k = td->key[h];
            if (k != pt) { if (k != ~0ull) continue; k = atomicCAS(&td->key[h], ~0ull, pt); if (k != ~0ull && k != pt) continue; }
            atomicAdd(&td->cnt[h], 1ull); return;
        }
        td->overflow = 1;
#endif
    }
    __device__ __forceinline__ void ldt(int64_t v) {
        if (!(seen & 2)) { min_ldt = max_ldt = v; seen |= 2; } else { min_ldt = v < min_ldt ? v : min_ldt; max_ldt = v > max_ldt ? v : max_ldt; }
        if (v != I64_MAX) tdrop(v);
    }
    __device__ __forceinline__ void live(const Live& l) { if (live_is_empty(l)) return; ts(l.ts); ttl(l.ttl); ldt(l.ldt); if (!live_is_live(l, now)) tombs++; }
    __device__ __forceinline__ void dt(const DT& d) { if (dt_is_live(d)) return; ts(d.mfda); ldt(d.ldt); tombs++; }
    __device__ __forceinline__ void cell(const MCell& m) { cells++; part_cells++; ts(m.ts); ttl(m.ttl); ldt(m.ldt); if (!(m.ldt == I64_MAX || (m.ttl != 0 && now < m.ldt))) tombs++; }
};

// ---- partition writer (SortedTablePartitionWriter + BigFormatPartitionWriter state) ------------------------------------------
template <bool EMIT> struct PWriter {
    Sink<EMIT> d;                 // Data stream, positioned at the partition start
    Sink<EMIT> ix;                // IndexInfo bytes of the promoted index (only emitted when nblocks_final > 1)
    uint8_t* ix_offs;             // where the int32 offsets array goes (EMIT and nblocks_final > 1)
    uint64_t start, header_len, prev_row_start, block_start;
    uint32_t nblocks, nblocks_final;
    bool started, have_first;
    CkRef first, last;
    DT open_marker;
    uint64_t rows_out;
    StatAcc* acc;                 // statistics side band (nullptr: not gathered in this pass)
    uint8_t* ix_entry; uint32_t ix_fixed;   // final emit into the Index.db entry itself: ix.base = ix_entry + ix_fixed + vint_size(header_len), set by pw_start
};

template <bool EMIT> __device__ __forceinline__ void write_partition_dt(Sink<EMIT>& s, const DT& d) {
    if (dt_is_live(d)) s.u8(0x80); else { s.be64((uint64_t)d.mfda); s.be32((uint32_t)d.ldt); }
}
template <bool EMIT> __device__ __forceinline__ void write_delta_dt(Sink<EMIT>& s, const CParams& P, const DT& d) {
    s.vint((uint64_t)d.mfda - (uint64_t)P.o_min_ts);
    s.vint((uint64_t)(int64_t)(int32_t)(d.ldt - P.o_min_ldt));
}
template <bool EMIT> __device__ __forceinline__ void write_prefix(Sink<EMIT>& s, const CParams& P, const CkRef& c) {   // ClusteringPrefix.Serializer.serialize :408-421
    s.u8(c.kind);
    if (c.kind != K_CLUSTERING) s.be16(c.n);
    s.copy(P.U + c.off, c.len);
}

template <bool EMIT> __device__ __forceinline__ void pw_add_index_block(PWriter<EMIT>& w, const CParams& P) {
    uint64_t cur = w.d.pos - w.start;
    bool emit_info = EMIT && w.ix.on;              // ix.on: this lane stores IndexInfos (final emit of a partition with > 1 block)
    if (emit_info && w.nblocks < w.nblocks_final) { uint32_t o = (uint32_t)w.ix.pos; uint8_t* q = w.ix_offs + 4 * w.nblocks; q[0] = (uint8_t)(o >> 24); q[1] = (uint8_t)(o >> 16); q[2] = (uint8_t)(o >> 8); q[3] = (uint8_t)o; }
    {                                              // the ix sink always counts; it stores only when ix.on
        write_prefix(w.ix, P, w.first); write_prefix(w.ix, P, w.last);
        w.ix.vint(w.block_start);
        w.ix.vint(zigzag_enc((int64_t)(cur - w.block_start) - 65536));
        w.ix.u8(dt_is_live(w.open_marker) ? 0 : 1);
        if (!dt_is_live(w.open_marker)) write_partition_dt(w.ix, w.open_marker);
    }
    w.nblocks++;
    w.have_first = false;
}

// book-keeping around one serialised unfiltered (SortedTablePartitionWriter.addUnfiltered :128-154, BigFormatPartitionWriter :208-215)
template <bool EMIT> __device__ __forceinline__ uint64_t pw_begin_unf(PWriter<EMIT>& w, const CkRef& ck) {
    uint64_t pos = w.d.pos - w.start;
    if (!w.have_first) { w.first = ck; w.block_start = pos; w.have_first = true; }
    return pos;
}
template <bool EMIT> __device__ __forceinline__ void pw_end_unf(PWriter<EMIT>& w, const CParams& P, const CkRef& ck, uint64_t pos) {
    w.last = ck; w.prev_row_start = pos; w.rows_out++;
    if ((w.d.pos - w.start) - w.block_start >= (uint64_t)P.column_index_size) pw_add_index_block(w, P);
}

struct CxVer { uint64_t cells, end; int64_t its, ildt; int32_t ittl; uint8_t flags, src; };      // one version of the row: where its columns start (behind the row header fields), its liveness (cells may say USE_ROW_TIMESTAMP / USE_ROW_TTL)
struct CxCol { DT cd; uint32_t ncells; uint8_t pre, post; };                                     // merged + purged complex deletion, cells after the purge; column exists before / after the purge
struct CxEmit { const CxVer* ver; int nver; bool as_is; DT active; const CxCol* col; const Purger* pg; bool stat = false; };      // stat: the static row (its columns are P.sfix / InDesc.smap)
template <bool E> __device__ int cx_merge(const CParams& P, const Purger& pg, const CxVer* ver, int nver, bool as_is, DT active, int j,
                                         const Live info, CxCol* sum, Sink<E>* s, bool row_has_cd, const CxCol* known, StatAcc* acc);      // (multi-cell columns, below)
// a merged counter cell has no bytes in an input stream: MCell.voff says so and carries what the header needs (counter columns, below)
constexpr uint64_t CTR_SYNTH = 1ull << 63, CTR_LEGACY = 1ull << 62;
template <bool E> __device__ int ctr_merge(const CParams& P, const CxVer* ver, int nver, DT active, int oc, MCell* sum, Sink<E>* s, int nhdr, bool stat = false);
// row body: UnfilteredSerializer.serializeRowBody :213-269 + Cell.Serializer.serialize S/db/rows/Cell.java:268-305
template <bool E, bool CX = false> __device__ __noinline__ uint64_t put_row_body(Sink<E> s, const CParams& P, int flags, Live info, DT del, const MCell* cells, int ncols, const int32_t* vfix, const CxEmit* cx = nullptr) {
    if (flags & 0x04) s.vint((uint64_t)info.ts - (uint64_t)P.o_min_ts);
    if (flags & 0x08) { s.vint((uint64_t)(int64_t)(info.ttl - P.o_min_ttl)); s.vint((uint64_t)(int64_t)(int32_t)(info.ldt - P.o_min_ldt)); }
    if (flags & 0x10) write_delta_dt(s, P, del);
    if (!(flags & 0x20)) {
        uint64_t missing = 0;
        for (int c = 0; c < ncols; c++) if (!cells[c].present) missing |= 1ull << c;
        s.vint(missing);
    }
    for (int c = 0; c < ncols; c++) {
        const MCell& m = cells[c]; if (!m.present) continue;
        if constexpr (CX) if (!cx->stat && c >= P.cx_first) {          // writeComplexColumn :271-280 (cells[c].present = the column exists)
            cx_merge<E>(P, *cx->pg, cx->ver, cx->nver, cx->as_is, cx->active, c - P.cx_first, info, nullptr, &s, (flags & 0x40) != 0, &cx->col[c - P.cx_first], nullptr);
            continue;
        }
        bool has_value = m.vlen > 0, deleted = m.ldt != I64_MAX && m.ttl == 0, expiring = m.ttl != 0;
        bool use_ts = !live_is_empty(info) && m.ts == info.ts;
        bool use_ttl = expiring && info.ttl != 0 && m.ttl == info.ttl && m.ldt == info.ldt;
        int cf = (has_value ? 0 : 0x04) | (deleted ? 0x01 : (expiring ? 0x02 : 0)) | (use_ts ? 0x08 : 0) | (use_ttl ? 0x10 : 0);
        s.u8(cf);
        if (!use_ts) s.vint((uint64_t)m.ts - (uint64_t)P.o_min_ts);
        if ((deleted || expiring) && !use_ttl) s.vint((uint64_t)(int64_t)(int32_t)(m.ldt - P.o_min_ldt));
        if (expiring && !use_ttl) s.vint((uint64_t)(int64_t)(m.ttl - P.o_min_ttl));
        if constexpr (CX) if (m.voff & CTR_SYNTH) {      // the merged context is written from the versions' contexts (ctr_merge)
            s.vint((uint64_t)m.vlen);
            ctr_merge<E>(P, cx->ver, cx->nver, cx->active, c, nullptr, &s, (int)(m.voff & 0xFFFF), cx->stat);
            continue;
        }
        if (has_value) { if (vfix[c] <= 0) s.vint((uint64_t)m.vlen); s.copy(P.U + m.voff, (uint32_t)m.vlen); }
    }
    return s.pos;
}

struct PartStats { uint64_t merged_unfiltereds; uint64_t rows_out; };

// decodes the row at cursor `c` : liveness + deletion; returns a reader positioned at the columns subset / cells
template <class CUR> __device__ __forceinline__ Rd row_header(const CParams& P, const CUR& c, Live& info, DT& del) {
    const InDesc& in = P.in[c.src];
    Rd r{P.U, c.pos + c.body_rel, c.next, 0};
    info = live_empty(); del = dt_live();
    if (c.flags & 0x04) info.ts = (int64_t)(r.vint() + (uint64_t)in.min_ts);
    if (c.flags & 0x08) { info.ttl = r.vint32() + in.min_ttl; info.ldt = decode_liveness_ldt((int64_t)r.vint32() + in.min_ldt, info.ttl); }      // :596-598
    if (c.flags & 0x10) del = read_delta_dt(r, in);
    return r;
}

// folds the cells of the row at cursor `c` into merged[] (ColumnDataReducer.getReduced :838-849)
template <class CUR, bool CX = false> __device__ __noinline__ int fold_cells_impl(const CParams& P, const CUR& c, Rd r, Live info, bool apply_deletion, DT active, MCell* merged, bool stat) {
    const InDesc& in = P.in[c.src];
    const int nin = stat ? in.nstat : in.ncols; const int32_t* const map = stat ? in.smap : in.colmap; const int32_t* const vfix = stat ? P.sfix : P.vfix;
    uint64_t missing = 0;
    if (!(c.flags & 0x20)) missing = r.vint();
    for (int i = 0; i < nin; i++) {
        if ((missing >> i) & 1) continue;
        int oc = map[i];
        if constexpr (CX) if (!stat && oc >= P.cx_first) break;      // the multi-cell columns follow the simple ones: merged by cx_merge
        uint32_t cf = r.u8();
        bool has_value = !(cf & 0x04), deleted = cf & 0x01, expiring = cf & 0x02, use_ts = cf & 0x08, use_ttl = cf & 0x10;
        MCell m; m.present = true;
        m.ts = use_ts ? info.ts : (int64_t)(r.vint() + (uint64_t)in.min_ts);
        m.ldt = use_ttl ? info.ldt : ((deleted || expiring) ? (int64_t)r.vint32() + in.min_ldt : I64_MAX);
        m.ttl = use_ttl ? info.ttl : (expiring ? r.vint32() + in.min_ttl : 0);
        m.voff = r.p; m.vlen = 0;
        if (has_value) {
            int64_t len = vfix[oc] > 0 ? vfix[oc] : (int64_t)r.vint32();
            if (len < 0) { r.err = PERR_CORRUPT; len = 0; }
            m.voff = r.p; m.vlen = (int32_t)len; r.skip((uint64_t)len);
        }
        if (m.ttl < 0) r.err = PERR_CORRUPT;
        if (m.ldt != I64_MAX) m.ldt = decode_ldt(m.ldt, m.ttl);
        if (r.err) return r.err;
        if (apply_deletion && dt_deletes(active, m.ts)) continue;
        if (!merged[oc].present || !reconcile_keep_left(P, merged[oc], m)) merged[oc] = m;
    }
    return r.err;
}
template <bool CX = false, class CUR> __device__ __forceinline__ void fold_cells(const CParams& P, const CUR& c, Rd& r, const Live& info, bool apply_deletion, const DT& active, MCell* merged, int& err, bool stat = false) {
    int e = fold_cells_impl<CUR, CX>(P, c, r, info, apply_deletion, active, merged, stat); if (e) err = e;
}

// BTreeRow.purge :457-499 + AbstractCell.purge :78-99. Returns the number of surviving cells, or -1 when the row disappears.
__device__ __forceinline__ int purge_row(const Purger& pg, Live& info, DT& del, MCell* cells, int ncols, int extra_present = 0) {      // extra_present: multi-cell columns left after their own purge
    if (pg.live(info)) info = live_empty();
    if (pg.dt(del)) del = dt_live();
    int present = 0;
    for (int c = 0; c < ncols; c++) {
        MCell& m = cells[c]; if (!m.present) continue;
        bool is_live = m.ldt == I64_MAX || (m.ttl != 0 && pg.now < m.ldt);
        if (!is_live) {
            if (pg.ts_ldt(m.ts, m.ldt)) { m.present = false; continue; }
            if (m.ttl != 0) {                       // expired TTL cell -> tombstone (ldt - ttl), value dropped, purged again
                m.ldt = m.ldt - m.ttl; m.ttl = 0; m.vlen = 0;
                if (pg.ts_ldt(m.ts, m.ldt)) { m.present = false; continue; }
            }
        }
        present++;
    }
    present += extra_present;
    if (live_is_empty(info) && dt_is_live(del) && present == 0) return -1;
    return present;
}

// ---- multi-cell (complex) columns: non-frozen map / set / list -------------------------------------------------------------------------
// One cell per element, each with a cell path; an optional complex deletion per column (S/db/rows/ComplexColumnData.java). They follow the simple
// columns in every row. Everything here is out of line and only runs for tables that have such columns (P.ncx > 0): the kernels' hot code
// stays what it was. A merged row's complex columns are merged straight from the versions' bytes — summary first (deletion, cell counts,
// whether the column exists before / after the purge: the row flags and the subset bitmap need them), then once more per serialisation.

__device__ __forceinline__ MCell purge_cell_fn(const Purger& pg, MCell m) {                     // AbstractCell.purge S/db/rows/AbstractCell.java:78-99
    if (!m.present) return m;
    bool is_live = m.ldt == I64_MAX || (m.ttl != 0 && pg.now < m.ldt);
    if (!is_live) {
        if (pg.ts_ldt(m.ts, m.ldt)) { m.present = false; return m; }
        if (m.ttl != 0) { m.ldt = m.ldt - m.ttl; m.ttl = 0; m.vlen = 0; if (pg.ts_ldt(m.ts, m.ldt)) m.present = false; }
    }
    return m;
}
// AbstractTimeUUIDType.compareCustom S/db/marshal/AbstractTimeUUIDType.java:58-87,126-144 (list cell paths); everything else: cmp_value
__device__ __noinline__ int cmp_path(int type, const uint8_t* a, int la, const uint8_t* b, int lb) {
    if (type == TYPE_TIMEUUID) {
        const bool pa = la == 16, pb = lb == 16;
        if (!(pa && pb)) return pa ? 1 : (pb ? -1 : 0);
        const uint64_t ma = load_be64(a), mb = load_be64(b);
        const int64_t ra = (int64_t)((ma << 48) | ((ma << 16) & 0xFFFF00000000ull) | (ma >> 32)), rb = (int64_t)((mb << 48) | ((mb << 16) & 0xFFFF00000000ull) | (mb >> 32));
        if (ra != rb) return ra < rb ? -1 : 1;
        const int64_t sa = (int64_t)(load_be64(a + 8) ^ 0x0080808080808080ull), sb = (int64_t)(load_be64(b + 8) ^ 0x0080808080808080ull);
        return sa == sb ? 0 : (sa < sb ? -1 : 1);
    }
    return cmp_value(type, a, la, b, lb);
}
// one cell at r (Cell.Serializer.deserialize S/db/rows/Cell.java:307-349); pfix < 0: a simple column's cell (no path), else the path's fixed length (0: vint length)
struct PCell { MCell m; uint64_t poff; int32_t plen; };
__device__ __noinline__ void cx_read_cell(const InDesc& in, Rd& r, const CxVer& v, int vfix, int pfix, PCell* out) {
    uint32_t cf = r.u8();
    bool has_value = !(cf & 0x04), deleted = cf & 0x01, expiring = cf & 0x02, use_ts = cf & 0x08, use_ttl = cf & 0x10;
    MCell m; m.present = true;
    m.ts = use_ts ? v.its : (int64_t)(r.vint() + (uint64_t)in.min_ts);
    m.ldt = use_ttl ? v.ildt : ((deleted || expiring) ? (int64_t)r.vint32() + in.min_ldt : I64_MAX);
    m.ttl = use_ttl ? v.ittl : (expiring ? r.vint32() + in.min_ttl : 0);
    out->poff = r.p; out->plen = 0;
    if (pfix >= 0) { int64_t pl = pfix > 0 ? pfix : (int64_t)r.vint32(); if (pl < 0) { r.err = PERR_CORRUPT; pl = 0; } out->poff = r.p; out->plen = (int32_t)pl; r.skip((uint64_t)pl); }
    m.voff = r.p; m.vlen = 0;
    if (has_value) { int64_t len = vfix > 0 ? vfix : (int64_t)r.vint32(); if (len < 0) { r.err = PERR_CORRUPT; len = 0; } m.voff = r.p; m.vlen = (int32_t)len; r.skip((uint64_t)len); }
    if (m.ttl < 0) r.err = PERR_CORRUPT;
    if (m.ldt != I64_MAX) m.ldt = decode_ldt(m.ldt, m.ttl);
    out->m = m;
}
// positions r at the cells of complex column `oc` in version v (UnfilteredSerializer.readComplexColumn :652-672); false: the version does not have it
__device__ __noinline__ bool cx_seek(const CParams& P, const CxVer& v, int oc, Rd& r, DT* cd, uint32_t* count) {
    const InDesc& in = P.in[v.src];
    r = Rd{P.U, v.cells, v.end, 0};
    uint64_t missing = 0;
    if (!(v.flags & 0x20)) missing = r.vint();
    for (int i = 0; i < in.ncols && !r.err; i++) {
        if ((missing >> i) & 1) continue;
        const int oci = in.colmap[i];
        PCell tmp;
        if (oci < P.cx_first) { cx_read_cell(in, r, v, P.vfix[oci], -1, &tmp); continue; }
        DT d = dt_live();
        if (v.flags & 0x40) { d = read_delta_dt(r, in); if (d.mfda == I64_MIN) d = dt_live(); }      // LIVE written beside another column's deletion (BTreeRow.java:770-778)
        const int32_t n = r.vint32();
        if (n < 0) { r.err = PERR_CORRUPT; return false; }
        if (oci == oc) { *cd = d; *count = (uint32_t)n; return true; }
        for (int32_t k = 0; k < n && !r.err; k++) cx_read_cell(in, r, v, P.vfix[oci], P.pfix[oci - P.cx_first], &tmp);
    }
    return false;
}
template <bool E> __device__ __forceinline__ void put_cell(Sink<E>& s, const CParams& P, const Live& info, const MCell& m, int vfix, const uint8_t* path, int plen, int pfix) {      // Cell.Serializer.serialize :268-305
    bool has_value = m.vlen > 0, deleted = m.ldt != I64_MAX && m.ttl == 0, expiring = m.ttl != 0;
    bool use_ts = !live_is_empty(info) && m.ts == info.ts;
    bool use_ttl = expiring && info.ttl != 0 && m.ttl == info.ttl && m.ldt == info.ldt;
    int cf = (has_value ? 0 : 0x04) | (deleted ? 0x01 : (expiring ? 0x02 : 0)) | (use_ts ? 0x08 : 0) | (use_ttl ? 0x10 : 0);
    s.u8(cf);
    if (!use_ts) s.vint((uint64_t)m.ts - (uint64_t)P.o_min_ts);
    if ((deleted || expiring) && !use_ttl) s.vint((uint64_t)(int64_t)(int32_t)(m.ldt - P.o_min_ldt));
    if (expiring && !use_ttl) s.vint((uint64_t)(int64_t)(m.ttl - P.o_min_ttl));
    if (pfix >= 0) { if (pfix == 0) s.vint((uint64_t)plen); s.copy(path, (uint32_t)plen); }          // :300-301: the path precedes the value
    if (has_value) { if (vfix <= 0) s.vint((uint64_t)m.vlen); s.copy(P.U + m.voff, (uint32_t)m.vlen); }
}
// ColumnDataReducer.getReduced, complex branch (S/db/rows/Row.java:851-883) + ComplexColumnData.purge (:212-216), for complex column j of the row
// whose versions are ver[0..nver). sum: fill the summary. s: serialise the column (its summary in `known`; header = [deletion when the row has
// any] count). acc: statistics (Rows.StatsAccumulation.accumulateOnColumnData S/db/rows/Rows.java:66-82). Returns an error code.
template <bool E> __device__ __noinline__ int cx_merge(const CParams& P, const Purger& pg, const CxVer* ver, int nver, bool as_is, DT active, int j,
                                                        const Live info, CxCol* sum, Sink<E>* s, bool row_has_cd, const CxCol* known, StatAcc* acc) {
    const int oc = P.cx_first + j, vfix = P.vfix[oc], pfix = P.pfix[j], ptype = P.ptype[j];
    uint64_t pos[MAXK]; uint32_t rem[MAXK];
    DT cd = dt_live();
    for (int v = 0; v < nver; v++) {
        Rd r; DT d = dt_live(); uint32_t n = 0; rem[v] = 0; pos[v] = 0;
        if (cx_seek(P, ver[v], oc, r, &d, &n)) { pos[v] = r.p; rem[v] = n; if (dt_supersedes(d, cd)) cd = d; }
        if (r.err) return r.err;
    }
    DT cell_del = dt_live();
    if (!as_is) { if (dt_supersedes(cd, active)) cell_del = cd; else { cd = dt_live(); cell_del = active; } }      // :867-876
    const bool cd_pre = !dt_is_live(cd);
    if (pg.dt(cd)) cd = dt_live();
    if (s) { if (row_has_cd) write_delta_dt(*s, P, known->cd); s->vint(known->ncells); }
    if (acc && !dt_is_live(cd)) acc->dt(cd);
    uint32_t npre = 0, npost = 0;
    for (;;) {
        // the smallest head in cell-path order (MergeIterator over Cell.comparator = column.cellPathComparator())
        int b = -1; PCell best;
        for (int v = 0; v < nver; v++) {
            if (!rem[v]) continue;
            Rd r{P.U, pos[v], ver[v].end, 0}; PCell c; cx_read_cell(P.in[ver[v].src], r, ver[v], vfix, pfix, &c);
            if (r.err) return r.err;
            if (b < 0 || cmp_path(ptype, P.U + c.poff, c.plen, P.U + best.poff, best.plen) < 0) { b = v; best = c; }
        }
        if (b < 0) break;
        MCell mc; mc.present = false; mc.ts = 0; mc.ldt = I64_MAX; mc.voff = 0; mc.ttl = 0; mc.vlen = 0;
        for (int v = 0; v < nver; v++) {                          // CellReducer :900-918, in source order
            if (!rem[v]) continue;
            Rd r{P.U, pos[v], ver[v].end, 0}; PCell c; cx_read_cell(P.in[ver[v].src], r, ver[v], vfix, pfix, &c);
            if (v != b && cmp_path(ptype, P.U + c.poff, c.plen, P.U + best.poff, best.plen) != 0) continue;
            pos[v] = r.p; rem[v]--;
            if (!as_is && dt_deletes(cell_del, c.m.ts)) continue;
            if (!mc.present || !reconcile_keep_left(P, mc, c.m)) mc = c.m;
        }
        if (!mc.present) continue;
        npre++;
        const MCell pc = purge_cell_fn(pg, mc);
        if (!pc.present) continue;
        npost++;
        if (s) put_cell(*s, P, info, pc, vfix, P.U + best.poff, best.plen, pfix);
        if (acc) acc->cell(pc);
    }
    if (sum) { sum->cd = cd; sum->ncells = npost; sum->pre = (cd_pre || npre) ? 1 : 0; sum->post = (!dt_is_live(cd) || npost) ? 1 : 0; }
    if (acc && npost) acc->cols++;
    return 0;
}

// ---- counter columns (CounterColumnType) -----------------------------------------------------------------------------------------------
// A counter cell's value is a context: [i16 n][n x i16 header element][shards of 32 bytes: 16-byte counter id, i64 clock, i64 count], shards in id
// order; element e >= 0 marks shard e LOCAL, e < 0 marks shard e + 32768 GLOBAL, the others are REMOTE (S/db/context/CounterContext.java:40-76).
// Live counter cells of one row are not picked but merged (Cells.resolveCounter S/db/rows/Cells.java:121-162 -> CounterContext.merge :296-447).
// The reference folds the versions pairwise; the per-id rules (:66-73: a global shard beats the others, the largest (clock, count) among globals;
// else the local shards ADD; else the largest (clock, count) among remotes) are associative and commutative, so the fold over the versions is
// one K-way merge by counter id — done here straight from the versions' bytes, twice: count (the value length and the header precede the
// shards), then write. The pairwise fold returns an input context UNCHANGED when it covers the other one; that equals the rebuilt context only
// for contexts in the form the reference itself writes (every header element meets its shard, ids strictly increasing, n >= 0): anything
// else in a merge is refused (PERR_UNSUPPORTED) rather than guessed at. Cells the active deletion covers are skipped BEFORE the merge
// (Row.java:838-849) — the merged cell carries the largest timestamp, so filtering afterwards would not be the same.
__device__ __noinline__ bool ctr_cell(const CParams& P, const CxVer& v, int oc, PCell* out, int* err, bool stat) {      // the cell of simple (or static) column oc in version v
    const InDesc& in = P.in[v.src];
    const int nin = stat ? in.nstat : in.ncols, lim = stat ? P.nstat : P.cx_first;
    const int32_t* const map = stat ? in.smap : in.colmap; const int32_t* const vfix = stat ? P.sfix : P.vfix;
    Rd r{P.U, v.cells, v.end, 0};
    uint64_t missing = 0;
    if (!(v.flags & 0x20)) missing = r.vint();
    for (int i = 0; i < nin && !r.err; i++) {
        if ((missing >> i) & 1) continue;
        const int oci = map[i];
        if (oci >= lim) break;
        cx_read_cell(in, r, v, vfix[oci], -1, out);
        if (r.err) break;
        if (oci == oc) return true;
    }
    if (r.err) *err = r.err;
    return false;
}
__device__ __forceinline__ int ctr_be16(const uint8_t* p) { return (int)(int16_t)(((uint32_t)p[0] << 8) | p[1]); }
// hasLegacyShards :595-608 (the caller has checked vlen >= 2)
__device__ __noinline__ bool ctr_has_legacy(const uint8_t* c, int len) {
    int n = ctr_be16(c); if (n < 0) n = -n;
    const int hl = 2 + 2 * n; if (hl > len) return false;
    if (n < (len - hl) / 32) return true;
    for (int i = 0; i < n; i++) if (ctr_be16(c + 2 + 2 * i) >= 0) return true;
    return false;
}
// sum != nullptr: what column oc of the merged row is (MCell; a merged context: voff = CTR_SYNTH | CTR_LEGACY? | header elements, vlen = its length).
// s != nullptr: write the merged context (the summary said CTR_SYNTH and how many header elements, nhdr). Returns an error code.
template <bool E> __device__ __noinline__ int ctr_merge(const CParams& P, const CxVer* ver, int nver, DT active, int oc, MCell* sum, Sink<E>* s, int nhdr, bool stat) {
    uint64_t base[MAXK]; uint16_t len[MAXK], hl[MAXK], bo[MAXK], ho[MAXK];
    int err = 0, ncand = 0, first = -1;
    MCell tomb, empty, one; tomb.present = empty.present = false; one.present = false;
    int64_t ts_max = I64_MIN;
    for (int v = 0; v < nver; v++) {
        base[v] = ~0ull; len[v] = hl[v] = bo[v] = ho[v] = 0;
        PCell c;
        if (!ctr_cell(P, ver[v], oc, &c, &err, stat)) { if (err) return err; continue; }
        if (dt_deletes(active, c.m.ts)) continue;
        ncand++; if (first < 0) { first = v; one = c.m; }
        if (c.m.ldt != I64_MAX && c.m.ttl == 0) { if (!tomb.present || !reconcile_keep_left(P, tomb, c.m)) tomb = c.m; continue; }     // tombstones among themselves: resolveRegular
        if (c.m.vlen == 0) { if (!empty.present || !(empty.ts > c.m.ts)) empty = c.m; continue; }                                    // :142-149
        if (c.m.ttl != 0) return PERR_UNSUPPORTED;                    // (a counter cell cannot expire)
        if (c.m.vlen < 2) return PERR_CORRUPT;
        if (c.m.vlen > 0xFFFF) return PERR_UNSUPPORTED;               // (2 047 shards and more: the 16-bit walk state below does not hold it)
        const int n = ctr_be16(P.U + c.m.voff);
        if (n < 0) return PERR_UNSUPPORTED;                           // "local shards to be cleared" marker (:618-628): only on streamed cells
        const int h = 2 + 2 * n;
        if (h > c.m.vlen || (c.m.vlen - h) % 32) return PERR_CORRUPT;
        base[v] = c.m.voff; len[v] = (uint16_t)c.m.vlen; hl[v] = bo[v] = (uint16_t)h; ho[v] = 2;
        ts_max = c.m.ts > ts_max ? c.m.ts : ts_max;
    }
    if (sum) {
        sum->present = ncand > 0;
        if (!ncand) return 0;
        if (ncand == 1) { *sum = one; return 0; }
        if (tomb.present) { *sum = tomb; return 0; }                 // a tombstone beats every counter cell whatever the timestamps (CASSANDRA-7346)
        if (empty.present) { *sum = empty; return 0; }
    }
    // K-way merge by counter id
    int ng = 0, nl = 0, nr = 0;
    Sink<E> hs{nullptr, 0, false, 0}, bs{nullptr, 0, false, 0};
    if (s) { hs = *s; bs = *s; bs.pos = s->pos + 2 + 2 * (uint64_t)nhdr; hs.be16((uint32_t)nhdr); }      // header elements and shards are written side by side
    for (;;) {
        int b = -1;
        for (int v = 0; v < nver; v++) {
            if (base[v] == ~0ull || bo[v] >= len[v]) continue;
            if (b < 0) { b = v; continue; }
            const uint8_t* x = P.U + base[v] + bo[v]; const uint8_t* y = P.U + base[b] + bo[b];
            const uint64_t x0 = load_be64(x), y0 = load_be64(y);
            if (x0 < y0 || (x0 == y0 && load_be64(x + 8) < load_be64(y + 8))) b = v;
        }
        if (b < 0) break;
        const uint8_t* id = P.U + base[b] + bo[b];
        const uint64_t id0 = load_be64(id), id1 = load_be64(id + 8);
        int kind = 0; int64_t clock = 0, count = 0; bool have = false;          // kind: 2 global, 1 local, 0 remote
        for (int v = 0; v < nver; v++) {
            if (base[v] == ~0ull || bo[v] >= len[v]) continue;
            const uint8_t* x = P.U + base[v] + bo[v];
            if (load_be64(x) != id0 || load_be64(x + 8) != id1) continue;
            int k = 0;
            if (ho[v] < hl[v]) {                                                // ContextState.updateIsGlobalOrLocal :810-822
                const int e = ctr_be16(P.U + base[v] + ho[v]), idx = (bo[v] - hl[v]) / 32;
                if (e == idx - 32768) k = 2; else if (e == idx) k = 1;
                if (k) ho[v] += 2;
            }
            const int64_t cl = (int64_t)load_be64(x + 16), cn = (int64_t)load_be64(x + 24);
            bo[v] += 32;
            if (bo[v] < len[v]) {                                               // ids strictly increasing inside one context
                const uint8_t* nx = P.U + base[v] + bo[v];
                const uint64_t n0 = load_be64(nx), n1 = load_be64(nx + 8);
                if (n0 < id0 || (n0 == id0 && n1 <= id1)) return PERR_UNSUPPORTED;
            } else if (ho[v] != hl[v]) return PERR_UNSUPPORTED;                 // a header element that met no shard
            if (!have || k > kind) { kind = k; clock = cl; count = cn; have = true; }
            else if (k == kind) {
                if (k == 1) { clock = (int64_t)((uint64_t)clock + (uint64_t)cl); count = (int64_t)((uint64_t)count + (uint64_t)cn); }
                else if (cl > clock || (cl == clock && cn > count)) { clock = cl; count = cn; }
            }
        }
        const int idx = ng + nl + nr;
        if (kind == 2) ng++; else if (kind == 1) nl++; else nr++;
        if (s) {
            bs.copy(id, 16); bs.be64((uint64_t)clock); bs.be64((uint64_t)count);
            if (kind) hs.be16((uint32_t)(kind == 2 ? idx - 32768 : idx) & 0xFFFF);
        }
    }
    if (ng + nl + nr > 0x7FFF) return PERR_UNSUPPORTED;                 // (a header element is an i16 shard index)
    if (sum) {
        sum->present = true; sum->ts = ts_max; sum->ldt = I64_MAX; sum->ttl = 0;
        sum->vlen = 2 + 2 * (ng + nl) + 32 * (ng + nl + nr);
        sum->voff = CTR_SYNTH | ((nl || nr) ? CTR_LEGACY : 0) | (uint64_t)(ng + nl);
    }
    if (s) s->pos = bs.pos;
    return 0;
}

// Tables with static columns carry a static row in every partition, the empty one included (SortedTableWriter.append :144-146,
// SortedTablePartitionWriter.addStaticRow :117-126, UnfilteredSerializer.serializeStaticRow :144-149): flags | EXTENSION, extended flags
// IS_STATIC, no clustering, previous size 0. scells == nullptr: the (merged, purged) static row is empty.
template <bool EMIT, bool CX = false> __device__ __noinline__ void write_static(PWriter<EMIT>& w, const CParams& P, const Live info, const DT del, const MCell* scells, int present, const CxEmit* cx = nullptr) {
    if (!scells) {                                   // no liveness, no deletion, every column missing
        const uint64_t mask = (1ull << P.nstat) - 1;
        w.d.u8(0x80); w.d.u8(0x01); w.d.vint(vint_size(mask) + 1); w.d.vint(0); w.d.vint(mask);
        return;
    }
    int flags = 0x80;
    if (!live_is_empty(info)) flags |= 0x04;
    if (info.ttl != 0) flags |= 0x08;
    if (!dt_is_live(del)) flags |= 0x10;
    if (present == P.nstat) flags |= 0x20;
    const uint64_t p0 = w.d.pos;                     // (size field guessed at one byte, see write_row)
    Sink<EMIT> b = w.d; b.pos = p0 + 2 + 1 + 1;
    uint64_t end = put_row_body<EMIT, CX>(b, P, flags, info, del, scells, P.nstat, P.sfix, cx);
    const uint64_t body = end - b.pos;
    const int vs = vint_size(body + 1);
    if (vs != 1) { b.pos = p0 + 2 + vs + 1; end = put_row_body<EMIT, CX>(b, P, flags, info, del, scells, P.nstat, P.sfix, cx); }
    w.d.u8(flags); w.d.u8(0x01);
    w.d.vint(body + 1); w.d.vint(0);
    w.d.pos = end;
    if (w.acc) {                                     // SortedTableWriter.addStaticRow :188-197: Rows.collectStats unless the row is empty
        w.acc->live(info); w.acc->dt(del);
        for (int c = 0; c < P.nstat; c++) if (scells[c].present) w.acc->cell(scells[c]);
        if constexpr (CX) for (uint64_t bits = P.sctr_mask; bits; bits &= bits - 1) {                     // Cells.collectStats :44-50
            const MCell& m = scells[__ffsll((long long)bits) - 1];
            if (!m.present || (m.ldt != I64_MAX && m.ttl == 0)) continue;
            if ((m.voff & CTR_SYNTH) ? (m.voff & CTR_LEGACY) != 0 : (m.vlen >= 2 && ctr_has_legacy(P.U + m.voff, m.vlen))) w.acc->seen |= 8;
        }
        w.acc->cols += (unsigned long long)present; w.acc->rows++;
    }
}
template <bool EMIT, bool CX = false> __device__ __forceinline__ void pw_start(PWriter<EMIT>& w, const CParams& P, uint64_t key_off, uint32_t klen, const DT& out_pdel,
                                                              const MCell* scells = nullptr, const Live& sinfo = Live{I64_MIN, I64_MAX, 0}, const DT& sdel = DT{I64_MIN, I64_MAX}, int spresent = 0,
                                                              const CxEmit* scx = nullptr) {
    w.d.be16(klen); w.d.copy(P.U + key_off, klen); write_partition_dt(w.d, out_pdel);      // SortedTablePartitionWriter.start :97-115
    w.started = true;
    if (w.acc) { w.acc->part_cells = 0; if (!dt_is_live(out_pdel)) { w.acc->pdel = 1; w.acc->dt(out_pdel); } }     // updatePartitionDeletion
    if (P.nstat > 0) { if constexpr (CX) { if (scx) write_static<EMIT, true>(w, P, sinfo, sdel, scells, spresent, scx); else write_static(w, P, sinfo, sdel, scells, spresent); } else write_static(w, P, sinfo, sdel, scells, spresent); }
    w.header_len = w.d.pos - w.start;
    // final emit with an Index.db slot: the IndexInfos start behind the entry's fixed part, whose size depends on headerLength
    if (EMIT && w.ix_entry) w.ix.base = w.ix_entry + w.ix_fixed + vint_size(w.header_len);
}

template <bool EMIT, bool CX = false> __device__ __forceinline__ void write_row(PWriter<EMIT>& w, const CParams& P, const CkRef& ck, const Live& info, const DT& del, const MCell* cells, int present, const CxEmit* cx = nullptr) {
    int flags = 0;
    if (!live_is_empty(info)) flags |= 0x04;
    if (info.ttl != 0) flags |= 0x08;
    if (!dt_is_live(del)) flags |= 0x10;
    if (present == P.ncols) flags |= 0x20;
    if constexpr (CX) for (int j = 0; j < P.ncx; j++) if (!dt_is_live(cx->col[j].cd)) flags |= 0x40;      // row.hasComplexDeletion() :166-167
    uint64_t pos = pw_begin_unf(w, ck);
    uint64_t prev = pos - w.prev_row_start;
    // The row size precedes the body it counts. Instead of serialising the body twice (count, then emit) it is emitted once behind a size
    // field assumed to take one byte — bodies of up to 126 bytes, i.e. nearly all of them — and emitted again only when that guess was wrong.
    const int vp = vint_size(prev);
    const uint64_t p0 = w.d.pos;
    Sink<EMIT> b = w.d; b.pos = p0 + 1 + ck.len + 1 + vp;
    uint64_t end = put_row_body<EMIT, CX>(b, P, flags, info, del, cells, P.ncols, P.vfix, cx);
    const uint64_t body = end - b.pos;
    const int vs = vint_size(body + vp);
    if (vs != 1) { b.pos = p0 + 1 + ck.len + vs + vp; end = put_row_body<EMIT, CX>(b, P, flags, info, del, cells, P.ncols, P.vfix, cx); }
    w.d.u8(flags); w.d.copy(P.U + ck.off, ck.len);
    w.d.vint(body + vp); w.d.vint(prev);
    w.d.pos = end;
    pw_end_unf(w, P, ck, pos);
    if (w.acc) {                                               // Rows.collectStats
        w.acc->live(info); w.acc->dt(del);
        const int nsimple = CX ? P.cx_first : P.ncols; int simple_present = 0;
        for (int c = 0; c < nsimple; c++) if (cells[c].present) { w.acc->cell(cells[c]); simple_present++; }
        if constexpr (CX) for (uint64_t bits = P.ctr_mask; bits; bits &= bits - 1) {                      // Cells.collectStats S/db/rows/Cells.java:44-50: updateHasLegacyCounterShards
            const MCell& m = cells[__ffsll((long long)bits) - 1];
            if (!m.present || (m.ldt != I64_MAX && m.ttl == 0)) continue;
            if ((m.voff & CTR_SYNTH) ? (m.voff & CTR_LEGACY) != 0 : (m.vlen >= 2 && ctr_has_legacy(P.U + m.voff, m.vlen))) w.acc->seen |= 8;
        }
        w.acc->cols += (unsigned long long)simple_present; w.acc->rows++;
        if constexpr (CX) for (int j = 0; j < P.ncx; j++) if (cells[P.cx_first + j].present)
            cx_merge<EMIT>(P, *cx->pg, cx->ver, cx->nver, cx->as_is, cx->active, j, info, nullptr, (Sink<EMIT>*)nullptr, false, nullptr, w.acc);
    }
}

// UnfilteredSerializer.serialize(RangeTombstoneMarker) :282-305
template <bool EMIT> __device__ __forceinline__ void write_marker(PWriter<EMIT>& w, const CParams& P, const CkRef& ck, const DT& m_close, const DT& m_open) {
    uint64_t pos = pw_begin_unf(w, ck);
    uint64_t prev = pos - w.prev_row_start;
    Sink<EMIT> cs{nullptr, 0, false, 0};
    bool boundary = kind_is_boundary(ck.kind), start = kind_is_start(ck.kind);
    if (boundary) { write_delta_dt(cs, P, m_close); write_delta_dt(cs, P, m_open); } else write_delta_dt(cs, P, start ? m_open : m_close);
    w.d.u8(0x02); w.d.u8(ck.kind); w.d.be16(ck.n); w.d.copy(P.U + ck.off, ck.len);
    w.d.vint(cs.pos + vint_size(prev)); w.d.vint(prev);
    if (boundary) { write_delta_dt(w.d, P, m_close); write_delta_dt(w.d, P, m_open); } else write_delta_dt(w.d, P, start ? m_open : m_close);
    w.open_marker = (boundary || start) ? m_open : dt_live();
    pw_end_unf(w, P, ck, pos);
    if (w.acc) { if (boundary) { w.acc->dt(m_close); w.acc->dt(m_open); } else w.acc->dt(start ? m_open : m_close); }
}

// PurgeFunction.applyToMarker :116-143. Returns false when the marker disappears; may turn a boundary into a bound.
__device__ __forceinline__ bool purge_marker(const Purger& pg, uint8_t& kind, DT& m_close, DT& m_open) {
    if (kind_is_boundary(kind)) {
        bool pc = pg.dt(m_close), po = pg.dt(m_open);
        if (pc) { if (po) return false; kind = (kind == K_EXCL_END_INCL_START) ? K_INCL_START : K_EXCL_START; m_close = dt_live(); return true; }
        if (po) { kind = (kind == K_EXCL_END_INCL_START) ? K_EXCL_END : K_INCL_END; m_open = dt_live(); }
        return true;
    }
    return !pg.dt(kind_is_start(kind) ? m_open : m_close);
}

template <class CUR> __device__ __forceinline__ void read_marker_dts(const CParams& P, const CUR& c, DT& m_close, DT& m_open, int& err) {
    const InDesc& in = P.in[c.src];
    Rd r{P.U, c.pos + c.body_rel, c.next, 0};
    m_close = dt_live(); m_open = dt_live();
    if (kind_is_boundary(c.kind)) { m_close = read_delta_dt(r, in); m_open = read_delta_dt(r, in); }
    else if (kind_is_start(c.kind)) m_open = read_delta_dt(r, in);
    else m_close = read_delta_dt(r, in);
    if (r.err) err = r.err;
}

// the purge evaluator's threshold for one output partition: per-key in the reference (CompactionController.getPurgeEvaluator
// S/db/compaction/CompactionController.java:247-286), here bucketed by token — first table bound >= the partition's token
__device__ __forceinline__ int64_t purge_threshold(const CParams& P, const uint64_t* __restrict__ contrib, uint64_t c0,
                                                   const uint64_t* __restrict__ pbase, const int64_t* __restrict__ part_tok) {
    if (!P.npurge) return P.purge_max_ts;
    const uint64_t e = contrib[c0];
    const int64_t t0 = part_tok[pbase[(int)((e >> 56) & 0x7F)] + (e & 0xFFFFFFFFFFull)];
    int64_t a = 0, b = P.npurge;
    while (a < b) { int64_t mid = (a + b) >> 1; if (P.purge_hi[mid] < t0) a = mid + 1; else b = mid; }
    return a < P.npurge ? P.purge_ts[a] : P.purge_max_ts;
}

struct PartOut { uint64_t dsize; uint32_t ipay, nblk, ihead; uint32_t ovf; uint32_t cells; };

// The merged static row of one output partition: cursors cur[v], v in sgrp, stand on their non-empty static rows (static_load).
// mergeStaticRows S/db/rows/UnfilteredRowIterators.java:484-505 -> Row.Merger.merge(partitionDeletion) S/db/rows/Row.java:730-781: runs for
// every fan-in (the merge iterator's constructor calls it), and its single-row shortcut counts every iterator, the ones with an empty
// static row too (merger.add(i, ...) for all i). Returns the number of merged cells, or -1 when nothing is left.
template <class CUR> __device__ __noinline__ int merge_static(const CParams& P, CUR* cur, uint64_t sgrp, uint32_t m, DT pdel, MCell* merged, Live* info_out, DT* del_out, int* err) {
    Live info = live_empty(); DT del = dt_live(); DT active = pdel;
    for (int k = 0; k < P.nstat; k++) merged[k].present = false;
    const bool as_is = m == 1 && dt_is_live(pdel);
    for (uint64_t bits = sgrp; bits; bits &= bits - 1) {
        int v = __ffsll((long long)bits) - 1;
        Live vi; DT vd; Rd r = row_header(P, cur[v], vi, vd); if (r.err) *err = r.err;
        if (live_supersedes(vi, info)) info = vi;
        if (dt_supersedes(vd, del)) del = vd;
    }
    if (!as_is) {
        if (dt_supersedes(del, active)) active = del; else del = dt_live();
        if (dt_deletes(active, info.ts)) info = live_empty();
    }
    for (uint64_t bits = sgrp; bits && !*err; bits &= bits - 1) {
        int v = __ffsll((long long)bits) - 1;
        Live vi; DT vd; Rd r = row_header(P, cur[v], vi, vd);
        fold_cells(P, cur[v], r, vi, !as_is, active, merged, *err, true);
    }
    *info_out = info; *del_out = del;
    int n = 0; for (int k = 0; k < P.nstat; k++) n += merged[k].present;
    return (live_is_empty(info) && dt_is_live(del) && n == 0) ? -1 : n;
}

// static counter columns of the merged static row: Cells.resolveCounter over the versions' cells (ctr_merge) in place of the winner fold_cells picked.
// Fills ver[] (the versions of the static row) and the deletion in force, both needed again when the row is written.
template <class CUR> __device__ __noinline__ int static_counters(const CParams& P, CUR* cur, uint64_t sgrp, uint32_t m, DT pdel, MCell* merged, CxVer* ver, int* nver, DT* active_out) {
    const bool as_is = m == 1 && dt_is_live(pdel);
    DT del = dt_live(); int nv = 0;
    for (uint64_t bits = sgrp; bits; bits &= bits - 1) {
        const int v = __ffsll((long long)bits) - 1;
        Live vi; DT vd; Rd r = row_header(P, cur[v], vi, vd); if (r.err) return r.err;
        if (dt_supersedes(vd, del)) del = vd;
        ver[nv++] = CxVer{r.p, (uint64_t)cur[v].next, vi.ts, vi.ldt, vi.ttl, (uint8_t)cur[v].flags, (uint8_t)cur[v].src};
    }
    DT active = pdel;
    if (!as_is && dt_supersedes(del, active)) active = del;
    *nver = nv; *active_out = active;
    if (as_is || nv < 2) return 0;
    for (uint64_t bits = P.sctr_mask; bits; bits &= bits - 1) {
        const int oc = __ffsll((long long)bits) - 1;
        const int e = ctr_merge<false>(P, ver, nv, active, oc, &merged[oc], (Sink<false>*)nullptr, 0, true);
        if (e) return e;
    }
    return 0;
}

// The whole life of one output partition. contrib[c0 .. c0+m) are its input partitions in source order.
// cur[0..m) / open_dt[0..m): per-source cursor state owned by this thread (the caller places it in shared memory);
// merged[0..ncols): scratch for the merged row.
__host__ __device__ int64_t murmur3_token(const uint8_t* key, uint32_t len);     // compact.cu

// where an input partition's bytes are, as an offset from P.U: the decompressed stream itself (XlateGlobal), or a tile of it that
// k_partition_staged copied into shared memory (XlateStaged: P.U then points at the tile)
struct XlateGlobal { __device__ __forceinline__ uint64_t operator()(int, uint64_t u) const { return u; } };
struct XlateStaged {
    const uint32_t* sbase; const uint64_t* g0;       // per source: offset of its staged range in the tile, stream offset that range starts at
    __device__ __forceinline__ uint64_t operator()(int src, uint64_t u) const { return sbase[src] + (u - g0[src]); }
};

// the versions of a row -> CxVer[], then the summary of every multi-cell column (see cx_merge)
template <class CUR> __device__ __noinline__ int cx_row_summary(const CParams& P, const Purger& pg, CUR* cur, uint64_t grp, bool as_is, DT active, CxVer* ver, CxCol* col,
                                                                MCell* merged, int* pre, int* post, int* nver_out) {
    int nv = 0;
    for (uint64_t bits = grp; bits; bits &= bits - 1) {
        const int v = __ffsll((long long)bits) - 1;
        Live vi; DT vd; Rd r = row_header(P, cur[v], vi, vd); if (r.err) return r.err;
        ver[nv++] = CxVer{r.p, (uint64_t)cur[v].next, vi.ts, vi.ldt, vi.ttl, (uint8_t)cur[v].flags, (uint8_t)cur[v].src};
    }
    for (int j = 0; j < P.ncx; j++) {
        const int e = cx_merge<false>(P, pg, ver, nv, as_is, active, j, live_empty(), &col[j], (Sink<false>*)nullptr, false, nullptr, nullptr);
        if (e) return e;
        merged[P.cx_first + j].present = col[j].post != 0; *pre += col[j].pre; *post += col[j].post;
    }
    // counter columns of a row with several versions: Cells.resolveCounter instead of the winner fold_cells picked (see ctr_merge)
    if (!as_is && nv > 1) for (uint64_t bits = P.ctr_mask; bits; bits &= bits - 1) {
        const int oc = __ffsll((long long)bits) - 1;
        const int e = ctr_merge<false>(P, ver, nv, active, oc, &merged[oc], (Sink<false>*)nullptr, 0);
        if (e) return e;
    }
    *nver_out = nv;
    return 0;
}

// CX: the table has multi-cell columns (a separate instantiation: the kernels of every other table compile to exactly the code they had)
template <bool EMIT, class CUR, class XL, int MCAP = MAXK, bool CX = false>
__device__ void process_partition(const CParams& P, const XL& xl, const uint64_t* __restrict__ contrib, uint64_t c0, uint32_t m,
                                  const uint64_t* __restrict__ part_upos, const uint64_t* __restrict__ pbase,
                                  const uint64_t* __restrict__ part_kp, const uint16_t* __restrict__ part_klen, const int64_t* __restrict__ part_tok,
                                  uint8_t* dout, uint64_t dcap, uint64_t dpos, uint8_t* iout, uint32_t nblocks_final, uint32_t ipay_final, uint32_t ixs_cap,
                                  CUR* cur, DT* open_dt, MCell* merged,
                                  PartOut& out, PartStats& st, int& err, StatAcc* acc = nullptr, uint32_t m_uni = 0) {
    // m_uni: a bound >= m that is the same for every lane of the warp (0: m itself). Loops over the cursors run to it with the lanes' own
    // m as a guard inside: lanes of different fan-in then leave those loops together. ptxas reconverges lanes that left a loop at different
    // trip counts only at the end of the enclosing region, i.e. after the whole partition — the staged kernel, whose warps mix fan-ins, ran
    // two lanes at a time that way.
    const uint32_t mu = m_uni > m ? m_uni : m;
    Purger pg{P.now, P.gc_before, purge_threshold(P, contrib, c0, pbase, part_tok)};
    DT pdel = dt_live();
    uint64_t key_off = 0; uint32_t klen = 0;
    uint64_t sgrp = 0;                                // contributors with a non-empty static row
    if (m > MAXK || (!CX && (P.ncx || P.ctr_mask || P.sctr_mask))) { err = PERR_UNSUPPORTED; return; }
    // prologue in three sweeps so that the m dependent chains (contrib -> upos -> Data bytes) overlap instead of serialising:
    // (1) resolve the input partitions, (2) prefetch their first lines, (3) parse the partition headers
    for (uint32_t v = 0; v < mu; v++) {
        if (v >= m) continue;
        uint64_t e = contrib[c0 + v];
        int src = (int)((e >> 56) & 0x7F); uint64_t g = pbase[src] + (e & 0xFFFFFFFFFFull);
        CUR& c = cur[v]; c.src = (uint8_t)src; c.pos = (decltype(c.pos))xl(src, part_upos[g]); c.end = (decltype(c.end))xl(src, part_upos[g + 1]); c.done = false;
        c.k0 = part_kp[g]; c.ckend_rel = part_klen[g];           // what Index.db said about this partition's key (checked below)
    }
#ifdef __CUDA_ARCH__
    if (sizeof(typename CUR::rel_t) == 4) for (uint32_t v = 0; v < m; v++) asm volatile("prefetch.global.L1 [%0];" :: "l"(P.U + cur[v].pos));
#endif
    for (uint32_t v = 0; v < mu; v++) {
        if (v >= m) continue;
        CUR& c = cur[v];
        uint64_t pos = c.pos;
        Rd r{P.U, pos, c.end, 0};
        uint32_t kl = r.be16();
        {   // Index.db <-> Data.db consistency (K2 only verified keys longer than 8 bytes): key length and 8-byte prefix must agree
            uint64_t pre = load_be64(P.U + pos + 2);
            if (kl < 8) pre &= kl ? (~0ull << (8 * (8 - kl))) : 0ull;
            if (kl != c.ckend_rel || pre != c.k0) { err = PERR_CORRUPT; return; }
        }
        r.skip(kl);
        DT pd = read_partition_dt(r);
        if (r.err) { err = r.err; return; }
        // keys longer than the 8-byte prefix: the token K2 computed from the Index.db key must be the token of the Data.db key
        if (kl > 8 && !P.partitioner) {
            const uint64_t e = contrib[c0 + v];
            if (murmur3_token(P.U + pos + 2, kl) != part_tok[pbase[(int)((e >> 56) & 0x7F)] + (e & 0xFFFFFFFFFFull)]) { err = PERR_CORRUPT; return; }
        }
        if (v == 0) { key_off = pos + 2; klen = kl; }
        if (!dt_supersedes(pdel, pd)) pdel = pd;                  // collectPartitionLevelDeletion :465-482
        c.pos = (decltype(c.pos))r.p; c.next = c.pos;
        if (P.in[c.src].nstat > 0) {                              // header.hasStatic(): this input's partitions carry a static row
            bool ne = false; int e = static_load(P, c, &ne);
            if (e) { err = e; return; }
            if (ne) sgrp |= 1ull << v;
        }
    }
    DT out_pdel = pg.dt(pdel) ? dt_live() : pdel;                 // PurgeFunction.applyToDeletion :95-99

    PWriter<EMIT> w;
    // ixs (scratch pass): iout is this partition's promoted-index slot (IXS_* layout), nblocks_final its block capacity, ixs_cap its IndexInfo capacity
    const bool ixs = EMIT && ixs_cap != 0;
    w.d.base = dout; w.d.pos = 0; w.d.on = true; w.d.cap = dcap; w.ix.on = EMIT && iout && (ixs || nblocks_final > 1); w.ix.cap = ixs ? (uint64_t)ixs_cap : ~0ull; w.start = 0; w.header_len = 0; w.prev_row_start = 0; w.block_start = 0;
    w.nblocks = 0; w.nblocks_final = nblocks_final; w.started = false; w.have_first = false; w.open_marker = dt_live(); w.rows_out = 0;
    w.first = CkRef{0, 0, 0, 0}; w.last = w.first; w.acc = acc;
    // index entry layout (EMIT): [u16 kl][key][vint dpos][vint ipay]{[vint headerLen][DT][vint nblocks][IndexInfo..][i32 offsets..]}
    uint32_t fixed = 2 + klen + vint_size(dpos) + vint_size(ipay_final);
    w.ix.base = nullptr; w.ix.pos = 0;
    w.ix_entry = (EMIT && iout && !ixs) ? iout : nullptr; w.ix_fixed = fixed + (dt_is_live(out_pdel) ? 1 : 12) + vint_size(nblocks_final);
    w.ix_offs = (EMIT && iout) ? iout + fixed + ipay_final - 4 * nblocks_final : nullptr;
    if (ixs) { w.ix_offs = iout + IXS_HEAD; w.ix.base = iout + IXS_HEAD + 4 * (size_t)nblocks_final; }
    // static row: merged and purged before anything else (the merge iterator's constructor does it); a non-empty one makes the partition
    // non-empty (UnfilteredRowIterator.isEmpty :63-68), so the partition starts here and now while merged[] still holds its cells
    if (P.nstat > 0 && sgrp) {
        Live sinfo; DT sdel;
        int n = merge_static(P, cur, sgrp, m, pdel, merged, &sinfo, &sdel, &err);
        if (err) return;
        bool done = false;
        if constexpr (CX) if (P.sctr_mask && n >= 0) {          // static counter columns: merged contexts, written from the versions (put_row_body<.., true>)
            CxVer sv[MCAP]; int snv = 0; DT sactive;
            { const int e = static_counters(P, cur, sgrp, m, pdel, merged, sv, &snv, &sactive); if (e) { err = e; return; } }
            n = 0; for (int k = 0; k < P.nstat; k++) n += merged[k].present;
            if (!(live_is_empty(sinfo) && dt_is_live(sdel) && n == 0)) {
                n = purge_row(pg, sinfo, sdel, merged, P.nstat);
                if (n >= 0) { CxEmit scx{sv, snv, false, sactive, nullptr, &pg, true}; pw_start<EMIT, true>(w, P, key_off, klen, out_pdel, merged, sinfo, sdel, n, &scx); }
            }
            done = true;
        }
        if (!done && n >= 0) { n = purge_row(pg, sinfo, sdel, merged, P.nstat); if (n >= 0) pw_start(w, P, key_off, klen, out_pdel, merged, sinfo, sdel, n); }
    }
    if (P.nstat > 0) for (uint32_t v = 0; v < m; v++) if (P.in[cur[v].src].nstat > 0) cur[v].pos = cur[v].next;      // step over the static rows

    // One code path for every fan-in. m == 1 is the reference's TrivialOneToOne case (UnfilteredRowIterators.java:552-556): rows
    // and markers pass through untouched (no Row.Merger, no marker merger) and only the purge transformation applies.
    const bool multi = m > 1;
    uint64_t has_open = 0; int biggest = -1;
    DT cur_open = dt_live();                       // open deletion in the merged stream
    for (uint32_t v = 0; v < mu; v++) if (v < m) cur_load(P, cur[v], err);
    while (!err) {
        // smallest head and the heads equal to it in one sweep (MergeIterator: equal items reduce together, in source order)
        int b = -1; uint64_t grp = 0;
        for (uint32_t v = 0; v < mu; v++) {
            if (v >= m || cur[v].done) continue;
            const int c = b < 0 ? -1 : cmp_heads(P, cur[v], cur[b]);
            if (c < 0) { b = (int)v; grp = 1ull << v; } else if (c == 0) grp |= 1ull << v;
        }
        if (b < 0) break;
        const int gcount = __popcll(grp), last = 63 - __clzll((long long)grp);
        if (!(cur[b].flags & 0x02)) {
            DT active = multi ? (dt_is_live(cur_open) ? pdel : cur_open) : dt_live();      // activeDeletion() :191-197
            const bool as_is = !multi || ((gcount == 1) && dt_is_live(active));            // Row.Merger.merge :734-739
            Live info = live_empty(); DT del = dt_live();
            for (int k = 0; k < P.ncols; k++) merged[k].present = false;
            // one sweep over the versions: row headers and cells together. Cells are reconciled first and the active deletion is applied to
            // the winners afterwards — the same result as ColumnDataReducer's skip-then-reconcile (:838-849), because Cells.reconcile orders by
            // timestamp first: a winner the deletion covers means every version was covered, a winner above it beat only lower timestamps.
            for (uint64_t bits = grp; bits && !err; bits &= bits - 1) {
                int v = __ffsll((long long)bits) - 1;
                Live vi; DT vd; Rd r = row_header(P, cur[v], vi, vd); if (r.err) err = r.err;
                if (gcount == 1) { info = vi; del = vd; }
                else { if (live_supersedes(vi, info)) info = vi; if (dt_supersedes(vd, del)) del = vd; }
                fold_cells<CX>(P, cur[v], r, vi, false, active, merged, err);
            }
            const int nsimple = CX ? P.cx_first : P.ncols;
            if (!as_is) {
                if (dt_supersedes(del, active)) active = del; else del = dt_live();
                if (dt_deletes(active, info.ts)) info = live_empty();
                for (int k = 0; k < nsimple; k++) if (merged[k].present && dt_deletes(active, merged[k].ts)) merged[k].present = false;
            }
            if (err) break;
            int npresent = 0; for (int k = 0; k < nsimple; k++) npresent += merged[k].present;
            if constexpr (CX) {
                // multi-cell columns: summary (deletion, cell counts, existence before / after the purge) now, the cells when the row is written
                CxVer cxv[MCAP]; CxCol cxc[MAXCX];
                int cx_pre = 0, cx_post = 0, cx_nver = 0;
                { int e = cx_row_summary(P, pg, cur, grp, as_is, active, cxv, cxc, merged, &cx_pre, &cx_post, &cx_nver); if (e) { err = e; break; } }
                if (P.ctr_mask) { npresent = 0; for (int k = 0; k < nsimple; k++) npresent += merged[k].present; }      // (the counter columns were merged there)
                if (!(live_is_empty(info) && dt_is_live(del) && npresent + cx_pre == 0)) {
                    st.merged_unfiltereds++;
                    CUR& f = cur[b];
                    CkRef ck{(uint64_t)f.pos + f.ck_rel, (uint32_t)(f.ckend_rel - f.ck_rel), K_CLUSTERING, (uint8_t)f.n};
                    int present = purge_row(pg, info, del, merged, nsimple, cx_post);
                    if (present >= 0) {
                        if (!w.started) pw_start(w, P, key_off, klen, out_pdel);
                        const CxEmit cxe{cxv, cx_nver, as_is, active, cxc, &pg};
                        write_row<EMIT, true>(w, P, ck, info, del, merged, present, &cxe);
                    }
                }
            } else if (!(live_is_empty(info) && dt_is_live(del) && npresent == 0)) {
                st.merged_unfiltereds++;
                CUR& f = cur[b];
                CkRef ck{(uint64_t)f.pos + f.ck_rel, (uint32_t)(f.ckend_rel - f.ck_rel), K_CLUSTERING, (uint8_t)f.n};
                int present = purge_row(pg, info, del, merged, P.ncols);
                if (present >= 0) { if (!w.started) pw_start(w, P, key_off, klen, out_pdel); write_row(w, P, ck, info, del, merged, present); }
            }
        } else {
            CUR& f = cur[last];                                       // `bound` = clustering of the last marker added (:99-103)
            CkRef ck{(uint64_t)f.pos + f.ck_rel, (uint32_t)(f.ckend_rel - f.ck_rel), (uint8_t)f.kind, (uint8_t)f.n};
            DT mc = dt_live(), mo = dt_live(); bool emit = false;
            if (!multi) { read_marker_dts(P, f, mc, mo, err); emit = true; }
            else {
                // RangeTombstoneMarker.Merger.merge :94-153
                for (uint64_t bits = grp; bits; bits &= bits - 1) {
                    int v = __ffsll((long long)bits) - 1;
                    DT a, o; read_marker_dts(P, cur[v], a, o, err);
                    bool is_open = kind_is_boundary(cur[v].kind) || kind_is_start(cur[v].kind);
                    if (is_open) { open_dt[v] = o; has_open |= 1ull << v; } else has_open &= ~(1ull << v);
                }
                biggest = -1;
                for (uint64_t bits = has_open; bits; bits &= bits - 1) { int v = __ffsll((long long)bits) - 1; if (biggest < 0 || dt_supersedes(open_dt[v], open_dt[biggest])) biggest = v; }
                DT now_open = (biggest >= 0 && dt_supersedes(open_dt[biggest], pdel)) ? open_dt[biggest] : dt_live();
                if (!dt_eq(cur_open, now_open)) {
                    bool before = kind_vs_clustering(f.kind) < 0;
                    if (dt_is_live(cur_open)) { ck.kind = before ? K_INCL_START : K_EXCL_START; mo = now_open; }
                    else if (dt_is_live(now_open)) { ck.kind = before ? K_EXCL_END : K_INCL_END; mc = cur_open; }
                    else { ck.kind = before ? K_EXCL_END_INCL_START : K_INCL_END_EXCL_START; mc = cur_open; mo = now_open; }
                    emit = true;
                }
                cur_open = now_open;
            }
            if (emit && !err) {
                st.merged_unfiltereds++;
                if (purge_marker(pg, ck.kind, mc, mo)) { if (!w.started) pw_start(w, P, key_off, klen, out_pdel); write_marker(w, P, ck, mc, mo); }
            }
        }
        for (uint64_t bits = grp; bits; bits &= bits - 1) { int v = __ffsll((long long)bits) - 1; cur[v].pos = cur[v].next; cur_load(P, cur[v], err); }
    }
    if (err) return;
    // partition.isEmpty() (UnfilteredRowIterator.java:63-68) / SortedTableWriter.append :134
    if (!w.started && !dt_is_live(out_pdel)) pw_start(w, P, key_off, klen, out_pdel);
    out.dsize = 0; out.ipay = 0; out.nblk = 0; out.ihead = 2 + klen; out.ovf = 0; out.cells = 0;
    if (w.started) {
        if (acc) out.cells = acc->part_cells;
        w.d.u8(0x01);                                                        // end of partition, then the trailing index block (finish() :217-243)
        if (w.rows_out && w.have_first) pw_add_index_block(w, P);
        out.dsize = w.d.pos; out.nblk = w.nblocks;
        if (w.nblocks > 1) out.ipay = vint_size(w.header_len) + (dt_is_live(out_pdel) ? 1 : 12) + vint_size(w.nblocks) + (uint32_t)w.ix.pos + 4 * w.nblocks;
        st.rows_out += w.rows_out;
        out.ovf = (EMIT && w.d.pos > dcap) ? 1 : 0;
        if (ixs) {                                                           // the entry itself is assembled by k_index_promoted once positions are known
            if (w.nblocks > 1) {
                if (w.ix.pos > w.ix.cap || w.nblocks > nblocks_final) out.ovf = 1;
                ((int64_t*)iout)[0] = out_pdel.mfda; ((int64_t*)iout)[1] = out_pdel.ldt; ((int64_t*)iout)[2] = (int64_t)w.header_len;
            }
        } else if (EMIT && !iout && w.nblocks > 1) out.ovf = 1;              // scratch pass without a slot: re-emit in mode 3
        else if (EMIT && iout) {                                             // RowIndexEntry.serialize :468-473, IndexedEntry.serialize :625-642
            Sink<true> e{iout, 0, true, ~0ull};
            e.be16(klen); e.copy(P.U + key_off, klen); e.vint(dpos); e.vint(ipay_final);
            if (nblocks_final > 1) { e.vint(w.header_len); write_partition_dt(e, out_pdel); e.vint(nblocks_final); }
        }
    }
}

} // namespace b200c
