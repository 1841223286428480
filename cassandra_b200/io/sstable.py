"""SSTable component files (big format, version `oa`) as the host side needs them: read the components of an input
sstable, derive what the C-ABI manifest carries (schema classes, EncodingStats, StatsMetadata minima), write outputs.

Mirrors what the Java shim gets for free from SSTableReader (`sstable.header`, `getSSTableMetadata()`, `getCompressionMetadata()`):
  Statistics.db layout  S/io/sstable/metadata/MetadataSerializer.java:67-112 (toc + per-component CRC)
  HEADER component      S/db/SerializationHeader.java:451-460 ; EncodingStats S/db/rows/EncodingStats.java:262-277
  STATS component       S/io/sstable/metadata/StatsMetadata.java:402-425
"""
import os, struct
from .. import native
from .compress import CompressionMetadata, ChecksumMetadata

TIMESTAMP_EPOCH = 1442880000000000      # EncodingStats.TIMESTAMP_EPOCH (2015-09-22T00:00Z in µs), EncodingStats.java:47-64
DELETION_TIME_EPOCH = 1442880000
NO_DELETION_TIME = (1 << 63) - 1
MARSHAL = "org.apache.cassandra.db.marshal."

def _vint(b, p):
    f = b[p]
    if f < 0x80: return f, p + 1
    extra = 8 if f == 0xFF else (8 - (f ^ 0xFF).bit_length())
    v = f & (0xFF >> extra)
    for i in range(extra): v = (v << 8) | b[p + 1 + i]
    return v, p + 1 + extra

def _vbytes(b, p):
    n, p = _vint(b, p); return b[p:p + n], p + n

def type_class(type_string: str):
    """AbstractType -> (B200C_TYPE_*, valueLengthIfFixed) for the comparison/layout classes the engine implements."""
    t = type_string
    if t.startswith(MARSHAL): t = t[len(MARSHAL):]
    # LongType / TimestampType / Int32Type compare as signed integers (LongType.compareLongs, S/db/marshal/LongType.java). DateType is the
    # pre-2.0 timestamp type: ComparisonType.BYTE_ORDER, i.e. UNSIGNED lexicographic (S/db/marshal/DateType.java) — pre-1970 values
    # sort after post-1970 ones — so it is a fixed-length bytes class, not a signed one.
    fixed_signed = {"LongType": 8, "TimestampType": 8, "Int32Type": 4}
    fixed_bytes = {"DateType": 8, "DoubleType": 8, "FloatType": 4, "BooleanType": 1, "UUIDType": 16, "TimeUUIDType": 16, "LexicalUUIDType": 16}
    if t in fixed_signed: return native.TYPE_FIXED_SIGNED, fixed_signed[t]
    if t in fixed_bytes: return native.TYPE_FIXED_BYTES, fixed_bytes[t]
    if t in ("ShortType", "ByteType"): return native.TYPE_VAR_SIGNED, 0
    if t in ("UTF8Type", "AsciiType", "BytesType"): return native.TYPE_BYTES, 0
    raise native.UnsupportedError(native.EUNSUPPORTED, "type outside the supported envelope: " + type_string)

def _split_args(inner: str):
    out, depth, cur = [], 0, ""
    for ch in inner:
        if ch == "(": depth += 1
        if ch == ")": depth -= 1
        if ch == "," and depth == 0: out.append(cur.strip()); cur = ""
        else: cur += ch
    if cur.strip(): out.append(cur.strip())
    return out

def is_complex(type_string: str) -> bool:
    """multi-cell column: a non-frozen collection (ColumnMetadata.isComplex = type.isMultiCell, S/schema/ColumnMetadata.java)"""
    t = type_string[len(MARSHAL):] if type_string.startswith(MARSHAL) else type_string
    return t.startswith(("MapType(", "SetType(", "ListType("))

def column_class(type_string: str):
    """(type, fixed_len) of a column for the manifest: simple columns as type_class; multi-cell collections as
    B200C_COLUMN_COMPLEX(value class, path class) / B200C_COLUMN_FIXED(value length, path length) — cell path = map key / set element /
    list timeuuid, cell value = map value / nothing / list element (CollectionType.nameComparator / valueComparator)."""
    t = type_string[len(MARSHAL):] if type_string.startswith(MARSHAL) else type_string
    if t.startswith("FrozenType("): return native.TYPE_BYTES, 0                    # a frozen collection / UDT is one opaque value
    if not is_complex(type_string):
        if t.startswith("CounterColumnType"): return native.TYPE_COUNTER, 0            # counter context, merged shard by shard (S/db/context/CounterContext.java)
        if t.startswith("UserType("): raise native.UnsupportedError(native.EUNSUPPORTED, "type outside the supported envelope: " + type_string)
        return type_class(type_string)
    kind, inner = t.split("(", 1); args = _split_args(inner[:-1])
    def cls(a):
        a2 = a[len(MARSHAL):] if a.startswith(MARSHAL) else a
        if a2.startswith("FrozenType("): return native.TYPE_BYTES, 0
        return type_class(a)
    if kind == "MapType": (pt, pl), (vt, vl) = cls(args[0]), cls(args[1])
    elif kind == "SetType": (pt, pl), (vt, vl) = cls(args[0]), (native.TYPE_BYTES, 0)
    else: (pt, pl), (vt, vl) = (native.TYPE_TIMEUUID, 16), cls(args[0])
    return vt | ((pt + 1) << 8), vl | (pl << 16)

PARTITIONER_IDS = {"org.apache.cassandra.dht.Murmur3Partitioner": native.PARTITIONER_MURMUR3,
                   "org.apache.cassandra.dht.ByteOrderedPartitioner": native.PARTITIONER_BYTE_ORDERED}

CLUSTERING_OK = {"LongType", "TimestampType", "DateType", "Int32Type", "ShortType", "ByteType", "UTF8Type", "AsciiType", "BytesType"}

# ---- Filter.db geometry: FilterFactory.getFilter(numElements, fpChance) (S/utils/FilterFactory.java:60-75) over BloomCalculations
# (S/utils/BloomCalculations.java:38-160). PROBS[buckets per element][K] = false-positive probability (published table, Cao et al.).
BLOOM_PROBS = [
    [1.0], [1.0, 1.0], [1.0, 0.393, 0.400], [1.0, 0.283, 0.237, 0.253], [1.0, 0.221, 0.155, 0.147, 0.160],
    [1.0, 0.181, 0.109, 0.092, 0.092, 0.101], [1.0, 0.154, 0.0804, 0.0609, 0.0561, 0.0578, 0.0638],
    [1.0, 0.133, 0.0618, 0.0423, 0.0359, 0.0347, 0.0364], [1.0, 0.118, 0.0489, 0.0306, 0.024, 0.0217, 0.0216, 0.0229],
    [1.0, 0.105, 0.0397, 0.0228, 0.0166, 0.0141, 0.0133, 0.0135, 0.0145], [1.0, 0.0952, 0.0329, 0.0174, 0.0118, 0.00943, 0.00844, 0.00819, 0.00846],
    [1.0, 0.0869, 0.0276, 0.0136, 0.00864, 0.0065, 0.00552, 0.00513, 0.00509], [1.0, 0.08, 0.0236, 0.0108, 0.00646, 0.00459, 0.00371, 0.00329, 0.00314],
    [1.0, 0.074, 0.0203, 0.00875, 0.00492, 0.00332, 0.00255, 0.00217, 0.00199, 0.00194],
    [1.0, 0.0689, 0.0177, 0.00718, 0.00381, 0.00244, 0.00179, 0.00146, 0.00129, 0.00121, 0.0012],
    [1.0, 0.0645, 0.0156, 0.00596, 0.003, 0.00183, 0.00128, 0.001, 0.000852, 0.000775, 0.000744],
    [1.0, 0.0606, 0.0138, 0.005, 0.00239, 0.00139, 0.000935, 0.000702, 0.000574, 0.000505, 0.00047, 0.000459],
    [1.0, 0.0571, 0.0123, 0.00423, 0.00193, 0.00107, 0.000692, 0.000499, 0.000394, 0.000335, 0.000302, 0.000287, 0.000284],
    [1.0, 0.054, 0.0111, 0.00362, 0.00158, 0.000839, 0.000519, 0.00036, 0.000275, 0.000226, 0.000198, 0.000183, 0.000176],
    [1.0, 0.0513, 0.00998, 0.00312, 0.0013, 0.000663, 0.000394, 0.000264, 0.000194, 0.000155, 0.000132, 0.000118, 0.000111, 0.000109],
    [1.0, 0.0488, 0.00906, 0.0027, 0.00108, 0.00053, 0.000303, 0.000196, 0.00014, 0.000108, 8.89e-05, 7.77e-05, 7.12e-05, 6.79e-05, 6.71e-05]]

def bloom_geometry(num_elements: int, fp_chance: float):
    """-> (hash_count, words): K hash functions over an OffHeapBitSet of `words` 64-bit words, or (0, 0) for fpChance 1.0 (AlwaysPresent)."""
    if fp_chance >= 1.0: return 0, 0
    probs = BLOOM_PROBS
    optk = []
    for row in probs:
        best = min(range(len(row)), key=lambda j: (row[j], j)); optk.append(max(1, best))
    max_buckets = min(len(probs) - 1, int(((1 << 63) - 1 - 20) / max(1, num_elements)))
    max_k = len(probs[max_buckets]) - 1
    if fp_chance >= probs[2][1]: k, buckets = 2, optk[2]                      # (the reference returns BloomSpecification(2, optK[2]) here, as is)
    else:
        if fp_chance < probs[max_buckets][max_k]: raise ValueError("fp chance not satisfiable")
        buckets = 2; k = optk[2]
        while probs[buckets][k] > fp_chance: buckets += 1; k = optk[buckets]
        while probs[buckets][k - 1] <= fp_chance: k -= 1
    num_bits = num_elements * buckets + 20                                     # FilterFactory.createFilter: BITSET_EXCESS
    return k, ((num_bits - 1) >> 6) + 1                                        # OffHeapBitSet(numBits): words

def parse_statistics(b: bytes):
    (n,) = struct.unpack_from(">i", b, 0)
    toc = {}
    p = 8                                              # count + crc
    for _ in range(n):
        t, pos = struct.unpack_from(">ii", b, p); p += 8; toc[t] = pos
    out = {}
    # VALIDATION (0): UTF partitioner class name | double bloomFilterFPChance (S/io/sstable/metadata/ValidationMetadata.java:64-78)
    if 0 in toc:
        p = toc[0]; (n,) = struct.unpack_from(">H", b, p); out["partitioner"] = b[p + 2:p + 2 + n].decode()
        (out["bloom_filter_fp_chance"],) = struct.unpack_from(">d", b, p + 2 + n)
    # STATS (2)
    p = toc[2]
    for _ in range(2):                                 # two EstimatedHistograms
        (sz,) = struct.unpack_from(">i", b, p); p += 4 + 16 * sz
    hists = []
    q = toc[2]
    for _ in range(2):                                 # EstimatedHistogram.serializer: i32 n | (i64 offset, i64 count) x n  (offset of bucket i = offsets[i-1], first = offsets[0])
        (sz,) = struct.unpack_from(">i", b, q); q += 4
        hists.append([struct.unpack_from(">qq", b, q + 16 * i)[1] for i in range(sz)]); q += 16 * sz
    out["partition_size_hist"], out["cells_per_partition_hist"] = hists
    p += 12                                            # CommitLogPosition
    mn_ts, mx_ts, mn_ldt, mx_ldt, mn_ttl, mx_ttl = struct.unpack_from(">qqIIii", b, p)
    out["min_timestamp"] = mn_ts; out["max_timestamp"] = mx_ts
    out["min_local_deletion_time"] = NO_DELETION_TIME if mn_ldt == 0xFFFFFFFF else mn_ldt
    out["max_local_deletion_time"] = NO_DELETION_TIME if mx_ldt == 0xFFFFFFFF else mx_ldt
    out["min_ttl"] = mn_ttl; out["max_ttl"] = mx_ttl
    q = p + 32
    (out["compression_ratio"],) = struct.unpack_from(">d", b, q); q += 8
    # TombstoneHistogram (oa: long points): i32 maxBinSize | i32 n | (i64 point, i32 count) x n ... versions differ; parsed defensively
    try:
        (_maxbin, n) = struct.unpack_from(">ii", b, q); q += 8
        td = []
        for _ in range(n):
            pt, cnt = struct.unpack_from(">qi", b, q); q += 12; td.append((pt, cnt))
        out["tombstone_drop_times"] = td
        (out["sstable_level"], out["repaired_at"]) = struct.unpack_from(">iq", b, q); q += 12
    except struct.error:
        pass
    # HEADER (3)
    p = toc[3]
    v, p = _vint(b, p); hts = v + TIMESTAMP_EPOCH
    v, p = _vint(b, p); hldt = (v & 0xFFFFFFFF) + DELETION_TIME_EPOCH if v < (1 << 32) else ((v - (1 << 64)) + DELETION_TIME_EPOCH)
    v, p = _vint(b, p); httl = v
    out["header_stats"] = (hts, hldt, httl)
    kt, p = _vbytes(b, p); out["key_type"] = kt.decode()
    nc, p = _vint(b, p); cl = []
    for _ in range(nc):
        t, p = _vbytes(b, p); cl.append(t.decode())
    out["clustering_types"] = cl
    cols = {}
    for kind in ("static_columns", "regular_columns"):
        k, p = _vint(b, p); lst = []
        for _ in range(k):
            name, p = _vbytes(b, p); t, p = _vbytes(b, p); lst.append((bytes(name), t.decode()))
        cols[kind] = lst
    out.update(cols)
    return out

class SSTable:
    """The components of one big-format sstable, in memory (what SSTableReader holds open for a compaction input)."""
    def __init__(self, data, index, compression: CompressionMetadata, header_stats, stats_min, clustering_types, regular_columns,
                 static_columns=(), key_type=MARSHAL + "BytesType", level=0, generation=0):
        self.data = data; self.index = index; self.compression = compression
        self.header_stats = tuple(header_stats)            # (minTimestamp, minLocalDeletionTime, minTTL) of the HEADER component
        self.stats_min = tuple(stats_min)                  # (minTimestamp, minLocalDeletionTime, minTTL) of the STATS component
        self.clustering_types = list(clustering_types)
        self.regular_columns = list(regular_columns)       # [(name bytes, type string)] in header order
        self.static_columns = list(static_columns)
        self.key_type = key_type; self.level = level; self.generation = generation
        self.summary_positions = None                      # Index.db offsets of the Summary.db samples (numpy uint64) when known
        self.partitioner = "org.apache.cassandra.dht.Murmur3Partitioner"

    @classmethod
    def open(cls, base_path: str, generation=0):
        """base_path: '<dir>/oa-1-big-' (descriptor prefix)."""
        rd = lambda c: open(base_path + c, "rb").read()
        st = parse_statistics(rd("Statistics.db"))
        data = rd("Data.db")
        # compression disabled: CRC.db stands in for CompressionInfo.db (ChecksummedSequentialWriter)
        meta = CompressionMetadata.parse(rd("CompressionInfo.db")) if os.path.exists(base_path + "CompressionInfo.db") else ChecksumMetadata.parse(rd("CRC.db"), len(data))
        t = cls(data, rd("Index.db"), meta, st["header_stats"],
                   (st["min_timestamp"], st["min_local_deletion_time"], st["min_ttl"]), st["clustering_types"],
                   st["regular_columns"], st["static_columns"], st["key_type"], generation=generation)
        if os.path.exists(base_path + "Summary.db"): t.summary_positions = parse_summary_positions(rd("Summary.db"))
        t.partitioner = st.get("partitioner", t.partitioner); t.bloom_filter_fp_chance = st.get("bloom_filter_fp_chance", 0.01)
        return t

def parse_summary_positions(buf: bytes):
    """Index.db offsets of the sampled entries of a Summary.db (IndexSummary.IndexSummarySerializer.serialize,
    S/io/sstable/indexsummary/IndexSummary.java:401-423): big-endian header (minIndexInterval, offsetCount, offHeapSize,
    samplingLevel, sizeAtFullSampling), then offsetCount native-order (little-endian) int32 offsets relative to the start of the
    offsets region, then per sample `key bytes | int64 Index.db position` (native order, :190-193)."""
    import numpy as np
    _min_interval, count, offheap, _level, _full = struct.unpack_from(">iiqii", buf, 0)
    base = 24
    offs = np.frombuffer(buf, dtype="<i4", count=count, offset=base).astype(np.int64)
    ends = np.append(offs[1:], offheap)
    pos = np.empty(count, dtype=np.uint64)
    for i in range(count):
        pos[i] = struct.unpack_from("<q", buf, base + int(ends[i]) - 8)[0]
    return pos

def index_summary_positions(index: bytes, interval: int = 128):
    """walks an Index.db image and returns the offset of every `interval`-th entry (what IndexSummaryBuilder.maybeAddEntry,
    S/io/sstable/indexsummary/IndexSummaryBuilder.java:200-228, records at the default min_index_interval). Python loop: for test-sized files."""
    import numpy as np
    out = []; o = 0; n = 0; L = len(index)
    while o < L:
        if n % interval == 0: out.append(o)
        kl = (index[o] << 8) | index[o + 1]; p = o + 2 + kl
        _, p = _vint(index, p)
        ps, p = _vint(index, p)
        o = p + ps; n += 1
    return np.asarray(out, dtype=np.uint64)

def write_components(base_path: str, data: bytes, index: bytes, compression: CompressionMetadata, digest: int):
    """Writes the components the engine produces (Data, Index, CompressionInfo or CRC.db, Digest). Statistics/Filter/Summary are
    SURVEY §8f 'next' rows and stay with the Java writer for now."""
    meta = "CRC.db" if isinstance(compression, ChecksumMetadata) else "CompressionInfo.db"
    for comp, payload in (("Data.db", data), ("Index.db", index), (meta, compression.serialize()),
                          ("Digest.crc32", str(digest).encode())):
        with open(base_path + comp, "wb") as f: f.write(payload)
