"""Mirror of org.apache.cassandra.db.compaction for the hot path: CompactionController (purge inputs), CompactionTask
(build the manifest from the input sstables, run the engine, hand back output components).

  CompactionTask.runMayThrow     S/db/compaction/CompactionTask.java:114-236
  SerializationHeader.make       S/db/SerializationHeader.java:77-100   (output EncodingStats + column union)
  CompactionController           S/db/compaction/CompactionController.java:76-96,247-286 (purge evaluator)
  CompactionManager.getDefaultGcBefore  S/db/compaction/CompactionManager.java:2001-2006

`engine` is any callable with the b200c_compact signature: the product passes the CUDA library (`GpuEngine`); the
tests additionally pass the CPU oracle to obtain the expected bytes from the same manifest.
"""
import ctypes as C, time
import numpy as np
from .. import native
from ..io import sstable as sst
from ..io.compress import CompressionMetadata, ChecksumMetadata, COMPRESSOR_IDS, COMPRESSOR_NAMES, check_chunk_length

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1

class CompactionController:
    """gcBefore and the purge evaluator. overlapping_min_timestamp = min timestamp over live sstables/memtables outside the
    compaction that may contain the keys (None = no overlaps: every tombstone older than gcBefore is purgeable)."""
    def __init__(self, now_in_sec, gc_grace_seconds=864000, overlapping_min_timestamp=None, purge_ranges=None):
        self.now_in_sec = now_in_sec
        self.gc_before = now_in_sec - gc_grace_seconds
        self.purge_max_timestamp = INT64_MAX if overlapping_min_timestamp is None else overlapping_min_timestamp
        # optional [(token_hi, min timestamp of the overlapping sstables that may hold keys up to token_hi)], ascending: the per-key
        # evaluator of getPurgeEvaluator bucketed by token range
        self.purge_ranges = list(purge_ranges or [])

class CompactionResult:
    def __init__(self): self.outputs = []; self.stats = {}

class OutputSSTable:
    def __init__(self, data, index, compression, digest, partitions, rows):
        self.data = data; self.index = index; self.compression = compression; self.digest = digest
        self.partitions = partitions; self.rows = rows
        self.filter = self.summary = self.first_key = self.last_key = None; self.stats = None
    def components(self):
        # compression disabled: CRC.db instead of CompressionInfo.db (DataComponent.buildWriter, S/io/sstable/format/DataComponent.java:43-60)
        meta = "CRC.db" if isinstance(self.compression, ChecksumMetadata) else "CompressionInfo.db"
        c = {"Data.db": self.data, "Index.db": self.index, meta: self.compression.serialize(), "Digest.crc32": str(self.digest).encode()}
        if self.filter is not None: c["Filter.db"] = self.filter
        if self.summary is not None: c["Summary.db"] = self.summary
        return c

STATS_SCALARS = ("min_timestamp", "max_timestamp", "min_local_deletion_time", "max_local_deletion_time", "min_ttl", "max_ttl", "total_rows",
                 "total_columns_set", "total_cells", "total_tombstones", "has_partition_level_deletions", "tdrop_overflow", "has_legacy_counter_shards")
def stats_dict(st):
    """b200c_sstable_stats -> plain dict (the MetadataCollector reductions, S/io/sstable/metadata/MetadataCollector.java:107-147)"""
    d = {k: int(getattr(st, k)) for k in STATS_SCALARS}
    d["partition_size_hist"] = [int(x) for x in st.partition_size_hist]; d["cells_per_partition_hist"] = [int(x) for x in st.cells_per_partition_hist]
    d["tombstone_drop_times"] = [(int(st.tdrop_point[i]), int(st.tdrop_count[i])) for i in range(st.ntdrop)]
    d["hll_registers"] = bytes(st.hll_registers)
    return d

def merged_encoding_stats(inputs):
    """SerializationHeader.make: EncodingStats.Collector over the inputs' StatsMetadata minima (S/db/rows/EncodingStats.java:150-236)."""
    ts = min(i.stats_min[0] for i in inputs)
    ldt = min(i.stats_min[1] for i in inputs)
    ttl = min(i.stats_min[2] for i in inputs)
    if ts == INT64_MIN: ts = sst.TIMESTAMP_EPOCH                    # LivenessInfo.NO_TIMESTAMP -> epoch (EncodingStats ctor :78-88)
    if ldt == sst.NO_DELETION_TIME: ldt = sst.DELETION_TIME_EPOCH
    return ts, ldt, ttl

def _name_key(name: bytes): return name                              # ColumnMetadata order within a group (simple / complex) = name bytes

class CompactionTask:
    def __init__(self, inputs, controller: CompactionController, compression=None, column_index_size=65536,
                 max_sstable_bytes=0, token_range=(INT64_MIN, INT64_MAX), bloom=None, min_index_interval=128, with_metadata=False):
        self.inputs = list(inputs); self.controller = controller
        c0 = self.inputs[0].compression
        if compression is None:
            compression = ChecksumMetadata(c0.chunk_length, 0, []) if isinstance(c0, ChecksumMetadata) else \
                          CompressionMetadata(c0.compressor_name, c0.chunk_length, c0.max_compressed_length, 0, [])
        self.compression = compression
        self.column_index_size = column_index_size; self.max_sstable_bytes = max_sstable_bytes; self.token_range = token_range
        # with_metadata: also produce Filter.db, Summary.db, first/last key and the Statistics.db side band (SURVEY §8 f1). bloom = (hash count,
        # 64-bit words) as FilterFactory would size the filter (io.sstable.bloom_geometry(estimated keys, fp chance)); None = 0.01 over the input keys
        self.with_metadata = with_metadata or bloom is not None; self.bloom = bloom; self.min_index_interval = min_index_interval
        self._keep = []

    def build_manifest(self):
        ins = self.inputs
        ct = ins[0].clustering_types
        if any(i.clustering_types != ct for i in ins): raise native.UnsupportedError(native.EUNSUPPORTED, "clustering types differ")
        union = {}
        for i in sorted(ins, key=lambda s: s.generation):            # newest generation's metadata wins (:91-99)
            for name, t in i.regular_columns: union[name] = t
        # ColumnMetadata.comparisonOrder: simple columns before complex (multi-cell) ones, each group by name (S/schema/ColumnMetadata.java:139-149)
        out_cols = sorted(union.items(), key=lambda kv: (sst.is_complex(kv[1]), _name_key(kv[0])))
        sunion = {}
        for i in sorted(ins, key=lambda s: s.generation):
            for name, t in i.static_columns: sunion[name] = t
        out_static = sorted(sunion.items(), key=lambda kv: _name_key(kv[0]))
        if len(out_static) > native.MAX_STATIC_COLUMNS: raise native.UnsupportedError(native.EUNSUPPORTED, "more than %d static columns" % native.MAX_STATIC_COLUMNS)
        for c in [i.compression for i in ins] + [self.compression]: check_chunk_length(c.chunk_length, isinstance(c, ChecksumMetadata))
        m = native.Manifest(); m.abi_version = native.ABI_VERSION; m.ninputs = len(ins)
        arr = (native.Input * len(ins))(); self._keep.append(arr)
        for k, s in enumerate(ins):
            a = arr[k]
            data = np.frombuffer(s.data, dtype=np.uint8); index = np.frombuffer(s.index, dtype=np.uint8)
            offs = np.asarray(s.compression.chunk_offsets, dtype=np.uint64)
            self._keep += [data, index, offs]
            a.data = data.ctypes.data if len(data) else None; a.data_len = len(data)
            a.index = index.ctypes.data if len(index) else None; a.index_len = len(index)
            a.chunk_offsets = offs.ctypes.data if len(offs) else None; a.nchunks = len(offs)
            a.data_length = s.compression.data_length; a.compressor = s.compression.compressor_id
            a.chunk_len = s.compression.chunk_length; a.max_compressed_len = s.compression.max_compressed_length
            a.ncolumns = len(s.regular_columns)
            names = [n for n, _ in out_cols]
            for ci, (name, _) in enumerate(s.regular_columns): a.column_map[ci] = names.index(name)
            a.nstatic_columns = len(s.static_columns)
            snames = [n for n, _ in out_static]
            for ci, (name, _) in enumerate(s.static_columns): a.static_column_map[ci] = snames.index(name)
            a.header_stats.min_timestamp, a.header_stats.min_local_deletion_time, a.header_stats.min_ttl = s.header_stats
            a.level = s.level
            sp = getattr(s, "summary_positions", None)
            if sp is not None and len(sp):
                sp = np.ascontiguousarray(sp, dtype=np.uint64); self._keep.append(sp)
                a.summary_positions = sp.ctypes.data; a.nsummary = len(sp)
            else: a.summary_positions = None; a.nsummary = 0
        m.inputs = arr
        m.nclustering = len(ct)
        for k, t in enumerate(ct):
            short = t[len(sst.MARSHAL):] if t.startswith(sst.MARSHAL) else t
            if short not in sst.CLUSTERING_OK: raise native.UnsupportedError(native.EUNSUPPORTED, "clustering type " + t)
            m.clustering[k].type, m.clustering[k].fixed_len = sst.type_class(t)
        m.ncolumns = len(out_cols)
        for k, (_, t) in enumerate(out_cols): m.columns[k].type, m.columns[k].fixed_len = sst.column_class(t)
        if sum(1 for _, t in out_cols if sst.is_complex(t)) > native.MAX_COMPLEX_COLUMNS: raise native.UnsupportedError(native.EUNSUPPORTED, "more than %d multi-cell columns" % native.MAX_COMPLEX_COLUMNS)
        if any(sst.is_complex(t) for _, t in out_static): raise native.UnsupportedError(native.EUNSUPPORTED, "multi-cell static column")
        m.nstatic_columns = len(out_static)
        for k, (_, t) in enumerate(out_static): m.static_columns[k].type, m.static_columns[k].fixed_len = sst.column_class(t)      # (simple columns; a static counter: TYPE_COUNTER)
        m.out_stats.min_timestamp, m.out_stats.min_local_deletion_time, m.out_stats.min_ttl = merged_encoding_stats(ins)
        m.out_compressor = self.compression.compressor_id; m.out_chunk_len = self.compression.chunk_length
        m.out_max_compressed_len = self.compression.max_compressed_length; m.column_index_size = self.column_index_size
        m.now_in_sec = self.controller.now_in_sec; m.gc_before = self.controller.gc_before
        m.purge_max_timestamp = self.controller.purge_max_timestamp
        m.tombstone_option = 0; m.enforce_strict_liveness = 0
        parts = {i.partitioner for i in ins}
        if len(parts) != 1 or next(iter(parts)) not in sst.PARTITIONER_IDS:
            raise native.UnsupportedError(native.EUNSUPPORTED, "partitioner " + ", ".join(sorted(parts)))
        m.partitioner = sst.PARTITIONER_IDS[next(iter(parts))]
        pr = self.controller.purge_ranges
        if pr:
            hi = np.asarray([a for a, _ in pr], dtype=np.int64); ts = np.asarray([b for _, b in pr], dtype=np.int64); self._keep += [hi, ts]
            m.npurge_ranges = len(pr); m.purge_range_hi = hi.ctypes.data; m.purge_range_max_ts = ts.ctypes.data
        m.token_lo, m.token_hi = self.token_range; m.max_sstable_bytes = self.max_sstable_bytes
        if self.with_metadata:
            k, words = self.bloom if self.bloom is not None else sst.bloom_geometry(max(1, sum(getattr(i, "partitions", 0) or 1 for i in ins)), 0.01)
            m.bloom_hash_count, m.bloom_words, m.min_index_interval = k, words, self.min_index_interval
        self.out_columns = out_cols
        return m

    def _result(self, m, nout, data_cap, index_cap, chunk_cap):
        """a b200c_result over `nout` output slots with buffers of the given capacities"""
        res = native.Result(); outs = (native.Output * nout)(); bufs = []; extra = []
        for o in outs:
            d = np.empty(data_cap, dtype=np.uint8); ix = np.empty(index_cap, dtype=np.uint8); co = np.zeros(chunk_cap, dtype=np.uint64)
            bufs.append((d, ix, co))
            o.data, o.data_cap, o.index, o.index_cap, o.chunk_offsets, o.chunk_cap = d.ctypes.data, data_cap, ix.ctypes.data, index_cap, co.ctypes.data, chunk_cap
            if self.with_metadata:
                kb = np.zeros(2 * 65535, dtype=np.uint8); fl = np.zeros(8 + 8 * int(m.bloom_words), dtype=np.uint8); sm = np.zeros(index_cap // 8 + (1 << 16), dtype=np.uint8)
                st = native.SSTableStats(); extra.append((kb, fl, sm, st))
                o.key_buf, o.key_cap, o.filter, o.filter_cap, o.summary, o.summary_cap = kb.ctypes.data, len(kb), fl.ctypes.data, len(fl), sm.ctypes.data, len(sm)
                o.stats = C.pointer(st)
        res.noutputs_cap = nout; res.outputs = outs
        return res, outs, bufs, extra

    def execute(self, engine, max_outputs=None):
        """Runs the compaction through `engine(manifest_ptr, result_ptr) -> rc` and returns a CompactionResult."""
        m = self.build_manifest()
        total_in = sum(i.compression.data_length for i in self.inputs)
        nout = max_outputs or (1 if not self.max_sstable_bytes else max(2, int(2 * total_in // max(self.max_sstable_bytes, 1)) + 2))
        cl = self.compression.chunk_length
        data_cap = native.lib().b200c_compress_bound(self.compression.compressor_id, total_in + 1024, cl) if engine.needs_lib_bound else total_in * 2 + (1 << 20)
        index_cap = sum(len(i.index) for i in self.inputs) * 2 + (1 << 16)
        chunk_cap = total_in // cl + 16
        # the merged stream can be longer than the inputs' streams (every row's deltas are re-encoded against the output header's minima,
        # which may lie far below an input's own): a call that finds the buffers too small reports what it needs and runs once more
        for attempt in (0, 1):
            res, outs, bufs, extra = self._result(m, nout, data_cap, index_cap, chunk_cap)
            t0 = time.perf_counter()
            try:
                engine(m, res)
                break
            except native.B200CError as e:
                if e.code != native.ETOOSMALL or attempt: raise
                data_cap = max(data_cap, int(res.required_data_cap)); index_cap = max(index_cap, int(res.required_index_cap))
                chunk_cap = max(chunk_cap, int(res.required_chunk_cap))
        wall = time.perf_counter() - t0
        r = CompactionResult()
        for k in range(res.noutputs):
            o = outs[k]; d, ix, co = bufs[k]
            if isinstance(self.compression, ChecksumMetadata): meta = ChecksumMetadata(cl, int(o.data_length), [int(x) for x in co[:o.nchunks]])
            else: meta = CompressionMetadata(self.compression.compressor_name, cl, self.compression.max_compressed_length, int(o.data_length),
                                             [int(x) for x in co[:o.nchunks]], self.compression.options)
            out = OutputSSTable(d[:o.data_len].tobytes(), ix[:o.index_len].tobytes(), meta, int(o.digest), int(o.partitions), int(o.rows))
            if self.with_metadata:
                kb, fl, sm, st = extra[k]
                out.first_key = kb[:o.first_key_len].tobytes(); out.last_key = kb[o.first_key_len:o.first_key_len + o.last_key_len].tobytes()
                out.filter = fl[:o.filter_len].tobytes(); out.summary = sm[:o.summary_len].tobytes(); out.stats = stats_dict(st)
            r.outputs.append(out)
        r.stats = dict(bytes_read=int(res.bytes_read), bytes_in_range=int(res.bytes_in_range), bytes_written=int(res.bytes_written), total_source_rows=int(res.total_source_rows),
                       input_partitions=int(res.input_partitions), merged_row_counts=[int(x) for x in res.merged_row_counts[:len(self.inputs)]],
                       kernel_ms=res.kernel_ms, total_ms=res.total_ms, kernel_launches=int(res.kernel_launches), index_slow_path_inputs=int(res.index_slow_path_inputs), wall_s=wall)
        return r

class GpuEngine:
    """b200c_compact on one device context."""
    needs_lib_bound = True
    def __init__(self, ctx, flags=0): self.ctx = ctx; self.flags = flags
    def __call__(self, manifest, result):
        rc = native.lib().b200c_compact(self.ctx.handle, C.byref(manifest), C.byref(result), self.flags)
        self.ctx.check(rc, result.corruption)
