"""ctypes binding of include/b200c.h. Fails loudly when libb200compact.so is missing or no CUDA device exists."""
import ctypes as C, os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200compact.so")

OK, EINVAL, ECUDA, ECORRUPT, ECANCELLED, EUNSUPPORTED, ENOMEM, ETOOSMALL = 0, -1, -2, -3, -4, -5, -6, -7
COMP_NONE, COMP_LZ4, COMP_SNAPPY, COMP_SNAPPY15 = 0, 1, 2, 3
COMP_UNCOMPRESSED = 4                 # compression disabled: Data.db + CRC.db (include/b200c.h)
FLAG_DEVICE_PTRS = 1
INT32_MAX = 0x7FFFFFFF
MAX_CLUSTERING, MAX_COLUMNS, MAX_INPUTS, MAX_STATIC_COLUMNS = 8, 64, 64, 16
ABI_VERSION = 2
PARTITIONER_MURMUR3, PARTITIONER_BYTE_ORDERED = 0, 1
PSIZE_BUCKETS, CELLS_BUCKETS, HLL_P, TDROP_CAP = 156, 119, 13, 512
TYPE_BYTES, TYPE_FIXED_SIGNED, TYPE_FIXED_BYTES, TYPE_VAR_SIGNED, TYPE_TIMEUUID, TYPE_COUNTER = 0, 1, 2, 3, 4, 5
MAX_COMPLEX_COLUMNS = 8

class B200CError(RuntimeError):
    def __init__(self, code, msg, corruption=None):
        super().__init__("b200c error %d: %s" % (code, msg)); self.code = code; self.corruption = corruption
class CorruptSSTableError(B200CError): pass          # CorruptSSTableException
class CompactionInterruptedError(B200CError): pass   # CompactionInterruptedException
class UnsupportedError(B200CError): pass

class Corruption(C.Structure):
    _fields_ = [("input", C.c_int32), ("kind", C.c_int32), ("chunk", C.c_uint64), ("offset", C.c_uint64)]
class Column(C.Structure):
    _fields_ = [("type", C.c_int32), ("fixed_len", C.c_int32)]
class EncodingStats(C.Structure):
    _fields_ = [("min_timestamp", C.c_int64), ("min_local_deletion_time", C.c_int64), ("min_ttl", C.c_int32), ("_pad", C.c_int32)]
class Input(C.Structure):
    _fields_ = [("data", C.c_void_p), ("data_len", C.c_uint64), ("index", C.c_void_p), ("index_len", C.c_uint64),
                ("chunk_offsets", C.c_void_p), ("nchunks", C.c_uint64), ("data_length", C.c_uint64),
                ("compressor", C.c_int32), ("chunk_len", C.c_int32), ("max_compressed_len", C.c_int32), ("ncolumns", C.c_int32),
                ("column_map", C.c_int32 * MAX_COLUMNS), ("header_stats", EncodingStats), ("_pad", C.c_int32), ("level", C.c_int32),
                ("summary_positions", C.c_void_p), ("nsummary", C.c_uint64),
                ("nstatic_columns", C.c_int32), ("static_column_map", C.c_int32 * MAX_STATIC_COLUMNS), ("_pad2", C.c_int32)]
class Manifest(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("ninputs", C.c_int32), ("inputs", C.POINTER(Input)),
                ("nclustering", C.c_int32), ("clustering", Column * MAX_CLUSTERING),
                ("ncolumns", C.c_int32), ("columns", Column * MAX_COLUMNS), ("nstatic_columns", C.c_int32),
                ("out_stats", EncodingStats), ("out_compressor", C.c_int32), ("out_chunk_len", C.c_int32),
                ("out_max_compressed_len", C.c_int32), ("column_index_size", C.c_int32),
                ("now_in_sec", C.c_int64), ("gc_before", C.c_int64), ("purge_max_timestamp", C.c_int64),
                ("tombstone_option", C.c_int32), ("enforce_strict_liveness", C.c_int32),
                ("token_lo", C.c_int64), ("token_hi", C.c_int64), ("max_sstable_bytes", C.c_uint64),
                ("partitioner", C.c_int32), ("npurge_ranges", C.c_int32), ("purge_range_hi", C.c_void_p), ("purge_range_max_ts", C.c_void_p),
                ("bloom_hash_count", C.c_int32), ("min_index_interval", C.c_int32), ("bloom_words", C.c_uint64),
                ("static_columns", Column * MAX_STATIC_COLUMNS)]
class SSTableStats(C.Structure):
    _fields_ = [("min_timestamp", C.c_int64), ("max_timestamp", C.c_int64),
                ("min_local_deletion_time", C.c_int64), ("max_local_deletion_time", C.c_int64),
                ("min_ttl", C.c_int32), ("max_ttl", C.c_int32),
                ("total_rows", C.c_uint64), ("total_columns_set", C.c_uint64), ("total_cells", C.c_uint64), ("total_tombstones", C.c_uint64),
                ("has_partition_level_deletions", C.c_int32), ("tdrop_overflow", C.c_int32),
                ("partition_size_hist", C.c_uint64 * PSIZE_BUCKETS), ("cells_per_partition_hist", C.c_uint64 * CELLS_BUCKETS),
                ("ntdrop", C.c_uint32), ("has_legacy_counter_shards", C.c_uint32),
                ("tdrop_point", C.c_int64 * TDROP_CAP), ("tdrop_count", C.c_uint64 * TDROP_CAP),
                ("hll_registers", C.c_uint8 * (1 << HLL_P))]
class Output(C.Structure):
    _fields_ = [("data", C.c_void_p), ("data_cap", C.c_uint64), ("data_len", C.c_uint64),
                ("index", C.c_void_p), ("index_cap", C.c_uint64), ("index_len", C.c_uint64),
                ("chunk_offsets", C.c_void_p), ("chunk_cap", C.c_uint64), ("nchunks", C.c_uint64),
                ("data_length", C.c_uint64), ("digest", C.c_uint32), ("_pad", C.c_uint32),
                ("partitions", C.c_uint64), ("rows", C.c_uint64),
                ("key_buf", C.c_void_p), ("key_cap", C.c_uint64), ("first_key_len", C.c_uint32), ("last_key_len", C.c_uint32),
                ("filter", C.c_void_p), ("filter_cap", C.c_uint64), ("filter_len", C.c_uint64),
                ("summary", C.c_void_p), ("summary_cap", C.c_uint64), ("summary_len", C.c_uint64),
                ("stats", C.POINTER(SSTableStats))]
class Result(C.Structure):
    _fields_ = [("noutputs_cap", C.c_int32), ("noutputs", C.c_int32), ("outputs", C.POINTER(Output)),
                ("bytes_read", C.c_uint64), ("bytes_in_range", C.c_uint64), ("bytes_written", C.c_uint64), ("total_source_rows", C.c_uint64),
                ("input_partitions", C.c_uint64), ("merged_row_counts", C.c_uint64 * MAX_INPUTS),
                ("required_data_cap", C.c_uint64), ("required_index_cap", C.c_uint64), ("required_chunk_cap", C.c_uint64),
                ("corruption", Corruption), ("kernel_ms", C.c_double), ("total_ms", C.c_double), ("kernel_launches", C.c_uint64),
                ("index_slow_path_inputs", C.c_uint64)]
class Progress(C.Structure):
    _fields_ = [("bytes_scanned", C.c_uint64), ("bytes_total", C.c_uint64), ("stage", C.c_int32), ("call_seq", C.c_int32)]

# every symbol include/b200c.h declares: (restype, argtypes)
_vp, _u64, _i, _u8p = C.c_void_p, C.c_uint64, C.c_int, C.c_void_p
SYMBOLS = {
    "b200c_abi_version": (C.c_int, []),
    "b200c_device_count": (C.c_int, []),
    "b200c_create": (_vp, [C.c_int, C.c_size_t]),
    "b200c_destroy": (None, [_vp]),
    "b200c_last_error": (C.c_char_p, [_vp]),
    "b200c_host_register": (C.c_int, [_vp, C.c_size_t]),
    "b200c_host_unregister": (C.c_int, [_vp]),
    "b200c_dev_alloc": (C.c_int, [_vp, C.c_size_t, C.POINTER(_vp)]),
    "b200c_dev_free": (C.c_int, [_vp, _vp]),
    "b200c_memcpy_h2d": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
    "b200c_memcpy_d2h": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
    "b200c_sync": (C.c_int, [_vp]),
    "b200c_last_kernel_ms": (C.c_double, [_vp]),
    "b200c_last_kernel_launches": (_u64, [_vp]),
    "b200c_total_kernel_launches": (_u64, [_vp]),
    "b200c_last_stage_ms": (C.c_int, [_vp, C.POINTER(C.c_double), C.c_int]),
    "b200c_compress_bound": (_u64, [_i, _u64, _i]),
    "b200c_chunk_count": (_u64, [_u64, _i]),
    "b200c_compress_chunks": (C.c_int, [_vp, _i, _u8p, _u64, _i, _i, _u8p, _u64, C.POINTER(_u64), _vp, C.POINTER(C.c_uint32), _i]),
    "b200c_decompress_chunks": (C.c_int, [_vp, _i, _u8p, _u64, _vp, _u64, _i, _i, _u64, _u8p, _i, C.POINTER(Corruption), _i]),
    "b200c_initial_compressed_buffer_length": (C.c_int, [_i, _i]),
    "b200c_compress": (C.c_int, [_vp, _i, _u8p, _i, _u8p, _i]),
    "b200c_uncompress": (C.c_int, [_vp, _i, _u8p, _i, _u8p, _i]),
    "b200c_compact": (C.c_int, [_vp, C.POINTER(Manifest), C.POINTER(Result), _i]),
    "b200c_token": (C.c_int64, [C.c_int, _u8p, C.c_uint32]),
    "b200c_poll": (C.c_int, [_vp, C.POINTER(Progress)]),
    "b200c_poll_inputs": (C.c_int, [_vp, C.POINTER(C.c_uint64), C.c_int]),
    "b200c_cancel": (None, [_vp]),
    "b200c_cancel_reset": (None, [_vp]),
}

_LIB = None
def lib():
    """Loads libb200compact.so (in-tree). Raises if it has not been built — there is no fallback implementation."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("libb200compact.so is not built (run ./build.sh or __graft_entry__.build()); "
                              "cassandra_b200 has no CPU fallback")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            f = getattr(L, name); f.restype = res; f.argtypes = args
        if L.b200c_abi_version() != ABI_VERSION:
            raise ImportError("libb200compact.so ABI mismatch")
        _LIB = L
    return _LIB

def _buf_addr(b):
    """address of a bytes / bytearray / numpy array / ctypes buffer (no copy)"""
    if b is None: return None
    if isinstance(b, bytes): return C.cast(C.c_char_p(b), C.c_void_p).value
    if hasattr(b, "ctypes"): return b.ctypes.data
    return C.addressof((C.c_char * len(b)).from_buffer(b))

class Context:
    """One engine context = one CUDA stream + workspace on one device (one per CompactionExecutor thread)."""
    def __init__(self, device=0, workspace_bytes=0):
        self._lib = lib()
        self._h = self._lib.b200c_create(device, workspace_bytes)
        if not self._h:
            raise B200CError(ECUDA, "b200c_create failed: no CUDA device %d (devices=%d); no CPU fallback exists"
                             % (device, self._lib.b200c_device_count()))
        self.device = device
    def close(self):
        if self._h: self._lib.b200c_destroy(self._h); self._h = None
    def __enter__(self): return self
    def __exit__(self, *a): self.close()
    def __del__(self):
        try: self.close()
        except Exception: pass
    @property
    def handle(self): return self._h
    def last_error(self): return self._lib.b200c_last_error(self._h).decode()
    def check(self, rc, corruption=None):
        if rc >= 0: return rc
        msg = self.last_error()
        if rc == ECORRUPT: raise CorruptSSTableError(rc, msg, corruption)
        if rc == ECANCELLED: raise CompactionInterruptedError(rc, msg)
        if rc == EUNSUPPORTED: raise UnsupportedError(rc, msg)
        raise B200CError(rc, msg)
    @property
    def last_kernel_ms(self): return self._lib.b200c_last_kernel_ms(self._h)
    @property
    def last_kernel_launches(self): return self._lib.b200c_last_kernel_launches(self._h)
    @property
    def total_kernel_launches(self): return self._lib.b200c_total_kernel_launches(self._h)
    def last_stage_ms(self):
        a = (C.c_double * 8)(); n = self._lib.b200c_last_stage_ms(self._h, a, 8); return [a[i] for i in range(n)]

    # ---- batched chunk codec -------------------------------------------------------------------------------------
    def compress_chunks(self, compressor, data, chunk_len=16384, max_compressed_len=INT32_MAX):
        """-> (Data.db image bytes, [chunk offsets], digest). Mirrors CompressedSequentialWriter over a whole stream."""
        import numpy as np
        n = len(data); L = self._lib
        cap = L.b200c_compress_bound(compressor, n, chunk_len); nch = L.b200c_chunk_count(n, chunk_len)
        out = np.empty(cap, dtype=np.uint8); offs = np.zeros(max(nch, 1), dtype=np.uint64)
        out_len = C.c_uint64(); dig = C.c_uint32()
        rc = L.b200c_compress_chunks(self._h, compressor, _buf_addr(data), n, chunk_len, max_compressed_len, out.ctypes.data, cap,
                                     C.byref(out_len), offs.ctypes.data, C.byref(dig), 0)
        self.check(rc)
        return out[:out_len.value].tobytes(), [int(x) for x in offs[:nch]], dig.value

    def decompress_chunks(self, compressor, image, chunk_offsets, data_length, chunk_len=16384, max_compressed_len=INT32_MAX, verify_crc=True):
        import numpy as np
        L = self._lib
        offs = np.asarray(chunk_offsets, dtype=np.uint64); out = np.empty(max(data_length, 1), dtype=np.uint8)
        where = Corruption()
        rc = L.b200c_decompress_chunks(self._h, compressor, _buf_addr(image), len(image), offs.ctypes.data, len(offs), chunk_len,
                                       max_compressed_len, data_length, out.ctypes.data, 1 if verify_crc else 0, C.byref(where), 0)
        self.check(rc, where)
        return out[:data_length].tobytes()
