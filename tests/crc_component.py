"""Plain restatement of the uncompressed Data.db + CRC.db format, independent of the engine (test helper). Only zlib.crc32 is shared.

  write_crc      ChecksummedSequentialWriter / ChecksumWriter.appendDirect   S/io/util/ChecksummedSequentialWriter.java,
                                                                             S/io/util/ChecksumWriter.java:48-89
  read_crc       what a reader that checks CRC.db does: every chunk against its entry (kind 1 on a mismatch)
  lcs_files      MaxSSTableSizeWriter.shouldSwitchWriterInCurrentLocation   S/db/compaction/writers/MaxSSTableSizeWriter.java:76-79
                 over an uncompressed writer, whose getEstimatedOnDiskBytesWritten() is position() (S/io/util/SequentialWriter.java:304-312)

Data.db is the partition stream itself. The writer's buffer (64 KiB by default, SequentialWriterOption.java:107) is flushed only when
it is full and the next byte arrives, and once more at the end, so every chunk is full but the last, and a file whose length is a
multiple of the chunk size has no empty trailing chunk. CRC.db is the BE i32 chunk size, then one BE i32 CRC32 per chunk. Digest.crc32
is the CRC32 of Data.db alone.

UncompressedOracle runs compactions with uncompressed inputs or output on the CPU oracle, which knows only compressed chunks: inputs are
checked against their CRC.db here and handed over NoopCompressor-framed; an uncompressed output is the oracle's NoopCompressor output
unframed, with its CRC.db written here and, for LCS, cut into files by lcs_files.
"""
import ctypes as C, struct, zlib
import numpy as np
import oracle_lib as O
from chunk_format import INT32_MAX, write_chunks, read_chunks
from cassandra_b200 import native

DEFAULT_CHUNK = 65536

def crc_entries(data, chunk_len):
    """CRC32 of every chunk [i * L, min((i + 1) * L, len)); none for an empty file, no empty chunk at an exact multiple"""
    return [zlib.crc32(bytes(data[i:i + chunk_len])) for i in range(0, len(data), chunk_len)]

def write_crc(data, chunk_len=DEFAULT_CHUNK):
    """-> (CRC.db bytes, CRC entries, Digest.crc32 value)"""
    crcs = crc_entries(data, chunk_len)
    return struct.pack(">i", chunk_len) + b"".join(struct.pack(">I", c) for c in crcs), crcs, zlib.crc32(bytes(data))

def parse_crc(crc_db):
    """-> (chunk size, CRC entries)"""
    (L,) = struct.unpack_from(">i", crc_db, 0)
    return L, list(struct.unpack_from(">%dI" % ((len(crc_db) - 4) // 4), crc_db, 4))

class CrcError(Exception):
    def __init__(self, chunk, offset):
        super().__init__("chunk %d at %d: CRC mismatch" % (chunk, offset)); self.chunk = chunk; self.offset = offset

def read_crc(data, crcs, chunk_len):
    """-> data, or CrcError(chunk, chunk * L) for the first chunk that does not match its entry; a table of the wrong length is refused"""
    if len(crcs) != (len(data) + chunk_len - 1) // chunk_len: raise ValueError("CRC.db has %d entries for %d chunks" % (len(crcs), (len(data) + chunk_len - 1) // chunk_len))
    for i, want in enumerate(crcs):
        if zlib.crc32(bytes(data[i * chunk_len:(i + 1) * chunk_len])) != want: raise CrcError(i, i * chunk_len)
    return bytes(data)

# ---- Index.db (big format): u16 key length | key | vint position | vint promoted size | promoted index (offsets inside it are relative
# to the partition start, so only the position changes when a file is cut) ---------------------------------------------------------------
def _vint(b, p):
    first = b[p]
    if first < 0x80: return first, p + 1
    extra = 8 if first == 0xFF else (8 - (~first & 0xFF).bit_length())
    v = first & (0xFF >> extra)
    for k in range(extra): v = (v << 8) | b[p + 1 + k]
    return v, p + 1 + extra

def _vint_bytes(v):
    for extra in range(9):
        if extra == 8 or v < (1 << (7 * (extra + 1))): break
    if extra == 0: return bytes([v])
    if extra == 8: return b"\xff" + v.to_bytes(8, "big")
    raw = v.to_bytes(extra + 1, "big")
    return bytes([raw[0] | (0xFF << (8 - extra) & 0xFF)]) + raw[1:]

def index_entries(index):
    """-> [(key, Data.db position, promoted index bytes)]"""
    out = []; o = 0
    while o < len(index):
        kl = (index[o] << 8) | index[o + 1]; key = bytes(index[o + 2:o + 2 + kl]); p = o + 2 + kl
        pos, p = _vint(index, p); ps, p = _vint(index, p)
        out.append((key, pos, bytes(index[p:p + ps]))); o = p + ps
    return out

def index_bytes(entries, base=0):
    return b"".join(struct.pack(">H", len(k)) + k + _vint_bytes(pos - base) + _vint_bytes(len(pr)) + pr for k, pos, pr in entries)

def lcs_files(starts, total, limit):
    """partition start positions of one merged stream -> [(first partition, end partition, start byte, end byte)] of the files an
    uncompressed LCS writer produces: before each partition but a file's first it switches when position() > limit"""
    files = []; j0 = 0
    while j0 < len(starts):
        j = j0 + 1
        while j < len(starts) and starts[j] - starts[j0] <= limit: j += 1
        files.append((j0, j, starts[j0], starts[j] if j < len(starts) else total)); j0 = j
    return files

# ---- the CPU oracle with uncompressed inputs and outputs ----------------------------------------------------------------------------------------
def _bytes_at(ptr, n):
    return C.string_at(ptr, n) if n else b""

class ParallelOracleEngine:
    """oracle/parallel.cc (orc_compact_parallel, one compaction cut into token ranges on several threads) behind O.OracleEngine's interface"""
    needs_lib_bound = False
    def __init__(self, threads=4, ranges=16): self.threads = threads; self.ranges = ranges
    def __call__(self, manifest, result):
        L = O.lib(); f = L.orc_compact_parallel
        f.restype = C.c_int
        f.argtypes = [C.POINTER(native.Manifest), C.POINTER(native.Result), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int64), C.c_char_p, C.c_int]
        err = C.create_string_buffer(256); tm = (C.c_double * 6)(); hi = C.c_int64((1 << 63) - 1)
        rc = f(C.byref(manifest), C.byref(result), self.threads, self.ranges, 0, tm, C.byref(hi), err, 256)
        if rc == native.ECORRUPT: raise native.CorruptSSTableError(rc, err.value.decode(), result.corruption)
        if rc == native.EUNSUPPORTED: raise native.UnsupportedError(rc, err.value.decode())
        if rc != 0: raise native.B200CError(rc, err.value.decode())

class UncompressedOracle:
    """O.OracleEngine (or `inner`, e.g. ParallelOracleEngine) for manifests with B200C_COMP_UNCOMPRESSED inputs or output (see the module
    docstring)"""
    needs_lib_bound = False
    def __init__(self, inner=None): self.inner = inner or O.OracleEngine()
    def __call__(self, manifest, result):
        n = manifest.ninputs; keep = []
        m2 = native.Manifest.from_buffer_copy(manifest)
        ins = (native.Input * n)()
        for k in range(n):
            a = native.Input.from_buffer_copy(manifest.inputs[k]); ins[k] = a
            if a.compressor != native.COMP_UNCOMPRESSED: continue
            data = _bytes_at(a.data, a.data_len)
            crcs = list(np.ctypeslib.as_array(C.cast(a.chunk_offsets, C.POINTER(C.c_uint64)), shape=(a.nchunks,))) if a.nchunks else []
            if a.data_length != a.data_len: raise native.B200CError(native.EINVAL, "data_length must equal data_len")
            try: read_crc(data, crcs, a.chunk_len)
            except ValueError as e: raise native.B200CError(native.EINVAL, str(e))
            except CrcError as e:
                result.corruption.input, result.corruption.kind, result.corruption.chunk, result.corruption.offset = k, 1, e.chunk, e.offset
                raise native.CorruptSSTableError(native.ECORRUPT, str(e), result.corruption)
            image, offs, _ = write_chunks(data, native.COMP_NONE, a.chunk_len, INT32_MAX)
            img = np.frombuffer(image, dtype=np.uint8); off = np.asarray(offs, dtype=np.uint64); keep += [img, off]
            ins[k].data = img.ctypes.data if len(img) else None; ins[k].data_len = len(img)
            ins[k].chunk_offsets = off.ctypes.data if len(off) else None
            ins[k].compressor = native.COMP_NONE; ins[k].max_compressed_len = INT32_MAX
        m2.inputs = ins
        if manifest.out_compressor != native.COMP_UNCOMPRESSED:
            self.inner(m2, result); return
        L = manifest.out_chunk_len; limit = manifest.max_sstable_bytes
        m2.out_compressor = native.COMP_NONE; m2.out_max_compressed_len = INT32_MAX; m2.max_sstable_bytes = 0
        r2 = native.Result(); o2 = (native.Output * 1)(); r2.noutputs_cap = 1; r2.outputs = o2
        o0 = result.outputs[0]
        cap = sum(ins[k].data_length for k in range(n)) * 2 + (1 << 20); icap = sum(ins[k].index_len for k in range(n)) * 2 + (1 << 16)
        d = np.empty(cap, dtype=np.uint8); ix = np.empty(icap, dtype=np.uint8); co = np.zeros(cap // L + 16, dtype=np.uint64)
        o2[0].data, o2[0].data_cap, o2[0].index, o2[0].index_cap, o2[0].chunk_offsets, o2[0].chunk_cap = d.ctypes.data, cap, ix.ctypes.data, icap, co.ctypes.data, len(co)
        for f in ("key_buf", "key_cap", "filter", "filter_cap", "summary", "summary_cap", "stats"): setattr(o2[0], f, getattr(o0, f))
        try: self.inner(m2, r2)
        finally:
            for f in ("bytes_read", "bytes_in_range", "bytes_written", "total_source_rows", "input_partitions", "merged_row_counts", "corruption"):
                setattr(result, f, getattr(r2, f))
        o = o2[0]
        stream = read_chunks(d[:o.data_len].tobytes(), [int(x) for x in co[:o.nchunks]], native.COMP_NONE, L, INT32_MAX, int(o.data_length)) if r2.noutputs else b""
        index = ix[:o.index_len].tobytes() if r2.noutputs else b""
        if not limit:
            files = [(stream, index, int(o.partitions), int(o.rows))] if r2.noutputs else []
            for f in ("first_key_len", "last_key_len", "filter_len", "summary_len"): setattr(o0, f, getattr(o, f))
        else:
            ents = index_entries(index)
            files = [(stream[a:b], index_bytes(ents[j0:j1], a), j1 - j0, None) for j0, j1, a, b in lcs_files([p for _, p, _ in ents], len(stream), limit)]
        if len(files) > result.noutputs_cap: raise native.B200CError(native.ETOOSMALL, "more output files than output slots")
        result.required_data_cap = max([len(f[0]) for f in files], default=0); result.required_index_cap = max([len(f[1]) for f in files], default=0)
        result.required_chunk_cap = max([(len(f[0]) + L - 1) // L for f in files], default=0)
        if any(result.required_data_cap > result.outputs[k].data_cap or result.required_index_cap > result.outputs[k].index_cap or
               result.required_chunk_cap > result.outputs[k].chunk_cap for k in range(len(files))):
            raise native.B200CError(native.ETOOSMALL, "output buffers too small")
        result.noutputs = len(files)
        for k, (data, idx, parts, rows) in enumerate(files):
            out = result.outputs[k]; crcs = crc_entries(data, L)
            C.memmove(out.data, data, len(data)); C.memmove(out.index, idx, len(idx))
            tab = np.asarray(crcs, dtype=np.uint64)
            if crcs: C.memmove(out.chunk_offsets, tab.ctypes.data, 8 * len(crcs))
            out.data_len = out.data_length = len(data); out.index_len = len(idx); out.nchunks = len(crcs); out.digest = zlib.crc32(data)
            out.partitions = parts; out.rows = rows if rows is not None else 0
