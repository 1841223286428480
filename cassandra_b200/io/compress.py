"""Mirror of org.apache.cassandra.io.compress for the GPU engine.

ICompressor (S/io/compress/ICompressor.java:28-86): initialCompressedBufferLength / compress / uncompress, stateless singletons
created by `create(options)` (S/schema/CompressionParams.java:266-283). The persisted class simple name stays
`LZ4Compressor` / `SnappyCompressor` so stock nodes can read the files (S/io/compress/CompressionMetadata.java:379).
CompressionMetadata: CompressionInfo.db reader/writer (S/io/compress/CompressionMetadata.java:113-160,375-431).
ChecksumMetadata: CRC.db, which stands in for CompressionInfo.db when a table's compression is disabled
(ChecksummedSequentialWriter, S/io/util/ChecksummedSequentialWriter.java).
"""
import struct
from .. import native

class ICompressor:
    compressor_id = native.COMP_NONE
    simple_name = "NoopCompressor"
    def __init__(self, ctx): self.ctx = ctx
    def initial_compressed_buffer_length(self, chunk_length):            # ICompressor.java:30
        return native.lib().b200c_initial_compressed_buffer_length(self.compressor_id, chunk_length)
    def compress(self, data: bytes) -> bytes:                            # ICompressor.java:51  (ByteBuffer in -> out)
        import ctypes as C
        cap = self.initial_compressed_buffer_length(max(len(data), 1)) + 8
        out = C.create_string_buffer(cap)
        n = native.lib().b200c_compress(self.ctx.handle, self.compressor_id, data, len(data), out, cap)
        self.ctx.check(n)
        return out.raw[:n]
    def uncompress(self, data: bytes, max_len=65536) -> bytes:           # ICompressor.java:37,58; IOException on malformed input
        import ctypes as C
        out = C.create_string_buffer(max(max_len, 1))
        n = native.lib().b200c_uncompress(self.ctx.handle, self.compressor_id, data, len(data), out, max_len)
        self.ctx.check(n)
        return out.raw[:n]
    def supported_options(self): return set()

class LZ4Compressor(ICompressor):
    """S/io/compress/LZ4Compressor.java — fast mode only (lz4_compressor_type = fast, :48,102-106)."""
    compressor_id = native.COMP_LZ4
    simple_name = "LZ4Compressor"
    @classmethod
    def create(cls, ctx, options=None):
        options = options or {}
        if options.get("lz4_compressor_type", "fast") != "fast":
            raise native.UnsupportedError(native.EUNSUPPORTED, "only lz4_compressor_type=fast is implemented on the GPU")
        return cls(ctx)
    def supported_options(self): return {"lz4_high_compressor_level", "lz4_compressor_type"}

class SnappyCompressor(ICompressor):
    """S/io/compress/SnappyCompressor.java — raw snappy. Byte parity with snappy-java is UNPINNED (no golden)."""
    compressor_id = native.COMP_SNAPPY
    simple_name = "SnappyCompressor"
    @classmethod
    def create(cls, ctx, options=None): return cls(ctx)

class NoopCompressor(ICompressor):
    """S/io/compress/NoopCompressor.java — the compressed format (CompressionInfo.db, inline CRCs) with a copy as its codec.
    CompressionParams.NOOP uses 4 KiB chunks."""
    compressor_id = native.COMP_NONE
    simple_name = "NoopCompressor"
    @classmethod
    def create(cls, ctx, options=None): return cls(ctx)

MAX_CHUNK_LENGTH = 1 << 20                  # chunk_length_in_kb up to 1024 (include/b200c.h: B200C_MAX_CHUNK_LEN)
MAX_CRC_CHUNK_LENGTH = 65536               # CRC.db of an uncompressed table (ChecksummedSequentialWriter writes 64 KiB)

def check_chunk_length(chunk_length, uncompressed=False):
    """CompressionParams accepts any power of two; the engine compacts chunks up to 1 MiB (CRC.db chunks up to 64 KiB) and refuses the rest."""
    limit = MAX_CRC_CHUNK_LENGTH if uncompressed else MAX_CHUNK_LENGTH
    if chunk_length <= 0 or chunk_length & (chunk_length - 1) or chunk_length > limit:
        raise native.UnsupportedError(native.EUNSUPPORTED, "chunk length %d: a power of two <= %d is supported" % (chunk_length, limit))

COMPRESSOR_IDS = {"LZ4Compressor": native.COMP_LZ4, "SnappyCompressor": native.COMP_SNAPPY, "NoopCompressor": native.COMP_NONE}
COMPRESSOR_NAMES = {v: k for k, v in COMPRESSOR_IDS.items()}

class CompressionMetadata:
    """CompressionInfo.db. Layout: UTF(simple class name) | i32 nOpts | (UTF k, UTF v)* | i32 chunkLength |
    i32 maxCompressedLength (version >= na) | i64 dataLength | i32 nChunks | i64 offset x n — all big-endian."""
    def __init__(self, compressor_name, chunk_length, max_compressed_length, data_length, chunk_offsets, options=None):
        self.compressor_name = compressor_name; self.chunk_length = chunk_length
        self.max_compressed_length = max_compressed_length; self.data_length = data_length
        self.chunk_offsets = list(chunk_offsets); self.options = dict(options or {})
    @property
    def compressor_id(self): return COMPRESSOR_IDS[self.compressor_name]
    @classmethod
    def parse(cls, b: bytes, has_max_compressed_length=True):
        p = 0
        (n,) = struct.unpack_from(">H", b, p); p += 2; name = b[p:p + n].decode(); p += n
        (nopt,) = struct.unpack_from(">i", b, p); p += 4; opts = {}
        for _ in range(nopt):
            (kl,) = struct.unpack_from(">H", b, p); p += 2; k = b[p:p + kl].decode(); p += kl
            (vl,) = struct.unpack_from(">H", b, p); p += 2; v = b[p:p + vl].decode(); p += vl
            opts[k] = v
        (cl,) = struct.unpack_from(">i", b, p); p += 4
        mcl = native.INT32_MAX
        if has_max_compressed_length: (mcl,) = struct.unpack_from(">i", b, p); p += 4
        (dl, nc) = struct.unpack_from(">qi", b, p); p += 12
        offs = list(struct.unpack_from(">%dq" % nc, b, p))
        return cls(name, cl, mcl, dl, offs, opts)
    def serialize(self) -> bytes:                                         # CompressionMetadata.Writer.writeHeader :375-398 + doPrepare :423-431
        name = self.compressor_name.encode()
        out = [struct.pack(">H", len(name)), name, struct.pack(">i", len(self.options))]
        for k, v in self.options.items():
            kb, vb = k.encode(), v.encode(); out += [struct.pack(">H", len(kb)), kb, struct.pack(">H", len(vb)), vb]
        out.append(struct.pack(">iiqi", self.chunk_length, self.max_compressed_length, self.data_length, len(self.chunk_offsets)))
        out.append(struct.pack(">%dq" % len(self.chunk_offsets), *self.chunk_offsets))
        return b"".join(out)

def write_compressed(ctx, compressor: ICompressor, stream: bytes, chunk_length=16384, max_compressed_length=native.INT32_MAX):
    """CompressedSequentialWriter over a whole uncompressed stream (S/io/compress/CompressedSequentialWriter.java:140-206):
    -> (Data.db bytes, CompressionInfo.db bytes, Digest.crc32 text)."""
    check_chunk_length(chunk_length)
    image, offs, digest = ctx.compress_chunks(compressor.compressor_id, stream, chunk_length, max_compressed_length)
    meta = CompressionMetadata(compressor.simple_name, chunk_length, max_compressed_length, len(stream), offs)
    return image, meta.serialize(), str(digest)

def read_compressed(ctx, data_db: bytes, compression_info: bytes, verify_crc=True) -> bytes:
    """CompressedChunkReader over a whole file (S/io/util/CompressedChunkReader.java:103-173) -> uncompressed stream."""
    meta = CompressionMetadata.parse(compression_info)
    return ctx.decompress_chunks(meta.compressor_id, data_db, meta.chunk_offsets, meta.data_length, meta.chunk_length,
                                 meta.max_compressed_length, verify_crc)

class ChecksumMetadata:
    """CRC.db of an sstable written with compression disabled: BE i32 chunk size, then one BE i32 CRC32 per chunk of Data.db
    (ChecksumWriter.writeChunkSize / appendDirect, S/io/util/ChecksumWriter.java:48-89). It takes CompressionMetadata's place in the
    manifest: compressor id B200C_COMP_UNCOMPRESSED, the chunk table holds the CRCs, data_length is the length of Data.db."""
    compressor_id = native.COMP_UNCOMPRESSED
    compressor_name = None
    max_compressed_length = native.INT32_MAX
    DEFAULT_CHUNK_LENGTH = 65536            # SequentialWriterOption's default buffer size (S/io/util/SequentialWriterOption.java:107)
    def __init__(self, chunk_length, data_length, crcs):
        self.chunk_length = chunk_length; self.data_length = data_length; self.chunk_offsets = list(crcs); self.options = {}
    @property
    def crcs(self): return self.chunk_offsets
    @classmethod
    def parse(cls, b: bytes, data_length: int):
        (cl,) = struct.unpack_from(">i", b, 0)
        n = (len(b) - 4) // 4
        return cls(cl, data_length, [x for x in struct.unpack_from(">%dI" % n, b, 4)])
    def serialize(self) -> bytes:
        return struct.pack(">i%dI" % len(self.chunk_offsets), self.chunk_length, *self.chunk_offsets)

def uncompressed_params(chunk_length=ChecksumMetadata.DEFAULT_CHUNK_LENGTH):
    """the output setting of a table with compression = {'enabled': false}"""
    return ChecksumMetadata(chunk_length, 0, [])

def write_uncompressed(ctx, stream: bytes, chunk_length=ChecksumMetadata.DEFAULT_CHUNK_LENGTH):
    """ChecksummedSequentialWriter over a whole stream -> (Data.db bytes, CRC.db bytes, Digest.crc32 text)."""
    data, crcs, digest = ctx.compress_chunks(native.COMP_UNCOMPRESSED, stream, chunk_length)
    return data, ChecksumMetadata(chunk_length, len(stream), crcs).serialize(), str(digest)

def read_uncompressed(ctx, data_db: bytes, crc_db: bytes, verify_crc=True) -> bytes:
    """Data.db of an uncompressed sstable, every chunk checked against CRC.db -> the stream."""
    meta = ChecksumMetadata.parse(crc_db, len(data_db))
    return ctx.decompress_chunks(native.COMP_UNCOMPRESSED, data_db, meta.crcs, len(data_db), meta.chunk_length, native.INT32_MAX, verify_crc)
