"""Chunks of 128 KiB to 1 MiB (test helper): the block codecs as the libraries write them, the chunk format over them, and inputs that
exercise what changes above 64 KiB.

  LZ4      the system liblz4.so.1, LZ4_compress_default (what lz4-java's JNI compressor calls): from LZ4_64Klimit = 65547 bytes on it hashes 5
           bytes into 4096 u32 slots (byU32) and refuses candidates more than 65535 bytes back; below it, the 16-bit regime of <= 64 KiB chunks
  Snappy   snappy::Compress: 64 KiB fragments compressed independently behind one varint length. Google's library (pyarrow) for the >= 1.2
           table generation; the oracle's fragment loop, which equals that library, for both generations
  decoding the oracle's block decoders (any block length)

write_chunks / reencode restate flushData (tests/chunk_format.py) over these codecs; chunk_format.read_chunks reads any chunk length.
"""
import ctypes as C, random, struct, zlib
import oracle_lib as O
from chunk_format import read_chunks
from cassandra_b200.io.compress import CompressionMetadata

COMP_NONE = 0
COMP_NAMES = {O.COMP_LZ4: "LZ4Compressor", O.COMP_SNAPPY: "SnappyCompressor", COMP_NONE: "NoopCompressor"}
LZ4_64KLIMIT = 65536 + 11
MASK64 = (1 << 64) - 1
_LZ4 = None

def liblz4():
    global _LZ4
    if _LZ4 is None:
        for n in ("liblz4.so.1", "liblz4.so"):
            try:
                L = C.CDLL(n); break
            except OSError:
                L = None
        if L is None: return None
        L.LZ4_compress_default.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int]; L.LZ4_compress_default.restype = C.c_int
        L.LZ4_decompress_safe.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int]; L.LZ4_decompress_safe.restype = C.c_int
        _LZ4 = L
    return _LZ4

def lz4_block(b: bytes) -> bytes:
    L = liblz4(); out = C.create_string_buffer(len(b) + len(b) // 255 + 16)
    n = L.LZ4_compress_default(b, out, len(b), len(out)); assert n > 0
    return out.raw[:n]

def snappy15(b: bytes) -> bytes:
    import pyarrow as pa
    return pa.Codec("snappy").compress(b, asbytes=True)

def chunk_compress(comp, b: bytes) -> bytes:
    """the compressor output of one chunk (LZ4Compressor: 4-byte LE length + block)"""
    if comp == O.COMP_LZ4: return struct.pack("<I", len(b)) + lz4_block(b)
    if comp in (O.COMP_SNAPPY, O.COMP_SNAPPY15): return O.chunk_compress(comp, b)
    return bytes(b)

def write_chunks(stream, comp, chunk_len, max_clen):
    """flushData over the stream -> (Data.db image, chunk offsets, Digest.crc32 value)"""
    image = bytearray(); offs = []
    for i in range(0, len(stream), chunk_len):
        u = bytes(stream[i:i + chunk_len])
        rec = chunk_compress(comp, u)
        if comp != COMP_NONE and len(rec) >= max_clen:
            rec = u if len(u) >= max_clen else u + bytes(max_clen - len(u))
        offs.append(len(image))
        image += rec + struct.pack(">I", zlib.crc32(rec))
    return bytes(image), offs, zlib.crc32(bytes(image))

def reencode(table, comp, chunk_len, max_clen=0x7FFFFFFF):
    """table.data / table.compression rewritten from table.uncompressed at another compressor and chunk length"""
    image, offs, _ = write_chunks(table.uncompressed, comp, chunk_len, max_clen)
    table.data = image
    table.compression = CompressionMetadata(COMP_NAMES[comp], chunk_len, max_clen, len(table.uncompressed), offs)
    return table

def stream_of(out):
    """the uncompressed stream of a compaction output"""
    c = out.compression
    return read_chunks(out.data, c.chunk_offsets, c.compressor_id, c.chunk_length, c.max_compressed_length, c.data_length)

def hash5(b5: bytes) -> int:
    """LZ4_hash5 of a 64-bit little-endian build, LZ4_HASHLOG 12"""
    return (((int.from_bytes(b5, "little") << 24) & MASK64) * 889523592379 & MASK64) >> 52

def corpus(n, rng):
    """(name, bytes) of length n: the shapes the byU32 regime and the fragment cut change"""
    runs = bytearray()
    while len(runs) < n: runs += bytes([rng.getrandbits(8)]) * rng.randint(1, 3000)
    out = [("incompressible", rng.randbytes(n)), ("runs", bytes(runs[:n]))]
    words = [rng.randbytes(rng.randint(3, 20)) for _ in range(300)]
    out.append(("words", b"".join(rng.choice(words) for _ in range(n // 8 + 2))[:n]))
    # a block repeated at distance d: matchable up to 65535 back, not at 65536 or 65537 (only nearer repeats inside the block remain)
    for d in (65535, 65536, 65537):
        blk = rng.randbytes(4096)
        b = bytearray(rng.randbytes(n))
        for at in range(0, n - d - len(blk), d + 4096 + 777): b[at + d:at + d + len(blk)] = b[at:at + len(blk)]
        out.append(("repeat at %d" % d, bytes(b)))
    # equal 4-byte prefixes with different fifth bytes (a match under the 4-byte key that hash5 keeps apart: for a fixed prefix the fifth
    # byte maps to distinct slots) next to a key of another prefix that shares hash5's slot with one of them (the 4-byte compare refuses it)
    prefix = rng.randbytes(4)
    keys = [prefix + bytes([x]) for x in rng.sample(range(256), 3)]
    other = None
    while other is None:
        k = rng.randbytes(5)
        if k[:4] != prefix and hash5(k) == hash5(keys[0]): other = k
    keys.append(other)
    b = bytearray(rng.randbytes(n))
    at = 0
    while at + 5 < n:
        k = rng.choice(keys); b[at:at + 5] = k; at += 5 + rng.choice([0, 1, 7, 60, 4000, 30000])
    out.append(("hash5 collisions", bytes(b)))
    assert all(len(d) == n for _, d in out)
    return out
