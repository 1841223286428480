"""Plain restatement of the compressed Data.db chunk format, independent of the oracle's and the engine's writers and readers
(test helper). Only the block codec itself (O.chunk_compress / O.chunk_decompress) is shared.

  write_chunks   CompressedSequentialWriter.flushData   S/io/compress/CompressedSequentialWriter.java:140-206
  read_chunks    CompressedChunkReader.readChunk        S/io/util/CompressedChunkReader.java:103-173, :200-230
  ratio_max_clen CompressionParams.calcMaxCompressedLength  S/schema/CompressionParams.java:186-189

A chunk whose compressed length is >= maxCompressedLength is stored raw; a raw chunk shorter than maxCompressedLength (only the file's
last chunk can be) is zero padded up to it. The reader decodes only records shorter than maxCompressedLength and copies the others.
"""
import math, random, struct, zlib
import oracle_lib as O
from cassandra_b200.io.compress import CompressionMetadata
from sstable_builder import Schema, Builder, Partition, Row, Cell

INT32_MAX = 0x7FFFFFFF
COMP_NAMES = {O.COMP_LZ4: "LZ4Compressor", O.COMP_SNAPPY: "SnappyCompressor"}

def ratio_max_clen(chunk_len, ratio):
    """(int) Math.ceil(Math.min(chunkLength / minCompressRatio, Integer.MAX_VALUE)); a ratio of 0 divides to +Infinity"""
    if ratio == 0: return INT32_MAX
    return int(math.ceil(min(chunk_len / ratio, INT32_MAX)))

def compressed_lengths(stream, comp, chunk_len):
    return [len(O.chunk_compress(comp, bytes(stream[i:i + chunk_len]))) for i in range(0, len(stream), chunk_len)]

def write_chunks(stream, comp, chunk_len, max_clen):
    """-> (Data.db image, chunk offsets, Digest.crc32 value)"""
    image = bytearray(); offs = []
    for i in range(0, len(stream), chunk_len):
        u = bytes(stream[i:i + chunk_len])
        rec = O.chunk_compress(comp, u)
        if len(rec) >= max_clen:                                    # :160 compressedLength >= maxCompressedLength
            rec = u if len(u) >= max_clen else u + bytes(max_clen - len(u))      # :163-175 raw, zero padded when shorter
        offs.append(len(image))
        image += rec + struct.pack(">I", zlib.crc32(rec))           # ChecksumWriter.appendDirect: CRC32 of the bytes as written, big-endian
    return bytes(image), offs, zlib.crc32(bytes(image))

class ChunkError(Exception):
    """kind 1: CRC mismatch; kind 2: malformed record (bad bounds, undecodable block, raw record shorter than the chunk)"""
    def __init__(self, chunk, kind):
        super().__init__("chunk %d kind %d" % (chunk, kind)); self.chunk = chunk; self.kind = kind

def read_chunks(image, offsets, comp, chunk_len, max_clen, data_length):
    """-> the uncompressed stream, or ChunkError(chunk, kind) for the first bad chunk"""
    out = bytearray(); n = len(offsets)
    if n != (data_length + chunk_len - 1) // chunk_len: raise ChunkError(0, 2)
    for i, off in enumerate(offsets):
        nxt = offsets[i + 1] if i + 1 < n else len(image)
        if off + 4 > nxt or nxt > len(image): raise ChunkError(i, 2)
        clen = nxt - off - 4
        rec = bytes(image[off:off + clen])
        if zlib.crc32(rec) != struct.unpack(">I", image[off + clen:nxt])[0]: raise ChunkError(i, 1)
        ulen = min(chunk_len, data_length - i * chunk_len)
        if clen < max_clen:                                         # :116 / :219 chunk.length < maxCompressedLength: decode
            try: u = O.chunk_decompress(comp, rec, ulen)
            except ValueError: raise ChunkError(i, 2)
            if len(u) != ulen: raise ChunkError(i, 2)
        else:                                                       # stored raw; the file length bounds what is used of the padding
            if clen < ulen: raise ChunkError(i, 2)
            u = rec[:ulen]
        out += u
    return bytes(out)

def census(image, offsets, max_clen, data_length, chunk_len, stream=None, comp=None):
    """what a written image holds: raw / compressed records, zero-padded short raw records, and (given the stream) chunks whose
    compressed length is exactly max_clen"""
    c = dict(chunks=len(offsets), raw=0, compressed=0, padded=0, boundary=0)
    for i, off in enumerate(offsets):
        clen = (offsets[i + 1] if i + 1 < len(offsets) else len(image)) - off - 4
        ulen = min(chunk_len, data_length - i * chunk_len)
        if clen >= max_clen:
            c["raw"] += 1
            if clen > ulen: c["padded"] += 1
        else: c["compressed"] += 1
    if stream is not None: c["boundary"] = sum(1 for x in compressed_lengths(stream, comp, chunk_len) if x == max_clen)
    return c

def boundary_max_clen(stream, comp, chunk_len, which=None):
    """a max_clen equal to the compressed length of one chunk (`which`, default: the median of the distinct lengths that CompressionParams
    accepts, <= chunk_len), so that the >= boundary is hit exactly: that chunk is stored raw, and some other chunk compresses to fewer bytes"""
    lens = compressed_lengths(stream, comp, chunk_len)
    if which is not None: m = lens[which]
    else:
        ok = sorted({x for x in lens if x <= chunk_len})
        assert len(ok) >= 2, "no two distinct admissible compressed lengths"
        m = ok[len(ok) // 2] if ok[len(ok) // 2] > ok[0] else ok[1]
    assert m <= chunk_len and min(lens) < m
    return m

def replace_record(image, offsets, i, rec):
    """the image with chunk i's record replaced by `rec` and a valid CRC after it -> (image, offsets)"""
    ends = list(offsets[1:]) + [len(image)]
    recs = [bytes(image[a:b]) for a, b in zip(offsets, ends)]
    recs[i] = rec + struct.pack(">I", zlib.crc32(rec))
    offs = [sum(map(len, recs[:k])) for k in range(len(recs))]
    return b"".join(recs), offs

def reencode(table, comp, chunk_len, max_clen):
    """rewrites table.data / table.compression from table.uncompressed; Index.db and Summary.db positions are uncompressed positions"""
    stream = table.uncompressed
    image, offs, _ = write_chunks(stream, comp, chunk_len, max_clen)
    table.data = image
    table.compression = CompressionMetadata(COMP_NAMES[comp], chunk_len, max_clen, len(stream), offs)
    return table

# ---- fixtures: raw and compressed chunks side by side -----------------------------------------------------------------------------------
MIXED = Schema(["LongType"], [("val", "BytesType")])

def mixed_table(seed, nkeys, chunk_len, gen=0, random_share=0.35, tail=None, keyspace=None):
    """a table whose partitions are text that compresses well or random BytesType values that do not. The partition with the largest token
    holds `tail` random bytes (default: a chunk and a half), so the file's last chunk is incompressible, and the tail is sized so that the
    last chunk is short (between a quarter and three quarters of chunk_len)."""
    rng = random.Random(seed)
    keys = [b"key-%05d" % k for k in (keyspace if keyspace is not None else range(nkeys))]
    last = max(keys, key=lambda k: (O.token(k), k))
    parts = []
    for k in keys:
        if k != last and rng.random() < 0.3: continue
        rows = []
        for ck in sorted(rng.sample(range(50), rng.randint(1, 4))):
            v = rng.randbytes(rng.randint(100, 2500)) if rng.random() < random_share else (b"value %s of %d; " % (k, ck)) * rng.randint(4, 120)
            rows.append(Row((struct.pack(">q", ck),), [Cell(0, 1000 + gen, v)], ts=1000 + gen))
        if len(parts) % 40 == 7:                    # runs of text longer than a 64 KiB chunk: chunks that compress more than 8 times
            rows.append(Row((struct.pack(">q", 60),), [Cell(0, 1000 + gen, (b"filler of %s; " % k) * 7000)], ts=1000 + gen))
        parts.append([k, rows])
    tail_len = tail if tail is not None else chunk_len + chunk_len // 2
    tail_bytes = rng.randbytes(tail_len + chunk_len)
    def build(n):
        ps = [Partition(k, rows if k != last else [Row((struct.pack(">q", 99),), [Cell(0, 1000 + gen, tail_bytes[:n])], ts=1000 + gen)]) for k, rows in parts]
        t = Builder(MIXED, (0, 0, 0)).build(ps, chunk_length=chunk_len, generation=gen)
        t.partitions = len(ps); return t
    t = build(tail_len)
    if tail is None:
        r = len(t.uncompressed) % chunk_len
        if not chunk_len // 4 <= r <= 3 * chunk_len // 4:
            t = build(tail_len + (chunk_len // 2 - r) % chunk_len)
        assert chunk_len // 4 - 8 <= len(t.uncompressed) % chunk_len <= 3 * chunk_len // 4 + 8
    return t
