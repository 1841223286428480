"""Chunks of 128 KiB to 1 MiB without a GPU.

K5's compressors for them (cassandra_b200/csrc/codec.cuh: k_compress_chunks_lz4_big over lz4.cuh's byU32 regime, k_snappy_big_fragments +
k_snappy_big_assemble) run on the CPU warp emulator (tests/native/codec_warp_big_host.cc) and must equal liblz4 and Google snappy byte for
byte; the decoders take what those libraries write and refuse damaged blocks; the chunk format (raw storage, short last chunk) is restated
over big chunks; the oracle compacts inputs stored at 128 KiB and 1 MiB into what it makes of the same tables at 64 KiB; chunk lengths above
1 MiB, CRC.db chunks above 64 KiB and non-powers of two are refused."""
import copy, ctypes as C, functools, os, random, shutil, struct, subprocess, zlib, pytest
import oracle_lib as O
import big_chunks as B
from chunk_format import INT32_MAX, ChunkError, read_chunks, ratio_max_clen, mixed_table, census
from cassandra_b200 import native
from cassandra_b200.io.compress import check_chunk_length, CompressionMetadata
from cassandra_b200.db.compaction import CompactionTask, CompactionController

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LZ4_SIZES = (65546, 65547, 65548, 128 << 10, 256 << 10, 1 << 20)
SNAPPY_SIZES = (65535, 65536, 65537, 3 * 65536 + 1, 1 << 20)

@pytest.fixture(scope="module")
def warp():
    if shutil.which("g++") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"): pytest.skip("needs g++ and the CUDA headers")
    out = os.path.join(ROOT, "tests", "native", "_build", "libcodecwarpbig.so")
    src = os.path.join(ROOT, "tests", "native", "codec_warp_big_host.cc")
    deps = [src, os.path.join(ROOT, "tests", "native", "warp_emu.h")] + [os.path.join(ROOT, "cassandra_b200", "csrc", f) for f in ("lz4.cuh", "snappy.cuh", "snappy_chain.cuh", "lz4_chain.cuh", "common.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        r = subprocess.run(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-fno-strict-aliasing", "-I/usr/local/cuda/include", "-Wno-attributes",
                            "-Wno-unknown-pragmas", "-o", out, src], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(out)
    L.warp_lz4_big.restype = C.c_int; L.warp_lz4_big.argtypes = [C.c_char_p, C.c_int, C.c_void_p]
    L.warp_snappy_big.restype = C.c_int; L.warp_snappy_big.argtypes = [C.c_int, C.c_char_p, C.c_int, C.c_void_p]
    return L

def need_liblz4():
    if B.liblz4() is None: pytest.skip("no system liblz4")

def cases(sizes, seed, big_cap):
    """the corpus at every size; at sizes above big_cap only the shapes that the emulator runs through quickly"""
    rng = random.Random(seed)
    for n in sizes:
        for name, d in B.corpus(n, rng):
            if n <= big_cap or name in ("incompressible", "runs", "repeat at 65535", "hash5 collisions"): yield n, name, d

@functools.lru_cache(None)
def lz4_cases(): return list(cases(LZ4_SIZES, 0xB16, 256 << 10))

@functools.lru_cache(None)
def snappy_cases(): return list(cases(SNAPPY_SIZES, 0x5B16, 3 * 65536 + 1))

def test_lz4_big_warp_source_equals_liblz4(warp):
    need_liblz4()
    for n, name, d in lz4_cases():
        out = C.create_string_buffer(n + n // 255 + 64)
        k = warp.warp_lz4_big(d, n, out)
        assert out.raw[:k] == B.lz4_block(d), (n, name)

def test_snappy_fragments_warp_source_equal_snappy(warp):
    pa = pytest.importorskip("pyarrow")
    if not pa.Codec.is_available("snappy"): pytest.skip("pyarrow built without snappy")
    for n, name, d in snappy_cases():
        out = C.create_string_buffer(n + n // 6 + 64)
        k = warp.warp_snappy_big(15, d, n, out)
        assert out.raw[:k] == B.snappy15(d) == O.chunk_compress(O.COMP_SNAPPY15, d), (n, name, "2^15")
        k = warp.warp_snappy_big(14, d, n, out)
        assert out.raw[:k] == O.chunk_compress(O.COMP_SNAPPY, d), (n, name, "2^14")

def test_decoders_round_trip_big_blocks_and_refuse_damage():
    need_liblz4()
    for n, name, d in lz4_cases():
        blk = B.lz4_block(d)
        assert O.lz4_decompress(blk, n) == d, (n, name)
    for n, name, d in snappy_cases():
        for comp in (O.COMP_SNAPPY, O.COMP_SNAPPY15):
            assert O.chunk_decompress(comp, O.chunk_compress(comp, d), n) == d, (n, name, comp)
    rng = random.Random(3); n = 256 << 10
    d = b"".join(rng.randbytes(rng.randint(1, 40)) * rng.randint(1, 9) for _ in range(40000))[:n]
    # LZ4: a match whose offset reaches before the start of the output; more output than the chunk holds
    lit = rng.randbytes(20)
    before = bytes([0x40 | 0x0]) + lit[:4] + struct.pack("<H", 5) + bytes([0x50]) + lit[:5]
    with pytest.raises(ValueError): O.lz4_decompress(before, 64)
    blk = B.lz4_block(d)
    with pytest.raises(ValueError): O.lz4_decompress(blk, n - 1)
    # Snappy: a varint that disagrees with the chunk (one more, one fewer byte than the fragments decode to)
    s = O.chunk_compress(O.COMP_SNAPPY, d)
    v = bytearray(); x = n + 1
    while x >= 0x80: v.append((x & 0x7f) | 0x80); x >>= 7
    v.append(x)
    hdr = 3                                                  # 262144 takes three varint bytes
    with pytest.raises(ValueError): O.chunk_decompress(O.COMP_SNAPPY, bytes(v) + s[hdr:], n + 1)
    with pytest.raises(ValueError): O.chunk_decompress(O.COMP_SNAPPY, s, n - 1)

@pytest.mark.parametrize("comp", [O.COMP_LZ4, O.COMP_SNAPPY, B.COMP_NONE])
@pytest.mark.parametrize("L", [128 << 10, 1 << 20])
def test_chunk_format_with_big_chunks(comp, L):
    """flushData's raw rule at a finite maxCompressedLength and a short last chunk: written and read back through the restatement"""
    if comp == O.COMP_LZ4: need_liblz4()
    rng = random.Random(L + comp)
    words = [rng.randbytes(rng.randint(3, 20)) for _ in range(200)]
    parts = []
    for k in range(7):                                       # compressible and incompressible chunks, then a short random last one
        parts.append(b"".join(rng.choice(words) for _ in range(L // 8))[:L] if k % 2 == 0 else rng.randbytes(L))
    stream = b"".join(parts) + rng.randbytes(L // 3)
    last = len(B.chunk_compress(comp, stream[len(stream) // L * L:]))     # a max_clen the short random last chunk reaches exactly: stored raw, padded
    for max_clen in (INT32_MAX, ratio_max_clen(L, 1.1), last):
        image, offs, digest = B.write_chunks(stream, comp, L, max_clen)
        assert digest == zlib.crc32(image) and len(offs) == (len(stream) + L - 1) // L
        assert read_chunks(image, offs, comp, L, max_clen, len(stream)) == stream
        c = census(image, offs, max_clen, len(stream), L)
        if comp != B.COMP_NONE and max_clen != INT32_MAX: assert c["raw"] >= 3 and c["compressed"] >= 3 and c["padded"] == (max_clen == last), c
        damaged = bytearray(image); damaged[offs[5] + 100] ^= 1
        with pytest.raises(ChunkError) as e: read_chunks(bytes(damaged), offs, comp, L, max_clen, len(stream))
        assert (e.value.chunk, e.value.kind) == (5, 1)

def test_unsupported_chunk_lengths_stay_refused():
    for L in (1 << 10, 64 << 10, 128 << 10, 256 << 10, 512 << 10, 1 << 20): check_chunk_length(L)
    for L in (0, -65536, 3 * 65536, 65536 + 16, 2 << 20, 4 << 20):
        with pytest.raises(native.UnsupportedError): check_chunk_length(L)
    check_chunk_length(65536, uncompressed=True)
    with pytest.raises(native.UnsupportedError): check_chunk_length(128 << 10, uncompressed=True)
    t = mixed_table(0xB1, 40, 16384)
    for L in (2 << 20, 3 * 65536):
        with pytest.raises(native.UnsupportedError):
            CompactionTask([t], CompactionController(1700000000), compression=CompressionMetadata("LZ4Compressor", L, INT32_MAX, 0, [])).build_manifest()

# ---- the oracle over inputs stored at big chunks ------------------------------------------------------------------------------------------
KEYS = range(120)

@functools.lru_cache(None)
def tables():
    return tuple(mixed_table(0xB60 + g, 0, 16384, gen=g, keyspace=KEYS) for g in range(3))

def restored(layout):
    return [B.reencode(copy.copy(t), comp, L) for t, (comp, L) in zip(tables(), layout)]

@pytest.mark.parametrize("layout", [
    ((O.COMP_LZ4, 128 << 10),) * 3, ((O.COMP_LZ4, 1 << 20),) * 3, ((O.COMP_SNAPPY, 128 << 10),) * 3, ((O.COMP_SNAPPY, 1 << 20),) * 3,
    ((B.COMP_NONE, 1 << 20),) * 3, ((O.COMP_LZ4, 16384), (O.COMP_SNAPPY, 1 << 20), (B.COMP_NONE, 128 << 10))],
    ids=["lz4-128k", "lz4-1m", "snappy-128k", "snappy-1m", "noop-1m", "mixed"])
@pytest.mark.parametrize("lcs", [False, True], ids=["one-file", "lcs"])
def test_oracle_compacts_big_chunk_inputs_as_at_64k(layout, lcs):
    need_liblz4()
    out = CompressionMetadata("SnappyCompressor", 65536, INT32_MAX, 0, [])
    kw = dict(max_sstable_bytes=60000) if lcs else {}
    def run(tabs): return CompactionTask(tabs, CompactionController(1700000000), compression=out, **kw).execute(O.OracleEngine(), max_outputs=64 if lcs else None).outputs
    want = run(restored(((O.COMP_LZ4, 65536),) * 3))
    got = run(restored(layout))
    assert len(got) == len(want) and (len(want) > 1) == lcs
    for g, w in zip(got, want):
        assert B.stream_of(g) == B.stream_of(w) and g.index == w.index and g.data == w.data
