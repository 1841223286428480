"""GPU parity for chunks of 128 KiB to 1 MiB (chunk_length_in_kb 128 to 1024): K5's big-chunk kernels (LZ4 in liblz4's byU32 regime, Snappy
one warp per 64 KiB fragment, Noop), K1's warp decoder over big chunks, and the codec entry points.

The reference of a compaction is the oracle's merged stream and Index.db (written at 64 KiB: both are independent of the chunk length) with
Data.db, the chunk offsets and the digest restated over liblz4 / Google snappy (tests/big_chunks.py). Every output must equal it byte for
byte on the host engine, the host engine cut into five token-range pieces, the device-resident engine, a device engine whose buffers sit
behind guard patterns, in token shards and under every K1 / K5 switch value."""
import copy, functools, os, struct, zlib, pytest
import numpy as np
import oracle_lib as O
import big_chunks as B
from chunk_format import INT32_MAX, ratio_max_clen, mixed_table, census
from test_gpu_compaction import DeviceEngine
from test_gpu_compression_params import PoisonedDeviceEngine
from cassandra_b200 import native
from cassandra_b200.io.compress import CompressionMetadata, LZ4Compressor, SnappyCompressor
from cassandra_b200.db.compaction import CompactionTask, CompactionController, GpuEngine

pytestmark = pytest.mark.gpu
NOW = 1700000000
KEYS = range(700)
KiB, MiB = 1 << 10, 1 << 20

@pytest.fixture(scope="module")
def ctx():
    if B.liblz4() is None: pytest.skip("no system liblz4")
    c = native.Context(0)
    yield c
    c.close()

def params(comp, L, max_clen=INT32_MAX): return CompressionMetadata(B.COMP_NAMES[comp], L, max_clen, 0, [])

def run(tables, engine, compression, **kw):
    return CompactionTask(tables, CompactionController(NOW), compression=compression, **kw).execute(engine, max_outputs=64 if kw.get("max_sstable_bytes") else None)

@functools.lru_cache(None)
def base_tables():
    """three overlapping tables of a few MiB each: compressible text, random values and 140 KiB text runs; the merged stream ends with the newest
    table's 1.5 MiB random value (chunks stored raw under a finite maxCompressedLength, a short last chunk)"""
    return tuple(mixed_table(0xB16C + g, 0, 16384, gen=g, tail=3 * MiB // 2 + 777, keyspace=KEYS) for g in range(3))

def tables(layout):
    return [B.reencode(copy.copy(t), comp, L) for t, (comp, L) in zip(base_tables(), layout)]

def expected(tabs, out, **kw):
    """the oracle's compaction, its chunks rewritten at the output's compressor, chunk length and maxCompressedLength"""
    w = run(tabs, O.OracleEngine(), params(O.COMP_LZ4, 65536), **kw)
    want = []
    for o in w.outputs:
        s = B.stream_of(o)
        image, offs, digest = B.write_chunks(s, out.compressor_id, out.chunk_length, out.max_compressed_length)
        want.append((o, s, image, offs, digest))
    return w, want

def same(got, ref, name):
    w, want = ref
    assert len(got.outputs) == len(want) >= 1, name
    for g, (o, s, image, offs, digest) in zip(got.outputs, want):
        assert g.compression.data_length == len(s) and g.index == o.index, name
        assert g.data == image and g.compression.chunk_offsets == offs and g.digest == digest == zlib.crc32(g.data), name
        assert g.partitions == o.partitions and g.rows == o.rows, name
        if o.filter is not None:
            assert g.filter == o.filter and g.summary == o.summary and (g.first_key, g.last_key) == (o.first_key, o.last_key), name
            for k in o.stats: assert g.stats[k] == o.stats[k], (name, k)
    for k in ("bytes_read", "bytes_in_range", "bytes_written", "total_source_rows", "merged_row_counts"):
        assert got.stats[k] == w.stats[k], (name, k)

def engines(ctx):
    return [("host", GpuEngine(ctx), {}), ("host pieces", GpuEngine(ctx), {"B200C_RANGES": "5"}), ("device", DeviceEngine(ctx), {}),
            ("poisoned device", PoisonedDeviceEngine(ctx), {})]

def on_every_engine(ctx, monkeypatch, tabs, out, **kw):
    ref = expected(tabs, out, **kw)
    for name, eng, env in engines(ctx):
        for k, v in env.items(): monkeypatch.setenv(k, v)
        try: same(run(tabs, eng, out, **kw), ref, name)
        finally:
            for k in env: monkeypatch.delenv(k)
    return ref

LAYOUTS = {"lz4 1m": ((O.COMP_LZ4, MiB),) * 3, "snappy 256k": ((O.COMP_SNAPPY, 256 * KiB),) * 3,
           "mixed": ((O.COMP_LZ4, 16 * KiB), (O.COMP_SNAPPY, MiB), (B.COMP_NONE, 128 * KiB))}
OUTS = {"lz4 256k": params(O.COMP_LZ4, 256 * KiB), "lz4 1m": params(O.COMP_LZ4, MiB), "snappy 128k": params(O.COMP_SNAPPY, 128 * KiB),
        "snappy 1m": params(O.COMP_SNAPPY, MiB), "noop 1m": params(B.COMP_NONE, MiB), "lz4 16k": params(O.COMP_LZ4, 16 * KiB)}

@pytest.mark.parametrize("layout,out", [("lz4 1m", "lz4 1m"), ("lz4 1m", "snappy 128k"), ("snappy 256k", "lz4 256k"), ("mixed", "snappy 1m"),
                                        ("mixed", "noop 1m"), ("mixed", "lz4 16k"), ("lz4 1m", "lz4 16k")])
def test_big_chunks_on_every_engine(ctx, monkeypatch, layout, out):
    on_every_engine(ctx, monkeypatch, tables(LAYOUTS[layout]), OUTS[out])

def test_side_band_with_big_chunks(ctx):
    tabs = tables(LAYOUTS["mixed"])
    same(run(tabs, GpuEngine(ctx), OUTS["lz4 1m"], with_metadata=True), expected(tabs, OUTS["lz4 1m"], with_metadata=True), "side band")

def test_raw_stored_big_chunks(ctx, monkeypatch):
    """finite maxCompressedLength at big output chunks: random chunks stored raw, the short last one zero padded"""
    tabs = tables(LAYOUTS["mixed"])
    for comp, L in ((O.COMP_LZ4, 128 * KiB), (O.COMP_SNAPPY, 256 * KiB)):
        for max_clen in (ratio_max_clen(L, 1.1), L - 1):
            out = params(comp, L, max_clen)
            w, want = on_every_engine(ctx, monkeypatch, tabs, out)
            o, s, image, offs, _ = want[0]
            c = census(image, offs, max_clen, len(s), L)
            assert c["raw"] >= 1 and c["compressed"] >= 1, (comp, L, max_clen, c)
    # inputs whose own chunks are stored raw
    raw_in = [B.reencode(copy.copy(t), O.COMP_LZ4, 256 * KiB, ratio_max_clen(256 * KiB, 1.1)) for t in base_tables()]
    assert any(census(t.data, t.compression.chunk_offsets, t.compression.max_compressed_length, t.compression.data_length, 256 * KiB)["raw"] for t in raw_in)
    on_every_engine(ctx, monkeypatch, raw_in, OUTS["lz4 1m"])

def test_token_shards_with_big_chunks(ctx):
    tabs = tables(LAYOUTS["mixed"])
    cuts = [-(1 << 63), -(1 << 62) - 12345, -7, (1 << 62) + 99, (1 << 63) - 1]
    for lo, hi in zip(cuts, cuts[1:]):
        ref = expected(tabs, OUTS["lz4 256k"], token_range=(lo, hi))
        for name, eng in (("host", GpuEngine(ctx)), ("device", DeviceEngine(ctx))):
            same(run(tabs, eng, OUTS["lz4 256k"], token_range=(lo, hi)), ref, (name, lo, hi))

@pytest.mark.parametrize("out", ["lz4 256k", "snappy 128k", "noop 1m"])
def test_lcs_files_with_big_chunks(ctx, out):
    """multi-file output: the files cut the merged stream into whole partitions, each file's Data.db is its stream written at the output's
    chunks, and the cut does not depend on how the inputs were stored"""
    p = OUTS[out]
    one = B.stream_of(expected(tables(LAYOUTS["mixed"]), p)[0].outputs[0])
    res = {}
    for layout in ("mixed", "lz4 1m"):
        got = run(tables(LAYOUTS[layout]), GpuEngine(ctx), p, max_sstable_bytes=3 * p.chunk_length // 2)
        assert len(got.outputs) > 1, layout
        streams = []
        for g in got.outputs:
            s = B.stream_of(g); streams.append(s)
            image, offs, digest = B.write_chunks(s, p.compressor_id, p.chunk_length, p.max_compressed_length)
            assert g.data == image and g.compression.chunk_offsets == offs and g.digest == digest, layout
        assert b"".join(streams) == one, layout
        res[layout] = [(g.data, g.index) for g in got.outputs]
    assert res["mixed"] == res["lz4 1m"]

def test_damaged_big_chunk_is_reported_like_a_small_one(ctx):
    """a flipped byte in chunk k of a 256 KiB-chunk input: (input, kind 1, chunk k) and the offset a 64 KiB-chunk input reports"""
    for L in (256 * KiB, 64 * KiB):
        tabs = tables(((O.COMP_LZ4, L),) * 3)
        k = len(tabs[1].compression.chunk_offsets) - 2
        d = bytearray(tabs[1].data); d[tabs[1].compression.chunk_offsets[k] + 77] ^= 0x10; tabs[1].data = bytes(d)
        with pytest.raises(native.CorruptSSTableError) as e: run(tabs, GpuEngine(ctx), OUTS["lz4 1m"])
        c = e.value.corruption
        assert (c.input, c.kind, c.chunk) == (1, 1, k), L
        if L == 64 * KiB: assert c.offset == big_offset
        big_offset = c.offset
        with pytest.raises(native.CorruptSSTableError) as e2: run(tabs, DeviceEngine(ctx), OUTS["lz4 1m"])
        assert (e2.value.corruption.input, e2.value.corruption.kind, e2.value.corruption.chunk) == (1, 1, k)
        with pytest.raises(native.CorruptSSTableError) as e3:
            ctx.decompress_chunks(O.COMP_LZ4, tabs[1].data, tabs[1].compression.chunk_offsets, tabs[1].compression.data_length, L)
        assert (e3.value.corruption.kind, e3.value.corruption.chunk) == (1, k)

# ---- codec entry points ------------------------------------------------------------------------------------------------------------------------
def codec_stream(seed, n):
    rng = np.random.default_rng(seed)
    words = [rng.bytes(int(rng.integers(3, 20))) for _ in range(300)]
    parts, size = [], 0
    while size < n:
        p = rng.bytes(int(rng.integers(1000, 200000))) if rng.random() < 0.3 else b"".join(words[i] for i in rng.integers(0, 300, 20000))
        parts.append(p); size += len(p)
    return b"".join(parts)[:n]

@pytest.mark.parametrize("comp", [O.COMP_LZ4, O.COMP_SNAPPY, O.COMP_SNAPPY15, B.COMP_NONE])
@pytest.mark.parametrize("L", [128 * KiB, 256 * KiB, MiB])
def test_codec_chunks_equal_the_libraries(ctx, comp, L):
    stream = codec_stream(L + comp, 5 * L + L // 3 + 7)
    for max_clen in (INT32_MAX, ratio_max_clen(L, 1.1)):
        image, offs, digest = ctx.compress_chunks(comp, stream, L, max_clen)
        want_image, want_offs, want_digest = B.write_chunks(stream, comp, L, max_clen)
        if comp == O.COMP_SNAPPY15: assert all(B.snappy15(stream[i:i + L]) == O.chunk_compress(O.COMP_SNAPPY15, stream[i:i + L]) for i in range(0, len(stream), L))
        assert image == want_image and list(offs) == want_offs and digest == want_digest, max_clen
        assert ctx.decompress_chunks(comp, image, offs, len(stream), L, max_clen) == stream

def test_single_buffer_codec_at_big_lengths(ctx):
    import random
    rng = random.Random(0x51B)
    for n in (65535, 65536, 65537, 65546, 65547, 65548, 3 * 65536 + 1, 128 * KiB, 256 * KiB, MiB):
        for name, d in B.corpus(n, rng):
            lz = LZ4Compressor(ctx); sn = SnappyCompressor(ctx)
            c = lz.compress(d)
            assert c == struct.pack("<I", n) + B.lz4_block(d), (n, name)
            assert lz.uncompress(c, n) == d, (n, name)
            c = sn.compress(d)
            assert c == O.chunk_compress(O.COMP_SNAPPY, d), (n, name)
            assert sn.uncompress(c, n) == d, (n, name)
        L = native.lib()
        assert L.b200c_initial_compressed_buffer_length(O.COMP_LZ4, n) == 4 + n + n // 255 + 16
        assert L.b200c_initial_compressed_buffer_length(O.COMP_SNAPPY, n) == 32 + n + n // 6
    assert native.lib().b200c_compress_bound(O.COMP_LZ4, 3 * MiB, MiB) >= 3 * (4 + MiB + MiB // 255 + 16 + 4)

def test_lengths_above_1mib_stay_refused(ctx):
    stream = codec_stream(5, 3 * MiB)
    for L in (2 * MiB, 3 * 65536):
        with pytest.raises(native.UnsupportedError): ctx.compress_chunks(O.COMP_LZ4, stream, L)
    with pytest.raises(native.UnsupportedError): ctx.compress_chunks(native.COMP_UNCOMPRESSED, stream, 128 * KiB)
    with pytest.raises(native.UnsupportedError): LZ4Compressor(ctx).compress(stream[:MiB + 1])
    tabs = tables(((O.COMP_LZ4, 16 * KiB),) * 3)
    with pytest.raises(native.UnsupportedError): run(tabs, GpuEngine(ctx), params(O.COMP_LZ4, 2 * MiB))

# ---- every switch value ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("env", [{"B200C_K1": "0", "B200C_K1_BATCH": "0"}, {"B200C_K1_BATCH": "2"}, {"B200C_K1": "2", "B200C_K1_BATCH": "2"},
                                 {"B200C_K5": "0"}, {"B200C_K5": "1"}, {"B200C_K5": "2"}, {"B200C_K5": "3"}])
def test_every_switch_value(env):
    """big chunks take their own kernels whatever a switch says, and the output may not depend on it; the switches are read once per process,
    so the compaction tests of this file run in a subprocess per setting"""
    import subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "tests/test_gpu_big_chunks.py", "-k", "every_engine or raw_stored or lcs"],
                       cwd=root, env=dict(os.environ, **env), capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]
