"""GPU parity for tables whose compression is disabled (Data.db + CRC.db: k_raw_ingest in K1, k_raw_checksum in K5) and for
NoopCompressor. Every compaction is compared byte for byte (Data, Index, CRC table or chunk offsets, digest, counters) with the oracle
composition that tests/test_oracle_uncompressed.py pins, on the host engine, the host engine cut into five token-range pieces, the
device-resident engine and a device engine whose buffers sit at 16- but not 32-byte aligned addresses behind a guard pattern."""
import ctypes as C, os, zlib, pytest
import numpy as np
import oracle_lib as O
from crc_component import write_crc, crc_entries, UncompressedOracle, DEFAULT_CHUNK
from test_oracle_uncompressed import (params, run, plain, encode, check_output, short_last, base_tables, golden, mixed_inputs, lcs_limits,
                                      corrupt_cases, growth_tables, SETTINGS, UNC)
from test_gpu_compaction import DeviceEngine
from test_gpu_compression_params import PoisonedDeviceEngine
from cassandra_b200 import native
from cassandra_b200.io.compress import uncompressed_params, write_uncompressed, read_uncompressed
from cassandra_b200.io.sstable import SSTable
from cassandra_b200.db.compaction import GpuEngine

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def ctx():
    c = native.Context(0)
    yield c
    c.close()

def engines(ctx):
    return [("host", GpuEngine(ctx), {}), ("host pieces", GpuEngine(ctx), {"B200C_RANGES": "5"}), ("device", DeviceEngine(ctx), {}),
            ("poisoned device", PoisonedDeviceEngine(ctx), {})]

def same(got, want, name, rows=True):
    assert len(got.outputs) == len(want.outputs) >= 1, name
    for g, w in zip(got.outputs, want.outputs):
        assert g.data == w.data and g.index == w.index, name
        assert g.compression.chunk_offsets == w.compression.chunk_offsets and g.compression.data_length == w.compression.data_length, name
        assert g.digest == w.digest == zlib.crc32(g.data), name
        assert g.partitions == w.partitions and (not rows or g.rows == w.rows), name
        if w.filter is not None:
            assert g.filter == w.filter and g.summary == w.summary and (g.first_key, g.last_key) == (w.first_key, w.last_key), name
            for k in w.stats: assert g.stats[k] == w.stats[k], (name, k)
    for k in ("bytes_read", "bytes_in_range", "bytes_written", "total_source_rows", "merged_row_counts"):
        assert got.stats[k] == want.stats[k], (name, k)

def on_every_engine(ctx, monkeypatch, tables, compression, rows=True, **kw):
    want = run(tables, UncompressedOracle(), compression, **kw)
    for name, eng, env in engines(ctx):
        for k, v in env.items(): monkeypatch.setenv(k, v)
        try: same(run(tables, eng, compression, **kw), want, name, rows)
        finally:
            for k in env: monkeypatch.delenv(k)
    return want

# ---- codec entry points -----------------------------------------------------------------------------------------------------------------------
def dev_codec(ctx, stream, chunk_len, crcs=None):
    """b200c_compress_chunks / b200c_decompress_chunks(UNCOMPRESSED) on device pointers -> (Data.db, CRC entries, digest, stream read back)"""
    L = native.lib(); allocs = []
    def alloc(n):
        d = C.c_void_p(); ctx.check(L.b200c_dev_alloc(ctx.handle, max(n, 1), C.byref(d))); allocs.append(d); return d
    try:
        n = len(stream); nch = L.b200c_chunk_count(n, chunk_len)
        assert L.b200c_compress_bound(UNC, n, chunk_len) == n
        d_in, d_out, d_crc, d_back = alloc(n), alloc(n), alloc((nch + 1) * 8), alloc(n)
        ctx.check(L.b200c_memcpy_h2d(ctx.handle, d_in, stream, n))
        out_len = C.c_uint64(); dig = C.c_uint32()
        ctx.check(L.b200c_compress_chunks(ctx.handle, UNC, d_in, n, chunk_len, 0, d_out, n, C.byref(out_len), d_crc, C.byref(dig), native.FLAG_DEVICE_PTRS))
        assert out_len.value == n
        data = C.create_string_buffer(max(n, 1)); tab = (C.c_uint64 * max(nch, 1))()
        ctx.check(L.b200c_memcpy_d2h(ctx.handle, data, d_out, n)); ctx.check(L.b200c_memcpy_d2h(ctx.handle, tab, d_crc, nch * 8))
        if crcs is not None:
            t = np.asarray(crcs, dtype=np.uint64); ctx.check(L.b200c_memcpy_h2d(ctx.handle, d_crc, t.ctypes.data, nch * 8))
        where = native.Corruption()
        rc = L.b200c_decompress_chunks(ctx.handle, UNC, d_out, n, d_crc, nch, chunk_len, 0, n, d_back, 1, C.byref(where), native.FLAG_DEVICE_PTRS)
        if rc == native.ECORRUPT: return data.raw[:n], list(tab)[:nch], dig.value, where
        ctx.check(rc)
        back = C.create_string_buffer(max(n, 1)); ctx.check(L.b200c_memcpy_d2h(ctx.handle, back, d_back, n))
        return data.raw[:n], list(tab)[:nch], dig.value, back.raw[:n]
    finally:
        for d in allocs: L.b200c_dev_free(ctx.handle, d)

def codec_stream(seed, n):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()

@pytest.mark.parametrize("chunk_len", [16, 1024, 4096, 16384, 65536])
def test_codec_is_the_checksummed_writer(ctx, chunk_len):
    for n in (0, 1, 15, chunk_len - 1, chunk_len, 3 * chunk_len, 5 * chunk_len + chunk_len // 3 + 7, 700_001):
        s = codec_stream(n + chunk_len, n)
        _, crcs, digest = write_crc(s, chunk_len)
        assert ctx.compress_chunks(UNC, s, chunk_len) == (s, crcs, digest), (chunk_len, n)
        assert ctx.decompress_chunks(UNC, s, crcs, n, chunk_len) == s, (chunk_len, n)
        assert dev_codec(ctx, s, chunk_len) == (s, crcs, digest, s), ("device", chunk_len, n)
        if n % chunk_len == 0 and n: assert len(crcs) == n // chunk_len          # no empty trailing entry at an exact multiple
    data, crc_db, dg = write_uncompressed(ctx, s, chunk_len)
    assert read_uncompressed(ctx, data, crc_db) == s and dg == str(zlib.crc32(s))

def test_codec_many_chunks_and_damage(ctx):
    """33 000 chunks of 1 KiB in one call (the last 1021 bytes); a flipped byte is (0, kind 1, chunk, chunk * L) on host and device pointers"""
    L = 1024; s = codec_stream(5, 32999 * L + 1021)
    _, crcs, digest = write_crc(s, L)
    assert len(crcs) == 33000
    assert ctx.compress_chunks(UNC, s, L) == (s, crcs, digest)
    assert dev_codec(ctx, s, L) == (s, crcs, digest, s)
    for pos in (1234567, len(s) - 3):
        bad = bytearray(s); bad[pos] ^= 1; bad = bytes(bad)
        with pytest.raises(native.CorruptSSTableError) as e:
            ctx.decompress_chunks(UNC, bad, crcs, len(s), L)
        c = e.value.corruption; assert (c.input, c.kind, c.chunk, c.offset) == (0, 1, pos // L, pos // L * L)
        *_, where = dev_codec(ctx, bad, L, crcs)
        assert (where.kind, where.chunk, where.offset) == (1, pos // L, pos // L * L)

def test_codec_refusals(ctx):
    L = native.lib()
    with pytest.raises(native.B200CError) as e: ctx.decompress_chunks(UNC, b"x" * 100, [0], 100, 64)      # 2 chunks, 1 entry
    assert e.value.code == native.EINVAL
    out = C.create_string_buffer(64)
    assert L.b200c_compress(ctx.handle, UNC, b"abc", 3, out, 64) == native.EINVAL
    assert L.b200c_uncompress(ctx.handle, UNC, b"abc", 3, out, 64) == native.EINVAL

# ---- compactions --------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["legacy_oa_simple", "legacy_oa_clust"])
def test_golden_uncompressed(ctx, monkeypatch, name):
    base = golden(name)
    t = SSTable.open(base); u = encode(t, UNC, DEFAULT_CHUNK)
    want = on_every_engine(ctx, monkeypatch, [u], uncompressed_params(), column_index_size=4096)
    assert want.outputs[0].data == plain(t) and want.outputs[0].index == open(base + "Index.db", "rb").read()

def test_every_input_and_output_setting(ctx, monkeypatch):
    tabs = base_tables()
    ref = run([encode(t, UNC, DEFAULT_CHUNK) for t in tabs], UncompressedOracle(), uncompressed_params()).outputs[0]
    for iname, ic, il in SETTINGS:
        ins = [encode(t, ic, il) for t in tabs]
        for oname, oc, ol in SETTINGS:
            if UNC not in (ic, oc) and native.COMP_NONE not in (ic, oc): continue        # (the compressed pairs: test_gpu_compression_params)
            want = on_every_engine(ctx, monkeypatch, ins, params(oc, ol))
            o = want.outputs[0]
            assert plain(o) == ref.data and o.index == ref.index, (iname, oname)
            if oc == UNC: check_output(o, ol)
            assert short_last(len(ref.data), ol)

def test_mixed_inputs(ctx, monkeypatch):
    ins = mixed_inputs()
    for L in (4096, 16384, 65536):
        o = on_every_engine(ctx, monkeypatch, ins, uncompressed_params(L)).outputs[0]
        check_output(o, L)
    on_every_engine(ctx, monkeypatch, ins, params(O.COMP_LZ4, 16384))
    on_every_engine(ctx, monkeypatch, ins, params(native.COMP_NONE, 4096))

class TooSmallCounter:
    """an engine that counts the calls it saw fail with B200C_ETOOSMALL (CompactionTask.execute then retries with the reported sizes)"""
    def __init__(self, eng): self.eng = eng; self.needs_lib_bound = eng.needs_lib_bound; self.too_small = 0
    def __call__(self, manifest, result):
        try: self.eng(manifest, result)
        except native.B200CError as e:
            if e.code == native.ETOOSMALL: self.too_small += 1
            raise

def test_output_longer_than_the_inputs(ctx, monkeypatch):
    """inputs whose headers' minimum timestamps differ by 1e11: the uncompressed output is longer than the inputs together, so buffers sized
    from the inputs are too small; the engine reports the sizes it needs and the second call matches the oracle"""
    ins = [encode(t, UNC, 4096) for t in growth_tables()]
    total_in = sum(len(t.data) for t in ins)
    want = on_every_engine(ctx, monkeypatch, ins, uncompressed_params())
    assert len(want.outputs[0].data) > total_in + 1024
    for name, eng, env in engines(ctx):
        for k, v in env.items(): monkeypatch.setenv(k, v)
        try:
            counted = TooSmallCounter(eng)
            same(run(ins, counted, uncompressed_params()), want, name)
            assert counted.too_small == 1, name
        finally:
            for k in env: monkeypatch.delenv(k)
    same(run(ins, GpuEngine(ctx), uncompressed_params(), max_sstable_bytes=len(want.outputs[0].data) // 3),
         run(ins, UncompressedOracle(), uncompressed_params(), max_sstable_bytes=len(want.outputs[0].data) // 3), "lcs", rows=False)

def test_token_shards_concatenate(ctx):
    tabs = [encode(t, UNC, DEFAULT_CHUNK) for t in base_tables()]
    whole = run(tabs, GpuEngine(ctx), uncompressed_params()).outputs[0]
    a = run(tabs, GpuEngine(ctx), uncompressed_params(), token_range=(-(1 << 63), 0)).outputs[0]
    b = run(tabs, GpuEngine(ctx), uncompressed_params(), token_range=(0, (1 << 63) - 1)).outputs[0]
    assert a.data + b.data == whole.data and a.partitions + b.partitions == whole.partitions
    for o in (a, b, whole): check_output(o)
    for o, tr in ((a, (-(1 << 63), 0)), (b, (0, (1 << 63) - 1))):
        same(run(tabs, GpuEngine(ctx), uncompressed_params(), token_range=tr), run(tabs, UncompressedOracle(), uncompressed_params(), token_range=tr), "shard")

def test_lcs_files(ctx, monkeypatch):
    tabs = [encode(t, UNC, DEFAULT_CHUNK) for t in base_tables()]
    whole = run(tabs, UncompressedOracle(), uncompressed_params()).outputs[0]
    _, cases = lcs_limits(whole.data, whole.index)
    for limit, end0 in cases:
        want = on_every_engine(ctx, monkeypatch, tabs, uncompressed_params(), rows=False, max_sstable_bytes=limit)
        assert len(want.outputs) >= 2 and len(want.outputs[0].data) == end0
        assert any(short_last(len(o.data), DEFAULT_CHUNK) for o in want.outputs)
        got = run(tabs, GpuEngine(ctx), uncompressed_params(), max_sstable_bytes=limit)
        assert sum(o.rows for o in got.outputs) == whole.rows
    ins = [encode(t, O.COMP_LZ4, 16384) for t in base_tables()]          # compressed inputs into uncompressed LCS files
    same(run(ins, GpuEngine(ctx), uncompressed_params(), max_sstable_bytes=cases[0][0]),
         run(ins, UncompressedOracle(), uncompressed_params(), max_sstable_bytes=cases[0][0]), "lz4 in", rows=False)

def test_metadata_side_band(ctx):
    """Filter / Summary / Statistics of an uncompressed single output equal those of the LZ4-output run"""
    tabs = [encode(t, UNC, DEFAULT_CHUNK) for t in base_tables()]
    lz4 = run(tabs, GpuEngine(ctx), params(O.COMP_LZ4, 16384), with_metadata=True).outputs[0]
    for eng in (GpuEngine(ctx), DeviceEngine(ctx)):
        o = run(tabs, eng, uncompressed_params(), with_metadata=True).outputs[0]
        assert o.filter == lz4.filter and o.summary == lz4.summary and (o.first_key, o.last_key) == (lz4.first_key, lz4.last_key)
        assert o.stats == lz4.stats and o.data == plain(lz4)

def test_damage(ctx, monkeypatch):
    for name, tabs, k, chunk, L in corrupt_cases():
        for ename, eng, env in [("oracle", UncompressedOracle(), {})] + engines(ctx):
            for kk, v in env.items(): monkeypatch.setenv(kk, v)
            try:
                with pytest.raises(native.CorruptSSTableError) as e:
                    run(tabs, eng, uncompressed_params())
            finally:
                for kk in env: monkeypatch.delenv(kk)
            c = e.value.corruption
            assert (c.input, c.kind, c.chunk, c.offset) == (k, 1, chunk, chunk * L), (name, ename)

# ---- every kernel variant --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("env", [{"B200C_K1": "0", "B200C_K1_BATCH": "0"}, {"B200C_K1_BATCH": "2"}, {"B200C_K1": "2", "B200C_K1_BATCH": "2"},
                                 {"B200C_K5": "0"}, {"B200C_K5": "1"}, {"B200C_K5": "3"}])
def test_every_kernel_variant(env):
    """Noop and uncompressed inputs next to LZ4 under every K1 / K5 variant (B200C_K1_BATCH=2 batches even tiny launches: neither may
    enter the LZ4 thread-per-chunk batch); the switches are read once per process, so the other tests run in a subprocess"""
    import subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "tests/test_gpu_uncompressed.py", "-k", "mixed or setting or damage or longer"],
                       cwd=root, env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]
