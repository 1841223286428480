"""GPU parity for compression parameters besides the defaults: raw-stored chunks (a finite maxCompressedLength; the file's last chunk
zero padded), chunk lengths from 1 to 64 KiB, and inputs that differ in compressor, chunk length and maxCompressedLength in one call.
Every case is compared byte for byte with the CPU oracle (pinned by tests/test_oracle_compression_params.py) on the host engine, the
host engine cut into token-range pieces, and the device-resident engine, and asserts that it saw the chunks it is about."""
import ctypes as C, os, zlib, pytest
import numpy as np
import oracle_lib as O
from chunk_format import INT32_MAX, MIXED, ratio_max_clen, write_chunks, census, boundary_max_clen, reencode, mixed_table
from sstable_builder import Builder
from test_oracle_compression_params import (params, run, stream_of, census_of, fresh, output_tables, input_tables, output_max_clens,
                                            check_census, input_encodings, encoded, corrupt_cases, DEFAULT_OUT, CHUNK_LENS, NOW)
from test_gpu_compaction import DeviceEngine
from cassandra_b200.db.compaction import GpuEngine

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def ctx():
    from cassandra_b200 import native
    c = native.Context(0)
    yield c
    c.close()

def engines(ctx):
    """(name, engine, environment): one piece, B200C_RANGES=5 (host-streamed pieces and OutStream), device-resident inputs and outputs"""
    return [("host", GpuEngine(ctx), {}), ("host pieces", GpuEngine(ctx), {"B200C_RANGES": "5"}), ("device", DeviceEngine(ctx), {})]

def same(got, want, name):
    assert len(got.outputs) == len(want.outputs) >= 1, name
    for g, w in zip(got.outputs, want.outputs):
        assert g.data == w.data, name
        assert g.index == w.index, name
        assert g.compression.chunk_offsets == w.compression.chunk_offsets and g.compression.data_length == w.compression.data_length, name
        assert g.digest == w.digest == zlib.crc32(g.data), name
        assert (g.partitions, g.rows) == (w.partitions, w.rows), name
        if w.filter is not None:
            assert g.filter == w.filter and g.summary == w.summary and (g.first_key, g.last_key) == (w.first_key, w.last_key), name
            for k in w.stats: assert g.stats[k] == w.stats[k], (name, k)
    for k in ("bytes_read", "bytes_in_range", "bytes_written", "total_source_rows", "merged_row_counts"):
        assert got.stats[k] == want.stats[k], (name, k)

def on_every_engine(ctx, monkeypatch, tables, compression=DEFAULT_OUT, **kw):
    """the oracle's result, after every engine has matched it"""
    want = run(tables, O.OracleEngine(), compression, **kw)
    for name, eng, env in engines(ctx):
        for k, v in env.items(): monkeypatch.setenv(k, v)
        try: same(run(tables, eng, compression, **kw), want, name)
        finally:
            for k in env: monkeypatch.delenv(k)
    return want

def output_census(o, stream=None):
    c = o.compression
    return census(o.data, c.chunk_offsets, c.max_compressed_length, c.data_length, c.chunk_length, stream, c.compressor_id if stream else None)

# ---- codec entry points -----------------------------------------------------------------------------------------------------------------------
def codec_stream(seed, chunk_len, nchunks=12):
    """chunks all random, all text, and random then text, ending in a short chunk (a quarter to three quarters of chunk_len) of random bytes"""
    rng = np.random.default_rng(seed)
    parts = []
    for i in range(nchunks):
        k = (chunk_len, 0, int(rng.integers(0, chunk_len)))[i % 3]
        parts += [rng.integers(0, 256, k, dtype=np.uint8).tobytes(), (b"chunk %d of %d " % (i, chunk_len) * chunk_len)[:chunk_len - k]]
    tail = int(rng.integers(chunk_len // 4, 3 * chunk_len // 4))
    return b"".join(parts) + rng.integers(0, 256, tail, dtype=np.uint8).tobytes()

def dev_codec(ctx, comp, stream, chunk_len, mcl):
    """b200c_compress_chunks / b200c_decompress_chunks with B200C_FLAG_DEVICE_PTRS -> (image, offsets, digest, stream decoded back)"""
    from cassandra_b200 import native
    L = native.lib(); allocs = []
    def alloc(n):
        d = C.c_void_p(); ctx.check(L.b200c_dev_alloc(ctx.handle, max(n, 1), C.byref(d))); allocs.append(d); return d
    try:
        n = len(stream); nch = L.b200c_chunk_count(n, chunk_len); cap = L.b200c_compress_bound(comp, n, chunk_len)
        d_in, d_img, d_offs, d_back = alloc(n), alloc(cap), alloc((nch + 1) * 8), alloc(n)
        ctx.check(L.b200c_memcpy_h2d(ctx.handle, d_in, stream, n))
        out_len = C.c_uint64(); dig = C.c_uint32()
        ctx.check(L.b200c_compress_chunks(ctx.handle, comp, d_in, n, chunk_len, mcl, d_img, cap, C.byref(out_len), d_offs, C.byref(dig), native.FLAG_DEVICE_PTRS))
        image = C.create_string_buffer(out_len.value); offs = (C.c_uint64 * nch)()
        ctx.check(L.b200c_memcpy_d2h(ctx.handle, image, d_img, out_len.value)); ctx.check(L.b200c_memcpy_d2h(ctx.handle, offs, d_offs, nch * 8))
        where = native.Corruption()
        ctx.check(L.b200c_decompress_chunks(ctx.handle, comp, d_img, out_len.value, d_offs, nch, chunk_len, mcl, n, d_back, 1, C.byref(where), native.FLAG_DEVICE_PTRS), where)
        back = C.create_string_buffer(n); ctx.check(L.b200c_memcpy_d2h(ctx.handle, back, d_back, n))
        return image.raw, list(offs), dig.value, back.raw
    finally:
        for d in allocs: L.b200c_dev_free(ctx.handle, d)

@pytest.mark.parametrize("comp", [O.COMP_LZ4, O.COMP_SNAPPY])
def test_codec_matches_the_reference_format(ctx, comp):
    for chunk_len in CHUNK_LENS:
        stream = codec_stream(chunk_len + comp, chunk_len)
        for name, mcl in output_max_clens(stream, comp, chunk_len):
            want = write_chunks(stream, comp, chunk_len, mcl)
            check_census(name, census(want[0], want[1], mcl, len(stream), chunk_len, stream, comp))
            assert ctx.compress_chunks(comp, stream, chunk_len, mcl) == want, (chunk_len, name)
            assert ctx.decompress_chunks(comp, want[0], want[1], len(stream), chunk_len, mcl) == stream, (chunk_len, name)
            image, offs, digest, back = dev_codec(ctx, comp, stream, chunk_len, mcl)
            assert (image, offs, digest) == want and back == stream, ("device", chunk_len, name)

def test_codec_thread_kernel_raw_chunks(ctx):
    """>= 32768 chunks of 1 KiB in one call: the thread-per-chunk decoder (k_decompress_chunks_thr) takes the raw branch for records at and
    above max_clen, the last chunk (1021 bytes) through its partial last word. Two settings: max_clen equal to a median chunk's compressed
    length (the writer's boundary: those chunks are stored raw), and max_clen = chunk_len (min_compress_ratio 1: every raw record is exactly
    max_clen long, the reader's boundary; the last one zero padded)"""
    rng = np.random.default_rng(7)
    n = 33000; L = 1024
    keep = rng.integers(0, L + 1, n); keep[-1] = L               # random bytes in the first `keep` bytes of a chunk, zeros after them
    a = rng.integers(0, 256, (n, L), dtype=np.uint8); a[np.arange(L)[None, :] >= keep[:, None]] = 0
    stream = a.reshape(-1).tobytes()[:(n - 1) * L + 1021]
    for setting, mcl in (("median", boundary_max_clen(stream, O.COMP_LZ4, L)), ("ratio 1", ratio_max_clen(L, 1.0))):
        want = write_chunks(stream, O.COMP_LZ4, L, mcl)
        c = census(want[0], want[1], mcl, len(stream), L, stream, O.COMP_LZ4)
        assert c["chunks"] >= 32768 and c["raw"] > 500 and c["compressed"] > 1000, c
        last = len(want[0]) - want[1][-1] - 4
        if setting == "median": assert c["boundary"] >= 10 and last == 1021, c            # the last chunk is stored raw, unpadded
        else: assert c["padded"] == 1 and last == mcl, c
        assert ctx.compress_chunks(O.COMP_LZ4, stream, L, mcl) == want, setting
        assert ctx.decompress_chunks(O.COMP_LZ4, want[0], want[1], len(stream), L, mcl) == stream, setting
        image, offs, digest, back = dev_codec(ctx, O.COMP_LZ4, stream, L, mcl)
        assert (image, offs, digest) == want and back == stream, setting

# ---- compactions --------------------------------------------------------------------------------------------------------------------------------
def test_raw_stored_inputs(ctx, monkeypatch):
    """finite max_clen on the inputs (ratios and exact boundaries, zero-padded last chunks), INT32_MAX on the output: the whole ring, a token
    sub-range and with_metadata"""
    tabs = input_tables()
    for rnd in input_encodings(tabs)[:2]:
        ins = encoded(tabs, rnd)
        on_every_engine(ctx, monkeypatch, ins)
        on_every_engine(ctx, monkeypatch, ins, token_range=(-(1 << 62), 1 << 61))
        on_every_engine(ctx, monkeypatch, ins, with_metadata=True)

OUTPUT_CASES = [(O.COMP_LZ4, 4096, "ratio 1.1"), (O.COMP_SNAPPY, 16384, "ratio 2"), (O.COMP_LZ4, 16384, "boundary last"), (O.COMP_SNAPPY, 16384, "boundary last"),
                (O.COMP_LZ4, 65536, "boundary last"), (O.COMP_SNAPPY, 65536, "boundary last")]

@pytest.mark.parametrize("comp,chunk_len,setting", OUTPUT_CASES)
def test_raw_stored_output(ctx, monkeypatch, comp, chunk_len, setting):
    """inputs with INT32_MAX; the output with a finite max_clen. 16 KiB: the two-pass compressors under B200C_K5=3 (Snappy's default);
    64 KiB: above LZ4C_MAX_CHUNK, the direct kernels"""
    tabs = fresh(output_tables(chunk_len))
    stream = stream_of(run(tabs, O.OracleEngine(), params(comp, chunk_len, INT32_MAX)).outputs[0])
    mcl = dict(output_max_clens(stream, comp, chunk_len))[setting]
    want = on_every_engine(ctx, monkeypatch, tabs, params(comp, chunk_len, mcl))
    check_census(setting, output_census(want.outputs[0], stream))

def test_lcs_with_raw_output(ctx, monkeypatch):
    """several output files, each ending in a short chunk; with ratio 1.1 raw chunks throughout, and with a max_clen found so that some
    file's short last chunk is stored raw and zero padded"""
    tabs = fresh(output_tables(4096, n=4))
    kw = dict(max_sstable_bytes=100_000)
    plain = run(tabs, O.OracleEngine(), params(O.COMP_LZ4, 4096, INT32_MAX), **kw)
    assert len(plain.outputs) >= 3
    cands = []
    for o in plain.outputs:                                      # the compressed length of a file's short last chunk, where it exceeds the chunk
        s = stream_of(o); last = s[len(s) // 4096 * 4096:]
        m = len(O.chunk_compress(O.COMP_LZ4, last))
        if len(last) < m <= 4096: cands.append(m)
    padded = None                                                # (raw chunks move the file boundaries: try each until one file ends padded)
    for mcl in cands:
        w = run(tabs, O.OracleEngine(), params(O.COMP_LZ4, 4096, mcl), **kw)
        if any(output_census(o)["padded"] for o in w.outputs): padded = mcl; break
    assert padded is not None, "no setting leaves a zero-padded short raw chunk at a file's end"
    for mcl in (ratio_max_clen(4096, 1.1), padded):
        want = on_every_engine(ctx, monkeypatch, tabs, params(O.COMP_LZ4, 4096, mcl), **kw)
        cs = [output_census(o) for o in want.outputs]
        assert len(want.outputs) >= 3 and sum(c["raw"] for c in cs) >= 3 and all(c["compressed"] for c in cs), cs
        if mcl == padded: assert sum(c["padded"] for c in cs) >= 1, cs

# ---- mixed inputs in one call -----------------------------------------------------------------------------------------------------------------------
def k1_tail_window(comp, chunk_len):
    """k1_tail.cuh: the bytes at a file's end whose chunks K1 decodes from a staged copy (chunk_max_compressed + chunk_len + 36)"""
    return (4 + chunk_len + chunk_len // 255 + 16 if comp == O.COMP_LZ4 else 32 + chunk_len + chunk_len // 6) + chunk_len + 36

def mixed_inputs():
    """LZ4 at 4, 16 and 64 KiB, Snappy at 16 KiB, finite and infinite max_clen, an empty input, and a 64 KiB input smaller than its tail window"""
    a, b, c, d = fresh(input_tables()[:3]) + [mixed_table(0x5E, 0, 16384, gen=3, keyspace=range(40, 200))]
    reencode(a, O.COMP_LZ4, 4096, ratio_max_clen(4096, 1.1))
    reencode(b, O.COMP_LZ4, 16384, boundary_max_clen(b.uncompressed, O.COMP_LZ4, 16384, which=-1))
    reencode(c, O.COMP_LZ4, 65536, INT32_MAX)
    reencode(d, O.COMP_SNAPPY, 16384, ratio_max_clen(16384, 2))
    empty = Builder(MIXED, (0, 0, 0)).build([], chunk_length=1024, generation=4); reencode(empty, O.COMP_LZ4, 1024, ratio_max_clen(1024, 1.0))
    small = mixed_table(0x5F, 0, 65536, gen=5, random_share=0.1, tail=30000, keyspace=range(100, 160))
    reencode(small, O.COMP_LZ4, 65536, boundary_max_clen(small.uncompressed, O.COMP_LZ4, 65536, which=-1))
    assert 0 < len(small.data) < k1_tail_window(O.COMP_LZ4, 65536) and len(small.compression.chunk_offsets) >= 2
    assert len(empty.data) == 0
    for t, kind in ((a, "ratio"), (b, "boundary last"), (d, "ratio"), (small, "boundary last")):
        ce = census_of(t); assert ce["raw"] >= 1 and ce["compressed"] >= 1, ce
        if kind == "boundary last": assert ce["boundary"] >= 1 and ce["padded"] == 1, ce
    return [a, b, c, d, empty, small]

MIXED_OUT = (O.COMP_SNAPPY, 8192, ratio_max_clen(8192, 1.1))

def test_mixed_inputs_in_one_call(ctx, monkeypatch):
    tabs = mixed_inputs()
    out = params(*MIXED_OUT)
    assert (out.compressor_name, out.chunk_length, out.max_compressed_length) != (tabs[0].compression.compressor_name, tabs[0].compression.chunk_length, tabs[0].compression.max_compressed_length)
    want = on_every_engine(ctx, monkeypatch, tabs, out)
    c = output_census(want.outputs[0]); assert c["raw"] >= 1 and c["compressed"] >= 1, c
    assert all(want.stats["merged_row_counts"][i] >= 0 for i in range(len(tabs)))
    on_every_engine(ctx, monkeypatch, tabs, out, with_metadata=True)

# ---- corruption in raw chunks -------------------------------------------------------------------------------------------------------------------------
def test_damaged_raw_chunks(ctx, monkeypatch):
    """a flipped byte in a raw chunk mid-file and in the (staged) tail, and a raw record shorter than its chunk with a valid CRC: every
    engine reports the oracle's (input, kind, chunk)"""
    from cassandra_b200 import native
    for name, tabs, inp, chunk, kind in corrupt_cases():
        for ename, eng, env in [("oracle", O.OracleEngine(), {})] + engines(ctx):
            for k, v in env.items(): monkeypatch.setenv(k, v)
            try:
                with pytest.raises(native.CorruptSSTableError) as e:
                    run(tabs, eng)
            finally:
                for k in env: monkeypatch.delenv(k)
            assert (e.value.corruption.input, e.value.corruption.kind, e.value.corruption.chunk) == (inp, kind, chunk), (name, ename)

# ---- device buffers as a caller keeps them -------------------------------------------------------------------------------------------------------------
PATTERN = 0xA5
DEVICE_SLACK = 256                                                    # B200C_DEVICE_SLACK (include/b200c.h)

class PoisonedDeviceEngine:
    """B200C_FLAG_DEVICE_PTRS with buffers as a caller may hand them over: every input at a 16-byte aligned address that is not 32-byte
    aligned inside one larger allocation, the bytes behind each buffer (its B200C_DEVICE_SLACK included) and the output buffers filled with
    a non-zero pattern. After the call the inputs must be unchanged and nothing behind an output's length + B200C_DEVICE_SLACK written."""
    needs_lib_bound = True
    GAP = 256 + 96                                                    # pattern bytes behind every buffer (>= B200C_DEVICE_SLACK)
    def __init__(self, ctx): self.ctx = ctx
    def __call__(self, manifest, result):
        from cassandra_b200 import native
        L = native.lib(); ctx = self.ctx
        bufs = []                                                     # (owner, field, host address, length)
        for k in range(manifest.ninputs):
            a = manifest.inputs[k]
            bufs += [(a, "data", a.data, a.data_len), (a, "index", a.index, a.index_len), (a, "chunk_offsets", a.chunk_offsets, a.nchunks * 8)]
            if a.nsummary: bufs.append((a, "summary_positions", a.summary_positions, a.nsummary * 8))
        place = []; pos = 0
        for b in bufs:
            pos = (pos + 31) // 32 * 32 + 16; place.append(pos); pos += b[3] + self.GAP
        arena = np.full(pos + 64, PATTERN, dtype=np.uint8)
        for (_, _, ptr, n), p in zip(bufs, place):
            if n: arena[p:p + n] = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(n,))
        d_in = C.c_void_p(); ctx.check(L.b200c_dev_alloc(ctx.handle, len(arena), C.byref(d_in)))
        allocs = [d_in]; outs = []                                    # outs: (output, field, host address, device buffer, bytes)
        try:
            ctx.check(L.b200c_memcpy_h2d(ctx.handle, d_in, arena.ctypes.data, len(arena)))
            for (owner, field, _, _), p in zip(bufs, place):
                setattr(owner, field, d_in.value + p); assert (d_in.value + p) % 32 == 16
            for k in range(result.noutputs_cap):
                o = result.outputs[k]
                for field, cap in (("data", o.data_cap), ("index", o.index_cap), ("chunk_offsets", o.chunk_cap * 8)):
                    n = cap + self.GAP; d = C.c_void_p(); ctx.check(L.b200c_dev_alloc(ctx.handle, n, C.byref(d))); allocs.append(d)
                    fill = np.full(n, PATTERN, dtype=np.uint8); ctx.check(L.b200c_memcpy_h2d(ctx.handle, d, fill.ctypes.data, n))
                    outs.append((k, field, getattr(o, field), d, n)); setattr(o, field, d.value)
            rc = L.b200c_compact(ctx.handle, C.byref(manifest), C.byref(result), native.FLAG_DEVICE_PTRS)
            back = np.empty_like(arena); ctx.check(L.b200c_memcpy_d2h(ctx.handle, back.ctypes.data, d_in, len(arena)))
            assert np.array_equal(back, arena), "an input buffer or the pattern behind it changed"
            for k, field, host, d, n in outs:
                o = result.outputs[k]
                used = {"data": o.data_len, "index": o.index_len, "chunk_offsets": o.nchunks * 8}[field] if rc == 0 and k < result.noutputs else 0
                got = np.empty(n, dtype=np.uint8); ctx.check(L.b200c_memcpy_d2h(ctx.handle, got.ctypes.data, d, n))
                if rc == 0: assert (got[used + DEVICE_SLACK:] == PATTERN).all(), "output %d %s written beyond its length + B200C_DEVICE_SLACK" % (k, field)
                if used: C.memmove(host, got.ctypes.data, used)
                setattr(o, field, host)
            for owner, field, ptr, _ in bufs: setattr(owner, field, ptr)
            ctx.check(rc, result.corruption)
        finally:
            for d in allocs: L.b200c_dev_free(ctx.handle, d)

def test_poisoned_device_buffers(ctx):
    """the mixed-input call (also in test_mixed_inputs_in_one_call) and a uniform LZ4 one: identical to the plain device engine"""
    from synth_util import synth_tables
    uni = synth_tables(0, 4, 0xB0150, 20000)
    for g, t in enumerate(uni): t.generation = g
    for tabs, out in ((uni, uni[0].compression), (mixed_inputs(), params(*MIXED_OUT))):
        want = run(tabs, DeviceEngine(ctx), out)
        got = run(tabs, PoisonedDeviceEngine(ctx), out)
        same(got, want, "poisoned vs plain device")
        same(got, run(tabs, O.OracleEngine(), out), "poisoned vs oracle")

# ---- every kernel variant --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("env", [{"B200C_K1": "0", "B200C_K1_BATCH": "0"}, {"B200C_K1_BATCH": "2"}, {"B200C_K1": "2", "B200C_K1_BATCH": "2"},
                                 {"B200C_K5": "0"}, {"B200C_K5": "1"}, {"B200C_K5": "3"}])
def test_every_kernel_variant(env):
    """the switches are read once per process: the file's other tests in a subprocess per setting. K1: warp per chunk, thread per chunk,
    two passes (all four raw-chunk branches); K5: all five compressors' raw fallback"""
    import subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "tests/test_gpu_compression_params.py", "-k", "not every_kernel_variant"],
                       cwd=root, env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]
