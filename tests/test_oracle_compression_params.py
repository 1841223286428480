"""Pins the CPU oracle's chunk writer and reader against the plain restatement of flushData / CompressedChunkReader in chunk_format.py,
for the compression parameters real tables carry besides the defaults: a finite maxCompressedLength (min_compress_ratio > 0, so that
chunks are stored raw, the file's last one zero padded), other chunk lengths, and inputs of one compaction that differ in compressor,
chunk length and maxCompressedLength (after ALTER TABLE ... WITH compression). The GPU tests compare the engine with this oracle."""
import copy, functools, pytest
import oracle_lib as O
from chunk_format import (INT32_MAX, COMP_NAMES, ChunkError, ratio_max_clen, write_chunks, read_chunks, census, boundary_max_clen,
                          replace_record, reencode, mixed_table)
from cassandra_b200 import native
from cassandra_b200.io.compress import CompressionMetadata
from cassandra_b200.db.compaction import CompactionTask, CompactionController

NOW = 1700000000
KEYS = range(160)
RATIOS = (0, 1.0, 1.1, 2, 8)
CHUNK_LENS = (1024, 4096, 16384, 65536)

def params(comp, chunk_len, max_clen): return CompressionMetadata(COMP_NAMES[comp], chunk_len, max_clen, 0, [])
DEFAULT_OUT = params(O.COMP_LZ4, 16384, INT32_MAX)

def run(tables, engine, compression=DEFAULT_OUT, **kw):
    return CompactionTask(tables, CompactionController(NOW), compression=compression, **kw).execute(engine, max_outputs=64 if kw.get("max_sstable_bytes") else None)

def stream_of(o):
    c = o.compression
    return read_chunks(o.data, c.chunk_offsets, c.compressor_id, c.chunk_length, c.max_compressed_length, c.data_length)

def census_of(t):
    c = t.compression
    return census(t.data, c.chunk_offsets, c.max_compressed_length, c.data_length, c.chunk_length, t.uncompressed, c.compressor_id)

def fresh(tables): return [copy.copy(t) for t in tables]

# ---- fixtures -----------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def output_tables(out_chunk_len, n=3):
    """n mixed tables over one key space (LZ4, 16 KiB, no finite max_clen). The merged stream ends with the newest table's last partition,
    a random value longer than one output chunk, sized so that the stream's last chunk of out_chunk_len is short: compressed, it is longer
    than itself, which is what a zero-padded raw chunk needs."""
    tail = max(out_chunk_len, 16384) * 3 // 2
    tabs = [mixed_table(0xC0 + g, 0, 16384, gen=g, tail=tail, keyspace=KEYS) for g in range(n)]
    r = run(tabs, O.OracleEngine()).outputs[0].compression.data_length % out_chunk_len
    if not out_chunk_len // 4 <= r <= 3 * out_chunk_len // 4:
        tabs[-1] = mixed_table(0xC0 + n - 1, 0, 16384, gen=n - 1, tail=tail + (out_chunk_len // 2 - r) % out_chunk_len, keyspace=KEYS)
    return tuple(tabs)

@functools.lru_cache(None)
def input_tables():
    """one key space, one table per chunk length; each file's last chunk is short and random"""
    return tuple(mixed_table(0x1A + g, 0, L, gen=g, keyspace=KEYS) for g, L in enumerate((4096, 16384, 65536, 1024)))

def output_max_clens(stream, comp, chunk_len):
    """(name, max_clen) of every output setting: the ratios, the exact length of the (short, random) last chunk and a median chunk length"""
    out = [("ratio %g" % r, ratio_max_clen(chunk_len, r)) for r in RATIOS]
    out.append(("boundary last", boundary_max_clen(stream, comp, chunk_len, which=-1)))
    out.append(("boundary median", boundary_max_clen(stream, comp, chunk_len)))
    return out

def check_census(name, c):
    """what each setting promises: finite max_clen -> raw and compressed chunks side by side; the boundary settings hit it exactly, and the
    last-chunk boundary leaves a zero-padded short raw chunk"""
    if name == "ratio 0": assert c["raw"] == 0 and c["compressed"] == c["chunks"], c
    else: assert c["raw"] >= 1 and c["compressed"] >= 1, (name, c)
    if name.startswith("boundary"): assert c["boundary"] >= 1, (name, c)
    if name == "boundary last": assert c["padded"] == 1, (name, c)

# ---- the oracle writes the reference format -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk_len", CHUNK_LENS)
@pytest.mark.parametrize("comp", [O.COMP_LZ4, O.COMP_SNAPPY])
def test_oracle_output_is_the_reference_format(comp, chunk_len):
    tabs = fresh(output_tables(chunk_len))
    plain = run(tabs, O.OracleEngine(), params(comp, chunk_len, INT32_MAX))
    stream = stream_of(plain.outputs[0])
    assert 3 * chunk_len <= len(stream) and chunk_len // 4 <= len(stream) % chunk_len <= 3 * chunk_len // 4
    for name, mcl in output_max_clens(stream, comp, chunk_len):
        r = run(tabs, O.OracleEngine(), params(comp, chunk_len, mcl))
        o = r.outputs[0]
        image, offs, digest = write_chunks(stream, comp, chunk_len, mcl)
        assert o.data == image, name
        assert o.compression.chunk_offsets == offs and o.compression.data_length == len(stream) and o.digest == digest, name
        assert o.index == plain.outputs[0].index and r.stats["bytes_written"] == plain.stats["bytes_written"]
        assert read_chunks(image, offs, comp, chunk_len, mcl, len(stream)) == stream
        check_census(name, census(image, offs, mcl, len(stream), chunk_len, stream, comp))

# ---- how the inputs are encoded does not change the result ---------------------------------------------------------------------------------
def input_encodings(tabs):
    """rounds of per-input (compressor, max_clen), each input at its own chunk length: every input different from the others in one call"""
    LZ, SN = O.COMP_LZ4, O.COMP_SNAPPY
    def b(t, comp, which): return boundary_max_clen(t.uncompressed, comp, t.compression.chunk_length, which)
    r = lambda t, x: ratio_max_clen(t.compression.chunk_length, x)
    t0, t1, t2, t3 = tabs
    return [
        [(LZ, r(t0, 1.1), "ratio"), (SN, r(t1, 2), "ratio"), (LZ, b(t2, LZ, -1), "boundary last"), (SN, r(t3, 1.0), "ratio")],
        [(SN, b(t0, SN, -1), "boundary last"), (LZ, b(t1, LZ, None), "boundary"), (SN, r(t2, 8), "ratio"), (LZ, INT32_MAX, "plain")],
        [(LZ, b(t0, LZ, -1), "boundary last"), (LZ, INT32_MAX, "plain"), (SN, b(t2, SN, -1), "boundary last"), (LZ, b(t3, LZ, -1), "boundary last")],
    ]

def check_input_census(kind, c):
    if kind == "plain": assert c["raw"] == 0, c; return
    assert c["raw"] >= 1 and c["compressed"] >= 1, (kind, c)
    if kind.startswith("boundary"): assert c["boundary"] >= 1, (kind, c)
    if kind == "boundary last": assert c["padded"] == 1, (kind, c)

def encoded(tabs, rnd):
    out = fresh(tabs)
    for t, (comp, mcl, kind) in zip(out, rnd):
        reencode(t, comp, t.compression.chunk_length, mcl)
        check_input_census(kind, census_of(t))
    return out

def test_input_encoding_does_not_change_the_result():
    tabs = input_tables()
    want = run(fresh(tabs), O.OracleEngine())
    assert len(want.outputs[0].data) > 0
    for rnd in input_encodings(tabs):
        for kw in ({}, dict(with_metadata=True)):
            got = run(encoded(tabs, rnd), O.OracleEngine(), **kw)
            g, w = got.outputs[0], want.outputs[0]
            assert (g.data, g.index, g.digest, g.compression.chunk_offsets) == (w.data, w.index, w.digest, w.compression.chunk_offsets)
            assert (g.partitions, g.rows) == (w.partitions, w.rows)
            for k in ("bytes_read", "bytes_in_range", "bytes_written", "total_source_rows", "input_partitions", "merged_row_counts"):
                assert got.stats[k] == want.stats[k], k

# ---- the parallel oracle agrees ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("comp,chunk_len,setting", [(O.COMP_LZ4, 16384, "boundary last"), (O.COMP_SNAPPY, 4096, "ratio 1.1"), (O.COMP_LZ4, 1024, "boundary median")])
def test_parallel_oracle_agrees_with_finite_max_compressed_length(comp, chunk_len, setting):
    from test_oracle_parallel import run_parallel
    tabs = fresh(output_tables(chunk_len))
    stream = stream_of(run(tabs, O.OracleEngine(), params(comp, chunk_len, INT32_MAX)).outputs[0])
    mcl = dict(output_max_clens(stream, comp, chunk_len))[setting]
    want = run(tabs, O.OracleEngine(), params(comp, chunk_len, mcl)); w = want.outputs[0]
    check_census(setting, census(w.data, w.compression.chunk_offsets, mcl, w.compression.data_length, chunk_len, stream, comp))
    data, index, offs, digest, parts, rows, stats, hi = run_parallel(CompactionTask(tabs, CompactionController(NOW), compression=params(comp, chunk_len, mcl)), 4, 7)
    assert data == w.data and index == w.index and offs == w.compression.chunk_offsets and digest == w.digest
    assert (parts, rows) == (w.partitions, w.rows)
    for k, v in stats.items(): assert want.stats[k] == v, k

# ---- corruption in raw chunks ------------------------------------------------------------------------------------------------------------------
def corrupt_cases():
    """(name, tables, input, chunk, kind): input 1 of three is damaged. Its chunks are 4 KiB LZ4, and max_clen is the compressed length of
    its short, random last chunk: that chunk is stored raw and zero padded, and so are the random chunks before it."""
    base = input_tables()
    t = copy.copy(base[0]); L = t.compression.chunk_length; assert L == 4096
    reencode(t, O.COMP_LZ4, L, boundary_max_clen(t.uncompressed, O.COMP_LZ4, L, which=-1))
    c = t.compression; n = len(c.chunk_offsets); mcl = c.max_compressed_length
    rec_len = lambda i: (c.chunk_offsets[i + 1] if i + 1 < n else len(t.data)) - c.chunk_offsets[i] - 4
    raw = [i for i in range(n) if rec_len(i) >= mcl]
    mid = next(i for i in raw if 2 < i < n - 4 and rec_len(i) == L)          # well before the file's tail window
    assert raw[-1] == n - 1 and rec_len(n - 1) == mcl > len(t.uncompressed) - (n - 1) * L      # the last chunk: raw, zero padded
    out = []
    for name, i in (("flipped byte, raw chunk mid-file", mid), ("flipped byte, padded raw last chunk", n - 1)):
        bad = copy.copy(t); img = bytearray(t.data); img[c.chunk_offsets[i] + 100] ^= 0x08; bad.data = bytes(img)
        out.append((name, bad, i, 1))
    short = copy.copy(t)
    img, offs = replace_record(t.data, c.chunk_offsets, mid, t.uncompressed[mid * L:mid * L + mcl + 10])      # >= max_clen, < the chunk: valid CRC
    short.data = img; short.compression = CompressionMetadata(c.compressor_name, L, c.max_compressed_length, c.data_length, offs)
    out.append(("short raw chunk", short, mid, 2))
    return [(name, [copy.copy(base[1]), bad, copy.copy(base[3])], 1, i, kind) for name, bad, i, kind in out]

def test_damaged_raw_chunks_are_reported_like_the_reader():
    for name, tabs, inp, chunk, kind in corrupt_cases():
        c = tabs[inp].compression
        with pytest.raises(ChunkError) as e:
            read_chunks(tabs[inp].data, c.chunk_offsets, c.compressor_id, c.chunk_length, c.max_compressed_length, c.data_length)
        assert (e.value.chunk, e.value.kind) == (chunk, kind), name
        with pytest.raises(native.CorruptSSTableError) as e2:
            run(tabs, O.OracleEngine())
        assert (e2.value.corruption.input, e2.value.corruption.kind, e2.value.corruption.chunk) == (inp, kind, chunk), name
