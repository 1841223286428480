"""Tables whose compression is disabled (Data.db + CRC.db) and tables written with NoopCompressor, on the CPU: pins crc_component.py's
restatement of ChecksummedSequentialWriter and of the uncompressed LCS switch, and the oracle composition built on it
(crc_component.UncompressedOracle), which the GPU tests in test_gpu_uncompressed.py compare the engine with."""
import copy, functools, os, struct, zlib, pytest
import oracle_lib as O
from chunk_format import INT32_MAX, COMP_NAMES, write_chunks, read_chunks, ratio_max_clen, mixed_table
from crc_component import (write_crc, parse_crc, read_crc, CrcError, crc_entries, lcs_files, index_entries, index_bytes, UncompressedOracle,
                           ParallelOracleEngine, DEFAULT_CHUNK)
from cassandra_b200 import native
from cassandra_b200.io.compress import CompressionMetadata, ChecksumMetadata, uncompressed_params, COMPRESSOR_IDS
from cassandra_b200.io.sstable import SSTable
from cassandra_b200.db.compaction import CompactionTask, CompactionController

NOW = 1700000000
NAMES = {**COMP_NAMES, native.COMP_NONE: "NoopCompressor"}
UNC = native.COMP_UNCOMPRESSED
# (name, compressor id, chunk length): every setting a table may carry here
SETTINGS = [("uncompressed", UNC, 65536), ("lz4", O.COMP_LZ4, 16384), ("snappy", O.COMP_SNAPPY, 16384), ("noop 4k", native.COMP_NONE, 4096),
            ("noop 16k", native.COMP_NONE, 16384)]

def params(comp, chunk_len, max_clen=INT32_MAX):
    return uncompressed_params(chunk_len) if comp == UNC else CompressionMetadata(NAMES[comp], chunk_len, max_clen, 0, [])

def run(tables, engine, compression, **kw):
    return CompactionTask(tables, CompactionController(NOW), compression=compression, **kw).execute(engine, max_outputs=64 if kw.get("max_sstable_bytes") else None)

def plain(t):
    """the uncompressed stream of a table or an output"""
    c = t.compression
    if isinstance(c, ChecksumMetadata): return read_crc(t.data, c.crcs, c.chunk_length)
    return read_chunks(t.data, c.chunk_offsets, c.compressor_id, c.chunk_length, c.max_compressed_length, c.data_length)

def encode(t, comp, chunk_len, max_clen=INT32_MAX):
    """a copy of table t stored with the given setting"""
    s = plain(t); t = copy.copy(t)
    if comp == UNC:
        t.data = s; t.compression = ChecksumMetadata(chunk_len, len(s), crc_entries(s, chunk_len))
    else:
        image, offs, _ = write_chunks(s, comp, chunk_len, max_clen)
        t.data = image; t.compression = CompressionMetadata(NAMES[comp], chunk_len, max_clen, len(s), offs)
    return t

def check_output(o, chunk_len=DEFAULT_CHUNK):
    """an uncompressed output is its own stream: CRC.db entries and digest as the restatement writes them"""
    assert isinstance(o.compression, ChecksumMetadata) and o.compression.data_length == len(o.data)
    crc_db, crcs, digest = write_crc(o.data, chunk_len)
    assert o.compression.crcs == crcs and o.digest == digest == zlib.crc32(o.data)
    assert o.compression.serialize() == crc_db
    comp = o.components(); assert "CRC.db" in comp and "CompressionInfo.db" not in comp and comp["CRC.db"] == crc_db

def short_last(n, chunk_len): return n % chunk_len != 0

# ---- fixtures ---------------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def base_tables():
    """three tables over one key space, random and text values. The first is 154 chunks of 4 KiB exactly; the others end in a short
    chunk at every chunk length used here"""
    return tuple(mixed_table(0x4C0 + g, 0, 16384, gen=g, keyspace=range(120)) for g in range(3))

@functools.lru_cache(None)
def growth_tables():
    """two tables with disjoint keys written 1e11 us apart, each header holding its own minimum timestamp. Merged, every row of the newer
    table re-encodes its timestamp delta against the older minimum in more bytes: the output stream is longer than the inputs' together."""
    from sstable_builder import Builder, Partition, Row, Cell
    from chunk_format import MIXED
    from cassandra_b200.io.sstable import DELETION_TIME_EPOCH
    tabs = []
    for g, ts in ((0, 1000), (1, 10 ** 11)):
        parts = [Partition(b"key-%05d" % (1000 * g + k), [Row((struct.pack(">q", ck),), [Cell(0, ts, b"v%d" % ck)], ts=ts) for ck in range(40)])
                 for k in range(60)]
        t = Builder(MIXED, (ts, DELETION_TIME_EPOCH, 0)).build(parts, chunk_length=4096, generation=g); t.partitions = len(parts)
        tabs.append(t)
    return tuple(tabs)

class SizedOracle(UncompressedOracle):
    """the oracle with output buffers sized as for the GPU engine (b200c_compress_bound of the inputs' length): exercises the retry with the
    sizes a call reports when its buffers are too small"""
    needs_lib_bound = True
    def __init__(self): super().__init__(); self.too_small = 0
    def __call__(self, manifest, result):
        try: super().__call__(manifest, result)
        except native.B200CError as e:
            if e.code == native.ETOOSMALL: self.too_small += 1
            raise

def golden(name): return os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "legacy-sstables", "oa", "legacy_tables", name, "oa-1-big-")

# ---- the restatement ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 65535, 65536, 65537, 3 * 65536, 3 * 65536 + 100])
def test_checksummed_writer(n):
    data = bytes((i * 131 + (i >> 9)) & 0xFF for i in range(n))
    crc_db, crcs, digest = write_crc(data)
    assert len(crcs) == (n + 65535) // 65536 and len(crc_db) == 4 + 4 * len(crcs)
    assert crc_db[:4] == struct.pack(">i", 65536) and digest == zlib.crc32(data)
    if n % 65536: assert crcs[-1] == zlib.crc32(data[n // 65536 * 65536:])                # the short last chunk
    elif n: assert crcs[-1] == zlib.crc32(data[-65536:])                                   # no empty trailing chunk at an exact multiple
    assert parse_crc(crc_db) == (65536, crcs) and read_crc(data, crcs, 65536) == data
    m = ChecksumMetadata.parse(crc_db, n); assert (m.chunk_length, m.crcs, m.serialize()) == (65536, crcs, crc_db)
    if crcs:
        assert digest != zlib.crc32(data + crc_db[4:]), "the digest covers Data.db alone"

def test_lcs_switch_rule():
    starts = [0, 10, 25, 40]
    assert lcs_files(starts, 50, 25) == [(0, 3, 0, 40), (3, 4, 40, 50)]          # position 25 == limit before partition 2: no switch
    assert lcs_files(starts, 50, 24) == [(0, 2, 0, 25), (2, 4, 25, 50)]          # one byte over: switch
    assert lcs_files(starts, 50, 0) == [(0, 1, 0, 10), (1, 2, 10, 25), (2, 3, 25, 40), (3, 4, 40, 50)]

def test_noop_is_the_compressed_format_with_a_copy():
    """a Noop chunk is never shorter than its data: flushData's raw-storage rule leaves every image unchanged at any maxCompressedLength"""
    s = plain(base_tables()[1])
    for L in (4096, 16384):
        want = write_chunks(s, native.COMP_NONE, L, INT32_MAX)
        assert short_last(len(s), L)
        for r in (1.0, 1.1, 2):
            assert write_chunks(s, native.COMP_NONE, L, ratio_max_clen(L, r)) == want
        assert COMPRESSOR_IDS["NoopCompressor"] == native.COMP_NONE

# ---- the oracle composition ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["legacy_oa_simple", "legacy_oa_clust"])
def test_golden_identity(name):
    """the reference's golden table stored uncompressed, compacted into an uncompressed output: Data.db is the golden Data.db decompressed
    and Index.db the golden Index.db"""
    base = golden(name)
    t = SSTable.open(base); u = encode(t, UNC, DEFAULT_CHUNK)
    r = run([u], UncompressedOracle(), uncompressed_params(), column_index_size=4096)
    o = r.outputs[0]
    assert o.data == plain(t) and o.index == open(base + "Index.db", "rb").read()
    check_output(o)

def test_cross_equalities():
    """every input setting x every output setting: the output decompressed is the uncompressed output's Data.db, Index.db is the same"""
    tabs = base_tables()
    ref = run([encode(t, UNC, DEFAULT_CHUNK) for t in tabs], UncompressedOracle(), uncompressed_params()).outputs[0]
    check_output(ref); assert short_last(len(ref.data), DEFAULT_CHUNK)
    assert ref.data == plain(run(list(tabs), O.OracleEngine(), params(O.COMP_LZ4, 16384)).outputs[0])
    for _, ic, il in SETTINGS:
        ins = [encode(t, ic, il) for t in tabs]
        for _, oc, ol in SETTINGS:
            o = run(ins, UncompressedOracle(), params(oc, ol)).outputs[0]
            assert plain(o) == ref.data and o.index == ref.index, (ic, il, oc, ol)

def mixed_inputs():
    """uncompressed at 4 (an exact multiple of the chunk size), 16 and 64 KiB, LZ4, Noop, and an empty uncompressed input"""
    a, b, c = base_tables()
    from sstable_builder import Builder
    from chunk_format import MIXED
    empty = Builder(MIXED, (0, 0, 0)).build([], chunk_length=4096, generation=9)
    return [encode(a, UNC, 4096), encode(b, UNC, 16384), encode(c, UNC, 65536), encode(a, O.COMP_LZ4, 16384), encode(b, native.COMP_NONE, 4096),
            encode(empty, UNC, 4096)]

def test_mixed_inputs_and_chunk_sizes():
    ins = mixed_inputs()
    assert len(ins[-1].data) == 0 and ins[-1].compression.crcs == []
    assert len(ins[0].data) % 4096 == 0 and len(ins[0].compression.crcs) == len(ins[0].data) // 4096      # no empty trailing entry
    for t in ins[1:3]: assert short_last(len(t.data), t.compression.chunk_length)
    ref = run(list(base_tables()) + [base_tables()[0], base_tables()[1]], O.OracleEngine(), params(O.COMP_LZ4, 16384)).outputs[0]
    for L in (4096, 16384, 65536):
        o = run(ins, UncompressedOracle(), uncompressed_params(L)).outputs[0]
        check_output(o, L); assert o.data == plain(ref) and o.index == ref.index and short_last(len(o.data), L)

def lcs_limits(stream, index):
    """(limit, first file end) pairs: a partition start exactly at the limit (no switch there) and one byte short of it (switch)"""
    starts = [p for _, p, _ in index_entries(index)]
    k = len(starts) // 3
    return starts, [(starts[k], starts[k + 1]), (starts[k] - 1, starts[k])]

def test_lcs_files_at_the_limit():
    tabs = [encode(t, UNC, DEFAULT_CHUNK) for t in base_tables()]
    whole = run(tabs, UncompressedOracle(), uncompressed_params()).outputs[0]
    starts, cases = lcs_limits(whole.data, whole.index)
    assert index_bytes(index_entries(whole.index)) == whole.index
    for limit, end0 in cases:
        r = run(tabs, UncompressedOracle(), uncompressed_params(), max_sstable_bytes=limit)
        assert len(r.outputs) >= 2 and len(r.outputs[0].data) == end0, (limit, [len(o.data) for o in r.outputs])
        assert b"".join(o.data for o in r.outputs) == whole.data
        assert sum(o.partitions for o in r.outputs) == whole.partitions
        for o in r.outputs: check_output(o)
        assert any(short_last(len(o.data), DEFAULT_CHUNK) for o in r.outputs)

def corrupt_cases():
    """(name, tables, input, chunk, chunk length): one flipped Data.db byte in an uncompressed input, mid-file and in the short last chunk"""
    out = []
    for name, k, where in (("mid", 1, 0.5), ("last", 2, 0.999)):
        tabs = [encode(t, UNC, 4096) for t in base_tables()]
        d = bytearray(tabs[k].data); pos = int(len(d) * where); d[pos] ^= 0x40; tabs[k].data = bytes(d)
        out.append((name, tabs, k, pos // 4096, 4096))
    return out

def test_damage():
    for name, tabs, k, chunk, L in corrupt_cases():
        with pytest.raises(native.CorruptSSTableError) as e:
            run(tabs, UncompressedOracle(), uncompressed_params())
        c = e.value.corruption
        assert (c.input, c.kind, c.chunk, c.offset) == (k, 1, chunk, chunk * L), name
    tabs = [encode(t, UNC, 4096) for t in base_tables()]
    tabs[0].compression = ChecksumMetadata(4096, len(tabs[0].data), tabs[0].compression.crcs[:-1])
    with pytest.raises(native.B200CError) as e:
        run(tabs, UncompressedOracle(), uncompressed_params())
    assert e.value.code == native.EINVAL

def test_noop_output_and_inputs_at_any_max_compressed_length():
    tabs = base_tables()
    want = run(list(tabs), O.OracleEngine(), params(native.COMP_NONE, 4096)).outputs[0]
    assert short_last(want.compression.data_length, 4096)
    for r in (1.1, 2):
        o = run(list(tabs), O.OracleEngine(), params(native.COMP_NONE, 4096, ratio_max_clen(4096, r))).outputs[0]
        assert o.data == want.data and o.compression.chunk_offsets == want.compression.chunk_offsets
        ins = [encode(t, native.COMP_NONE, 4096, ratio_max_clen(4096, r)) for t in tabs]
        assert run(ins, O.OracleEngine(), params(native.COMP_NONE, 4096)).outputs[0].data == want.data

def test_output_longer_than_the_inputs():
    """an uncompressed output longer than all inputs together: the first call finds its buffers too small, reports the sizes it needs, and the
    second call writes the same stream as the LZ4 output decompressed"""
    tabs = growth_tables()
    assert tabs[0].header_stats[0] != tabs[1].header_stats[0]
    ins = [encode(t, UNC, 4096) for t in tabs]
    total_in = sum(len(t.data) for t in ins)
    eng = SizedOracle()
    o = run(ins, eng, uncompressed_params()).outputs[0]
    assert len(o.data) > total_in + 1024 and eng.too_small == 1, (len(o.data), total_in)
    check_output(o)
    assert o.data == plain(run(list(tabs), O.OracleEngine(), params(O.COMP_LZ4, 16384)).outputs[0])

@pytest.mark.parametrize("out", [(UNC, DEFAULT_CHUNK), (UNC, 4096), (O.COMP_LZ4, 16384), (native.COMP_NONE, 4096)])
def test_parallel_oracle_agrees(out):
    """the same composition over oracle/parallel.cc gives the single-threaded oracle's bytes"""
    for ins in (mixed_inputs(), [encode(t, UNC, 4096) for t in growth_tables()]):
        a = run(ins, UncompressedOracle(), params(*out)); b = run(ins, UncompressedOracle(ParallelOracleEngine()), params(*out))
        assert len(a.outputs) == len(b.outputs) == 1
        x, y = a.outputs[0], b.outputs[0]
        assert (x.data, x.index, x.compression.chunk_offsets, x.digest, x.partitions, x.rows) == (y.data, y.index, y.compression.chunk_offsets, y.digest, y.partitions, y.rows)
        for k in ("bytes_read", "bytes_written", "total_source_rows", "merged_row_counts"): assert a.stats[k] == b.stats[k], k
