"""GPU parity tests of b200c_compact through the C ABI: for the same manifest the CUDA engine must return the same Data.db,
Index.db, chunk offsets, Digest.crc32 and counters as the CPU oracle (itself pinned by the reference's golden SSTables),
and reproduce the golden `oa` files directly."""
import os, random, struct, zlib, pytest
import oracle_lib as O
from sstable_builder import *
from synth_util import synth_tables, decompress_output
from cassandra_b200.io.sstable import SSTable
from cassandra_b200.db.compaction import CompactionTask, CompactionController, GpuEngine

pytestmark = pytest.mark.gpu
NOW = 1700000000
I32 = lambda v: struct.pack(">i", v)

@pytest.fixture(scope="module")
def ctx():
    from cassandra_b200 import native
    c = native.Context(0)
    yield c
    c.close()

def both(ctx, tables, controller, **kw):
    for g, t in enumerate(tables): t.generation = g
    want = CompactionTask(tables, controller, **kw).execute(O.OracleEngine())
    got = CompactionTask(tables, controller, **kw).execute(GpuEngine(ctx))
    assert len(got.outputs) == len(want.outputs) == 1
    g, w = got.outputs[0], want.outputs[0]
    if g.data != w.data:                      # localise the first difference in the uncompressed stream for the report
        a, b = decompress_output(g), decompress_output(w)
        i = next((k for k in range(min(len(a), len(b))) if a[k] != b[k]), min(len(a), len(b)))
        raise AssertionError("Data stream differs at %d (len %d vs %d): gpu %s | oracle %s" % (i, len(a), len(b), a[max(0, i - 24):i + 16].hex(), b[max(0, i - 24):i + 16].hex()))
    assert g.index == w.index
    assert g.compression.chunk_offsets == w.compression.chunk_offsets and g.compression.data_length == w.compression.data_length
    assert g.digest == w.digest == zlib.crc32(g.data)
    assert (g.partitions, g.rows) == (w.partitions, w.rows)
    if w.filter is not None:                  # with_metadata: Filter.db, Summary.db, first/last key and every MetadataCollector reduction
        assert g.filter == w.filter and g.summary == w.summary and (g.first_key, g.last_key) == (w.first_key, w.last_key)
        for k in w.stats: assert g.stats[k] == w.stats[k], k
    for k in ("bytes_read", "bytes_in_range", "bytes_written", "total_source_rows", "input_partitions", "merged_row_counts"):
        assert got.stats[k] == want.stats[k], k
    assert got.stats["kernel_launches"] > 0
    assert got.stats["index_slow_path_inputs"] == 0, "Index.db speculation fell back to the sequential walk"
    if len(tables) <= 6 and any(getattr(t, "summary_positions", None) is not None for t in tables):
        # same compaction without Summary.db positions: K2 then speculates on entry starts with Data.db's help (and cannot stream)
        saved = [t.summary_positions for t in tables]
        try:
            for t in tables: t.summary_positions = None
            g2 = CompactionTask(tables, controller, **kw).execute(GpuEngine(ctx))
        finally:
            for t, sp in zip(tables, saved): t.summary_positions = sp
        o2 = g2.outputs[0]
        assert o2.data == w.data and o2.index == w.index and o2.digest == w.digest and g2.stats["index_slow_path_inputs"] == 0
    return got, want

def _golden(golden_dir, name): return os.path.join(golden_dir, "oa", "legacy_tables", name, "oa-1-big-")

@pytest.mark.parametrize("name", ["legacy_oa_simple", "legacy_oa_clust"])
def test_golden_identity_compaction(ctx, golden_dir, name):
    base = _golden(golden_dir, name)
    got, _ = both(ctx, [SSTable.open(base)], CompactionController(NOW), column_index_size=4096)
    comp = got.outputs[0].components()
    for c in ("Data.db", "Index.db", "CompressionInfo.db", "Digest.crc32"):
        assert comp[c] == open(base + c, "rb").read(), c

def test_golden_self_merge(ctx, golden_dir):
    base = _golden(golden_dir, "legacy_oa_clust")
    got, _ = both(ctx, [SSTable.open(base, 1), SSTable.open(base, 2), SSTable.open(base, 3)], CompactionController(NOW), column_index_size=4096)
    assert got.outputs[0].data == open(base + "Data.db", "rb").read()
    assert got.stats["merged_row_counts"] == [0, 0, 5]

@pytest.mark.parametrize("schema,n,universe,rpp,cis", [(0, 4, 20000, 0, 65536), (0, 16, 6000, 0, 65536), (1, 3, 60, 1000, 65536), (1, 4, 80, 300, 4096)])
def test_synthetic_configs_match_oracle(ctx, schema, n, universe, rpp, cis):
    tabs = synth_tables(schema, n, 0xCA550000 + schema + n, universe, rows_per_partition=rpp, column_index_size=cis)
    got, want = both(ctx, tabs, CompactionController(NOW), column_index_size=cis)
    assert want.stats["bytes_written"] < want.stats["bytes_read"]
    # nothing purgeable / expired: a different code path through purge
    both(ctx, tabs, CompactionController(0, 0), column_index_size=cis)
    # overlapping-sstable rule blocks part of the purge
    both(ctx, tabs, CompactionController(NOW, overlapping_min_timestamp=1600000000000000 + 1500000000), column_index_size=cis)

def test_snappy_output_and_input(ctx):
    tabs = synth_tables(0, 3, 11, 5000, comp=O.COMP_SNAPPY)
    both(ctx, tabs, CompactionController(NOW))

def test_sixty_four_inputs(ctx):
    tabs = synth_tables(0, 64, 64, 3000, p=0.3)
    got, _ = both(ctx, tabs, CompactionController(NOW))
    assert sum(got.stats["merged_row_counts"][32:]) >= 0

def test_random_range_tombstone_merges(ctx):
    S1 = Schema(["Int32Type"], [("val", "UTF8Type")])
    rng = random.Random(99); b = Builder(S1, (0, 0, 0))
    for it in range(25):
        parts_per_table = []
        nsrc = rng.randint(1, 5)
        for s in range(nsrc):
            parts = []
            for key in (b"p1", b"p2", b"p3", b"key-%d" % rng.randint(0, 3)):
                if rng.random() < 0.3: continue
                us = []; pos = 0; open_dt = None
                while pos < 60:
                    pos += rng.randint(1, 5); r = rng.random()
                    if open_dt is None and r < 0.3:
                        t = rng.randint(100, 200); us.append(Marker(rng.choice((K_INCL_START, K_EXCL_START)), (I32(pos),), None, (t, NOW - rng.randint(0, 2000000)))); open_dt = us[-1].open
                    elif open_dt is not None and r < 0.35:
                        if rng.random() < 0.3:
                            t = (rng.randint(100, 200), NOW - rng.randint(0, 2000000))
                            us.append(Marker(rng.choice((K_EXCL_END_INCL_START, K_INCL_END_EXCL_START)), (I32(pos),), open_dt, t)); open_dt = t
                        else:
                            us.append(Marker(rng.choice((K_INCL_END, K_EXCL_END)), (I32(pos),), open_dt, None)); open_dt = None
                    else:
                        kind = rng.random()
                        ts = rng.randint(90, 210)
                        if kind < 0.15: us.append(Row((I32(pos),), [], deletion=(ts, NOW - rng.randint(0, 2000000))))
                        elif kind < 0.3: us.append(Row((I32(pos),), [Cell.tombstone(0, ts, NOW - rng.randint(0, 2000000))], ts=rng.randint(90, 210)))
                        elif kind < 0.45: us.append(Row((I32(pos),), [Cell(0, ts, b"ttl", 3600, NOW + rng.randint(-5000, 5000))], ts=ts, ttl=3600, ldt=NOW + rng.randint(-5000, 5000)))
                        else: us.append(Row((I32(pos),), [Cell(0, rng.randint(90, 210), rng.choice([b"", b"v", b"value-%d" % it]))], ts=ts if rng.random() < 0.8 else NO_TS))
                if open_dt is not None: us.append(Marker(K_INCL_END, (I32(pos + 1),), open_dt, None))
                pd = (rng.randint(100, 160), NOW - rng.randint(0, 2000000)) if rng.random() < 0.25 else None
                if us or pd: parts.append(Partition(key, us, pd))
            if not parts: parts = [Partition(b"p1", [Row((I32(1),), [Cell(0, 100, b"x")], ts=100)])]
            uniq = {p.key: p for p in parts}
            parts_per_table.append(b.build(list(uniq.values())))
        both(ctx, parts_per_table, CompactionController(NOW, rng.choice([864000, 0, 10**9])))

def test_mixed_types_variable_keys(ctx):
    rng = random.Random(5)
    s = Schema(["LongType", "UTF8Type"], [("a", "LongType"), ("b", "UTF8Type"), ("c", "Int32Type"), ("d", "DoubleType")])
    tables = []
    keys = sorted({bytes(rng.getrandbits(8) for _ in range(rng.choice([1, 3, 8, 9, 17, 40]))) for _ in range(300)} | {b""})     # a key occurs once per sstable
    for t in range(5):
        parts = []
        for k in keys:
            if rng.random() < 0.5: continue
            us = []
            for ck in sorted({(rng.randint(-3, 3), rng.choice([b"", b"x", b"yy", b"zzzzzzzz" * 30])) for _ in range(rng.randint(1, 12))}):
                cells = [Cell(ci, 1000 + rng.randint(0, 5), v) for ci, v in ((0, struct.pack(">q", rng.getrandbits(40))), (1, rng.choice([b"", b"hello", b"w" * 200])),
                         (2, I32(rng.randint(-9, 9))), (3, struct.pack(">d", rng.random()))) if rng.random() < 0.7]
                us.append(Row((struct.pack(">q", ck[0]), ck[1]), cells, ts=1000 + rng.randint(0, 5) if (rng.random() < 0.8 or not cells) else NO_TS))
            parts.append(Partition(k, us, (1002, NOW) if rng.random() < 0.1 else None))
        tables.append(Builder(s, (1000 - t, 0, 0), column_index_size=1024).build(parts))
    both(ctx, tables, CompactionController(NOW, 10**9), column_index_size=1024)
    both(ctx, tables[:1], CompactionController(NOW, 10**9), column_index_size=1024)

def test_token_range_shards_partition_the_output(ctx):
    tabs = synth_tables(0, 4, 21, 8000)
    full, _ = both(ctx, tabs, CompactionController(NOW))
    cuts = [-(1 << 63), -(1 << 62), 0, 1 << 61, (1 << 63) - 1]
    parts = rows = 0; streams = b""
    for lo, hi in zip(cuts, cuts[1:]):
        g, _ = both(ctx, tabs, CompactionController(NOW), token_range=(lo, hi))
        parts += g.outputs[0].partitions; rows += g.outputs[0].rows; streams += decompress_output(g.outputs[0])
    assert (parts, rows) == (full.outputs[0].partitions, full.outputs[0].rows)
    assert streams == decompress_output(full.outputs[0])          # partition records are position independent: shards concatenate exactly

def test_corrupt_chunk_is_reported_with_its_input(ctx):
    from cassandra_b200 import native
    tabs = synth_tables(0, 3, 31, 4000)
    bad = bytearray(tabs[1].data); bad[tabs[1].compression.chunk_offsets[2] + 9] ^= 0x10; tabs[1].data = bytes(bad)
    with pytest.raises(native.CorruptSSTableError) as e:
        CompactionTask(tabs, CompactionController(NOW)).execute(GpuEngine(ctx))
    assert (e.value.corruption.input, e.value.corruption.kind, e.value.corruption.chunk) == (1, 1, 2)
    with pytest.raises(native.CorruptSSTableError) as e2:
        CompactionTask(tabs, CompactionController(NOW)).execute(O.OracleEngine())
    assert (e2.value.corruption.input, e2.value.corruption.chunk) == (1, 2)

def test_corrupt_index_is_rejected(ctx):
    from cassandra_b200 import native
    tabs = synth_tables(0, 2, 32, 3000)
    bad = bytearray(tabs[0].index); bad[len(bad) // 2] ^= 0xFF; tabs[0].index = bytes(bad)
    with pytest.raises(native.CorruptSSTableError):
        CompactionTask(tabs, CompactionController(NOW)).execute(GpuEngine(ctx))

def test_unsupported_is_refused_not_faked(ctx):
    from cassandra_b200 import native
    class ComplexDeletion(Builder):                  # HAS_COMPLEX_DELETION (0x40): complex columns are outside the envelope
        def row(self, u, prev_size, columns, vfixed, static):
            b = bytearray(super().row(u, prev_size, columns, vfixed, static)); b[0] |= 0x40; return bytes(b)
    t = ComplexDeletion(Schema(["Int32Type"], [("val", "UTF8Type")]), (0, 0, 0)).build([Partition(b"k", [Row((I32(1),), [Cell(0, 5, b"v")], ts=5)])])
    with pytest.raises(native.UnsupportedError):
        CompactionTask([t], CompactionController(NOW)).execute(GpuEngine(ctx))
    with pytest.raises(native.UnsupportedError):
        CompactionTask([t], CompactionController(NOW)).execute(O.OracleEngine())
    # a header that promises static columns over a stream without static rows is corruption, not something to guess around
    t = Builder(Schema(["Int32Type"], [("val", "UTF8Type")]), (0, 0, 0)).build([Partition(b"k", [Row((I32(1),), [Cell(0, 5, b"v")], ts=5)])])
    t.static_columns = [(b"s", "org.apache.cassandra.db.marshal.UTF8Type")]
    with pytest.raises(native.CorruptSSTableError):
        CompactionTask([t], CompactionController(NOW)).execute(GpuEngine(ctx))

@pytest.mark.parametrize("limit,n,universe", [(200_000, 6, 30000), (1 << 20, 8, 60000), (50_000, 3, 8000)])
def test_lcs_output_switching_matches_oracle(ctx, limit, n, universe):
    """MaxSSTableSizeWriter: a new output file starts before the first partition that sees more than `limit` flushed on-disk bytes.
    Every file (Data, Index with file-relative positions, chunk offsets, digest, counters) must equal the oracle's."""
    tabs = synth_tables(0, n, 0x1C5 + n, universe)
    kw = dict(max_sstable_bytes=limit)
    want = CompactionTask(tabs, CompactionController(NOW), **kw).execute(O.OracleEngine(), max_outputs=64)
    got = CompactionTask(tabs, CompactionController(NOW), **kw).execute(GpuEngine(ctx), max_outputs=64)
    assert len(want.outputs) >= 3 and len(got.outputs) == len(want.outputs)
    for g, w in zip(got.outputs, want.outputs):
        assert g.data == w.data and g.index == w.index and g.digest == w.digest
        assert g.compression.chunk_offsets == w.compression.chunk_offsets and g.compression.data_length == w.compression.data_length
        assert (g.partitions, g.rows) == (w.partitions, w.rows)
    if w.filter is not None:                  # with_metadata: Filter.db, Summary.db, first/last key and every MetadataCollector reduction
        assert g.filter == w.filter and g.summary == w.summary and (g.first_key, g.last_key) == (w.first_key, w.last_key)
        for k in w.stats: assert g.stats[k] == w.stats[k], k
    for k in ("bytes_read", "bytes_written", "total_source_rows", "merged_row_counts"): assert got.stats[k] == want.stats[k]

def test_lcs_wide_partitions(ctx):
    tabs = synth_tables(1, 3, 0x1C9, 120, rows_per_partition=1000)
    kw = dict(max_sstable_bytes=1 << 20)
    want = CompactionTask(tabs, CompactionController(NOW), **kw).execute(O.OracleEngine(), max_outputs=64)
    got = CompactionTask(tabs, CompactionController(NOW), **kw).execute(GpuEngine(ctx), max_outputs=64)
    assert len(want.outputs) >= 2 and len(got.outputs) == len(want.outputs)
    for g, w in zip(got.outputs, want.outputs):
        assert g.data == w.data and g.index == w.index and g.digest == w.digest and g.compression.chunk_offsets == w.compression.chunk_offsets

def test_empty_result_and_tiny_inputs(ctx):
    S1 = Schema(["Int32Type"], [("val", "UTF8Type")]); b = Builder(S1, (0, 0, 0))
    t = b.build([Partition(b"k", [], (5, 7))])                      # only a purgeable partition deletion -> empty output
    got, _ = both(ctx, [t], CompactionController(NOW))
    assert got.outputs[0].data == b"" and got.outputs[0].index == b"" and got.outputs[0].partitions == 0
    t2 = b.build([Partition(b"k", [Row((I32(1),), [Cell(0, 5, b"v")], ts=5)])])
    both(ctx, [t2], CompactionController(NOW)); both(ctx, [t2, t], CompactionController(NOW))

def test_scratch_overflow_partitions_are_re_emitted(ctx):
    """the single serialisation pass writes into a scratch slot sized from the input partitions (+25 %); re-basing the deltas to a much
    smaller output minTimestamp makes rows grow past that, which must be caught and re-emitted exactly"""
    S1 = Schema(["Int32Type"], [("val", "UTF8Type")])
    base = 1600000000000000
    a = Builder(S1, (base, 0, 0)).build([Partition(b"grow-%d" % p, [Row((I32(i),), [Cell(0, base + i, b"")], ts=base + i) for i in range(200)]) for p in range(40)])
    b = Builder(S1, (0, 0, 0)).build([Partition(b"other", [Row((I32(1),), [Cell(0, 5, b"v")], ts=5)])])
    got, want = both(ctx, [a, b], CompactionController(NOW, 10**9))
    assert want.stats["bytes_written"] > 1.3 * a.compression.data_length

def test_two_pass_mode_matches(golden_dir):
    """A/B switch B200C_K4_TWO_PASS=1 (size pass + emit pass) must produce the same bytes as the default scratch + gather path"""
    import subprocess, sys, textwrap
    code = textwrap.dedent('''
        import sys; sys.path.insert(0, "tests"); sys.path.insert(0, ".")
        import oracle_lib as O
        from synth_util import synth_tables
        from cassandra_b200 import native
        from cassandra_b200.db.compaction import CompactionTask, CompactionController, GpuEngine
        for schema, n, u, rpp, cis in ((0, 6, 8000, 0, 65536), (1, 3, 50, 400, 4096)):
            tabs = synth_tables(schema, n, 5 + schema, u, rows_per_partition=rpp, column_index_size=cis)
            with native.Context(0) as ctx:
                g = CompactionTask(tabs, CompactionController(1700000000), column_index_size=cis).execute(GpuEngine(ctx)).outputs[0]
            w = CompactionTask(tabs, CompactionController(1700000000), column_index_size=cis).execute(O.OracleEngine()).outputs[0]
            assert g.data == w.data and g.index == w.index and g.digest == w.digest
        print("ok")
    ''')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], cwd=root, env=dict(os.environ, B200C_K4_TWO_PASS="1"), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]

def test_config0_full_size_4x64mb(ctx):
    """BASELINE.json configs[0]: STCS 4 SSTables x 64 MB, LZ4, single token range — full size, byte for byte against the oracle"""
    import synth
    tabs = synth_tables(0, 4, 0xCA550001, synth.universe_for(0, 64 << 20, 0.5))
    got, want = both(ctx, tabs, CompactionController(NOW))
    assert want.stats["bytes_read"] > 4 * 60 * (1 << 20)

def test_wide_partitions_medium(ctx):
    """schema W at ~70 KB per partition: every partition has a promoted index (2 column-index blocks) and takes the re-emit route"""
    tabs = synth_tables(1, 4, 0xCA550005, 400, rows_per_partition=1000)
    got, want = both(ctx, tabs, CompactionController(NOW))
    assert len(want.outputs[0].index) > want.outputs[0].partitions * 90        # promoted index present on every partition

def test_output_buffers_too_small_reports_required_sizes(ctx):
    import ctypes as C, numpy as np
    from cassandra_b200 import native
    tabs = synth_tables(0, 2, 41, 3000)
    task = CompactionTask(tabs, CompactionController(NOW)); m = task.build_manifest()
    res = native.Result(); outs = (native.Output * 1)(); tiny = np.empty(64, dtype=np.uint8); co = np.zeros(4, dtype=np.uint64)
    outs[0].data, outs[0].data_cap, outs[0].index, outs[0].index_cap, outs[0].chunk_offsets, outs[0].chunk_cap = tiny.ctypes.data, 64, tiny.ctypes.data, 64, co.ctypes.data, 4
    res.noutputs_cap = 1; res.outputs = outs
    rc = native.lib().b200c_compact(ctx.handle, C.byref(m), C.byref(res), 0)
    assert rc == native.ETOOSMALL
    assert res.required_data_cap > 64 and res.required_index_cap > 64 and res.required_chunk_cap >= 1

def test_poll_reports_progress(ctx):
    import ctypes as C
    from cassandra_b200 import native
    tabs = synth_tables(0, 2, 42, 3000)
    CompactionTask(tabs, CompactionController(NOW)).execute(GpuEngine(ctx))
    p = native.Progress()
    assert native.lib().b200c_poll(ctx.handle, C.byref(p)) == 0
    assert p.stage == 6 and p.bytes_scanned == p.bytes_total == sum(t.compression.data_length for t in tabs)

def test_config2_shape_lcs_l0_l1_snappy(ctx):
    """BASELINE.json configs[2] at reduced scale: LCS L0->L1, 32 overlapping inputs (4 L0 tables over the whole ring + 28 L1 tables
    in 8 disjoint token bands), Snappy in and out, output switched at a fixed on-disk size. Byte parity is against the oracle's
    Snappy restatement (parity with snappy-java itself is unpinned, DESIGN.md §1c)."""
    tabs = synth_tables(0, 32, 0xCA550003, 40000, p=0.25, comp=O.COMP_SNAPPY, band_count=8, l0_count=4)
    kw = dict(max_sstable_bytes=160 * 1024)
    want = CompactionTask(tabs, CompactionController(NOW), **kw).execute(O.OracleEngine(), max_outputs=64)
    got = CompactionTask(tabs, CompactionController(NOW), **kw).execute(GpuEngine(ctx), max_outputs=64)
    assert len(want.outputs) >= 3 and len(got.outputs) == len(want.outputs)
    for g, w in zip(got.outputs, want.outputs):
        assert g.data == w.data and g.index == w.index and g.digest == w.digest and g.compression.chunk_offsets == w.compression.chunk_offsets
        assert g.compression.compressor_name == "SnappyCompressor"
    assert got.stats["merged_row_counts"] == want.stats["merged_row_counts"]

def test_edge_shapes(ctx):
    """ragged and extreme shapes the reference's own tests exercise: empty input file, 65535-byte key, 60 columns with sparse rows,
    8 clustering columns with empty / long components, values larger than a chunk and than column_index_size, single-row tables"""
    rng = random.Random(17)
    # (1) wide schema: 8 clustering columns, 60 regular columns
    s = Schema(["Int32Type", "UTF8Type", "LongType", "BytesType", "Int32Type", "UTF8Type", "LongType", "BytesType"],
               [("c%02d" % i, ("UTF8Type", "LongType", "Int32Type", "DoubleType")[i % 4]) for i in range(60)])
    def val(ci):
        t = ci % 4
        return (rng.choice([b"", b"x" * rng.randint(1, 40)]), struct.pack(">q", rng.getrandbits(50)), I32(rng.randint(-5, 5)), struct.pack(">d", rng.random()))[t]
    def ck():
        return (I32(rng.randint(0, 3)), rng.choice([b"", b"a", b"b" * 70]), struct.pack(">q", rng.randint(-2, 2)), rng.choice([b"", b"\x00", b"\xff\xfe"]),
                I32(rng.randint(0, 1)), rng.choice([b"k", b""]), struct.pack(">q", rng.randint(0, 1)), rng.choice([b"", b"zz"]))
    tables = []
    for t in range(3):
        parts = []
        for k in (b"\x01", b"k" * 65535, b"mid-key", b"another"):
            if rng.random() < 0.3: continue
            rows = {}
            for _ in range(rng.randint(1, 10)):
                c = ck(); cols = rng.sample(range(60), rng.randint(0, 12))
                rows[c] = Row(c, [Cell(ci, 1000 + rng.randint(0, 3), val(ci)) for ci in cols], ts=1000 + rng.randint(0, 3))
            def sk(c):   # clustering order: ints signed, text/bytes unsigned lexicographic
                return (struct.unpack(">i", c[0])[0], c[1], struct.unpack(">q", c[2])[0], c[3], struct.unpack(">i", c[4])[0], c[5], struct.unpack(">q", c[6])[0], c[7])
            parts.append(Partition(k, [rows[c] for c in sorted(rows, key=sk)]))
        if not parts: parts = [Partition(b"\x01", [Row(ck(), [Cell(0, 1000, b"v")], ts=1000)])]
        tables.append(Builder(s, (1000, 0, 0), column_index_size=512).build(parts))
    both(ctx, tables, CompactionController(NOW, 10**9), column_index_size=512)
    # (2) values larger than a chunk / an index block; an input file with no partitions at all
    s2 = Schema(["Int32Type"], [("val", "BytesType")])
    big = Builder(s2, (0, 0, 0)).build([Partition(b"p%d" % i, [Row((I32(j),), [Cell(0, 10 + j, bytes(rng.getrandbits(8) for _ in range(rng.choice([10, 40000, 70000]))))], ts=10 + j) for j in range(3)]) for i in range(4)])
    empty = Builder(s2, (0, 0, 0)).build([])
    one = Builder(s2, (0, 0, 0)).build([Partition(b"p1", [Row((I32(1),), [Cell(0, 99, b"newer")], ts=99)])])
    both(ctx, [big, empty, one], CompactionController(NOW, 10**9))
    both(ctx, [empty, one], CompactionController(NOW, 10**9))
    g, _ = both(ctx, [empty], CompactionController(NOW, 10**9))
    assert g.outputs[0].data == b"" and g.outputs[0].partitions == 0


@pytest.mark.parametrize("ranges", [2, 5, 16])
def test_token_range_streaming_matches_oracle(ctx, ranges, monkeypatch):
    """host-buffer compactions are cut into token-range pieces (Data.db copies, K1, K3-K5 and the read-back overlap piece by piece);
    B200C_RANGES forces the piece count on inputs that would otherwise run as one piece. Every output byte must stay the same."""
    monkeypatch.setenv("B200C_RANGES", str(ranges))
    tabs = synth_tables(0, 6, 0x57E + ranges, 20000)
    got, _ = both(ctx, tabs, CompactionController(NOW))
    assert got.outputs[0].partitions > 1000
    wide = synth_tables(1, 3, 0x57F + ranges, 60, rows_per_partition=600, column_index_size=4096)
    both(ctx, wide, CompactionController(NOW), column_index_size=4096)
    both(ctx, tabs[:1], CompactionController(NOW))                       # single input
    # a token sub-range on top of the pieces
    lo, hi = -(1 << 62), (1 << 61)
    want = CompactionTask(tabs, CompactionController(NOW), token_range=(lo, hi)).execute(O.OracleEngine()).outputs[0]
    g = CompactionTask(tabs, CompactionController(NOW), token_range=(lo, hi)).execute(GpuEngine(ctx)).outputs[0]
    assert g.data == want.data and g.index == want.index and g.digest == want.digest and g.compression.chunk_offsets == want.compression.chunk_offsets

def test_token_range_streaming_tiny_and_empty(ctx, monkeypatch):
    monkeypatch.setenv("B200C_RANGES", "4")
    S1 = Schema(["Int32Type"], [("val", "UTF8Type")]); b = Builder(S1, (0, 0, 0))
    few = b.build([Partition(b"k%d" % i, [Row((I32(1),), [Cell(0, 5, b"v" * (i % 7))], ts=5)]) for i in range(9)])
    both(ctx, [few, few], CompactionController(NOW))
    gone = b.build([Partition(b"k", [], (5, 7))])
    got, _ = both(ctx, [gone], CompactionController(NOW))
    assert got.outputs[0].data == b""


def test_wrong_summary_positions_only_cost_the_sequential_walk(ctx):
    """Summary positions are hints: the Index.db walk is proven against the sequential parse, so garbage hints must not change a byte"""
    import numpy as np
    tabs = synth_tables(0, 3, 0x5AD, 5000)
    for g, t in enumerate(tabs): t.generation = g
    want = CompactionTask(tabs, CompactionController(NOW)).execute(O.OracleEngine()).outputs[0]
    tabs[1].summary_positions = np.asarray([0, 7, 1001, len(tabs[1].index) // 2 + 1], dtype=np.uint64)
    got = CompactionTask(tabs, CompactionController(NOW)).execute(GpuEngine(ctx))
    g = got.outputs[0]
    assert g.data == want.data and g.index == want.index and g.digest == want.digest
    assert got.stats["index_slow_path_inputs"] == 1

@pytest.mark.parametrize("env", [{"B200C_K1_BATCH": "2"}, {"B200C_K1": "0", "B200C_K1_BATCH": "0"}, {"B200C_K1": "2", "B200C_K1_BATCH": "2"}, {"B200C_K5": "3"}, {"B200C_K5": "1"}])
def test_alternate_codec_kernels_match(env):
    """K1 mappings stay selectable for A/B (B200C_K1: 0 = warp per chunk, 1 = thread per chunk for launches of >= 32768 chunks;
    2 = two passes, lz4_batch.cuh; B200C_K1_BATCH: 1 = all inputs' chunk ranges in one launch, 2 = even for tiny launches; B200C_K5: 1 = LZ4 with
    the hash table in shared memory, 3 = two passes, lz4_chain.cuh): parity must hold for all"""
    import subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "tests/test_gpu_codec.py", "tests/test_gpu_compaction.py",
                        "-k", "(test_gpu_codec or golden or synthetic_configs or lcs_wide or streaming_matches) and not alternate"], cwd=root,
                       env=dict(os.environ, **env), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]

# ---- round 2 --------------------------------------------------------------------------------------------------------------------------
def test_wrong_partition_order_is_rejected_whatever_the_file_size(ctx, golden_dir):
    """no small-file exemption: 5 byte-ordered keys declared as a Murmur3 file are out of token order -> ECORRUPT (markSuspect), as the oracle"""
    from cassandra_b200 import native
    s = SSTable.open(_golden(golden_dir, "legacy_oa_simple"))
    s.partitioner = "org.apache.cassandra.dht.Murmur3Partitioner"
    for eng in (GpuEngine(ctx), O.OracleEngine()):
        with pytest.raises(native.CorruptSSTableError):
            CompactionTask([s], CompactionController(NOW), column_index_size=4096).execute(eng)
    # a Murmur3 table fed as ByteOrdered is refused as well
    t = synth_tables(0, 1, 77, 300)[0]; t.partitioner = "org.apache.cassandra.dht.ByteOrderedPartitioner"
    with pytest.raises(native.CorruptSSTableError):
        CompactionTask([t], CompactionController(NOW)).execute(GpuEngine(ctx))

def test_byte_ordered_long_keys_and_ties(ctx):
    """ByteOrderedPartitioner: keys sharing their first 8 bytes are ordered (and merged) on the remaining bytes and the length"""
    S1 = Schema(["Int32Type"], [("val", "UTF8Type")]); b = Builder(S1, (0, 0, 0))
    keys = sorted([b"prefix00", b"prefix00\x00", b"prefix00a", b"prefix00ab", b"prefix0", b"a", b"", b"zzzzzzzzzzzzzzzzzzzz", b"prefix01"])
    def table(sel, ts):
        parts = [Partition(k, [Row((I32(1),), [Cell(0, ts, b"v%d" % ts)], ts=ts)]) for k in keys if k in sel]
        t = b.build(parts)                      # the builder orders by token: rebuild in byte order
        return t
    import sstable_builder as sb
    saved = O.token
    try:
        O.token = lambda k: 0                   # Builder.build sorts by (token, key): constant token = pure byte order
        sb.O.token = O.token
        t1 = table(set(keys[::2]) | {b"prefix00a"}, 5); t2 = table(set(keys[1::2]) | {b"prefix00a", b""}, 6)
    finally:
        O.token = saved; sb.O.token = saved
    for t in (t1, t2): t.partitioner = "org.apache.cassandra.dht.ByteOrderedPartitioner"
    got, want = both(ctx, [t1, t2], CompactionController(NOW))
    assert got.stats["merged_row_counts"][:2] == [len(keys) - 2, 2]

def test_datetype_clustering_is_unsigned_byte_order(ctx):
    from test_oracle_compaction import datetype_tables
    sc, tabs, want = datetype_tables()
    got, _ = both(ctx, tabs, CompactionController(0, 0))
    parts = decode_stream(sc, decompress_output(got.outputs[0]), (0, 0, 0))
    assert [u.ck[0] for u in parts[0].unfiltereds] == want

def test_lcs_switch_counts_only_flushed_chunks(ctx):
    from test_oracle_compaction import lcs_boundary_tables
    sc, t = lcs_boundary_tables(256)
    kw = dict(max_sstable_bytes=1000)
    want = CompactionTask([t], CompactionController(0, 0), **kw).execute(O.OracleEngine(), max_outputs=64)
    got = CompactionTask([t], CompactionController(0, 0), **kw).execute(GpuEngine(ctx), max_outputs=64)
    assert [o.partitions for o in got.outputs] == [o.partitions for o in want.outputs] and len(want.outputs) > 3
    for g, w in zip(got.outputs, want.outputs):
        assert g.data == w.data and g.index == w.index and g.digest == w.digest and g.compression.chunk_offsets == w.compression.chunk_offsets

def test_purge_table_per_token_range(ctx):
    tabs = synth_tables(0, 4, 0xCA551234, 3000)
    cuts = [-(1 << 62), 0, 1 << 62]; base = 1600000000000000
    thr = [base + 500000000, base + 2500000000, (1 << 63) - 1]
    ctl = CompactionController(NOW, overlapping_min_timestamp=base + 1500000000, purge_ranges=list(zip(cuts, thr)))
    got, want = both(ctx, tabs, ctl)
    flat, _ = both(ctx, tabs, CompactionController(NOW, overlapping_min_timestamp=base + 1500000000))
    assert flat.outputs[0].data != got.outputs[0].data

def _big_host_task(n=8, universe=400000):
    tabs = synth_tables(0, n, 0xCA55CA, universe)
    return tabs, CompactionTask(tabs, CompactionController(NOW))

def test_cancel_before_and_during_the_call(ctx):
    """b200c_cancel from another thread: the running call returns ECANCELLED with nothing in flight; a request that lands before the
    call starts is not lost (sticky), and b200c_cancel_reset clears a stale one. The context stays usable."""
    import ctypes as C, threading, time
    from cassandra_b200 import native
    L = native.lib()
    tabs, task = _big_host_task()
    # (1) sticky: cancel first, then call
    L.b200c_cancel(ctx.handle)
    with pytest.raises(native.CompactionInterruptedError):
        task.execute(GpuEngine(ctx))
    # (2) consumed by the call that reported it: the next call runs
    ok = task.execute(GpuEngine(ctx)); want = ok.outputs[0]
    # (3) reset clears a stale request
    L.b200c_cancel(ctx.handle); L.b200c_cancel_reset(ctx.handle)
    again = task.execute(GpuEngine(ctx)); assert again.outputs[0].data == want.data
    # (4) mid-run, from a second thread, at several delays; at least one must land while the call is running
    os.environ["B200C_RANGES"] = "16"
    try:
        interrupted = 0
        for delay in (0.002, 0.01, 0.03, 0.08):
            err = []
            def run():
                try: task.execute(GpuEngine(ctx)); err.append(None)
                except native.CompactionInterruptedError as e: err.append(e)
            th = threading.Thread(target=run); th.start(); time.sleep(delay); L.b200c_cancel(ctx.handle); th.join()
            if err[0] is not None:
                interrupted += 1
                assert err[0].code == native.ECANCELLED
            L.b200c_cancel_reset(ctx.handle)
        assert interrupted >= 1
    finally:
        del os.environ["B200C_RANGES"]
    final = task.execute(GpuEngine(ctx)); assert final.outputs[0].data == want.data and final.outputs[0].digest == want.digest

def test_poll_while_running(ctx):
    """b200c_poll / b200c_poll_inputs from another thread during the call: bytes never decrease, stages advance, per-input positions
    (ISSTableScanner.getCurrentPosition) end at each input's uncompressed length"""
    import ctypes as C, threading, time
    from cassandra_b200 import native
    L = native.lib()
    tabs, task = _big_host_task()
    os.environ["B200C_RANGES"] = "8"
    try:
        seen = []; done = threading.Event()
        def poller():
            p = native.Progress(); pos = (C.c_uint64 * 64)()
            while not done.is_set():
                L.b200c_poll(ctx.handle, C.byref(p)); k = L.b200c_poll_inputs(ctx.handle, pos, 64)
                seen.append((p.bytes_scanned, p.bytes_total, p.stage, tuple(pos[i] for i in range(k)), p.call_seq))
                time.sleep(0.001)
        p0 = native.Progress(); L.b200c_poll(ctx.handle, C.byref(p0))
        th = threading.Thread(target=poller); th.start()
        task.execute(GpuEngine(ctx)); done.set(); th.join()
    finally:
        del os.environ["B200C_RANGES"]
    total = sum(t.compression.data_length for t in tabs)
    run = [s for s in seen if s[4] == p0.call_seq + 1 and s[1] == total]               # (samples before the call still show the previous call: other call_seq)
    assert len(run) >= 3
    assert all(a[0] <= b[0] for a, b in zip(run, run[1:]))
    assert len({s[2] for s in run}) >= 2                       # saw more than one stage
    pos = (C.c_uint64 * 64)(); k = L.b200c_poll_inputs(ctx.handle, pos, 64)
    assert k == len(tabs) and [pos[i] for i in range(k)] == [t.compression.data_length for t in tabs]
    mids = [s[3] for s in run if len(s[3]) == len(tabs) and any(0 < v < t.compression.data_length for v, t in zip(s[3], tabs))]
    assert mids, "never observed an input mid-file"
    for a, b in zip(mids, mids[1:]): assert all(x <= y for x, y in zip(a, b))

def test_more_than_32768_chunks_default_switches(ctx):
    """the thread-per-chunk K1 (k_decompress_multi_thr) engages from 32768 chunks per launch: a byte-for-byte comparison at that
    size with no environment override (6 x 96 MiB = 36864 chunks in the device-resident one-launch path, and the streamed host path)"""
    import synth
    tabs = synth_tables(0, 6, 0xCA55B16, synth.universe_for(0, 96 << 20, 0.5))
    assert sum(len(t.compression.chunk_offsets) for t in tabs) >= 32768
    got, want = both(ctx, tabs, CompactionController(NOW))


# ---- SURVEY §8 f1: the rest of the sstable on the GPU ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["legacy_oa_simple", "legacy_oa_clust"])
def test_golden_filter_summary_statistics(ctx, golden_dir, name):
    """identity compaction on the GPU: Filter.db and Summary.db byte for byte as the Cassandra release wrote them, statistics = the oracle's
    (which tests/test_oracle_compaction.py pins against the golden Statistics.db)"""
    from test_oracle_compaction import golden_meta_task
    base, s, task = golden_meta_task(golden_dir, name)
    got, want = both(ctx, [s], CompactionController(NOW), column_index_size=4096, bloom=task.bloom)
    o = got.outputs[0]
    assert o.filter == open(base + "Filter.db", "rb").read()
    assert o.summary == open(base + "Summary.db", "rb").read()
    assert (o.first_key, o.last_key) == (b"0", b"4")

@pytest.mark.parametrize("ranges", [0, 5])
def test_metadata_matches_oracle_on_synthetic_tables(ctx, ranges, monkeypatch):
    if ranges: monkeypatch.setenv("B200C_RANGES", str(ranges))
    tabs = synth_tables(0, 6, 0x3E7A + ranges, 20000)
    got, want = both(ctx, tabs, CompactionController(NOW), with_metadata=True, min_index_interval=16)
    st = got.outputs[0].stats
    assert st["total_tombstones"] > 0 and len(st["tombstone_drop_times"]) > 0 and st["max_ttl"] > 0
    wide = synth_tables(1, 3, 0x3E7B + ranges, 60, rows_per_partition=400, column_index_size=4096)
    both(ctx, wide, CompactionController(NOW), column_index_size=4096, with_metadata=True)
    both(ctx, tabs, CompactionController(0, 0), with_metadata=True)               # nothing purged: other tombstone / TTL paths

class DeviceEngine:
    """b200c_compact with B200C_FLAG_DEVICE_PTRS: inputs uploaded to HBM first, outputs produced there and read back (the path bench.py's `value` times)"""
    needs_lib_bound = True
    def __init__(self, ctx): self.ctx = ctx
    def __call__(self, manifest, result):
        import ctypes as C
        from cassandra_b200 import native
        L = native.lib(); ctx = self.ctx; allocs = []
        def up(ptr, n):
            d = C.c_void_p(); ctx.check(L.b200c_dev_alloc(ctx.handle, max(n, 1), C.byref(d))); allocs.append(d)
            if n and ptr: ctx.check(L.b200c_memcpy_h2d(ctx.handle, d, ptr, n))
            return d.value
        try:
            host_in = []
            for k in range(manifest.ninputs):
                a = manifest.inputs[k]; host_in.append((a.data, a.index, a.chunk_offsets, a.summary_positions))
                a.data = up(a.data, a.data_len); a.index = up(a.index, a.index_len); a.chunk_offsets = up(a.chunk_offsets, a.nchunks * 8)
                if a.nsummary: a.summary_positions = up(a.summary_positions, a.nsummary * 8)
            host_out = []
            for k in range(result.noutputs_cap):
                o = result.outputs[k]; host_out.append((o.data, o.index, o.chunk_offsets))
                o.data = up(None, o.data_cap); o.index = up(None, o.index_cap); o.chunk_offsets = up(None, o.chunk_cap * 8)
            rc = L.b200c_compact(ctx.handle, C.byref(manifest), C.byref(result), native.FLAG_DEVICE_PTRS)
            for k in range(result.noutputs_cap):
                o = result.outputs[k]; hd, hi, hc = host_out[k]
                if rc == 0 and k < result.noutputs:
                    if o.data_len: ctx.check(L.b200c_memcpy_d2h(ctx.handle, hd, o.data, o.data_len))
                    if o.index_len: ctx.check(L.b200c_memcpy_d2h(ctx.handle, hi, o.index, o.index_len))
                    if o.nchunks: ctx.check(L.b200c_memcpy_d2h(ctx.handle, hc, o.chunk_offsets, o.nchunks * 8))
                o.data, o.index, o.chunk_offsets = hd, hi, hc
            for k in range(manifest.ninputs):
                a = manifest.inputs[k]; a.data, a.index, a.chunk_offsets, a.summary_positions = host_in[k]
            ctx.check(rc, result.corruption)
        finally:
            for d in allocs: L.b200c_dev_free(ctx.handle, d)

def test_device_resident_inputs_whole_ring_and_token_shards(ctx):
    """B200C_FLAG_DEVICE_PTRS (what bench.py's `value` and the sharded multi-GPU run use): the whole ring, and token sub-ranges, for which
    only the Index.db slice between the bracketing Summary.db samples is walked and only the chunks the range crosses are decoded.
    Shards must equal the oracle's and concatenate to the whole-ring output."""
    tabs = synth_tables(0, 5, 0xD37, 30000)
    for g, t in enumerate(tabs): t.generation = g
    want = CompactionTask(tabs, CompactionController(NOW)).execute(O.OracleEngine()).outputs[0]
    got = CompactionTask(tabs, CompactionController(NOW)).execute(DeviceEngine(ctx)).outputs[0]
    assert got.data == want.data and got.index == want.index and got.digest == want.digest and got.compression.chunk_offsets == want.compression.chunk_offsets
    cuts = [-(1 << 63), -(1 << 62) - 12345, -7, (1 << 62) + 99, (1 << 63) - 1]
    stream = b""
    for lo, hi in zip(cuts, cuts[1:]):
        w = CompactionTask(tabs, CompactionController(NOW), token_range=(lo, hi)).execute(O.OracleEngine())
        for eng in (DeviceEngine(ctx), GpuEngine(ctx)):
            g = CompactionTask(tabs, CompactionController(NOW), token_range=(lo, hi)).execute(eng)
            assert g.outputs[0].data == w.outputs[0].data and g.outputs[0].index == w.outputs[0].index and g.outputs[0].digest == w.outputs[0].digest
            assert g.stats["bytes_in_range"] == w.stats["bytes_in_range"] and g.stats["merged_row_counts"] == w.stats["merged_row_counts"]
        stream += decompress_output(w.outputs[0])
    assert stream == decompress_output(want)
    # the same without the slices (A/B switch): identical bytes
    os.environ["B200C_NO_INDEX_SLICES"] = "1"
    try:
        g = CompactionTask(tabs, CompactionController(NOW), token_range=(cuts[1], cuts[2])).execute(GpuEngine(ctx))
        w = CompactionTask(tabs, CompactionController(NOW), token_range=(cuts[1], cuts[2])).execute(O.OracleEngine())
        assert g.outputs[0].data == w.outputs[0].data and g.outputs[0].index == w.outputs[0].index
    finally:
        del os.environ["B200C_NO_INDEX_SLICES"]
    # a range that holds nothing, and one that ends before the first / starts after the last key
    for lo, hi in ((5, 6), (-(1 << 63), -(1 << 63) + 5), ((1 << 63) - 7, (1 << 63) - 1)):
        w = CompactionTask(tabs, CompactionController(NOW), token_range=(lo, hi)).execute(O.OracleEngine())
        g = CompactionTask(tabs, CompactionController(NOW), token_range=(lo, hi)).execute(GpuEngine(ctx))
        assert g.outputs[0].data == w.outputs[0].data and g.outputs[0].partitions == w.outputs[0].partitions


# ---- static rows (SURVEY §8 f3) ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,wide,cis", [(1, False, 2048), (2, False, 65536), (3, True, 1024)])
def test_static_rows_match_oracle(ctx, seed, wide, cis):
    from static_tables import static_tables
    tabs = static_tables(seed, ntables=5, nkeys=400, wide=wide, cis=cis)
    both(ctx, tabs, CompactionController(NOW, 864000), column_index_size=cis, with_metadata=True)
    both(ctx, tabs, CompactionController(NOW, 10**9), column_index_size=cis)
    both(ctx, tabs, CompactionController(NOW, 864000, overlapping_min_timestamp=1015), column_index_size=cis)
    both(ctx, tabs[:1], CompactionController(NOW, 864000), column_index_size=cis)     # one source: the partition deletion still shadows static cells
    both(ctx, tabs[2:3], CompactionController(NOW, 864000), column_index_size=cis)    # no static columns in the only input

def test_static_rows_every_kernel_variant(ctx, monkeypatch):
    from static_tables import static_tables
    many = static_tables(7, ntables=20, nkeys=300, cis=2048)                          # fan-in above 16: the warp-per-partition kernel
    both(ctx, many, CompactionController(NOW, 864000), column_index_size=2048, with_metadata=True)
    tabs = static_tables(8, ntables=6, nkeys=2000, cis=2048)
    for env in ({"B200C_K4_STAGED": "1"}, {"B200C_K4_STAGED": "0"}, {"B200C_RANGES": "5"}, {"B200C_K4_WIDE_WARP": "2048"}):
        for k, v in env.items(): monkeypatch.setenv(k, v)
        both(ctx, tabs, CompactionController(NOW, 864000), column_index_size=2048, with_metadata=True)
        for k in env: monkeypatch.delenv(k)
    # LCS output switching and a token sub-range with static rows
    want = CompactionTask(tabs, CompactionController(NOW), column_index_size=2048, max_sstable_bytes=60000).execute(O.OracleEngine())
    got = CompactionTask(tabs, CompactionController(NOW), column_index_size=2048, max_sstable_bytes=60000).execute(GpuEngine(ctx))
    assert len(got.outputs) == len(want.outputs) > 1
    for g, w in zip(got.outputs, want.outputs): assert g.data == w.data and g.index == w.index and g.digest == w.digest
    lo, hi = -(1 << 62), (1 << 61)
    w = CompactionTask(tabs, CompactionController(NOW), token_range=(lo, hi)).execute(O.OracleEngine()).outputs[0]
    g = CompactionTask(tabs, CompactionController(NOW), token_range=(lo, hi)).execute(GpuEngine(ctx)).outputs[0]
    assert g.data == w.data and g.index == w.index and g.digest == w.digest

# ---- multi-cell (complex) columns (SURVEY §8 f3) ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,ntab,big,cis", [(1, 5, False, 65536), (2, 20, False, 65536), (3, 3, True, 2048), (4, 40, False, 65536)])
def test_complex_columns_match_oracle(ctx, seed, ntab, big, cis):
    """a map, a set and a list beside simple columns: complex deletions, cells merged in cell-path order (TimeUUID order for the list), purge,
    HAS_COMPLEX_DELETION / subset bitmap, statistics; fan-ins up to 40 (the 64-cursor instantiation), wide partitions with a promoted index"""
    from complex_tables import complex_tables
    tabs = complex_tables(seed, ntables=ntab, nkeys=60 if not big else 6, cis=cis, big=big)
    both(ctx, tabs, CompactionController(NOW, 864000), column_index_size=cis, with_metadata=True)
    both(ctx, tabs, CompactionController(NOW, 10 ** 9), column_index_size=cis)          # nothing purgeable
    both(ctx, tabs[:1], CompactionController(NOW, 864000), column_index_size=cis)       # single source: pass-through + purge
    both(ctx, tabs, CompactionController(NOW, 0), column_index_size=cis, with_metadata=True)

def test_complex_columns_streamed_and_sharded(ctx, monkeypatch):
    from complex_tables import complex_tables
    tabs = complex_tables(9, ntables=6, nkeys=2500)
    monkeypatch.setenv("B200C_RANGES", "4")
    both(ctx, tabs, CompactionController(NOW, 864000))
    lo, hi = -(1 << 62), (1 << 61)
    for g, t in enumerate(tabs): t.generation = g
    want = CompactionTask(tabs, CompactionController(NOW), token_range=(lo, hi)).execute(O.OracleEngine()).outputs[0]
    g = CompactionTask(tabs, CompactionController(NOW), token_range=(lo, hi)).execute(GpuEngine(ctx)).outputs[0]
    assert g.data == want.data and g.index == want.index and g.digest == want.digest

# ---- counter columns (SURVEY §8 f3) ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,ntab,big,cis,legacy,static", [(1, 5, False, 65536, True, False), (2, 20, False, 65536, False, False), (3, 3, True, 2048, True, False),
                                                             (4, 40, False, 65536, True, False), (5, 6, False, 65536, True, True), (6, 3, True, 2048, True, True), (7, 24, False, 65536, True, True)])
def test_counter_columns_match_oracle(ctx, seed, ntab, big, cis, legacy, static):
    """counter contexts merged shard by shard (the K-way merge of partition.cuh against the oracle's pairwise fold): global / local / remote rules,
    tombstones and empty values, cells under a deletion left out of the merge, the merged timestamp, hasLegacyCounterShards; fan-ins up to 40"""
    from counter_tables import counter_tables
    tabs = counter_tables(seed, ntables=ntab, nkeys=60 if not big else 6, cis=cis, big=big, legacy=legacy, static=static)      # static: two static counter columns as well
    both(ctx, tabs, CompactionController(NOW, 864000), column_index_size=cis, with_metadata=True)
    both(ctx, tabs, CompactionController(NOW, 10 ** 9), column_index_size=cis)
    both(ctx, tabs[:1], CompactionController(NOW, 864000), column_index_size=cis, with_metadata=True)
    both(ctx, tabs, CompactionController(NOW, 0), column_index_size=cis, with_metadata=True)

@pytest.mark.parametrize("name", ["legacy_oa_simple_counter", "legacy_oa_clust_counter"])
def test_golden_counter_tables(ctx, golden_dir, name):
    """the reference's own counter tables (written by a 5.0 node): identity compaction and the three-way self merge reproduce the files"""
    base = _golden(golden_dir, name)
    s = SSTable.open(base)
    r = CompactionTask([s], CompactionController(NOW), column_index_size=4096).execute(GpuEngine(ctx))
    comp = r.outputs[0].components()
    for c in ("Data.db", "Index.db", "CompressionInfo.db", "Digest.crc32"):
        assert comp[c] == open(base + c, "rb").read(), c
    r3 = CompactionTask([SSTable.open(base, 1), SSTable.open(base, 2), SSTable.open(base, 3)], CompactionController(NOW), column_index_size=4096).execute(GpuEngine(ctx))
    assert r3.outputs[0].components()["Data.db"] == open(base + "Data.db", "rb").read()

def test_counter_columns_streamed_and_unsupported_forms(ctx, monkeypatch):
    from counter_tables import counter_tables, SCTR, ctx as cctx, cid, G, T0
    from cassandra_b200 import native
    tabs = counter_tables(9, ntables=6, nkeys=2500)
    monkeypatch.setenv("B200C_RANGES", "4")
    both(ctx, tabs, CompactionController(NOW, 864000))
    monkeypatch.delenv("B200C_RANGES")
    # a context whose header element meets no shard is not what the reference writes: in a merge the engine refuses it instead of guessing
    odd = struct.pack(">hh", 1, 5) + cid(1) + struct.pack(">qq", 1, 1)
    good = cctx([(cid(1), 2, 2, G)])
    t = [Builder(SCTR).build([Partition(b"k", [Row((struct.pack(">i", 1),), [Cell(0, T0, v)])])]) for v in (odd, good)]
    for g_, tb in enumerate(t): tb.generation = g_
    with pytest.raises(native.UnsupportedError):
        CompactionTask(t, CompactionController(NOW)).execute(GpuEngine(ctx))
    r = CompactionTask(t[:1], CompactionController(NOW)).execute(GpuEngine(ctx))             # alone it passes through untouched, as in the reference
    assert odd in decompress_output(r.outputs[0])
