"""Multi-cell (complex) columns — non-frozen map / set / list — through the oracle: known answers and a randomised comparison with an independent
Python restatement of the reference's rules (this file), both written from the Java, not from oracle/compaction.cc:
  Row.Merger.merge / ColumnDataReducer.getReduced   S/db/rows/Row.java:730-781, 838-883   (complex deletion vs active deletion, cells merged in cell-path order)
  CellReducer                                        S/db/rows/Row.java:893-918
  ComplexColumnData.purge / Builder.build            S/db/rows/ComplexColumnData.java:212-216, 350-356
  UnfilteredSerializer.serialize / writeComplexColumn S/db/rows/UnfilteredSerializer.java:151-186, 213-280   (HAS_COMPLEX_DELETION, HAS_ALL_COLUMNS, subset bitmap)
  Cell.Serializer.serialize                          S/db/rows/Cell.java:268-305   (the path precedes the value)
  AbstractTimeUUIDType.compareCustom                 S/db/marshal/AbstractTimeUUIDType.java:58-87   (list cell paths)
No reference-held `oa` fixture carries a multi-cell column: the expected outputs are produced by sstable_builder.py from the model's rows and compared
with the oracle's Data.db bytes. The reference's own known answers for such rows — RowsTest.merge and mergeComplexDeletionSupersededByRowDeletion
(T/unit/org/apache/cassandra/db/rows/RowsTest.java:460-508) — are the last two tests."""
import random, struct, pytest
import oracle_lib as O
from sstable_builder import *
from cassandra_b200.db.compaction import CompactionTask, CompactionController, merged_encoding_stats

NOW = 1700000000
I32 = lambda v: struct.pack(">i", v)
I64 = lambda v: struct.pack(">q", v)
SM = Schema(["Int32Type"], [("a", "UTF8Type"), ("m", "MapType(UTF8Type,Int32Type)"), ("s", "SetType(LongType)")])
A, M, S_ = 0, 1, 2

def raw_of(t):
    o = t
    return b"".join(O.chunk_decompress(O.COMP_LZ4, o.data[a:(b if b else len(o.data)) - 4], 16384)
                    for a, b in zip(o.compression.chunk_offsets, o.compression.chunk_offsets[1:] + [None]))

def oracle_compact(tables, now=NOW, gc_grace=864000):
    for g, t in enumerate(tables): t.generation = g
    r = CompactionTask(tables, CompactionController(now, gc_grace)).execute(O.OracleEngine())
    return raw_of(r.outputs[0]) if r.outputs and r.outputs[0].data else b""

# ---- the model: row merge and purge (row_model.py), partitions here --------------------------------------------------------------
from row_model import LIVE_DT, dt_sup, dt_deletes, live_sup, reconcile, timeuuid_key, path_key, model_merge, model_purge

def model_compact(schema, tables_parts, now=NOW, gc_grace=864000):
    """tables_parts: per table the list of Partitions (no range tombstones, no static rows here)"""
    keys = {}
    for parts in tables_parts:
        for p in parts: keys.setdefault(p.key, []).append(p)
    out = []
    for key in sorted(keys, key=lambda k: (O.token(k), k)):
        ps = keys[key]
        pdel = LIVE_DT
        for p in ps:
            if p.deletion is not None and not dt_sup(pdel, p.deletion): pdel = p.deletion
        cks = sorted({u.ck for p in ps for u in p.unfiltereds}, key=lambda ck: struct.unpack(">i", ck[0])[0])
        rows = []
        for ck in cks:
            vs = [u for p in ps for u in p.unfiltereds if u.ck == ck]
            m = model_merge(schema, vs, pdel if len(ps) > 1 else LIVE_DT) if len(ps) > 1 else vs[0]
            if m is not None:
                import copy
                m = model_purge(copy.deepcopy(m), now, now - gc_grace)
            if m is not None: rows.append(m)
        out_pdel = pdel if pdel != LIVE_DT and not (pdel[1] < now - gc_grace) else None
        if rows or out_pdel is not None: out.append(Partition(key, rows, out_pdel))
    return out

def check(schema, tables_parts, stats_list=None, now=NOW, gc_grace=864000):
    tabs = [Builder(schema, (st if st else (TIMESTAMP_EPOCH, DELETION_TIME_EPOCH, 0))).build(parts) for parts, st in zip(tables_parts, stats_list or [None] * len(tables_parts))]
    got = oracle_compact(tabs, now, gc_grace)
    want_parts = model_compact(schema, tables_parts, now, gc_grace)
    want = raw_of(Builder(schema, merged_encoding_stats(tabs)).build(want_parts)) if want_parts else b""
    assert got == want
    return got

T0 = 1_600_000_000_000_000
def mcell(k, v, ts, **kw): return Cell(M, ts, I32(v), path=k, **kw)
def scell(e, ts, **kw): return Cell(S_, ts, b"", path=I64(e), **kw)

def test_union_and_reconcile_by_path():
    t1 = [Partition(b"k", [Row((I32(1),), [Cell(A, T0, b"x"), mcell(b"a", 1, T0), mcell(b"c", 3, T0)], ts=T0)])]
    t2 = [Partition(b"k", [Row((I32(1),), [mcell(b"a", 9, T0 + 5), mcell(b"b", 2, T0 + 5), scell(-7, T0 + 5), scell(4, T0 + 5)], ts=T0 + 5)])]
    raw = check(SM, [t1, t2])
    assert raw.count(b"\x00\x00\x00\x09") == 1 and b"\x00\x00\x00\x01" not in raw.replace(I32(1), b"", 1)      # a -> 9 won, 1 only as the clustering value

def test_complex_deletion_shadows_older_cells_and_is_kept():
    t1 = [Partition(b"k", [Row((I32(1),), [mcell(b"a", 1, T0), mcell(b"b", 2, T0 + 20), scell(1, T0)], ts=T0)])]
    t2 = [Partition(b"k", [Row((I32(1),), [mcell(b"z", 5, T0 + 11)], complex_deletions={M: (T0 + 10, NOW - 5)})])]
    check(SM, [t1, t2])                                             # a (ts <= deletion) goes, b and z stay; flag 0x40: the set's column carries a LIVE deletion

def test_row_deletion_supersedes_the_complex_deletion():
    t1 = [Partition(b"k", [Row((I32(1),), [mcell(b"a", 1, T0 + 50), mcell(b"b", 1, T0 + 5)], complex_deletions={M: (T0 + 10, NOW - 5)})])]
    t2 = [Partition(b"k", [Row((I32(1),), [], deletion=(T0 + 20, NOW - 5))])]
    check(SM, [t1, t2])                                             # the complex deletion is dropped, only a (ts > row deletion) survives

def test_deletion_only_column_and_single_source_pass_through():
    t1 = [Partition(b"k", [Row((I32(1),), [Cell(A, T0, b"x")], complex_deletions={S_: (T0 + 1, NOW - 5)}),
                           Row((I32(2),), [scell(3, T0)], complex_deletions={M: (T0 + 1, NOW - 5)})])]
    check(SM, [t1])                                                 # TrivialOneToOne: untouched but for the purge
    t2 = [Partition(b"k", [Row((I32(1),), [scell(8, T0 + 2)])])]
    check(SM, [t1, t2])

def test_purge_of_complex_deletions_and_cells():
    old = NOW - 20 * 86400
    t1 = [Partition(b"k", [Row((I32(1),), [mcell(b"a", 1, T0, ttl=100, ldt=old), mcell(b"b", 2, T0 + 30), Cell.tombstone(M, T0 + 30, old, path=b"c")],
                               complex_deletions={M: (T0 + 10, old)})]),
          Partition(b"l", [Row((I32(1),), [], complex_deletions={S_: (T0 + 10, old)})])]
    t2 = [Partition(b"k", [Row((I32(1),), [mcell(b"d", 4, T0 + 40, ttl=1000, ldt=NOW + 900)])])]
    check(SM, [t1, t2])                                             # purgeable deletion -> gone, partition l disappears, expired cell a was shadowed, tombstone c purged
    check(SM, [t1, t2], gc_grace=10 ** 9)                           # nothing purgeable: deletions stay, expired cell becomes a tombstone with its path

def test_list_paths_order_by_timeuuid_time_not_by_bytes():
    SL = Schema(["Int32Type"], [("l", "ListType(UTF8Type)")])
    def tu(ts100ns, node): return struct.pack(">IHHQ", ts100ns & 0xFFFFFFFF, (ts100ns >> 32) & 0xFFFF, 0x1000 | ((ts100ns >> 48) & 0x0FFF), node)
    p1, p2, p3 = tu(0x0000_0001_FFFF_FFFF, 0x8000000000000001), tu(0x0000_0002_0000_0000, 0x8000000000000001), tu(0x0000_0002_0000_0000, 0x80FF000000000001)
    assert p2 < p1                                                  # byte order would put p2 first; time order puts p1 first
    t1 = [Partition(b"k", [Row((I32(1),), [Cell(0, T0, b"one", path=p1)], ts=T0)])]
    assert timeuuid_key(p3) < timeuuid_key(p2)                     # equal timestamps: the other 8 bytes compare as SIGNED bytes (0xFF < 0x00)
    t2 = [Partition(b"k", [Row((I32(1),), [Cell(0, T0 + 1, b"three", path=p3), Cell(0, T0 + 1, b"two", path=p2)], ts=T0 + 1)])]
    raw = check(SL, [t1, t2])
    assert raw.index(b"one") < raw.index(b"three") < raw.index(b"two")

def test_randomised_against_the_model():
    rng = random.Random(0xC0113C7)
    for it in range(60):
        ntab = rng.randint(1, 4); tables = []
        for t in range(ntab):
            parts = []
            for key in sorted({b"k%d" % rng.randint(0, 4) for _ in range(3)}, key=lambda k: (O.token(k), k)):
                rows = []
                for ck in sorted({rng.randint(0, 3) for _ in range(3)}):
                    cells = []
                    if rng.random() < 0.5: cells.append(Cell(A, T0 + rng.randint(0, 40), rng.choice([b"", b"x", b"yy"])))
                    for k in sorted({rng.choice([b"a", b"b", b"c", b"dd"]) for _ in range(rng.randint(0, 3))}):
                        r = rng.random(); ts = T0 + rng.randint(0, 40)
                        if r < 0.7: cells.append(mcell(k, rng.randint(0, 9), ts))
                        elif r < 0.85: cells.append(Cell.tombstone(M, ts, NOW - rng.choice([5, 30 * 86400]), path=k))
                        else: cells.append(mcell(k, 1, ts, ttl=50, ldt=NOW + rng.choice([-30 * 86400, -100, 500])))
                    for e in sorted({rng.randint(-3, 3) for _ in range(rng.randint(0, 3))}): cells.append(scell(e, T0 + rng.randint(0, 40)))
                    cd = {}
                    if rng.random() < 0.3: cd[M] = (T0 + rng.randint(0, 40), NOW - rng.choice([5, 30 * 86400]))
                    if rng.random() < 0.15: cd[S_] = (T0 + rng.randint(0, 40), NOW - rng.choice([5, 30 * 86400]))
                    dele = (T0 + rng.randint(0, 40), NOW - rng.choice([5, 30 * 86400])) if rng.random() < 0.1 else None
                    ts = T0 + rng.randint(0, 40) if (rng.random() < 0.7 or not (cells or cd or dele)) else NO_TS
                    rows.append(Row((I32(ck),), cells, ts=ts, deletion=dele, complex_deletions=cd))
                parts.append(Partition(key, rows, (T0 + rng.randint(0, 40), NOW - 5) if rng.random() < 0.1 else None))
            tables.append(parts)
        check(SM, tables, gc_grace=rng.choice([864000, 10 ** 9, 0]))

# ---- the reference's own known answers for rows with a multi-cell column (T/unit/org/apache/cassandra/db/rows/RowsTest.java) ------------------------------
# Table kcvm there: clustering c, regular v, m map<..>, (:60-66; IntegerType there, Int32Type here — the cases do not depend on the value comparison).
SKV = Schema(["Int32Type"], [("v", "Int32Type"), ("m", "MapType(Int32Type,Int32Type)")])
def _expect_rows(tables_parts, want_rows, schema=SKV):
    tabs = [Builder(schema).build(p) for p in tables_parts]
    got = oracle_compact(tabs, NOW, 10 ** 9)
    want = raw_of(Builder(schema, merged_encoding_stats(tabs)).build([Partition(b"k", want_rows)])) if want_rows else b""
    assert got == want

def test_reference_rows_merge_with_complex_deletion():
    """RowsTest.merge :460-489: the update's value and map cell win, its complex deletion shadows the existing map cell"""
    now1, now2 = NOW - 100, NOW - 99; ts1, ts2 = now1 * 1000000, now2 * 1000000
    existing = Row((I32(1),), [Cell(0, ts1, I32(1)), Cell(1, ts1, I32(1), path=I32(1))], ts=ts1, complex_deletions={1: (ts1 - 1, now1)})     # createBuilder(c1, now1, BB1, BB1, BB1) :222-238
    update = Row((I32(1),), [Cell(0, ts2, I32(2)), Cell(1, ts2, I32(2), path=I32(1))], ts=ts2, complex_deletions={1: (ts2 - 1, now2)})
    merged = Row((I32(1),), [Cell(0, ts2, I32(2)), Cell(1, ts2, I32(2), path=I32(1))], ts=ts2, complex_deletions={1: (ts2 - 1, now2)})
    _expect_rows([[Partition(b"k", [existing])], [Partition(b"k", [update])]], [merged])

def test_reference_complex_deletion_superseded_by_row_deletion():
    """RowsTest.mergeComplexDeletionSupersededByRowDeletion :491-508: the row deletion stays, no complex deletion, no cells"""
    now1 = NOW - 100; now3 = now1 + 2; ts1 = now1 * 1000000
    existing = Row((I32(1),), [Cell(1, ts1, I32(2), path=I32(2))], ts=ts1, complex_deletions={1: (ts1 - 1, now1)})                           # createBuilder(c1, now1, null, BB2, BB2)
    update = Row((I32(1),), [], deletion=(now3 * 1000000, now3))
    _expect_rows([[Partition(b"k", [existing])], [Partition(b"k", [update])]], [Row((I32(1),), [], deletion=(now3 * 1000000, now3))])
