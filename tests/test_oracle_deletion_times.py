"""Local deletion times of 2^31 and above (expiry after 2038-01-19, INVALID_DELETION_TIME) through the oracle and the K4 source built for the host.
Known answers are written from the Java (cited beside each), the randomised cases are checked against deletion_times.model_compact, byte for byte:
the model's partitions are written by sstable_builder with the merged header and compared with the oracle's Data.db stream."""
import ctypes as C, os, random, shutil, struct, subprocess
import numpy as np, pytest
import oracle_lib as O
from sstable_builder import *
from synth_util import decompress_output
from deletion_times import *
from deletion_times import _pos
from cassandra_b200 import native
from cassandra_b200.db.compaction import CompactionTask, CompactionController, merged_encoding_stats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRACE = 864000
W = 2_300_000_000                                    # expires in 2042: a delta of 2^31 or more against a header minimum of 0
S1 = Schema(["Int32Type"], [("val", "UTF8Type")])
M = COMPLEX.col_index("m")

def run(tables, now=NOW, gc_grace=GRACE, meta=False):
    for g, t in enumerate(tables): t.generation = g
    r = CompactionTask(tables, CompactionController(now, gc_grace), with_metadata=meta).execute(O.OracleEngine())
    o = r.outputs[0]
    return (decompress_output(o) if o.data else b""), r

def table(parts, base=0, schema=S1): return Builder(schema, (0, base, 0)).build(parts)

def parts_of(tables, now=NOW, gc_grace=GRACE, schema=S1):
    raw, r = run(tables, now, gc_grace)
    return decode_output(schema, raw, merged_encoding_stats(tables)), r

def row_of(tables, **kw):
    parts, _ = parts_of(tables, **kw)
    assert len(parts) == 1 and len(parts[0].unfiltereds) == 1, [len(p.unfiltereds) for p in parts]
    return parts[0].unfiltereds[0]

# ---- the rules themselves ----------------------------------------------------------------------------------------------------------------
def test_rules_restate_the_java():
    assert write_delta(W, 0) == W - (1 << 32) and write_delta(W, NOW - 1000) == W - NOW + 1000          # (int) cast: wraps at 2^31
    assert decode_ldt(W - (1 << 32), 600_000_000) == W                                                  # negative: its unsigned value
    assert decode_ldt(5, 600_000_000) == INVALID_DELETION_TIME and decode_ldt(5, EXPIRED_LIVENESS_TTL) == 5
    assert build_dt(7, W - (1 << 32)) == (7, INVALID_DELETION_TIME) and build_dt(7, MAX_DELETION_TIME) == (7, MAX_DELETION_TIME)
    assert build_dt(7, MAX_DELETION_TIME + 1) == (7, INVALID_DELETION_TIME) and build_dt(7, (1 << 32) - 1) == (7, INVALID_DELETION_TIME)
    assert complex_dt(7, W - (1 << 32)) == (7, INVALID_DELETION_TIME)                                   # build runs first: the unsigned repair never fires
    assert as_read(W, 0, "cell", 600_000_000) == W and as_read(W, 0, "deletion") == INVALID_DELETION_TIME and as_read(W, NOW - 1000, "deletion") == W

# ---- one known answer per rule (header minima (0, 0, 0), nowInSec 1.7e9, gc grace 864000 s) --------------------------------------------------
def test_row_liveness_past_2038_stays_live():
    """UnfilteredSerializer.deserializeRowBody :596-598 decodes the liveness ldt as a cell's: the wrapped delta reads as 2.3e9, the row is live"""
    r = row_of([table([Partition(b"k", [Row((I32(1),), [], ts=5, ttl=600_000_000, ldt=W)])])])
    assert (r.ts, r.ttl, r.ldt, r.deletion) == (5, 600_000_000, W, None)

def test_row_deletion_with_a_wrapped_delta_reads_as_invalid_and_is_never_purged():
    """header.readDeletionTime -> DeletionTime.build (DeletionTime.java:54-58): the negative ldt is an InvalidDeletionTime, ldt 2^32 - 2"""
    r = row_of([table([Partition(b"k", [Row((I32(1),), [], deletion=(7, W))])])])
    assert (r.ts, r.deletion) == (NO_TS, (7, INVALID_DELETION_TIME))

def test_the_same_rows_without_a_wrapped_delta_come_out_unchanged():
    rows = [Row((I32(1),), [], ts=5, ttl=600_000_000, ldt=W), Row((I32(2),), [], deletion=(7, W))]
    parts, _ = parts_of([table([Partition(b"k", rows)], base=NOW - 1000)])
    a, b = parts[0].unfiltereds
    assert (a.ts, a.ttl, a.ldt) == (5, 600_000_000, W) and b.deletion == (7, W)

def test_expiring_cell_with_a_wrapped_delta_stays_live():
    """Cell.decodeLocalDeletionTime (Cell.java:221-239, 347): decode_stream alone shows the raw negative read, the rule gives 2.3e9 back"""
    t = table([Partition(b"k", [Row((I32(1),), [Cell(0, 5, b"v", 600_000_000, W)])])])
    raw, _ = run([t])
    assert decode_stream(S1, raw, (0, 0, 0))[0].unfiltereds[0].cells[0].ldt == -1_994_967_296
    c = decode_output(S1, raw, (0, 0, 0))[0].unfiltereds[0].cells[0]
    assert (c.ts, c.ttl, c.ldt, c.value) == (5, 600_000_000, W, b"v")

def test_cell_ldt_below_its_ttl_reads_as_invalid_unless_the_liveness_expired():
    """decodeLocalDeletionTime :234-237: 0 <= ldt < ttl cannot happen without corruption -> INVALID_DELETION_TIME (so: live for ever)"""
    c = row_of([table([Partition(b"k", [Row((I32(1),), [Cell(0, 5, b"v", 600_000_000, 1000)])])])]).cells[0]
    assert (c.ttl, c.ldt, c.value) == (600_000_000, INVALID_DELETION_TIME, b"v")
    r = row_of([table([Partition(b"k", [Row((I32(1),), [Cell(0, 5, b"v")], ts=5, ttl=EXPIRED_LIVENESS_TTL, ldt=NOW - 5)])])], gc_grace=10 ** 9)
    assert (r.ts, r.ttl, r.ldt) == (5, EXPIRED_LIVENESS_TTL, NOW - 5)                               # EXPIRED_LIVENESS_TTL keeps its ldt

def test_range_tombstone_markers_with_wrapped_deltas_read_as_invalid():
    """markers are read with header.readDeletionTime too (UnfilteredSerializer.deserializeMarkerBody :531-536)"""
    us = [Marker(K_INCL_START, (I32(1),), None, (7, W)), Marker(K_INCL_END, (I32(3),), (7, W), None)]
    parts, _ = parts_of([table([Partition(b"k", us)])])
    assert [(m.kind, m.close, m.open) for m in parts[0].unfiltereds] == [(K_INCL_START, None, (7, INVALID_DELETION_TIME)), (K_INCL_END, (7, INVALID_DELETION_TIME), None)]
    # a boundary whose open side is purgeable: the close side (wrapped, INVALID) stays as a bound (PurgeFunction.applyToMarker :117-128)
    old = (8, NOW - 10 ** 7)
    us = [Marker(K_INCL_START, (I32(1),), None, (7, W)), Marker(K_EXCL_END_INCL_START, (I32(3),), (7, W), old), Marker(K_INCL_END, (I32(5),), old, None)]
    parts, _ = parts_of([table([Partition(b"k", us)])])
    assert [(m.kind, m.close, m.open) for m in parts[0].unfiltereds] == [(K_INCL_START, None, (7, INVALID_DELETION_TIME)), (K_EXCL_END, (7, INVALID_DELETION_TIME), None)]

def test_complex_deletion_with_a_wrapped_delta_reads_as_invalid():
    """readComplexColumn (UnfilteredSerializer.java:668-676) takes header.readDeletionTime, i.e. DeletionTime.build: INVALID, not the unsigned value"""
    row = Row((I32(1),), [Cell(M, 9, I32(1), path=b"a")], complex_deletions={M: (7, W)})
    raw, _ = run([table([Partition(b"k", [row])], schema=COMPLEX)])
    want = Row((I32(1),), [Cell(M, 9, I32(1), path=b"a")], complex_deletions={M: (7, INVALID_DELETION_TIME)})
    assert raw == Builder(COMPLEX, (0, 0, 0)).build([Partition(b"k", [want])]).uncompressed
    raw, _ = run([table([Partition(b"k", [row])], base=NOW - 1000, schema=COMPLEX)])                  # no wrap: 2.3e9 as written
    assert raw == Builder(COMPLEX, (0, NOW - 1000, 0)).build([Partition(b"k", [row])]).uncompressed

def test_partition_deletion_is_a_raw_uint32():
    """DeletionTime.Serializer.deserialize (DeletionTime.java:222-243): 12 bytes, the ldt unsigned; 2^31 and above are ordinary times"""
    for ldt in (1 << 31, W, MAX_DELETION_TIME):
        parts, _ = parts_of([table([Partition(b"k", [], deletion=(7, ldt))])])
        assert parts[0].deletion == (7, ldt)
        parts, _ = parts_of([table([Partition(b"k", [], deletion=(7, ldt))])], now=ldt + 10, gc_grace=10)      # gcBefore = ldt: kept
        assert parts[0].deletion == (7, ldt)
        parts, _ = parts_of([table([Partition(b"k", [], deletion=(7, ldt))])], now=ldt + 11, gc_grace=10)      # gcBefore = ldt + 1: purged
        assert parts == []

# ---- purge and liveness boundaries past 2038 ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("now", [(1 << 31) + 1000, 2_200_000_000])
def test_purge_is_strictly_before_gc_before(now):
    gcb = now - GRACE
    for base in (0, gcb - 10):                      # wrapped deltas read as INVALID (never purged); unwrapped ones purge at gcb - 1
        for ldt, purged in ((gcb, False), (gcb - 1, True)):
            wrapped = base == 0 and ldt >= 1 << 31
            t = table([Partition(b"k", [Row((I32(1),), [Cell.tombstone(0, 5, ldt)]), Row((I32(2),), [], deletion=(7, ldt)),
                                        Marker(K_INCL_START, (I32(3),), None, (7, ldt)), Marker(K_INCL_END, (I32(5),), (7, ldt), None)])], base)
            parts, _ = parts_of([t], now=now)
            us = parts[0].unfiltereds if parts else []
            cell = [u for u in us if isinstance(u, Row) and _pos(u.ck) == 1]
            assert bool(cell) != purged and (not cell or cell[0].cells[0].ldt == ldt), (base, ldt)      # cells decode the wrap: the time itself
            dele = [u for u in us if isinstance(u, Row) and _pos(u.ck) == 2]
            marks = [u for u in us if isinstance(u, Marker)]
            if wrapped: assert dele[0].deletion == (7, INVALID_DELETION_TIME) and len(marks) == 2
            else: assert bool(dele) != purged and bool(marks) != purged and (not dele or dele[0].deletion == (7, ldt))

def test_expiry_at_now_and_conversion_to_a_tombstone_below_2038():
    """AbstractCell.isLive: now < ldt; an expired TTL cell becomes a tombstone at ldt - ttl (AbstractCell.purge :88-97)"""
    ldt = (1 << 31) + 5; ttl = MAX_TTL
    for base in (0, NOW):
        for now, live in ((ldt - 1, True), (ldt, False)):
            c = row_of([table([Partition(b"k", [Row((I32(1),), [Cell(0, 5, b"v", ttl, ldt)])])], base)], now=now, gc_grace=10 ** 9).cells[0]
            assert (c.ttl, c.ldt, c.value) == ((ttl, ldt, b"v") if live else (0, ldt - ttl, b"")), (base, now)
            assert live or c.ldt < 1 << 31
    # the tombstone at ldt - ttl is itself purgeable once gcBefore passes it
    parts, _ = parts_of([table([Partition(b"k", [Row((I32(1),), [Cell(0, 5, b"v", ttl, ldt)])])])], now=ldt, gc_grace=ldt - (ldt - ttl) - 1)
    assert parts == []
    # row liveness past 2038: live at ldt - 1, expired (and purged: no other content) at ldt with gcBefore past it
    r = row_of([table([Partition(b"k", [Row((I32(1),), [Cell(0, 5, b"x")], ts=5, ttl=ttl, ldt=ldt)])])], now=ldt - 1)
    assert (r.ts, r.ttl, r.ldt) == (5, ttl, ldt)
    r = row_of([table([Partition(b"k", [Row((I32(1),), [Cell(0, 5, b"x")], ts=5, ttl=ttl, ldt=ldt)])])], now=ldt + 10, gc_grace=5)
    assert (r.ts, len(r.cells)) == (NO_TS, 1)

def test_supersedes_ties_are_decided_on_the_unsigned_ldt():
    """DeletionTime.supersedes (:158-161): equal markedForDeleteAt -> the greater ldt, compared as the widened unsigned value, so 2^31 + 5
    beats 100 (as int32 it would be negative). Headers keep both deltas unwrapped."""
    big, small = (7, (1 << 31) + 5), (7, 100)
    for order in ((big, small), (small, big)):
        tabs = [table([Partition(b"k", [Row((I32(1),), [], deletion=d)])], base=d[1] - 10) for d in order]
        assert row_of(tabs, gc_grace=10 ** 9).deletion == big
        tabs = [table([Partition(b"k", [Marker(K_INCL_START, (I32(1),), None, d), Marker(K_INCL_END, (I32(5),), d, None)])], base=d[1] - 10) for d in order]
        parts, _ = parts_of(tabs, gc_grace=10 ** 9)
        assert [(m.kind, m.close, m.open) for m in parts[0].unfiltereds] == [(K_INCL_START, None, big), (K_INCL_END, big, None)]
        tabs = [table([Partition(b"k", [Row((I32(1),), [Cell(0, 5, b"v")], ts=5)], deletion=d)]) for d in order]
        parts, _ = parts_of(tabs, gc_grace=10 ** 9)
        assert parts[0].deletion == big
    # cells: equal timestamps, both tombstones -> the greater ldt (Cells.reconcile), 2^31 + 5 over 100
    tabs = [table([Partition(b"k", [Row((I32(1),), [Cell.tombstone(0, 5, ldt)])])], base) for ldt, base in (((1 << 31) + 5, 0), (100, 0))]
    assert row_of(tabs, gc_grace=10 ** 9).cells[0].ldt == (1 << 31) + 5

def test_metadata_local_deletion_times_and_drop_times_past_2038():
    """MetadataCollector: min / max local deletion time and the 60 s-rounded drop times (ceilKey) of values of 2^31 and above"""
    t = table([Partition(b"k", [Row((I32(1),), [Cell.tombstone(0, 5, (1 << 31) + 1)]), Row((I32(2),), [Cell(0, 5, b"v", MAX_TTL, W)]),
                                Row((I32(3),), [], deletion=(7, W))], deletion=(3, MAX_DELETION_TIME))])
    raw, r = run([t], meta=True)
    st = r.outputs[0].stats
    want = model_metadata(decode_output(S1, raw, (0, 0, 0)), NOW)
    assert (st["min_local_deletion_time"], st["max_local_deletion_time"], st["tombstone_drop_times"]) == want
    assert want == ((1 << 31) + 1, INVALID_DELETION_TIME, [(2147483700, 1), (2300000040, 1), (4294967340, 2)])     # 2^32 - 3 and 2^32 - 2 share a minute

# ---- randomised against the model ---------------------------------------------------------------------------------------------------------
def _check_model(schema, logical, now, gc_grace):
    tabs = build_tables(schema, logical)
    raw, r = run(tabs, now, gc_grace, meta=True)
    want_parts = expected(schema, logical, now, gc_grace)
    want = Builder(schema, merged_encoding_stats(tabs)).build(want_parts).uncompressed if want_parts else b""
    assert raw == want, "oracle output differs from the model"
    if want_parts:
        st = r.outputs[0].stats
        assert (st["min_local_deletion_time"], st["max_local_deletion_time"], st["tombstone_drop_times"]) == model_metadata(want_parts, now)
    return tabs

CASES = [(seed, schema) for seed in range(20) for schema in ("simple", "static", "complex")]

def case(seed, schema, zero_headers=False):
    rng = random.Random(0xD7 * 1000 + seed)
    sch = {"simple": SIMPLE, "static": STATIC, "complex": COMPLEX}[schema]
    now = NOWS[seed % 4]; gc_grace = rng.choice([0, GRACE, 10 ** 9])
    logical = gen_tables(rng, sch, rng.randint(1, 4), now, now - gc_grace, ranges=schema != "complex" or seed % 2 == 0)
    if zero_headers: logical = [(p, (st[0], 0, 0)) for p, st in logical]
    return sch, logical, now, gc_grace

@pytest.mark.parametrize("seed,schema", CASES)
def test_randomised_against_the_model(seed, schema):
    _check_model(*case(seed, schema))

@pytest.mark.parametrize("seed", range(6))
def test_randomised_with_zero_header_minima(seed):
    for schema in ("simple", "static", "complex"): _check_model(*case(100 + seed, schema, zero_headers=True))

# ---- the K4 source built for the host, on the same tables -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def k4lib():
    if shutil.which("g++") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"): pytest.skip("needs g++ and the CUDA headers")
    out = os.path.join(ROOT, "tests", "native", "_build", "libk4host.so")
    srcs = [os.path.join(ROOT, "tests", "native", "k4_host.cc"), os.path.join(ROOT, "oracle", "codec.cc")]
    deps = srcs + [os.path.join(ROOT, "cassandra_b200", "csrc", f) for f in ("partition.cuh", "common.cuh")] + [os.path.join(ROOT, "include", "b200c.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        r = subprocess.run(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-fno-strict-aliasing", "-I/usr/local/cuda/include", "-Wno-attributes",
                            "-Wno-unknown-pragmas", "-o", out] + srcs, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(out)
    L.k4host_compact.restype = C.c_int
    L.k4host_compact.argtypes = [C.POINTER(native.Manifest), C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                 C.POINTER(C.c_uint64), C.c_char_p, C.c_int]
    return L

def host_k4(L, tables, controller):
    task = CompactionTask(tables, controller)
    m = task.build_manifest()
    total = sum(t.compression.data_length for t in tables)
    ucap = int(total * 1.5) + 4096; icap = sum(len(t.index) for t in tables) * 2 + 4096
    u = np.zeros(ucap, dtype=np.uint8); ix = np.zeros(icap, dtype=np.uint8); ul = C.c_uint64(); il = C.c_uint64(); st = (C.c_uint64 * 3)(); err = C.create_string_buffer(256)
    rc = L.k4host_compact(C.byref(m), u.ctypes.data, ucap, C.byref(ul), ix.ctypes.data, icap, C.byref(il), st, err, 256)
    assert rc == 0, err.value
    return bytes(u[:ul.value]), bytes(ix[:il.value])

def k4_check(L, tables, now, gc_grace):
    for g, t in enumerate(tables): t.generation = g
    w = CompactionTask(tables, CompactionController(now, gc_grace)).execute(O.OracleEngine()).outputs[0]
    data, index = host_k4(L, tables, CompactionController(now, gc_grace))
    assert data == (decompress_output(w) if w.data else b""), "Data stream of the K4 host build differs from the oracle"
    assert index == w.index

def test_k4_host_known_answers(k4lib):
    # the two confirmed cases (live row past 2038, wrapped row deletion), markers, complex deletion, ties, the boundary purge
    k4_check(k4lib, [table([Partition(b"k", [Row((I32(1),), [], ts=5, ttl=600_000_000, ldt=W)])])], NOW, GRACE)
    k4_check(k4lib, [table([Partition(b"k", [Row((I32(1),), [], deletion=(7, W))])])], NOW, GRACE)
    old = (8, NOW - 10 ** 7)
    k4_check(k4lib, [table([Partition(b"k", [Marker(K_INCL_START, (I32(1),), None, (7, W)), Marker(K_EXCL_END_INCL_START, (I32(3),), (7, W), old),
                                             Marker(K_INCL_END, (I32(5),), old, None)])])], NOW, GRACE)
    k4_check(k4lib, [table([Partition(b"k", [Row((I32(1),), [Cell(M, 9, I32(1), path=b"a")], complex_deletions={M: (7, W)})])], schema=COMPLEX)], NOW, GRACE)
    big, small = (7, (1 << 31) + 5), (7, 100)
    for order in ((big, small), (small, big)):
        k4_check(k4lib, [table([Partition(b"k", [Row((I32(1),), [], deletion=d)])], base=d[1] - 10) for d in order], NOW, 10 ** 9)
        k4_check(k4lib, [table([Partition(b"k", [Marker(K_INCL_START, (I32(1),), None, d), Marker(K_INCL_END, (I32(5),), d, None)])], base=d[1] - 10) for d in order], NOW, 10 ** 9)
    now = 2_200_000_000; gcb = now - GRACE
    for ldt in (gcb, gcb - 1):
        k4_check(k4lib, [table([Partition(b"k", [Row((I32(1),), [Cell.tombstone(0, 5, ldt)]), Row((I32(2),), [], deletion=(7, ldt))])], gcb - 10)], now, GRACE)

@pytest.mark.parametrize("seed,schema", CASES[::2])
def test_k4_host_randomised(k4lib, seed, schema):
    sch, logical, now, gc_grace = case(seed, schema)
    k4_check(k4lib, build_tables(sch, logical), now, gc_grace)
