"""Local deletion times past 2038: the `oa` reading and writing rules of the reference restated in Python (test helper), a decoder that applies
them to a merged Data.db stream, a logical compaction model and a generator of tables whose deletion times sit on the boundaries that matter.

Since 5.0 (CASSANDRA-14227) a local deletion time is an unsigned 32-bit value: Cell.MAX_DELETION_TIME = 2^32 - 3, INVALID_DELETION_TIME = 2^32 - 2
(S/db/rows/Cell.java:51-55), and a TTL reaches 20 years (Attributes.MAX_TTL). Row bodies store them as deltas against the header's
minLocalDeletionTime, and the writer's (int) cast wraps a delta of 2^31 or more into a negative int, which every reader repairs by its own rule:

  what is read                         rule                                                         Java
  writing any delta                    writeUnsignedVInt32((int) (ldt - min)), sign-extended vint   S/db/SerializationHeader.java:170-173, S/utils/vint/VIntCoding.java:329-332
  reading any delta                    readUnsignedVInt32() (int) + min (long)                      S/db/SerializationHeader.java:191-194
  cell                                 Cell.decodeLocalDeletionTime                                 S/db/rows/Cell.java:221-239, 347
  row primary-key liveness             Cell.decodeLocalDeletionTime                                 S/db/rows/UnfilteredSerializer.java:596-598
  row deletion, range tombstone marker header.readDeletionTime -> DeletionTime.build               S/db/SerializationHeader.java:201-206, S/db/DeletionTime.java:54-58
  complex deletion                     DeletionTime.build, then "negative -> unsigned" (unreachable: S/db/rows/UnfilteredSerializer.java:668-676
                                       build never returns a negative ldt)
  partition deletion                   raw uint32                                                   S/db/DeletionTime.java:222-243
"""
import copy, random, struct
import oracle_lib as O
from sstable_builder import *
from row_model import LIVE_DT, dt_sup, dt_deletes, model_merge, model_purge

MAX_DELETION_TIME = (1 << 32) - 3
INVALID_DELETION_TIME = (1 << 32) - 2
EXPIRED_LIVENESS_TTL = (1 << 31) - 1                 # LivenessInfo.EXPIRED_LIVENESS_TTL
MAX_TTL = 630_720_000                                # Attributes.MAX_TTL: 20 years
NOW = 1_700_000_000
NOWS = (1_700_000_000, (1 << 31) - 1, 1 << 31, 2_200_000_000)

# ---- the rules -----------------------------------------------------------------------------------------------------------------------------
def write_delta(ldt, base):
    """the int the writer stores for ldt against the header minimum: (int) (ldt - min)"""
    return ((ldt - base + (1 << 31)) % (1 << 32)) - (1 << 31)

def read_ldt(delta, base):
    """SerializationHeader.readLocalDeletionTime: the int delta plus the long minimum"""
    return delta + base

def decode_ldt(ldt, ttl):
    """Cell.decodeLocalDeletionTime (messaging version >= 5.0), for cells and for row liveness"""
    if ldt >= ttl: return ldt
    if ldt < 0: return ldt & 0xFFFFFFFF              # deletionTimeUnsignedIntegerToLong((int) ldt)
    if ttl == EXPIRED_LIVENESS_TTL: return ldt
    return INVALID_DELETION_TIME

def build_dt(mfda, ldt):
    """DeletionTime.build: a negative ldt or one above MAX_DELETION_TIME is an InvalidDeletionTime, whose ldt is INVALID_DELETION_TIME"""
    return (mfda, INVALID_DELETION_TIME if ldt < 0 or ldt > MAX_DELETION_TIME else ldt)

def complex_dt(mfda, ldt):
    """readComplexColumn: header.readDeletionTime (build) first, then a negative ldt would be taken as its unsigned value. A deletion stamped
    Long.MIN_VALUE (LIVE, written for a column without one when another column of the row has one) is then dropped by BTreeRow.Builder's
    CellResolver (S/db/rows/BTreeRow.java:770-778): LIVE."""
    if mfda == NO_TS: return LIVE_DT
    d = build_dt(mfda, ldt)
    return (d[0], d[1] & 0xFFFFFFFF) if d[1] < 0 else d

def as_read(ldt, base, rule, ttl=0):
    """the value the reader hands to the merge for a logical ldt the writer stored against `base`"""
    raw = read_ldt(write_delta(ldt, base), base)
    if rule == "cell": return decode_ldt(raw, ttl)
    if rule == "deletion": return build_dt(0, raw)[1]
    if rule == "complex": return complex_dt(0, raw)[1]
    raise ValueError(rule)

def dt_supersedes(a, b):
    """DeletionTime.supersedes: markedForDeleteAt first, then the (unsigned, widened) local deletion time"""
    return a[0] > b[0] or (a[0] == b[0] and a[1] > b[1])

def purgeable(ldt, gc_before): return ldt < gc_before        # DeletionPurger / PurgeFunction: strictly before gcBefore (no overlapping sstables)

# ---- logical partitions as the reader sees them -----------------------------------------------------------------------------------------
def read_partitions(schema, parts, stats):
    """the logical partitions written by Builder(schema, stats), as the reader decodes them (deep copy)"""
    base = stats[1]; out = []
    def row(r, static=False):
        r = copy.deepcopy(r)
        if r.ttl: r.ldt = as_read(r.ldt, base, "cell", r.ttl)
        if r.deletion is not None: r.deletion = (r.deletion[0], as_read(r.deletion[1], base, "deletion"))
        r.complex_deletions = {c: (d[0], as_read(d[1], base, "complex")) for c, d in r.complex_deletions.items()}
        for c in r.cells:
            if c.ldt != NO_DELETION_TIME: c.ldt = as_read(c.ldt, base, "cell", c.ttl)
        return r
    for p in parts:
        us = []
        for u in p.unfiltereds:
            if isinstance(u, Marker):
                f = lambda d: None if d is None else (d[0], as_read(d[1], base, "deletion"))
                us.append(Marker(u.kind, u.ck, f(u.close), f(u.open)))
            else: us.append(row(u))
        out.append(Partition(p.key, us, p.deletion, None if p.static is None else row(p.static, True)))
    return out

def decode_output(schema, data, stats):
    """a merged Data.db stream -> logical partitions with the reading rules applied (sstable_builder.decode_stream returns the raw
    readLocalDeletionTime values: int delta + long minimum). Simple columns only, as decode_stream."""
    parts = decode_stream(schema, data, stats)
    for p in parts:
        rows = [u for u in p.unfiltereds if isinstance(u, Row)] + ([p.static] if p.static is not None else [])
        for r in rows:
            if r.ldt != NO_DELETION_TIME: r.ldt = decode_ldt(r.ldt, r.ttl)
            if r.deletion is not None: r.deletion = build_dt(*r.deletion)
            for c in r.cells:
                if c.ldt != NO_DELETION_TIME: c.ldt = decode_ldt(c.ldt, c.ttl)
        for u in p.unfiltereds:
            if isinstance(u, Marker):
                if u.close is not None: u.close = build_dt(*u.close)
                if u.open is not None: u.open = build_dt(*u.open)
    return parts

# ---- the compaction model ---------------------------------------------------------------------------------------------------------------
def _pos(ck): return struct.unpack(">i", ck[0])[0]
OPEN_OF = {K_EXCL_END_INCL_START: K_INCL_START, K_INCL_END_EXCL_START: K_EXCL_START}      # RangeTombstoneBoundaryMarker.createCorrespondingOpenMarker
CLOSE_OF = {K_EXCL_END_INCL_START: K_EXCL_END, K_INCL_END_EXCL_START: K_INCL_END}         # .createCorrespondingCloseMarker

def _remark(m, close, open_):
    """a marker whose sides may have gone: a boundary left with one side becomes that side's bound, with none it disappears"""
    if close is None and open_ is None: return None
    if m.kind in OPEN_OF:
        if close is None: return Marker(OPEN_OF[m.kind], m.ck, None, open_)
        if open_ is None: return Marker(CLOSE_OF[m.kind], m.ck, close, None)
    return Marker(m.kind, m.ck, close, open_)

class _Static:
    def __init__(self, schema): self.columns = schema.static_columns; self.complex = [False] * len(schema.static_columns)

def model_compact(schema, tables_parts, now, gc_before):
    """tables_parts: per input, its partitions AS READ (read_partitions). Range tombstones: one source's ranges never overlap another's and
    markers sit at odd clustering positions, rows at even ones, so RangeTombstoneMarker.Merger only re-emits each source's markers, less the
    sides the partition deletion covers (UnfilteredRowIterators.MergeReducer :160-168). One source: TrivialOneToOne, rows pass unmerged."""
    keys = {}
    for parts in tables_parts:
        for p in parts: keys.setdefault(p.key, []).append(p)
    out = []
    for key in sorted(keys, key=lambda k: (O.token(k), k)):
        ps = keys[key]; multi = len(ps) > 1
        pdel = LIVE_DT
        for p in ps:
            if p.deletion is not None and dt_sup(p.deletion, pdel): pdel = p.deletion
        # static row: merged against the partition deletion whatever the fan-in (UnfilteredRowIterators.mergeStaticRows :484-505)
        st = None
        svs = [p.static for p in ps if p.static is not None]
        if svs:
            st = model_merge(_Static(schema), svs, pdel)
            if st is not None: st = model_purge(copy.deepcopy(st), now, gc_before)
        # range deletions in force at each even position, per source
        cover = {}                                    # position -> deletion
        markers = []
        for p in ps:
            open_dt = None; last = None
            for u in p.unfiltereds:
                if not isinstance(u, Marker): continue
                pos = _pos(u.ck)
                if open_dt is not None:
                    for x in range(last + 1, pos): cover[x] = open_dt
                keep = lambda d: d if d is not None and (not multi or dt_sup(d, pdel)) else None
                m = _remark(u, keep(u.close), keep(u.open))
                if m is not None and multi and m.close == m.open: m = None      # both sides read the same (e.g. two INVALIDs): the merger emits only on change
                if m is not None: markers.append(m)
                open_dt = u.open; last = pos
        rows = {}
        for p in ps:
            for u in p.unfiltereds:
                if isinstance(u, Row): rows.setdefault(_pos(u.ck), []).append(u)
        us = []
        for pos, vs in rows.items():
            if multi:
                active = pdel
                if pos in cover and dt_sup(cover[pos], active): active = cover[pos]
                m = model_merge(schema, vs, active)
            else: m = vs[0]
            if m is not None: m = model_purge(copy.deepcopy(m), now, gc_before)
            if m is not None: us.append(m)
        for m in markers:                              # PurgeFunction.applyToMarker :108-135
            pm = _remark(m, None if m.close is None or purgeable(m.close[1], gc_before) else m.close,
                         None if m.open is None or purgeable(m.open[1], gc_before) else m.open)
            if pm is not None: us.append(pm)
        us.sort(key=lambda u: _pos(u.ck))
        out_pdel = pdel if pdel != LIVE_DT and not purgeable(pdel[1], gc_before) else None
        if us or st is not None or out_pdel is not None: out.append(Partition(key, us, out_pdel, st))
    return out

def model_metadata(parts, now):
    """MetadataCollector's local-deletion-time reductions over the written partitions (S/io/sstable/metadata/MetadataCollector.java:208-268):
    (min, max, [(drop time rounded up to 60 s (StreamingTombstoneHistogramBuilder.ceilKey), count)]). Non-expiring liveness and live cells count
    as NO_DELETION_TIME in min / max, never in the histogram."""
    vals = []
    def row(r):
        if r.ts != NO_TS: vals.append(r.ldt if r.ttl else NO_DELETION_TIME)
        if r.deletion is not None: vals.append(r.deletion[1])
        vals.extend(d[1] for _, d in sorted(r.complex_deletions.items()))
        vals.extend(c.ldt for c in r.cells)
    for p in parts:
        if p.deletion is not None: vals.append(p.deletion[1])
        if p.static is not None: row(p.static)
        for u in p.unfiltereds:
            if isinstance(u, Marker): vals.extend(d[1] for d in (u.close, u.open) if d is not None)
            else: row(u)
    if not vals: return NO_DELETION_TIME, NO_DELETION_TIME, []
    hist = {}
    for v in vals:
        if v == NO_DELETION_TIME: continue
        k = v if v % 60 == 0 else v + 60 - v % 60
        hist[k] = hist.get(k, 0) + 1
    return min(vals), max(vals), sorted(hist.items())

# ---- the generator ----------------------------------------------------------------------------------------------------------------------
T0 = 1_600_000_000_000_000
SIMPLE = Schema(["Int32Type"], [("a", "UTF8Type"), ("b", "Int32Type")])
STATIC = Schema(["Int32Type"], [("a", "UTF8Type")], static_columns=[("s", "UTF8Type")])
COMPLEX = Schema(["Int32Type"], [("a", "UTF8Type"), ("m", "MapType(UTF8Type,Int32Type)")])
I32 = lambda v: struct.pack(">i", v)

def boundary_ldts(now, gc_before):
    return [(1 << 31) - 1, 1 << 31, (1 << 31) + 1, MAX_DELETION_TIME, INVALID_DELETION_TIME, now - 1, now, now + 1, gc_before - 1, gc_before]

def gen_tables(rng, schema, ntables, now, gc_before, keys=None, fanin=None, ranges=True):
    """logical inputs (per table its partitions, and its header minima). Deletion times come from boundary_ldts, TTLs reach MAX_TTL, header minima
    make the deltas wrap (0, far below) or not (the table's own minimum, one just under 2^31). fanin: every key appears in exactly that many tables."""
    B = [v for v in boundary_ldts(now, gc_before) if 0 <= v <= INVALID_DELETION_TIME]
    keys = keys or [b"k%d" % i for i in range(4)]
    ts = lambda: T0 + rng.randint(0, 6)                   # few distinct timestamps: ties decided on the local deletion time
    member = {k: set(rng.sample(range(ntables), fanin)) if fanin else {t for t in range(ntables) if rng.random() < 0.6} or {rng.randrange(ntables)} for k in keys}
    cx = [i for i, c in enumerate(schema.complex) if c]
    def cell(col, path=None):
        r = rng.random()
        val = I32(rng.randint(0, 9)) if schema.columns[col][1].endswith("Int32Type") and path is None else rng.choice([b"x", b"yy", b""])
        if path is not None: val = I32(rng.randint(0, 9))
        if r < 0.35: return Cell(col, ts(), val, path=path)
        if r < 0.6: return Cell.tombstone(col, ts(), rng.choice(B), path=path)
        return Cell(col, ts(), val or b"v", rng.choice([1, 3600, MAX_TTL]), rng.choice(B), path=path)
    def row(pos):
        cells = []
        for col in range(len(schema.columns)):
            if col in cx:
                for k in sorted({rng.choice([b"a", b"b", b"c"]) for _ in range(rng.randint(0, 2))}): cells.append(cell(col, k))
            elif rng.random() < 0.6: cells.append(cell(col))
        r = Row((I32(pos),), cells)
        x = rng.random()
        if x < 0.5: r.ts = ts()
        elif x < 0.75:
            r.ts = ts(); r.ldt = rng.choice(B); r.ttl = rng.choice([1, 3600, MAX_TTL])
        elif x < 0.8:
            r.ts = ts(); r.ttl = EXPIRED_LIVENESS_TTL; r.ldt = rng.choice([now - 5, now - 10 ** 7])       # an expired-liveness row (view)
        if rng.random() < 0.25: r.deletion = (ts(), rng.choice(B))
        for col in cx:
            if rng.random() < 0.3: r.complex_deletions[col] = (ts(), rng.choice(B))
        if r.ts == NO_TS and r.deletion is None and not r.cells and not r.complex_deletions: r.ts = ts()
        return r
    tables = [[] for _ in range(ntables)]
    for key in sorted(keys, key=lambda k: (O.token(k), k)):
        owners = sorted(member[key])
        lanes = {t: (20 * i, 20 * i + 19) for i, t in enumerate(owners)}      # each owner's range tombstones stay inside its own lane
        for t in range(ntables):
            if t not in member[key]: continue
            us = [row(2 * rng.randint(0, 4 * len(owners) + 10)) for _ in range(rng.randint(1, 4))]
            us = list({_pos(u.ck): u for u in us}.values())
            if ranges and rng.random() < 0.5:
                lo, hi = lanes[t]; a = lo + 1; b = a + 2 * rng.randint(1, 4); c = b + 2 * rng.randint(1, 3)
                d1 = (ts(), rng.choice(B)); d2 = (ts(), rng.choice(B))
                if d2 == d1: d2 = (d1[0] + 1, d1[1])
                if rng.random() < 0.5:
                    us += [Marker(rng.choice((K_INCL_START, K_EXCL_START)), (I32(a),), None, d1), Marker(rng.choice((K_INCL_END, K_EXCL_END)), (I32(b),), d1, None)]
                else:
                    us += [Marker(K_INCL_START, (I32(a),), None, d1), Marker(rng.choice((K_EXCL_END_INCL_START, K_INCL_END_EXCL_START)), (I32(b),), d1, d2),
                           Marker(K_INCL_END, (I32(c),), d2, None)]
            us.sort(key=lambda u: _pos(u.ck))
            st = None
            if schema.static_columns and rng.random() < 0.7: st = Row((), [Cell(0, ts(), b"s")] if rng.random() < 0.5 else [Cell.tombstone(0, ts(), rng.choice(B))])
            pdel = (ts(), rng.choice(B + [now - 10 ** 7])) if rng.random() < 0.2 else None
            tables[t].append(Partition(key, us, pdel, st))
    out = []
    for parts in tables:
        ldts = table_ldts(parts)
        base = rng.choice([0, 1000, (1 << 31) - 5, min(ldts) if ldts else 0])
        out.append((parts, (T0 - 10, base, 0)))
    return out

def table_ldts(parts):
    vals = []
    for p in parts:
        for u in p.unfiltereds + ([p.static] if p.static is not None else []):
            if isinstance(u, Marker): vals += [d[1] for d in (u.close, u.open) if d is not None]; continue
            if u.ttl: vals.append(u.ldt)
            if u.deletion is not None: vals.append(u.deletion[1])
            vals += [d[1] for d in u.complex_deletions.values()]
            vals += [c.ldt for c in u.cells if c.ldt != NO_DELETION_TIME]
    return vals

def build_tables(schema, logical, cis=65536):
    """Builder-written tables of gen_tables' output (generation = position)"""
    tabs = []
    for g, (parts, stats) in enumerate(logical):
        t = Builder(schema, stats, column_index_size=cis).build(parts); t.generation = g; tabs.append(t)
    return tabs

def expected(schema, logical, now, gc_grace):
    """the model's merged partitions for gen_tables' output"""
    return model_compact(schema, [read_partitions(schema, parts, st) for parts, st in logical], now, now - gc_grace)
