"""The reference's row-level merge and purge rules restated in Python, independently of oracle/compaction.cc (test helper):
  Row.Merger.merge / ColumnDataReducer.getReduced   S/db/rows/Row.java:730-781, 838-883
  CellReducer / Cells.reconcile                      S/db/rows/Row.java:893-918, S/db/rows/Cells.java:58-120
  LivenessInfo.supersedes, DeletionTime.supersedes   S/db/LivenessInfo.java:216-225, S/db/DeletionTime.java:158-161
  BTreeRow.purge / AbstractCell.purge                S/db/rows/BTreeRow.java:457-499, S/db/rows/AbstractCell.java:78-99
  ComplexColumnData.purge / Builder.build            S/db/rows/ComplexColumnData.java:212-216, 350-356
Values are logical (as the reader hands them to the merge): local deletion times are plain integers, unsigned 32-bit in range."""
import struct
from sstable_builder import Row, Cell, NO_TS, NO_DELETION_TIME, MARSHAL

LIVE_DT = (NO_TS, NO_DELETION_TIME)
def dt_sup(a, b): return a[0] > b[0] or (a[0] == b[0] and a[1] > b[1])              # DeletionTime.supersedes
def dt_deletes(d, ts): return ts <= d[0]
def live_sup(a, b):                                                                  # LivenessInfo.supersedes on (ts, ttl, ldt); EMPTY = (NO_TS, 0, NO_DEL)
    if a[0] != b[0]: return a[0] > b[0]
    ae, be = a[1] == 0x7FFFFFFF, b[1] == 0x7FFFFFFF
    if ae != be: return ae
    if (a[1] != 0) == (b[1] != 0): return a[2] > b[2]
    return a[1] != 0
def reconcile(l, r):                                                                 # Cells.reconcile
    if l.ts != r.ts: return l if l.ts > r.ts else r
    le, re_ = l.ldt != NO_DELETION_TIME, r.ldt != NO_DELETION_TIME
    if le or re_:
        if le != re_: return l if le else r
        lt, rt = l.ttl == 0, r.ttl == 0
        if lt != rt: return l if lt else r
        if l.ldt != r.ldt: return l if l.ldt > r.ldt else r
    return l if l.value >= r.value else r
def timeuuid_key(b):
    msb, lsb = struct.unpack(">QQ", b)
    re = ((msb << 48) | ((msb << 16) & 0xFFFF00000000) | (msb >> 32)) & ((1 << 64) - 1)
    sgn = lambda x: x - (1 << 64) if x >= 1 << 63 else x
    return (sgn(re), sgn(lsb ^ 0x0080808080808080))
def path_key(schema, col):
    t = schema.columns[col][1]
    if "ListType" in t: return timeuuid_key
    inner = t.split("(", 1)[1]
    if inner.startswith(MARSHAL + "LongType") or inner.startswith(MARSHAL + "Int32Type") or inner.startswith("LongType") or inner.startswith("Int32Type"):
        return lambda b: int.from_bytes(b, "big", signed=True)
    return lambda b: b

def model_merge(schema, versions, active):
    """versions: Rows of one clustering in source order; active: the deletion in force around them. Returns the merged Row or None."""
    if len(versions) == 1 and active == LIVE_DT: return versions[0]
    info, dele = (NO_TS, 0, NO_DELETION_TIME), LIVE_DT
    for v in versions:
        vi = (v.ts, v.ttl, v.ldt)
        if live_sup(vi, info): info = vi
        vd = v.deletion or LIVE_DT
        if dt_sup(vd, dele): dele = vd
    if dt_sup(dele, active): active = dele
    else: dele = LIVE_DT
    if dt_deletes(active, info[0]): info = (NO_TS, 0, NO_DELETION_TIME)
    out = Row(versions[0].ck, [], info[0], info[1], info[2], None if dele == LIVE_DT else dele)
    for col in range(len(schema.columns)):
        if not schema.complex[col]:
            m = None
            for v in versions:
                for c in v.cells:
                    if c.col == col and not dt_deletes(active, c.ts): m = c if m is None else reconcile(m, c)
            if m is not None: out.cells.append(m)
            continue
        cd = LIVE_DT
        for v in versions:
            d = v.complex_deletions.get(col, LIVE_DT)
            if dt_sup(d, cd): cd = d
        cell_del = active
        if dt_sup(cd, active): cell_del = cd; out.complex_deletions[col] = cd
        key = path_key(schema, col); by_path = {}
        for v in versions:
            for c in v.cells:
                if c.col == col and not dt_deletes(cell_del, c.ts):
                    k = key(c.path); by_path[k] = c if k not in by_path else reconcile(by_path[k], c)
        out.cells += [by_path[k] for k in sorted(by_path)]
    if out.ts == NO_TS and out.deletion is None and not out.cells and not out.complex_deletions: return None
    return out

def model_purge(row, now, gc_before):
    def purgeable(ts, ldt): return ldt < gc_before
    info_live = row.ts != NO_TS and not (row.ttl == 0x7FFFFFFF) and (row.ttl == 0 or now < row.ldt)
    if row.ts != NO_TS and not info_live and purgeable(row.ts, row.ldt): row.ts, row.ttl, row.ldt = NO_TS, 0, NO_DELETION_TIME
    if row.deletion is not None and purgeable(*row.deletion): row.deletion = None
    kept = []
    for c in row.cells:
        live = c.ldt == NO_DELETION_TIME or (c.ttl != 0 and now < c.ldt)
        if not live:
            if purgeable(c.ts, c.ldt): continue
            if c.ttl != 0:
                c = Cell(c.col, c.ts, b"", 0, c.ldt - c.ttl, c.path)
                if purgeable(c.ts, c.ldt): continue
        kept.append(c)
    row.cells = kept
    row.complex_deletions = {k: d for k, d in row.complex_deletions.items() if not purgeable(*d)}
    if row.ts == NO_TS and row.deletion is None and not row.cells and not row.complex_deletions: return None
    return row
