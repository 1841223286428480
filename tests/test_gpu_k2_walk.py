"""K2 with Summary.db samples walks Index.db one Summary interval per thread, in one launch over all inputs, and checks the partition order as
it emits (k_index_walk_count / k_index_walk_emit). B200C_K2_LEGACY=1 keeps the speculate-chain-verify path with its separate order check
selectable: both must produce the same outputs, counters and corruption reports."""
import os, pytest
import oracle_lib as O
from synth_util import synth_tables
from cassandra_b200.io.sstable import SSTable
from cassandra_b200.db.compaction import CompactionTask, CompactionController, GpuEngine

pytestmark = pytest.mark.gpu
NOW = 1700000000

@pytest.fixture(scope="module")
def ctx():
    from cassandra_b200 import native
    c = native.Context(0)
    yield c
    c.close()

def _run(engine, tables, monkeypatch, legacy, **kw):
    if legacy: monkeypatch.setenv("B200C_K2_LEGACY", "1")
    else: monkeypatch.delenv("B200C_K2_LEGACY", raising=False)
    return CompactionTask(tables, CompactionController(NOW), **kw).execute(engine)

def _same(a, b):
    assert len(a.outputs) == len(b.outputs)
    for x, y in zip(a.outputs, b.outputs):
        assert x.data == y.data and x.index == y.index and x.digest == y.digest
        assert x.compression.chunk_offsets == y.compression.chunk_offsets and (x.partitions, x.rows) == (y.partitions, y.rows)
    for k in ("bytes_read", "bytes_in_range", "bytes_written", "total_source_rows", "input_partitions", "merged_row_counts", "index_slow_path_inputs"):
        assert a.stats[k] == b.stats[k], k

CASES = {
    "schema_n_16_inputs": dict(args=(0, 16, 0xB2, 6000), kw={}),
    "schema_w_promoted": dict(args=(1, 4, 0xB3, 80), synth=dict(rows_per_partition=300, column_index_size=4096), kw=dict(column_index_size=4096)),
    "token_range": dict(args=(0, 5, 0xB4, 20000), kw=dict(token_range=(-(1 << 62) - 12345, (1 << 61) + 99))),
    "streamed_pieces": dict(args=(0, 6, 0xB5, 30000), kw={}, env={"B200C_RANGES": "5"}),
}

@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_walk_by_interval_matches_legacy_path(ctx, monkeypatch, case, device):
    from test_gpu_compaction import DeviceEngine
    c = CASES[case]
    if device and "env" in c: pytest.skip("device-resident inputs run as one piece")
    for k, v in c.get("env", {}).items(): monkeypatch.setenv(k, v)
    tabs = synth_tables(*c["args"], **c.get("synth", {}))
    for g, t in enumerate(tabs): t.generation = g
    eng = DeviceEngine(ctx) if device else GpuEngine(ctx)
    new = _run(eng, tabs, monkeypatch, False, **c["kw"])
    old = _run(eng, tabs, monkeypatch, True, **c["kw"])
    _same(new, old)
    assert new.stats["index_slow_path_inputs"] == 0
    want = CompactionTask(tabs, CompactionController(NOW), **c["kw"]).execute(O.OracleEngine())
    assert new.outputs[0].data == want.outputs[0].data and new.outputs[0].index == want.outputs[0].index

def test_walk_by_interval_on_golden_files(ctx, monkeypatch, golden_dir):
    for name in ("legacy_oa_simple", "legacy_oa_clust", "legacy_oa_simple_counter", "legacy_oa_clust_counter"):
        base = os.path.join(golden_dir, "oa", "legacy_tables", name, "oa-1-big-")
        tabs = [SSTable.open(base, 1), SSTable.open(base, 2)]
        _same(_run(GpuEngine(ctx), tabs, monkeypatch, False, column_index_size=4096), _run(GpuEngine(ctx), tabs, monkeypatch, True, column_index_size=4096))

def test_order_errors_are_reported_like_the_legacy_path(ctx, monkeypatch, golden_dir):
    """files in another partitioner's order: the first bad pair (input, Data.db offset) is the same whichever path checks the order"""
    from cassandra_b200 import native
    s = SSTable.open(os.path.join(golden_dir, "oa", "legacy_tables", "legacy_oa_simple", "oa-1-big-"))
    s.partitioner = "org.apache.cassandra.dht.Murmur3Partitioner"
    tabs = synth_tables(0, 3, 0xB6, 3000)
    for t in tabs: t.partitioner = "org.apache.cassandra.dht.ByteOrderedPartitioner"
    for case in ([s], tabs):
        for g, t in enumerate(case): t.generation = g
        seen = []
        for legacy in (False, True):
            with pytest.raises(native.CorruptSSTableError) as e:
                _run(GpuEngine(ctx), case, monkeypatch, legacy)
            cr = e.value.corruption
            seen.append((cr.input, cr.kind, cr.chunk, cr.offset))
        assert seen[0] == seen[1] and seen[0][1] == 3
