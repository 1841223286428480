"""Local deletion times of 2^31 and above through b200c_compact: every K4 route against the oracle (test_gpu_compaction.both, with the Statistics
side band) and against the model of deletion_times.py. Keys are spread so that each appears in exactly the fan-in a route takes."""
import os, random, subprocess, sys, pytest
import oracle_lib as O
from sstable_builder import Builder
from synth_util import decompress_output
from deletion_times import *
from test_gpu_compaction import both, DeviceEngine
from cassandra_b200.db.compaction import CompactionTask, CompactionController, merged_encoding_stats

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def ctx():
    from cassandra_b200 import native
    c = native.Context(0)
    yield c
    c.close()

SCHEMAS = {"simple": SIMPLE, "static": STATIC, "complex": COMPLEX}

def tables_for(seed, schema, ntables, fanin, nkeys=24, now=None):
    rng = random.Random(0xDE1 * 100 + seed)
    now = now or NOWS[seed % 4]; gc_grace = rng.choice([0, 864000, 10 ** 9])
    logical = gen_tables(rng, SCHEMAS[schema], ntables, now, now - gc_grace, keys=[b"key%03d" % i for i in range(nkeys)], fanin=fanin)
    return SCHEMAS[schema], logical, build_tables(SCHEMAS[schema], logical), now, gc_grace

def check(ctx, schema, logical, tabs, now, gc_grace):
    got, want = both(ctx, tabs, CompactionController(now, gc_grace), with_metadata=True)
    want_parts = expected(schema, logical, now, gc_grace)
    raw = decompress_output(got.outputs[0]) if got.outputs[0].data else b""
    assert raw == (Builder(schema, merged_encoding_stats(tabs)).build(want_parts).uncompressed if want_parts else b""), "GPU output differs from the model"
    if want_parts:
        st = got.outputs[0].stats
        mn, mx, drops = model_metadata(want_parts, now)
        assert (st["min_local_deletion_time"], st["max_local_deletion_time"], st["tombstone_drop_times"]) == (mn, mx, drops)
    return got

# fan-in 1 (TrivialOneToOne: as_is), <= 8, 9-12, 13-16 (thread kernels), above 16 (k_partition_warp)
@pytest.mark.parametrize("ntables,fanin", [(3, 1), (4, 3), (8, 8), (12, 10), (16, 14), (20, 18)])
@pytest.mark.parametrize("schema", ["simple", "static", "complex"])
def test_every_fan_in_route(ctx, ntables, fanin, schema):
    for seed in range(2):
        check(ctx, *tables_for(seed + 10 * fanin, schema, ntables, fanin))

@pytest.mark.parametrize("now", NOWS)
def test_now_past_2038_and_zero_header_minima(ctx, now):
    for schema in SCHEMAS:
        s, logical, _, _, gc_grace = tables_for(7, schema, 5, 3, now=now)
        logical = [(p, (st[0], 0, 0)) for p, st in logical]
        check(ctx, s, logical, build_tables(s, logical), now, gc_grace)

@pytest.mark.parametrize("env", [{"B200C_K4_STAGED": "1"}, {"B200C_K4_WIDE_WARP": "2048"}, {"B200C_RANGES": "5"}])
def test_kernel_variants(ctx, monkeypatch, env):
    for k, v in env.items(): monkeypatch.setenv(k, v)
    for schema in SCHEMAS:
        for ntables, fanin in ((6, 4), (20, 18)):
            check(ctx, *tables_for(3 + fanin, schema, ntables, fanin, nkeys=60))

def test_device_resident_inputs(ctx):
    for schema in SCHEMAS:
        s, logical, tabs, now, gc_grace = tables_for(5, schema, 6, 4, nkeys=40)
        w = CompactionTask(tabs, CompactionController(now, gc_grace)).execute(O.OracleEngine()).outputs[0]
        g = CompactionTask(tabs, CompactionController(now, gc_grace)).execute(DeviceEngine(ctx)).outputs[0]
        assert g.data == w.data and g.index == w.index and g.digest == w.digest
        want_parts = expected(s, logical, now, gc_grace)
        assert decompress_output(g) == Builder(s, merged_encoding_stats(tabs)).build(want_parts).uncompressed

def test_two_pass_mode():
    """B200C_K4_TWO_PASS is read once per process: a child process with it set runs the same tables (the two-pass merge refuses multi-cell columns)"""
    code = '''
import sys; sys.path.insert(0, "tests"); sys.path.insert(0, ".")
import oracle_lib as O
from test_gpu_deletion_times import tables_for
from cassandra_b200 import native
from cassandra_b200.db.compaction import CompactionTask, CompactionController, GpuEngine
with native.Context(0) as ctx:
    for schema in ("simple", "static"):
        for ntables, fanin in ((3, 1), (6, 4), (20, 18)):
            s, logical, tabs, now, gc_grace = tables_for(11 + fanin, schema, ntables, fanin, nkeys=40)
            g = CompactionTask(tabs, CompactionController(now, gc_grace)).execute(GpuEngine(ctx)).outputs[0]
            w = CompactionTask(tabs, CompactionController(now, gc_grace)).execute(O.OracleEngine()).outputs[0]
            assert g.data == w.data and g.index == w.index and g.digest == w.digest, (schema, fanin)
print("ok")
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], cwd=root, env=dict(os.environ, B200C_K4_TWO_PASS="1"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]
