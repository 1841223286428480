"""K2 walks Index.db through a window of aligned 16-byte loads (IdxCursor / iw_entry, index_walk.cuh), which reads up to 15 bytes past the
entries it parses. Here that reader runs on the CPU under AddressSanitizer against a byte-wise parse with idx_entry's checks, over buffers
that end exactly IW_PAD bytes past the input: the golden `oa` Index.db files, synthetic ones of schema N and W (promoted index entries)
and random ones must parse entry for entry the same, damaged and truncated copies must stop both parsers at the same offset, and the
window's Murmur3 must equal the oracle's for keys of every length 0..80."""
import glob, os, shutil, subprocess, pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

def _index_files(tmp_path):
    """(path, Data.db length) pairs: the golden `oa` tables and synthetic schema N / W tables"""
    import synth
    from cassandra_b200.io.sstable import SSTable
    out = []
    for p in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "legacy-sstables", "oa", "legacy_tables", "*", "oa-1-big-Index.db"))):
        t = SSTable.open(p[:-len("Index.db")])
        out.append((p, t.compression.data_length))
    for schema, universe, rpp, cis in ((0, 6000, 1000, 65536), (1, 40, 600, 4096)):
        raw = synth.generate_raw(schema, 0, 2, 0x1D3A + schema, universe, 0.5, rows_per_partition=rpp, column_index_size=cis, threads=4)
        p = str(tmp_path / ("synth%d-Index.db" % schema))
        open(p, "wb").write(raw["index"])
        out.append((p, len(raw["stream"])))
    return out

@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_index_walk_reads_match_the_bytewise_parse(tmp_path):
    exe = str(tmp_path / "index_walk_host")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=address", "-fno-omit-frame-pointer", "-fno-strict-aliasing",
           "-Wno-unknown-pragmas", "-o", exe, os.path.join(ROOT, "tests", "native", "index_walk_host.cc"), os.path.join(ROOT, "oracle", "codec.cc")]
    b = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert b.returncode == 0, b.stderr[-2000:]
    files = _index_files(tmp_path)
    assert len(files) >= 6
    args = [exe, "200"] + [str(x) for pair in files for x in pair]
    r = subprocess.run(args, capture_output=True, text=True, timeout=900, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1"))
    assert r.returncode == 0 and "index_walk_host ok" in r.stdout, (r.stdout + r.stderr)[-3000:]
    assert "runtime error" not in r.stderr, r.stderr[-3000:]
