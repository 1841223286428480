"""K1 reads device-resident inputs where the caller keeps them, and a caller's buffer may end exactly at its last byte. The chunks
near the end of a file are therefore read from a staged copy of the file's tail (k1_src / k1_tail_window, k1_tail.cuh). Here K1's
per-chunk steps run on the CPU under AddressSanitizer over file images that end exactly at data_len: valid files must decode exactly,
damaged last chunks must be refused or decoded, and no read may leave the file or the staged tail."""
import os, shutil, subprocess, pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_k1_reads_stay_inside_an_exact_length_buffer(tmp_path):
    exe = str(tmp_path / "k1_tail_host")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=address", "-fno-omit-frame-pointer", "-fno-strict-aliasing",
           "-o", exe, os.path.join(ROOT, "tests", "native", "k1_tail_host.cc"), os.path.join(ROOT, "oracle", "codec.cc")]
    b = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert b.returncode == 0, b.stderr[-2000:]
    r = subprocess.run([exe, "300"], capture_output=True, text=True, timeout=600, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1"))
    assert r.returncode == 0 and "k1_tail_host ok" in r.stdout, (r.stdout + r.stderr)[-3000:]
    assert "runtime error" not in r.stderr, r.stderr[-3000:]
