"""The in-place LZ4 compressor K5 launches by default (lz4_compress_warp<true>, cassandra_b200/csrc/lz4.cuh) asks for the bytes of catch-up, of
the first 32 literals and of the first 32 bytes of the match length in ONE round of loads after a hit, and takes the candidate of an attempt
whose hash an earlier lane of the same window holds from that lane's register. On the CPU warp emulator it must still equal liblz4's output
byte for byte on the shapes those changes touch: back-extension that stops at the anchor, at position 0, after more than 32 bytes; literal runs
and matches shorter than, equal to and longer than one 32-byte step; matches whose source overlaps them (offsets 1 to 3 and below 32); immediate
matches; and, under AddressSanitizer, chunks whose buffer ends at their last byte and starts 4- but not 16-byte aligned."""
import os, random, shutil, subprocess, pytest
import oracle_lib as O
from test_codec_warp_host import warp, run                  # the emulator build of tests/native/codec_warp_host.cc (mode 1 = in place)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

def shapes(seed=0xF37C4, rounds=3):
    """(name, bytes) pairs; also the input of tests/test_gpu_k5_window.py"""
    rng = random.Random(seed)
    rnd = lambda n: bytes(rng.getrandbits(8) for _ in range(n))
    out = []
    for r in range(rounds):
        blk = rnd(rng.choice([40, 150, 400]))
        # an accelerated search (long incompressible stretch) lands inside the repeated block: catch-up runs back to the block's start, which
        # is position 0 of the chunk for the first and the anchor for the second (the copies follow each other)
        out.append(("back_to_zero", blk + rnd(rng.randint(700, 1500)) + blk + blk + rnd(20)))
        out.append(("back_past_32", rnd(9) + blk + rnd(1200) + blk[:-1] + b"\x00" + rnd(900) + blk + rnd(13)))
        for k in (1, 2, 3, 5, 31, 32, 33):                             # source overlaps the match; lengths around one and two 32-byte steps
            per = rnd(k)
            for ml in (28, 35, 36, 37, 67, 68, 69, 300):
                out.append((f"period{k}_len{ml}", rnd(rng.randint(0, 70)) + (per * (ml // k + 2))[:ml + k] + rnd(rng.randint(0, 40))))
        for lit in (0, 1, 14, 15, 31, 32, 33, 64, 65, 270, 300):       # literal runs around the token nibble, one 32-byte step and one length byte
            out.append((f"lit{lit}", blk[:24] + rnd(lit) + blk[:24] + rnd(lit) + blk[4:24] + rnd(12)))
        out.append(("immediate", b"".join(blk[:12] + bytes([i]) for i in range(40))))     # a match ends where the next one begins
        out.append(("ends_in_match", rnd(50) + bytes(rng.choice([13, 17, 36, 37, 38, 100]))))
        words = [rnd(rng.randint(2, 9)) for _ in range(12)]
        out.append(("words", b"".join(rng.choice(words) for _ in range(700))[:4000]))
    return out

def test_one_round_of_loads_per_hit_equals_the_oracle(warp):
    for name, d in shapes():
        assert run(warp, 1, d) == O.lz4_compress(d), (name, len(d))

def test_random_differential_in_place(warp):
    """the shapes of test_lz4_chain_random_differential, for the in-place compressor"""
    rng = random.Random(0x17C4A1)
    alphabet = [bytes(rng.getrandbits(8) for _ in range(rng.randint(1, 9))) for _ in range(30)]
    sizes = [1, 4, 11, 12, 13, 14, 15, 16, 17, 31, 32, 33, 44, 45, 63, 64, 65, 66, 67, 100, 255, 256, 257, 1000, 4095, 4096, 4097, 8192, 16383, 16384]
    for it in range(120):
        n = rng.choice(sizes)
        kind = rng.random()
        if kind < 0.2: d = bytes(rng.getrandbits(8) for _ in range(n))
        elif kind < 0.5: d = b"".join(rng.choice(alphabet) for _ in range(n))[:n]
        elif kind < 0.65: d = bytes(rng.choice(b"ab\x00") for _ in range(n))
        elif kind < 0.8: d = (bytes(rng.getrandbits(8) for _ in range(rng.randint(1, 40))) * n)[:n]
        elif kind < 0.9:
            blk = bytes(rng.getrandbits(8) for _ in range(rng.randint(8, 300)))
            d = b"".join((bytes(rng.getrandbits(8) for _ in range(rng.randint(0, 900))) + blk) for _ in range(n // 200 + 1))[:n]
        else: d = bytes(n)
        assert run(warp, 1, d) == O.lz4_compress(d), (it, n, kind)

@pytest.mark.skipif(shutil.which("g++") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"), reason="needs g++ and the CUDA headers")
def test_reads_stay_inside_a_chunk_that_ends_with_its_buffer(tmp_path):
    exe = str(tmp_path / "lz4_fetch_host")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address", "-fno-omit-frame-pointer", "-fno-strict-aliasing", "-I/usr/local/cuda/include",
           "-Wno-attributes", "-Wno-unknown-pragmas", "-o", exe, os.path.join(ROOT, "tests", "native", "lz4_fetch_host.cc"), os.path.join(ROOT, "oracle", "codec.cc")]
    b = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert b.returncode == 0, b.stderr[-2000:]
    r = subprocess.run([exe, "60"], capture_output=True, text=True, timeout=900, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0"))
    assert r.returncode == 0 and "lz4_fetch_host ok" in r.stdout, (r.stdout + r.stderr)[-3000:]
