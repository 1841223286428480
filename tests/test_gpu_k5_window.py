"""K5's default LZ4 kernel (k_compress_chunks_lz4_direct) on the GPU over the shapes of tests/test_lz4_window_host.py — the cases its one round of
loads per hit must get right — and over chunks that are stored raw: Data.db image, chunk offsets and digest equal the CPU oracle's."""
import random, struct, zlib, pytest
import oracle_lib as O
from test_lz4_window_host import shapes

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def ctx():
    from cassandra_b200 import native
    c = native.Context(0)
    yield c
    c.close()

def _oracle_image(stream, chunk_len, max_clen):
    image = bytearray(); offs = []
    for i in range(0, len(stream), chunk_len):
        u = stream[i:i + chunk_len]
        c = O.chunk_compress(O.COMP_LZ4, u)
        if len(c) >= max_clen: c = u + bytes(max(0, max_clen - len(u)))      # CompressedSequentialWriter.flushData: stored raw, zero padded
        offs.append(len(image)); image += c + struct.pack(">I", O.crc32(c))
    return bytes(image), offs, zlib.crc32(bytes(image))

def test_each_shape_alone_in_its_chunk(ctx):
    """one chunk per call: the chunk ends where the shape ends (matches that run to the last five bytes, last literals)"""
    from cassandra_b200 import native
    for name, d in shapes(rounds=1):
        assert ctx.compress_chunks(native.COMP_LZ4, d, 16384) == _oracle_image(d, 16384, native.INT32_MAX), name

@pytest.mark.parametrize("max_clen", [None, 3000])
def test_shapes_as_one_stream(ctx, max_clen):
    """every shape padded to a 4 KiB chunk of one stream, so that chunks start at every alignment of 4 KiB a slot sees; with a finite
    max_compressed_length the chunks that random padding keeps above it are stored raw"""
    from cassandra_b200 import native
    rng = random.Random(0x4B5)
    stream = b"".join(d + bytes(rng.getrandbits(8) for _ in range(4096 - len(d))) if i % 3 else (d * (4096 // len(d) + 1))[:4096] for i, (_, d) in enumerate(shapes()))
    stream = stream[:-1111]                                                  # ragged last chunk
    mcl = max_clen or native.INT32_MAX
    want = _oracle_image(stream, 4096, mcl)
    if max_clen: assert any(b - a - 4 == max_clen or b - a - 4 == 4096 for a, b in zip(want[1], want[1][1:])), "no raw chunk in the fixture"
    assert ctx.compress_chunks(native.COMP_LZ4, stream, 4096, mcl) == want
    assert ctx.decompress_chunks(native.COMP_LZ4, want[0], want[1], len(stream), 4096, mcl) == stream
