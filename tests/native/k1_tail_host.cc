// CPU check of how K1 reads a device-resident input in place (compact.cu, codec.cuh: k1_src / k1_tail_window in k1_tail.cuh), meant to be built with
// -fsanitize=address,undefined. Test infrastructure only.
// Every file image lives in a heap buffer that ends exactly at data_len (no slack behind it, as a caller's tensor may have none); its
// last k1_tail_window() bytes are staged in a copy with 64 bytes of slack, as compact.cu stages them. Each chunk then goes through
// K1's per-thread steps on the bytes k1_src points at: the size checks of decompress_chunk_thread, the CRC over the chunk and the
// decoder (lz4_decompress_thread, or the word copy of a stored chunk). Valid files must decode exactly; damaged last chunks must fail
// or decode, and no read may leave [data, data + data_len) or the staged tail.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <random>
#include "../../cassandra_b200/csrc/lz4_thread.cuh"
#include "../../cassandra_b200/csrc/k1_tail.cuh"
#include "../../oracle/codec.h"

using namespace b200c;

static std::vector<uint8_t> make_data(std::mt19937_64& rng, int n, int kind) {
    std::vector<uint8_t> d(n);
    switch (kind) {
    case 0: for (auto& b : d) b = (uint8_t)rng(); break;                                           // incompressible: stored when max_clen allows
    case 1: { uint8_t v = (uint8_t)rng(); for (int i = 0; i < n; i++) { if (rng() % 97 == 0) v = (uint8_t)rng(); d[i] = v; } } break;
    case 2: { int period = 2 + (int)(rng() % 14); for (int i = 0; i < n; i++) d[i] = i < period ? (uint8_t)rng() : (rng() % 53 ? d[i - period] : (uint8_t)rng()); } break;
    default: { std::vector<std::vector<uint8_t>> words(48); for (auto& w : words) { w.resize(3 + rng() % 20); for (auto& b : w) b = (uint8_t)rng(); }
               int i = 0; while (i < n) { auto& w = words[rng() % words.size()]; for (uint8_t b : w) { if (i < n) d[i++] = b; } } } break;
    }
    return d;
}

struct File { std::vector<uint8_t> image, plain; std::vector<uint64_t> offs; int chunk_len, max_clen; };

// CompressedSequentialWriter's layout: per chunk [LZ4 length prefix + block | raw bytes (zero padded to max_clen)] + big-endian CRC32
static File make_file(std::mt19937_64& rng, int it) {
    File f; f.chunk_len = 256 << (rng() % 5); f.max_clen = (rng() % 2) ? 0x7fffffff : f.chunk_len - (int)(rng() % 64);
    const int nch = 1 + (int)(rng() % 5);
    const int n = (nch - 1) * f.chunk_len + 1 + (int)(rng() % f.chunk_len);
    f.plain = make_data(rng, n, it % 4);
    std::vector<uint8_t> buf(oracle::chunk_max_compressed(oracle::COMP_LZ4, f.chunk_len) + f.chunk_len + 16);
    for (int s = 0; s < n; s += f.chunk_len) {
        const int ulen = std::min(f.chunk_len, n - s);
        int c = oracle::chunk_compress(oracle::COMP_LZ4, f.plain.data() + s, ulen, buf.data());
        if (c >= f.max_clen) { memcpy(buf.data(), f.plain.data() + s, ulen); c = ulen; if (ulen < f.max_clen) { memset(buf.data() + ulen, 0, f.max_clen - ulen); c = f.max_clen; } }
        const uint32_t crc = oracle::crc32_ieee(0, buf.data(), c);
        f.offs.push_back(f.image.size());
        f.image.insert(f.image.end(), buf.begin(), buf.begin() + c);
        for (int k = 3; k >= 0; k--) f.image.push_back((uint8_t)(crc >> (8 * k)));
    }
    return f;
}

// K1 on one chunk: 0 decoded, 1 CRC mismatch, 2 malformed (decompress_chunk_thread's order of checks)
static int k1_chunk(const uint8_t* data, uint64_t data_len, const uint8_t* tail, uint64_t tail_off, const File& f, uint64_t chunk, uint8_t* out) {
    const uint64_t nchunks = f.offs.size(), data_length = f.plain.size();
    const uint64_t off = f.offs[chunk], next = chunk + 1 < nchunks ? f.offs[chunk + 1] : data_len, ustart = chunk * (uint64_t)f.chunk_len;
    const int max_c = oracle::chunk_max_compressed(oracle::COMP_LZ4, f.chunk_len);
    if (off + 4 > next || next > data_len || ustart >= data_length || next - off - 4 > (uint64_t)(max_c + f.chunk_len)) return 2;
    const int clen = (int)(next - off - 4), ulen = (int)std::min<uint64_t>(f.chunk_len, data_length - ustart);
    const uint8_t* src = k1_src(data, tail, tail_off, off);
    const uint32_t stored = ((uint32_t)src[clen] << 24) | ((uint32_t)src[clen + 1] << 16) | ((uint32_t)src[clen + 2] << 8) | src[clen + 3];
    const bool crc_ok = oracle::crc32_ieee(0, src, clen) == stored;
    uint8_t* dst = out + ustart;
    int got;                                          // (decoded even after a CRC mismatch: the reads must stay inside either way)
    if (clen >= f.max_clen) {
        if (clen < ulen) return crc_ok ? 2 : 1;
        WordSink w{dst, 0, 0ull};
        int i = 0;
        for (; i + 8 <= ulen; i += 8) w.put(ld_le64(src + i), 8);
        if (i < ulen) w.put(low_bytes(ld_le64(src + i), ulen - i), ulen - i);
        w.flush_bytes();
        got = ulen;
    } else {
        const int plen = clen >= 4 ? (int)((uint32_t)src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24)) : -1;
        got = plen == ulen ? lz4_decompress_thread(src + 4, clen - 4, dst, ulen) : -1;
    }
    return !crc_ok ? 1 : (got == ulen ? 0 : 2);
}

// the file as compact.cu hands it to K1: the caller's buffer (ending exactly at data_len, `align` bytes into its allocation) + staged tail
static int run_file(const File& f, const std::vector<uint8_t>& image, int align, std::vector<int>& kinds) {
    const uint64_t data_len = image.size();
    uint8_t* alloc = (uint8_t*)malloc(align + data_len);              // ends at data + data_len
    uint8_t* data = alloc + align;
    memcpy(data, image.data(), data_len);
    const uint64_t win = std::min<uint64_t>(data_len, k1_tail_window(oracle::chunk_max_compressed(oracle::COMP_LZ4, f.chunk_len), f.chunk_len));
    uint8_t* tail = (uint8_t*)malloc(win + 64);
    memcpy(tail, data + (data_len - win), win); memset(tail + win, 0xA5, 64);
    uint8_t* out = nullptr; if (posix_memalign((void**)&out, 8, f.plain.size() + 16)) return -1;
    int bad = 0;
    kinds.clear();
    for (uint64_t c = 0; c < f.offs.size(); c++) { int k = k1_chunk(data, data_len, tail, data_len - win, f, c, out); kinds.push_back(k); bad |= k; }
    if (!bad && memcmp(out, f.plain.data(), f.plain.size())) { fprintf(stderr, "decoded bytes differ\n"); exit(4); }
    free(out); free(tail); free(alloc);
    return bad;
}

int main(int argc, char** argv) {
    const int iters = argc > 1 ? atoi(argv[1]) : 300;
    std::mt19937_64 rng(0xB200C71);
    long valid = 0, damaged = 0, stored = 0;
    std::vector<int> kinds;
    for (int it = 0; it < iters; it++) {
        File f = make_file(rng, it);
        if (f.max_clen != 0x7fffffff) stored++;
        for (int align = 0; align < 16; align += 1 + (int)(rng() % 7))
            if (run_file(f, f.image, align, kinds) != 0) { fprintf(stderr, "valid file rejected (it %d)\n", it); return 3; }
        valid++;
        // damaged last chunk: flipped bytes, truncated image (K1 must refuse or decode, reading nothing outside)
        std::vector<uint8_t> d = f.image;
        const uint64_t last = f.offs.back();
        for (int k = 0; k < 3; k++) d[last + rng() % (d.size() - last)] ^= (uint8_t)(1 + rng() % 255);
        run_file(f, d, (int)(rng() % 16), kinds);
        std::vector<uint8_t> t(f.image.begin(), f.image.end() - (1 + rng() % std::min<uint64_t>(12, f.image.size() - last)));
        if (t.size() > last) run_file(f, t, (int)(rng() % 16), kinds);
        damaged++;
    }
    printf("k1_tail_host ok: %ld valid files, %ld with stored chunks, %ld damaged\n", valid, stored, damaged);
    return 0;
}
