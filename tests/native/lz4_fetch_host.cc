// lz4_compress_warp<true> (cassandra_b200/csrc/lz4.cuh) on the warp emulator, reading each chunk from a heap buffer that ENDS at the chunk's last
// byte and starts 4- but not 16-byte aligned, as the chunks of every output file after the first do; and lz4_compress_warp<false> on the chunk +
// 16 bytes, which is what k_compress_chunks stages. TEST INFRASTRUCTURE: built with
// AddressSanitizer by tests/test_lz4_window_host.py; the output must equal the oracle's byte for byte and no load may leave the buffer.
#include <cstdio>
#include <cstdlib>
#include <random>
#include "codec_warp_host.cc"
#include "../../oracle/codec.h"

static int check(const std::vector<uint8_t>& d, int lead, const char* what) {
    const int n = (int)d.size();
    uint8_t* buf = (uint8_t*)malloc((size_t)lead + n);                  // malloc: 16-byte aligned, so buf + lead is the alignment asked for
    memcpy(buf + lead, d.data(), n);
    std::vector<uint16_t> tab(LZ4_TABLE_ENTRIES, 0xDEAD);
    std::vector<uint8_t> got(lz4_compress_bound(n)), want(oracle::lz4_compress_bound(n));
    int r = -1;
    warp_emu::run([&](int lane) { int x = lz4_compress_warp<true>(buf + lead, n, tab.data(), got.data(), lane); if (lane == 0) r = x; });
    free(buf);
    const int w = oracle::lz4_compress_block(d.data(), n, want.data(), (int)want.size());
    if (r != w || memcmp(got.data(), want.data(), w)) { printf("MISMATCH %s n=%d lead=%d got=%d want=%d\n", what, n, lead, r, w); return 1; }
    // the shared-memory variant: k_compress_chunks gives it the chunk and 16 zeroed bytes, and the attempts of a search window that lie
    // beyond the chunk's end (an accelerated search overshoots by hundreds of bytes) must not be read
    buf = (uint8_t*)calloc((size_t)n + 16, 1);
    memcpy(buf, d.data(), n);
    warp_emu::run([&](int lane) { int x = lz4_compress_warp<false>(buf, n, tab.data(), got.data(), lane); if (lane == 0) r = x; });
    free(buf);
    if (r != w || memcmp(got.data(), want.data(), w)) { printf("MISMATCH (shared) %s n=%d got=%d want=%d\n", what, n, r, w); return 1; }
    return 0;
}

int main(int argc, char** argv) {
    const int iters = argc > 1 ? atoi(argv[1]) : 40;
    std::mt19937 rng(0x1F47C4);
    auto rnd = [&](int n) { std::vector<uint8_t> v(n); for (auto& b : v) b = (uint8_t)rng(); return v; };
    int bad = 0;
    for (int it = 0; it < iters; it++) {
        const int sizes[] = {1, 12, 13, 16, 17, 33, 64, 67, 100, 257, 1000, 2500, 4097};
        const int n = sizes[rng() % 13], lead = 4 * (1 + rng() % 3);
        std::vector<uint8_t> d;
        switch (rng() % 5) {
        case 0: d = rnd(n); break;
        case 1: d.assign(n, 0); break;                                                             // the match runs to matchlimit = n - 5
        case 2: { auto p = rnd(1 + rng() % 40); for (int i = 0; i < n; i++) d.push_back(p[i % p.size()]); break; }
        case 3: { auto b = rnd(8 + rng() % 90); while ((int)d.size() < n) { auto g = rnd(rng() % 50); d.insert(d.end(), g.begin(), g.end()); d.insert(d.end(), b.begin(), b.end()); } d.resize(n); break; }
        default: for (int i = 0; i < n; i++) d.push_back("ab\0"[rng() % 3]); break;
        }
        bad += check(d, lead, "random");
    }
    if (!bad) printf("lz4_fetch_host ok\n");
    return bad ? 1 : 0;
}
