// Host build of K5's compressors for chunks above 64 KiB (cassandra_b200/csrc/codec.cuh: k_compress_chunks_lz4_big, k_snappy_big_fragments +
// k_snappy_big_assemble) on the 32-fiber warp emulator of warp_emu.h. TEST INFRASTRUCTURE: the device source itself, byte-compared on the CPU with
// liblz4 and Google snappy.
#include <cstdint>
#include <cstring>
#include <vector>
#include <cuda_runtime.h>
#include "warp_emu.h"
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned s) {
    unsigned long long pool = ((unsigned long long)b << 32) | a; unsigned r = 0;
    for (int i = 0; i < 4; i++) r |= (unsigned)((pool >> (8 * ((s >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
}
static inline unsigned atomicOr(unsigned* p, unsigned v) { unsigned o = *p; *p = o | v; return o; }       // (one fiber runs at a time)
static inline unsigned atomicAnd(unsigned* p, unsigned v) { unsigned o = *p; *p = o & v; return o; }
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) { sh &= 31; return sh ? (lo >> sh) | (hi << (32 - sh)) : lo; }
template <typename T> static inline T __ldg(const T* p) { return *p; }
static inline int min(int a, int b) { return a < b ? a : b; }
#include "../../cassandra_b200/csrc/lz4.cuh"
#include "../../cassandra_b200/csrc/snappy.cuh"
#include "../../cassandra_b200/csrc/snappy_chain.cuh"

using namespace b200c;

// k_compress_chunks_lz4_big's block of one chunk without its 4-byte length prefix: byU32 from LZ4_64KLIMIT on, byU16 below
extern "C" int warp_lz4_big(const uint8_t* in, int n, uint8_t* out) {
    std::vector<uint32_t> src((size_t)n / 4 + 16, 0); memcpy(src.data(), in, n);      // 4-byte aligned, slack behind the chunk as in device memory
    std::vector<uint32_t> tab(1 << LZ4_HASHLOG_U32, 0xDEADBEEFu);                      // the kernel zeroes it
    int result = -1;
    warp_emu::run([&](int lane) {
        const uint8_t* s = (const uint8_t*)src.data();
        const int r = n >= LZ4_64KLIMIT ? lz4_compress_warp<true, true>(s, n, tab.data(), out, lane) : lz4_compress_warp<true>(s, n, (uint16_t*)tab.data(), out, lane);
        if (lane == 0) result = r;
    });
    return result;
}

// k_snappy_big_fragments (one warp per 64 KiB fragment, each with its own table) followed by k_snappy_big_assemble's varint + concatenation
extern "C" int warp_snappy_big(int max_bits, const uint8_t* in, int n, uint8_t* out) {
    std::vector<uint32_t> src((size_t)n / 4 + 16, 0); memcpy(src.data(), in, n);
    std::vector<uint16_t> tab(1 << 15, 0xDEAD);
    std::vector<uint8_t> frag((size_t)snappy_max_compressed_length(65536) + 64);
    int op = 0;
    { uint32_t v = (uint32_t)n; while (v >= 0x80) { out[op++] = (uint8_t)(v | 0x80); v >>= 7; } out[op++] = (uint8_t)v; }
    for (int start = 0; start < n; start += 65536) {
        const int len = n - start < 65536 ? n - start : 65536, tsz = snappy_table_size(len, max_bits);
        int flen = -1;
        warp_emu::run([&](int lane) {
            for (int i = lane; i < tsz / 2; i += 32) ((uint32_t*)tab.data())[i] = 0;
            __syncwarp();
            const int r = snappy_compress_fragment_warp<true>((const uint8_t*)src.data() + start, 0, len, tab.data(), tsz, max_bits, frag.data(), 0, lane);
            if (lane == 0) flen = r;
        });
        if (flen < 0) return -1;
        memcpy(out + op, frag.data(), flen); op += flen;
    }
    return op;
}
