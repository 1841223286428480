// common.cuh — shared device helpers for the H100 (sm_90a) SSTable compaction engine.
// Integer/byte work only: vint codec, CRC32 (IEEE) as a warp-parallel linear map, small warp utilities.
#pragma once
#include <cstdint>
#include <cstddef>
#include <cuda_runtime.h>

#define FULL_MASK 0xFFFFFFFFu

namespace b200c {

// Constant tables built on the host at context creation (engine.cu: build_tables) and kept in global memory.
struct DevTables {
    uint32_t crc_t[4][256];      // slice-by-4: crc_t[k][b] = register after byte b then k zero bytes
    uint32_t crc_adv128[4][256]; // advance a CRC register through 128 zero bytes, byte-sliced
    uint32_t xp_lane[32];        // x^(8*4*(32-l)) mod P  (reflected)
    uint32_t xp_pow2[64];        // x^(8*2^k) mod P
    uint32_t crc_adv512[4][256]; // advance a CRC register through 512 zero bytes (one warp row of 16-byte words), byte-sliced
    uint32_t xp_lane16[32];      // x^(8*16*(31-l)) mod P: bytes behind lane l's 16-byte word in a 512-byte row
};

__host__ __device__ __forceinline__ uint32_t gf2_mulmod(uint32_t a, uint32_t b) {
    // polynomial product mod the CRC32 polynomial, reflected bit order (bit31 = x^0)
    uint32_t r = 0;
#pragma unroll 8
    for (int i = 0; i < 32; i++) {
        r ^= (a & 0x80000000u) ? b : 0u;
        a <<= 1;
        b = (b >> 1) ^ ((b & 1u) ? 0xEDB88320u : 0u);
    }
    return r;
}

// x^(8*n) mod P using the precomputed squares; n < 2^63
__device__ __forceinline__ uint32_t gf2_xpow8n(const DevTables* T, uint64_t n) {
    uint32_t r = 0x80000000u;
    for (int k = 0; n; k++, n >>= 1)
        if (n & 1) r = gf2_mulmod(r, T->xp_pow2[k]);
    return r;
}

// ---- vint (S/utils/vint/VIntCoding.java:303-327,535-540) -------------------------------------------------------
__host__ __device__ __forceinline__ int vint_size(uint64_t v) {
#ifdef __CUDA_ARCH__
    int magnitude = __clzll((long long)(v | 1));
#else
    int magnitude = __builtin_clzll(v | 1);
#endif
    return (639 - magnitude * 9) >> 6;
}
__host__ __device__ __forceinline__ uint64_t zigzag_enc(int64_t n) { return ((uint64_t)n << 1) ^ (uint64_t)(n >> 63); }
__host__ __device__ __forceinline__ int64_t zigzag_dec(uint64_t n) { return (int64_t)(n >> 1) ^ -(int64_t)(n & 1); }

// reads an unsigned vint at p (caller guarantees 9 readable bytes or checks `end`); returns bytes consumed, 0 on overrun
__device__ __forceinline__ int vint_read(const uint8_t* p, const uint8_t* end, uint64_t* v) {
    if (p >= end) return 0;
    uint32_t first = p[0];
    if (first < 0x80) { *v = first; return 1; }
    int extra = __clz((int)(~(first << 24))) ;       // leading one bits of the first byte (8 for 0xFF)
    if (first == 0xFF) extra = 8;
    if (p + 1 + extra > end) return 0;
    uint64_t r = first & (0xffu >> extra);
    for (int i = 0; i < extra; i++) r = (r << 8) | p[1 + i];
    *v = r;
    return 1 + extra;
}

// ---- warp-parallel CRC32 ------------------------------------------------------------------------------------------
// CRC is linear over GF(2): the message is cut into 4-byte words, lane l folds words l, l+32, l+64, ... with a
// "advance 128 zero bytes" operator (4 table lookups per word, coalesced word loads), and the 32 lane registers are
// then advanced by their distance to the end and XOR-reduced. The message is virtually front-padded with zeroes to a
// multiple of 128 bytes (leading zeroes do not change a zero-initialised CRC); the 0xFFFFFFFF init is added by linearity.

__device__ __forceinline__ uint32_t crc_adv128(const uint32_t (*A)[256], uint32_t x) {
    return A[0][x & 0xff] ^ A[1][(x >> 8) & 0xff] ^ A[2][(x >> 16) & 0xff] ^ A[3][x >> 24];
}

// little-endian word of message bytes [o, o+4); bytes outside [0, len) read as zero. buf may be unaligned.
__device__ __forceinline__ uint32_t crc_msg_word(const uint8_t* buf, int len, int o) {
    if (o <= -4 || o >= len) return 0;
    if (o < 0 || o + 4 > len) {
        uint32_t w = 0;
        for (int b = 0; b < 4; b++) { int i = o + b; if (i >= 0 && i < len) w |= (uint32_t)buf[i] << (8 * b); }
        return w;
    }
    uintptr_t addr = (uintptr_t)(buf + o);
    const uint32_t* ap = (const uint32_t*)(addr & ~(uintptr_t)3);
    int sh = (int)(addr & 3);
    uint32_t lo = ap[0];
    uint32_t hi = sh ? ap[1] : 0u;       // the engine keeps >= 8 readable slack bytes after every buffer
    return __funnelshift_r(lo, hi, sh * 8);
}

// Raw (zero-init, no final xor) CRC register of buf[0..len) — all lanes return the value. s_adv: the adv128 tables
// (shared or global memory).
__device__ __forceinline__ uint32_t warp_crc32_raw(const DevTables* T, const uint32_t (*s_adv)[256],
                                                   const uint8_t* buf, int len, int lane) {
    int pad = (128 - (len & 127)) & 127;
    int nrows = (len + pad) >> 7;                 // rows of 32 words
    uint32_t u = 0;
    int o = 4 * lane - pad;
    for (int k = 0; k < nrows; k++, o += 128)
        u = crc_adv128(s_adv, u) ^ crc_msg_word(buf, len, o);
    uint32_t r = gf2_mulmod(u, T->xp_lane[lane]);
#pragma unroll
    for (int d = 16; d; d >>= 1) r ^= __shfl_xor_sync(FULL_MASK, r, d);
    return r;
}

// x^(8*len) for warp-uniform len < 2^32, product-reduced across lanes
__device__ __forceinline__ uint32_t warp_xpow8n(const DevTables* T, uint32_t len, int lane) {
    uint32_t f = ((len >> lane) & 1u) ? T->xp_pow2[lane] : 0x80000000u;
#pragma unroll
    for (int d = 16; d; d >>= 1) f = gf2_mulmod(f, __shfl_xor_sync(FULL_MASK, f, d));
    return f;
}

// zlib-compatible CRC32 of buf[0..len); all lanes return it
__device__ __forceinline__ uint32_t warp_crc32(const DevTables* T, const uint32_t (*s_adv)[256],
                                               const uint8_t* buf, int len, int lane) {
    uint32_t raw = warp_crc32_raw(T, s_adv, buf, len, lane);
    uint32_t init = gf2_mulmod(0xFFFFFFFFu, warp_xpow8n(T, (uint32_t)len, lane));
    return ~(raw ^ init);
}

// 8 bytes at an arbitrary address as a big-endian integer (p[0] in the most significant byte): two aligned 8-byte loads + shifts.
// Reads up to 15 bytes past p's 8-byte-aligned start: every engine buffer carries >= 64 bytes of slack.
__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
    uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
}
__device__ __forceinline__ uint64_t load_be64(const uint8_t* p) {
    uintptr_t a = (uintptr_t)p; const uint64_t* q = (const uint64_t*)(a & ~(uintptr_t)7); uint32_t sh = (uint32_t)(a & 7) * 8;
    uint64_t lo = q[0];
    if (sh) lo = (lo >> sh) | (q[1] << (64 - sh));
    return bswap64(lo);
}
// 16 bytes at an arbitrary address as two big-endian words (three aligned 8-byte loads)
__device__ __forceinline__ void load_be128(const uint8_t* p, uint64_t& w0, uint64_t& w1) {
    uintptr_t a = (uintptr_t)p; const uint64_t* q = (const uint64_t*)(a & ~(uintptr_t)7); uint32_t sh = (uint32_t)(a & 7) * 8;
    uint64_t q0 = q[0], q1 = q[1];
    if (sh) { uint64_t q2 = q[2]; q0 = (q0 >> sh) | (q1 << (64 - sh)); q1 = (q1 >> sh) | (q2 << (64 - sh)); }
    w0 = bswap64(q0); w1 = bswap64(q1);
}

// unaligned little-endian 32-bit read from a 4-byte aligned base (shared or global); needs base[.. p+7] readable
__device__ __forceinline__ uint32_t rd32_at(const uint32_t* base32, int p) {
    uint32_t lo = base32[p >> 2];
    uint32_t hi = base32[(p >> 2) + 1];
    return __funnelshift_r(lo, hi, (p & 3) * 8);
}

// ---- bulk asynchronous copies global -> shared memory (the TMA unit's 1-D path: cp.async.bulk, SASS UBLKCP) with an mbarrier that
// counts the bytes as they land. Source, destination and size must be multiples of 16 bytes. ------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t arrivals) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(arrivals) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src), "r"(bytes), "r"((uint32_t)__cvta_generic_to_shared(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0; const uint32_t a = (uint32_t)__cvta_generic_to_shared(bar);
    while (!done) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(a), "r"(parity) : "memory");
}
#endif

} // namespace b200c
