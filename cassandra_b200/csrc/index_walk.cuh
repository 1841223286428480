// index_walk.cuh — K2's Index.db walk on 16-byte words. Plain C++ for host and device: tests/native/index_walk_host.cc runs it on the CPU
// under AddressSanitizer against a byte-wise parse, over buffers that end IW_PAD bytes past the input.
//
// One thread walks the ~2 KB between two Summary.db samples entry by entry. Reading that byte by byte costs one load per byte (the lanes of a
// warp sit kilobytes apart, so every load is its own L1 wavefront); here the thread keeps a window of two aligned 16-byte chunks in registers,
// moves it forward one chunk at a time as the walk advances, and takes every field (key length, key, both vints) out of the window by shifts.
// A skipped payload (the promoted index of a wide partition) moves the window by address without reading what it skips.
#pragma once
#include <cstdint>
#include <cstring>
#ifdef __CUDACC__
#define B200C_IW_HD __host__ __device__ __forceinline__
#else
#define B200C_IW_HD inline
#endif

namespace b200c {

// The cursor loads an aligned chunk only when its first byte lies inside the input: it reads at most 15 bytes past the input's last byte, and
// from the aligned address at or below its first byte. The buffer holding an input's Index.db must be readable that far.
enum { IW_PAD = 16 };

// ---- Murmur3 mixing (Cassandra variant, S/utils/MurmurHash.java:178-260) ------------------------------------------------------------
B200C_IW_HD uint64_t rotl64(uint64_t v, int n) { return (v << n) | (v >> (64 - n)); }
B200C_IW_HD uint64_t fmix64(uint64_t k) { k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33; return k; }
enum : uint64_t { MM3_C1 = 0x87c37b91114253d5ULL, MM3_C2 = 0x4cf5ad432745937fULL };
B200C_IW_HD void mm3_mix_k1(uint64_t& h1, uint64_t k1) { k1 *= MM3_C1; k1 = rotl64(k1, 31); k1 *= MM3_C2; h1 ^= k1; }
B200C_IW_HD void mm3_mix_k2(uint64_t& h2, uint64_t k2) { k2 *= MM3_C2; k2 = rotl64(k2, 33); k2 *= MM3_C1; h2 ^= k2; }
B200C_IW_HD void mm3_block(uint64_t& h1, uint64_t& h2, uint64_t k1, uint64_t k2) {
    mm3_mix_k1(h1, k1); h1 = rotl64(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729;
    mm3_mix_k2(h2, k2); h2 = rotl64(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5;
}
B200C_IW_HD int64_t mm3_finish(uint64_t h1, uint64_t h2, uint32_t len) {
    h1 ^= (uint64_t)len; h2 ^= (uint64_t)len;
    h1 += h2; h2 += h1; h1 = fmix64(h1); h2 = fmix64(h2); h1 += h2;
    const int64_t v = (int64_t)h1;
    return v == INT64_MIN ? INT64_MAX : v;                    // Murmur3Partitioner.getToken: MINIMUM is not a key's token
}
// XOR of bytes 0..n-1 of w, each sign-extended to 64 bits and shifted to its place (the tail of MurmurHash.hash3_x64_128 reads signed bytes)
B200C_IW_HD uint64_t mm3_signed_tail(uint64_t w, int n) {
    uint64_t r = n >= 8 ? w : (w & ((1ull << (8 * n)) - 1));
#pragma unroll
    for (int i = 0; i < 7; i++) if (i < n && ((w >> (8 * i + 7)) & 1)) r ^= ~0ull << (8 * (i + 1));
    return r;
}

B200C_IW_HD uint64_t iw_bswap64(uint64_t x) {
#ifdef __CUDA_ARCH__
    const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
#else
    return __builtin_bswap64(x);
#endif
}
B200C_IW_HD int iw_leading_ones8(uint32_t b) {          // of a byte >= 0x80: 1..8
#ifdef __CUDA_ARCH__
    return __clz((int)~(b << 24));
#else
    return __builtin_clz(~(b << 24));
#endif
}

// ---- the cursor ----------------------------------------------------------------------------------------------------------------------
struct IdxCursor {
    uintptr_t base, end;                 // the input's first byte and one past its last
    uintptr_t wa;                        // the window holds bytes [wa, wa + 32) in w0..w3 (little-endian); wa is 16-byte aligned
    uint64_t w0, w1, w2, w3;

    B200C_IW_HD void init(const uint8_t* p, uint64_t len) { base = (uintptr_t)p; end = base + len; wa = ~(uintptr_t)63; w0 = w1 = w2 = w3 = 0; }
    B200C_IW_HD void chunk(uintptr_t a, uint64_t& lo, uint64_t& hi) const {
        if (a >= end) { lo = hi = 0; return; }
#ifdef __CUDA_ARCH__
        const ulonglong2 v = __ldg((const ulonglong2*)a); lo = v.x; hi = v.y;
#else
        memcpy(&lo, (const void*)a, 8); memcpy(&hi, (const void*)(a + 8), 8);
#endif
    }
    // bytes [o, o + 16) of the input as two little-endian words; those at or past the end of the input are unspecified. The window slides
    // by one chunk when o has moved into its second half and is reloaded when o lies anywhere else.
    B200C_IW_HD void peek16(uint64_t o, uint64_t& lo, uint64_t& hi) {
        const uintptr_t x = base + o;
        uintptr_t d = x - wa;
        if (d >= 16) {
            if (d < 32) { w0 = w2; w1 = w3; wa += 16; chunk(wa + 16, w2, w3); }
            else { wa = x & ~(uintptr_t)15; chunk(wa, w0, w1); chunk(wa + 16, w2, w3); }
            d = x - wa;
        }
        const bool h = (d & 8) != 0;
        const uint64_t a0 = h ? w1 : w0, a1 = h ? w2 : w1, a2 = h ? w3 : w2;
        const uint32_t s = (uint32_t)(d & 7) * 8;
        lo = s ? (a0 >> s) | (a1 << (64 - s)) : a0;
        hi = s ? (a1 >> s) | (a2 << (64 - s)) : a1;
    }
    // vint_read (common.cuh) at offset p: bytes consumed, 0 when the vint runs past the end of the input
    B200C_IW_HD int vint(uint64_t p, uint64_t* v) {
        const uint64_t len = end - base;
        if (p >= len) return 0;
        uint64_t lo, hi; peek16(p, lo, hi);
        const uint32_t first = (uint32_t)(lo & 0xFF);
        if (first < 0x80) { *v = first; return 1; }
        const int extra = iw_leading_ones8(first);
        if (p + 1 + extra > len) return 0;
        uint64_t r = iw_bswap64((lo >> 8) | (hi << 56)) >> (8 * (8 - extra));      // bytes 1..extra, big-endian
        if (extra < 8) r |= (uint64_t)(first & (0xFFu >> extra)) << (8 * extra);
        *v = r;
        return 1 + extra;
    }
    // Murmur3 token of the `len` key bytes at offset k: murmur3_token (compact.cu) on the window's bytes
    B200C_IW_HD int64_t murmur3(uint64_t k, uint32_t len) {
        if (len == 0) return INT64_MIN;
        uint64_t h1 = 0, h2 = 0, lo, hi;
        const uint32_t nblocks = len >> 4;
        for (uint32_t i = 0; i < nblocks; i++) { peek16(k + 16ull * i, lo, hi); mm3_block(h1, h2, lo, hi); }
        const int rem = (int)(len & 15);
        if (rem) {
            peek16(k + 16ull * nblocks, lo, hi);
            if (rem > 8) mm3_mix_k2(h2, mm3_signed_tail(hi, rem - 8));
            mm3_mix_k1(h1, mm3_signed_tail(lo, rem < 8 ? rem : 8));
        }
        return mm3_finish(h1, h2, len);
    }
};

// One Index.db entry = u16 keyLen | key | vint dataPosition | vint32 payloadSize | payload (RowIndexEntry.java:468-473).
struct IdxEntry {
    uint64_t pos;          // dataPosition
    uint32_t kl;           // key length
    uint64_t pre;          // KEY: the first 8 key bytes, big-endian, zero padded (order_token_of's prefix)
    int64_t tok;           // KEY: the Murmur3 token of the key, or the sign-flipped prefix (byte-ordered partitioner)
};
// The entry at offset o, with idx_entry's structural checks (compact.cu): every field inside the input, payloadSize <= 0x7FFFFFFF, and a
// dataPosition that leaves room for the partition's key in the input's ulen bytes of Data.db. Returns the entry's length, 0 = not an entry.
// KEY also fills pre / tok (murmur: Murmur3 partitioner).
template <bool KEY>
B200C_IW_HD uint64_t iw_entry(IdxCursor& c, uint64_t o, uint64_t ulen, bool murmur, IdxEntry& e) {
    const uint64_t ilen = c.end - c.base;
    if (o + 2 > ilen) return 0;
    uint64_t lo, hi; c.peek16(o, lo, hi);
    const uint32_t kl = (uint32_t)(((lo & 0xFF) << 8) | ((lo >> 8) & 0xFF));
    uint64_t p = o + 2 + kl;
    if (p + 2 > ilen) return 0;
    if (KEY) {
        uint64_t k8 = (lo >> 16) | (hi << 48);                 // key bytes 0..7 (little-endian)
        if (kl < 8) k8 &= (1ull << (8 * kl)) - 1;
        e.pre = iw_bswap64(k8);
        e.tok = murmur ? c.murmur3(o + 2, kl) : (int64_t)(e.pre ^ 0x8000000000000000ull);
    }
    uint64_t pos, ps;
    int n = c.vint(p, &pos); if (!n) return 0; p += n;
    n = c.vint(p, &ps); if (!n) return 0; p += n;
    if (ps > 0x7FFFFFFFull || p + ps > ilen) return 0;
    if (pos >= ulen || pos + 2 + kl + 2 > ulen) return 0;
    e.pos = pos; e.kl = kl;
    return p + ps - o;
}

} // namespace b200c
