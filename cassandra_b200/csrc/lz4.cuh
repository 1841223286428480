// lz4.cuh — warp-cooperative LZ4 block codec for sm_90a, bit-exact with liblz4's LZ4_compress_default: below 64 KiB + 11 bytes in the
// 16-bit-index hash table regime every SSTable chunk length <= 64 KiB falls in (byU16), above it in the 32-bit-index regime of chunks of
// 128 KiB to 1 MiB (byU32: 4096 entries hashed from 5 bytes, candidates farther back than 65535 bytes are not matches).
//
// Replaces the JNI boundary of S/io/compress/LZ4Compressor.java:113-134 (compress) and :136-190 (uncompress).
// One warp owns one chunk. The greedy match finder is sequential by definition (the hash table state after position i
// decides what position i+1 sees), so the warp speculates: 32 consecutive search attempts are evaluated at once —
// hashes, table probes and 4-byte compares in parallel, intra-window table dependencies resolved with match.any —
// and the first hit in attempt order wins, which is exactly what the sequential loop would have found. Literal runs,
// match extension and back-tracking ("catch up") are done 32 bytes per step with ballots.
#pragma once
#include "common.cuh"

namespace b200c {

enum { LZ4_MINMATCH = 4, LZ4_MFLIMIT = 12, LZ4_LASTLITERALS = 5, LZ4_MINLENGTH = 13, LZ4_HASHLOG_U16 = 13,
       LZ4_TABLE_ENTRIES = 1 << LZ4_HASHLOG_U16, LZ4_64KLIMIT = 65536 + 11, LZ4_HASHLOG_U32 = 12, LZ4_DISTANCE_MAX = 65535 };

__host__ __device__ __forceinline__ int lz4_compress_bound(int n) { return n + n / 255 + 16; }
__device__ __forceinline__ uint32_t lz4_hash_u16(uint32_t seq) { return (seq * 2654435761u) >> (32 - LZ4_HASHLOG_U16); }
// LZ4_hash5 of a 64-bit build: the 5 bytes at the position (seq = the first four, b4 = the fifth) times prime5bytes, top 12 bits
__device__ __forceinline__ uint32_t lz4_hash_u32(uint32_t seq, uint32_t b4) {
    return (uint32_t)((((((uint64_t)b4 << 32) | seq) << 24) * 889523592379ull) >> (64 - LZ4_HASHLOG_U32));
}
// the table entry type of a regime: byU16 for inputs below LZ4_64KLIMIT, byU32 from there on (LZ4_compress_fast_extState)
template <bool U32> struct Lz4Tab { typedef uint16_t T; };
template <> struct Lz4Tab<true> { typedef uint32_t T; };

// distance from the search start of attempt a: steps are 1 for the first 64 attempts after the initial one, then grow by one
// every 64 attempts (LZ4_skipTrigger = 6, acceleration = 1)
__device__ __forceinline__ int lz4_attempt_offset(int a) {
    if (a <= 65) return a;
    int m = a - 1, q = m >> 6, r = m & 63;
    return 1 + 32 * q * (q + 1) + r * (q + 1);
}

// Writes `len` (>= 15 case handled by caller) extension bytes: (len/255) x 0xFF then len%255. Returns bytes written.
__device__ __forceinline__ int lz4_emit_len_ext(uint8_t* out, int rem, int lane) {
    int nff = rem / 255;
    for (int i = lane; i < nff; i += 32) out[i] = 255;
    if (lane == 0) out[nff] = (uint8_t)(rem - nff * 255);
    return nff + 1;
}

// s_in: chunk bytes (4-byte aligned, >= n + 8 readable bytes); s_tab: 8192 x u16 in shared memory (zeroed here);
// out: destination (global), capacity >= lz4_compress_bound(n). Returns the compressed size (warp-uniform).
// GLOBAL = false: s_in is a shared-memory copy of the chunk. GLOBAL = true: s_in is the chunk where it lies in global memory, read
// through the read-only L1 path (ld.global.nc): only the hash table occupies shared memory then, which doubles the chunks an SM holds
// — and this kernel is a chain of dependent instructions per chunk, so chunks in flight are what buys throughput. No byte beyond
// position n - 1 influences the result (searches stop at n - 12, matches at n - 5), so what follows the chunk in memory is irrelevant.
// With 13 one-warp blocks on an SM the time is the number of L2 round trips one warp waits for one after the other, so the GLOBAL path
// issues reads as soon as their addresses are known: three dependent trips per sequence (the search window's bytes, the candidates'
// bytes, then catch-up + literals + match length in one round) where reading each when it is used makes five. No load is past byte n - 1.
template <bool GLOBAL> __device__ __forceinline__ uint32_t lz4_rd32(const uint32_t* in32, int p) {
    if (!GLOBAL) return rd32_at(in32, p);
    uint32_t lo = __ldg(in32 + (p >> 2)), hi = __ldg(in32 + (p >> 2) + 1);
    return __funnelshift_r(lo, hi, (p & 3) * 8);
}
template <bool GLOBAL> __device__ __forceinline__ uint32_t lz4_rd8(const uint8_t* in, int p) { return GLOBAL ? (uint32_t)__ldg(in + p) : (uint32_t)in[p]; }

// s_dup (optional, LZ4_DUP_ENTRIES bytes of shared memory, any content): lets a search window prove in five instructions that no two of its
// attempts share a hash — the usual case — instead of building the same-hash masks with 13 ballots.
// U32 (needs GLOBAL, n >= LZ4_64KLIMIT): liblz4's byU32 regime — s_tab is 4096 x u32 (16 KiB as well), the hash reads a fifth byte (the
// high word the GLOBAL read fetched anyway) and a candidate more than LZ4_DISTANCE_MAX bytes back is no match (its slot is still updated).
enum { LZ4_DUP_ENTRIES = 2048 };
template <bool GLOBAL, bool U32 = false> __device__ int lz4_compress_warp(const uint8_t* s_in, int n, typename Lz4Tab<U32>::T* s_tab, uint8_t* out, int lane,
                                                                         uint8_t* s_dup = nullptr) {
    static_assert(GLOBAL || !U32, "the byU32 regime reads the chunk in place");
    constexpr int HASHLOG = U32 ? LZ4_HASHLOG_U32 : LZ4_HASHLOG_U16;
    const uint32_t* in32 = (const uint32_t*)s_in;
    {   // zero the hash table: 16 KiB, 16 bytes per lane per step
        uint4* t4 = (uint4*)s_tab;
        for (int i = lane; i < (LZ4_TABLE_ENTRIES * 2) / 16; i += 32) t4[i] = make_uint4(0, 0, 0, 0);
    }
    __syncwarp();
    int anchor = 0, op = 0;
    const int mfl1 = n - LZ4_MFLIMIT + 1;        // mflimitPlusOne
    const int matchlimit = n - LZ4_LASTLITERALS;
    const uint32_t lt_mask = (1u << lane) - 1u;

    if (n >= LZ4_MINLENGTH) {
        // "First byte": position 0 is inserted with value 0 — already the zeroed state.
        // After every match liblz4 (1) inserts position ip-2, (2) tests position ip (lookup + insert; a hit is an immediate match
        // with no literals and no back-tracking), (3) otherwise resumes the search at ip+1. Those three steps are folded into
        // the FIRST window after a match: lane 0 = insert-only ip-2, lane 1 = the test of ip, lanes 2..31 = search attempts 0..29.
        // The lane order equals the sequential order, so the same-hash resolution below needs no special case.
        int fwd = 1; bool have_prefix = false; int pre_ip = 0;
        for (;;) {
            int ip = 0, match = 0, token_pos; bool ended = false, immediate = false;
            // ---- search: up to 32 attempts per step -----------------------------------------------------------------
            int a0 = 0;
            for (bool first = true;; first = false) {
                const bool prefixed = first && have_prefix;
                int p; bool valid, putonly = false;
                if (prefixed && lane < 2) { p = lane == 0 ? pre_ip - 2 : pre_ip; valid = true; putonly = lane == 0; }
                else {
                    int a = a0 + lane - (prefixed ? 2 : 0);
                    p = fwd + lz4_attempt_offset(a);
                    int pn = fwd + lz4_attempt_offset(a + 1);
                    valid = pn <= mfl1;
                }
                uint32_t seq, h;
                if constexpr (U32) {
                    const uint32_t lo = valid ? __ldg(in32 + (p >> 2)) : 0u, hi = valid ? __ldg(in32 + (p >> 2) + 1) : 0u, sh = (p & 3) * 8;
                    seq = __funnelshift_r(lo, hi, sh);
                    h = lz4_hash_u32(seq, (hi >> sh) & 0xffu);
                } else {
                    seq = valid ? lz4_rd32<GLOBAL>(in32, p) : 0u;
                    h = lz4_hash_u16(seq);
                }
                int cand = valid ? (int)s_tab[h] : 0;
                // the table's candidate is nearly always the one compared: ask for its bytes before the same-hash masks are built, so that
                // the round trip runs under the ballots; a lane whose candidate is an earlier lane of this window takes that lane's `seq`
                uint32_t cseq = GLOBAL ? lz4_rd32<GLOBAL>(in32, cand) : 0u;
                // lanes with the same hash. match.any costs several hundred cycles here (one pass per distinct value); 13 ballots, one
                // per hash bit, are independent of each other and give the same mask. Invalid lanes form a suffix that neither
                // `prev` (lower lanes only) nor the masked `later_same` tests below can reach, so they need no special key.
                uint32_t same = FULL_MASK;
                bool unique = false;
                if (s_dup) {
                    // every valid lane writes its number into the slot of its hash (one of the writers of a slot wins): a lane that reads back
                    // another number shares the slot, i.e. possibly the hash, with someone; no such lane = all hashes distinct
                    const uint32_t dh = h & (LZ4_DUP_ENTRIES - 1);
                    if (valid) s_dup[dh] = (uint8_t)lane;
                    __syncwarp();
                    const bool shared = valid && s_dup[dh] != (uint8_t)lane;
                    unique = !__any_sync(FULL_MASK, shared);
                }
                if (unique) same = 1u << lane;
                else {
#pragma unroll
                    for (int b = 0; b < HASHLOG; b++) { uint32_t mb = __ballot_sync(FULL_MASK, (h >> b) & 1u); same &= ((h >> b) & 1u) ? mb : ~mb; }
                }
                uint32_t prev = same & lt_mask;
                int src = prev ? (31 - __clz(prev)) : lane;
                int pc = __shfl_sync(FULL_MASK, p, src);
                if (prev) cand = pc;
                if (GLOBAL) { const uint32_t sseq = __shfl_sync(FULL_MASK, seq, src); if (prev) cseq = sseq; }   // that lane read those four bytes
                // (an invalid lane's `cand` may be an invalid lane's p, beyond the chunk: it must not be read)
                bool hit = valid && !putonly && ((GLOBAL ? cseq : lz4_rd32<GLOBAL>(in32, cand)) == seq);
                if constexpr (U32) hit = hit && p - cand <= LZ4_DISTANCE_MAX;
                uint32_t hits = __ballot_sync(FULL_MASK, hit);
                uint32_t inval = __ballot_sync(FULL_MASK, !valid);
                int first_hit = hits ? (__ffs(hits) - 1) : 32;
                int first_inv = inval ? (__ffs(inval) - 1) : 32;
                if (first_hit < first_inv) {
                    uint32_t le = (first_hit == 31) ? FULL_MASK : ((2u << first_hit) - 1u);
                    uint32_t later_same = same & le & ~lt_mask & ~(1u << lane);
                    if (lane <= first_hit && !later_same) s_tab[h] = (typename Lz4Tab<U32>::T)p;
                    ip = __shfl_sync(FULL_MASK, p, first_hit);
                    match = __shfl_sync(FULL_MASK, cand, first_hit);
                    immediate = prefixed && first_hit == 1;
                    break;
                }
                if (first_inv < 32) { ended = true; break; }
                {
                    uint32_t later_same = same & ~lt_mask & ~(1u << lane);
                    if (!later_same) s_tab[h] = (typename Lz4Tab<U32>::T)p;
                }
                __syncwarp();
                a0 += prefixed ? 30 : 32;
            }
            if (ended) break;
            __syncwarp();

            int lit_nibble = 0, mc = 0;
            if (GLOBAL) {
                // One round of loads instead of three dependent ones. The backward extension, the first 32 literals and the first 32 bytes
                // of the match length read at addresses that the hit alone decides: the forward compare starts at the hit's ip + 4
                // wherever catch-up ends (the bytes between are known to be equal), and the literals start at anchor. Every chunk
                // byte is a round trip to L2 here, so the three are asked for together and only the long cases loop.
                const int ip0 = ip, m0 = match;
                const bool bk = !immediate && ip0 - 1 - lane >= anchor && m0 - 1 - lane >= 0;
                const bool fw = ip0 + LZ4_MINMATCH + lane < matchlimit;
                const bool lt = !immediate && anchor + lane < ip0;
                const uint32_t bi = bk ? lz4_rd8<GLOBAL>(s_in, ip0 - 1 - lane) : 0u, bm = bk ? lz4_rd8<GLOBAL>(s_in, m0 - 1 - lane) : 1u;
                const uint32_t fi = fw ? lz4_rd8<GLOBAL>(s_in, ip0 + LZ4_MINMATCH + lane) : 0u, fm = fw ? lz4_rd8<GLOBAL>(s_in, m0 + LZ4_MINMATCH + lane) : 1u;
                const uint32_t lb = lt ? lz4_rd8<GLOBAL>(s_in, anchor + lane) : 0u;
                // ---- catch up ---------------------------------------------------------------------------------------
                uint32_t b = __ballot_sync(FULL_MASK, bi == bm);
                while (b == FULL_MASK) {
                    ip -= 32; match -= 32;
                    const int j = lane + 1;
                    const bool ok = (ip - j >= anchor) && (match - j >= 0) && (lz4_rd8<GLOBAL>(s_in, ip - j) == lz4_rd8<GLOBAL>(s_in, match - j));
                    b = __ballot_sync(FULL_MASK, ok);
                }
                { const int steps = __ffs(~b) - 1; ip -= steps; match -= steps; }
                // ---- literals ---------------------------------------------------------------------------------------
                token_pos = op++;
                if (!immediate) {
                    const int lit = ip - anchor;
                    if (lit >= 15) op += lz4_emit_len_ext(out + op, lit - 15, lane);
                    if (lane < lit) out[op + lane] = (uint8_t)lb;
                    for (int i = lane + 32; i < lit; i += 32) out[op + i] = (uint8_t)lz4_rd8<GLOBAL>(s_in, anchor + i);
                    op += lit;
                    lit_nibble = lit < 15 ? lit : 15;
                }
                // ---- the match: offset, length beyond MINMATCH limited by matchlimit (LZ4_count) ----------------------
                if (lane == 0) { int off = ip - match; out[op] = (uint8_t)off; out[op + 1] = (uint8_t)(off >> 8); }
                op += 2;
                const int pi = ip0 + LZ4_MINMATCH, pm = m0 + LZ4_MINMATCH;
                b = __ballot_sync(FULL_MASK, fi == fm);
                int fc = 0;
                while (b == FULL_MASK) {
                    fc += 32;
                    const int i = fc + lane;
                    const bool eq = (pi + i < matchlimit) && (lz4_rd8<GLOBAL>(s_in, pi + i) == lz4_rd8<GLOBAL>(s_in, pm + i));
                    b = __ballot_sync(FULL_MASK, eq);
                }
                fc += __ffs(~b) - 1;
                mc = (ip0 - ip) + fc;                     // liblz4 counts from the caught-up ip + 4: the bytes up to the hit's ip + 4 are equal
            } else {                                       // the chunk in shared memory: each step reads when it knows where
                if (!immediate) {
                    // ---- catch up: extend the match backwards -------------------------------------------------------
                    for (;;) {
                        int j = lane + 1;
                        bool ok = (ip - j >= anchor) && (match - j >= 0) && (lz4_rd8<GLOBAL>(s_in, ip - j) == lz4_rd8<GLOBAL>(s_in, match - j));
                        uint32_t b = __ballot_sync(FULL_MASK, ok);
                        int steps = (b == FULL_MASK) ? 32 : (__ffs(~b) - 1);
                        ip -= steps; match -= steps;
                        if (steps < 32) break;
                    }
                    // ---- literals -----------------------------------------------------------------------------------
                    int lit = ip - anchor;
                    token_pos = op++;
                    if (lit >= 15) op += lz4_emit_len_ext(out + op, lit - 15, lane);
                    for (int i = lane; i < lit; i += 32) out[op + i] = (uint8_t)lz4_rd8<GLOBAL>(s_in, anchor + i);
                    op += lit;
                    lit_nibble = lit < 15 ? lit : 15;
                } else token_pos = op++;                  // immediate match: token with literal length 0
                // ---- the match: offset, length beyond MINMATCH limited by matchlimit (LZ4_count) ----------------------
                if (lane == 0) { int off = ip - match; out[op] = (uint8_t)off; out[op + 1] = (uint8_t)(off >> 8); }
                op += 2;
                int pi = ip + LZ4_MINMATCH, pm = match + LZ4_MINMATCH;
                for (;;) {
                    int i = mc + lane;
                    bool eq = (pi + i < matchlimit) && (lz4_rd8<GLOBAL>(s_in, pi + i) == lz4_rd8<GLOBAL>(s_in, pm + i));
                    uint32_t b = __ballot_sync(FULL_MASK, eq);
                    if (b == FULL_MASK) { mc += 32; continue; }
                    mc += __ffs(~b) - 1;
                    break;
                }
            }
            ip += mc + LZ4_MINMATCH;
            if (lane == 0) out[token_pos] = (uint8_t)((lit_nibble << 4) | (mc < 15 ? mc : 15));
            if (mc >= 15) op += lz4_emit_len_ext(out + op, mc - 15, lane);
            anchor = ip;
            if (ip >= mfl1) break;
            have_prefix = true; pre_ip = ip; fwd = ip + 1;
        }
    }
    // ---- last literals ------------------------------------------------------------------------------------------
    {
        int last = n - anchor;
        if (lane == 0) out[op] = (uint8_t)((last < 15 ? last : 15) << 4);
        op++;
        if (last >= 15) op += lz4_emit_len_ext(out + op, last - 15, lane);
        for (int i = lane; i < last; i += 32) out[op + i] = (uint8_t)lz4_rd8<GLOBAL>(s_in, anchor + i);
        op += last;
    }
    return op;
}

// LZ4_decompress_safe semantics. src: compressed block (global, n bytes); s_out: destination (global or shared memory, cap bytes).
// Returns decoded size or -1 on malformed input (warp-uniform). Literal and match copies run 32 bytes per step.
__device__ int lz4_decompress_warp(const uint8_t* __restrict__ src, int n, uint8_t* s_out, int cap, int lane) {
    int ip = 0, op = 0;
    if (n == 0) return cap == 0 ? 0 : -1;
    for (;;) {
        if (ip >= n) return -1;
        uint32_t token = src[ip++];
        int len = token >> 4;
        if (len == 15) { uint32_t s; do { if (ip >= n) return -1; s = src[ip++]; len += (int)s; } while (s == 255 && len < (1 << 24)); }
        if (n - ip < len || cap - op < len) return -1;
        for (int i = lane; i < len; i += 32) s_out[op + i] = src[ip + i];
        op += len; ip += len;
        if (ip == n) break;
        if (n - ip < 2) return -1;
        int offset = (int)src[ip] | ((int)src[ip + 1] << 8); ip += 2;
        if (offset == 0 || offset > op) return -1;
        int ml = token & 15;
        if (ml == 15) { uint32_t s; do { if (ip >= n) return -1; s = src[ip++]; ml += (int)s; } while (s == 255 && ml < (1 << 24)); }
        ml += LZ4_MINMATCH;
        if (cap - op < ml) return -1;
        __syncwarp();
        const uint8_t* m = s_out + op - offset;
        for (int i = lane; i < ml; i += 32) { int j = i; if (j >= offset) j %= offset; s_out[op + i] = m[j]; }
        op += ml;
        __syncwarp();
    }
    __syncwarp();
    return op;
}

} // namespace b200c
