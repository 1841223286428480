// codec.cuh — chunk codec kernels (K1 decompress + CRC verify, K5 compress fused with CRC32, pack, digest).
//
// K5 replaces CompressedSequentialWriter.flushData (S/io/compress/CompressedSequentialWriter.java:140-206): one warp
// per 16 KiB chunk compresses it (LZ4 bit-exact with liblz4 / Snappy), writes the chunk into a fixed-stride slot,
// computes the CRC32 of the bytes as written (ChecksumWriter.appendDirect, S/io/util/ChecksumWriter.java:62-89) in the
// same kernel while the bytes are still in L1/L2, and appends it big-endian. A scan over the chunk sizes gives the
// CompressionInfo.db offsets (CompressionMetadata.Writer.addOffset), k_pack_chunks moves the slots into the dense
// Data.db image and k_digest folds the per-chunk CRCs into Digest.crc32 with x^(8n) shifts (no re-read of the bytes).
// K1 replaces CompressedChunkReader.readChunk (S/io/util/CompressedChunkReader.java:103-173).
#pragma once
#include "common.cuh"
#include "lz4.cuh"
#include "lz4_chain.cuh"
#include "snappy_chain.cuh"
#include "snappy.cuh"
#include "codec_defs.cuh"
#include "lz4_thread.cuh"
#include "lz4_batch.cuh"

namespace b200c {

// ---- K5: compress + CRC ------------------------------------------------------------------------------------------
// grid = nchunks blocks of one warp. dynamic smem: [hash table tab_bytes][chunk bytes chunk_len + 16]
__global__ void __launch_bounds__(32) k_compress_chunks(const DevTables* __restrict__ T, int comp, int tab_bytes,
        const uint8_t* __restrict__ in, uint64_t n, int chunk_len, int max_clen,
        uint8_t* __restrict__ slots, int slot_stride, uint32_t* __restrict__ file_len, uint32_t* __restrict__ seg_raw) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint16_t* s_tab = (uint16_t*)smem;
    uint8_t* s_in = smem + tab_bytes;     // lz4: 8192 x u16 (16 KiB); snappy: 16384 x u16 (32 KiB)
    const int lane = threadIdx.x;
    const uint64_t chunk = blockIdx.x;
    const uint64_t start = chunk * (uint64_t)chunk_len;
    const int ulen = (int)min((uint64_t)chunk_len, n - start);
    const uint8_t* src = in + start;

    // stage the chunk in shared memory (16-byte vectors when aligned), zero the slack
    if ((((uintptr_t)src) & 15) == 0) {
        const uint4* s4 = (const uint4*)src; uint4* d4 = (uint4*)s_in;
        int nv = ulen >> 4;
        for (int i = lane; i < nv; i += 32) d4[i] = __ldg(s4 + i);
        for (int i = (nv << 4) + lane; i < ulen; i += 32) s_in[i] = src[i];
    } else {
        for (int i = lane; i < ulen; i += 32) s_in[i] = src[i];
    }
    if (lane < 16) s_in[ulen + lane] = 0;
    __syncwarp();

    uint8_t* slot = slots + chunk * (uint64_t)slot_stride;
    int clen;
    if (comp == COMP_LZ4) {
        if (lane == 0) { slot[0] = (uint8_t)ulen; slot[1] = (uint8_t)(ulen >> 8); slot[2] = (uint8_t)(ulen >> 16); slot[3] = (uint8_t)(ulen >> 24); }
        clen = 4 + lz4_compress_warp<false>(s_in, ulen, s_tab, slot + 4, lane);
    } else if (comp_is_snappy(comp)) {
        clen = snappy_compress_warp(s_in, ulen, s_tab, comp == COMP_SNAPPY15 ? 15 : 14, slot, lane);
    } else {
        clen = ulen;
        for (int i = lane; i < ulen; i += 32) slot[i] = s_in[i];
    }
    // flushData :158-177 — store raw when compression did not help enough (never with the default ratio)
    if (comp != COMP_NONE && clen >= max_clen) {
        for (int i = lane; i < ulen; i += 32) slot[i] = s_in[i];
        clen = ulen;
        if (ulen < max_clen) { for (int i = ulen + lane; i < max_clen; i += 32) slot[i] = 0; clen = max_clen; }
    }
    __syncwarp();
    __threadfence_block();
    // CRC32 over the bytes as written, appended big-endian
    uint32_t raw = warp_crc32_raw(T, T->crc_adv128, slot, clen, lane);
    uint32_t init = gf2_mulmod(0xFFFFFFFFu, warp_xpow8n(T, (uint32_t)clen, lane));
    uint32_t crc = ~(raw ^ init);
    if (lane == 0) {
        slot[clen] = (uint8_t)(crc >> 24); slot[clen + 1] = (uint8_t)(crc >> 16); slot[clen + 2] = (uint8_t)(crc >> 8); slot[clen + 3] = (uint8_t)crc;
        file_len[chunk] = (uint32_t)clen + 4;
        // zero-init register of (chunk bytes || 4 CRC bytes): advance (raw ^ LE word of the CRC bytes) by 4 bytes
        uint32_t x = raw ^ __byte_perm(crc, 0, 0x0123);
        seg_raw[chunk] = T->crc_t[3][x & 0xff] ^ T->crc_t[2][(x >> 8) & 0xff] ^ T->crc_t[1][(x >> 16) & 0xff] ^ T->crc_t[0][x >> 24];
    }
}

// LZ4 with only the 16 KiB hash table in shared memory: the chunk is read where it lies (L1 read-only path), 13 blocks of one warp per
// SM instead of 7: 3 warps per scheduler, so the time is the length of one warp's chain of L2 round trips, which lz4_compress_warp<true>
// keeps to three per sequence (lz4.cuh). Needs a 4-byte aligned stream start and chunk length (every caller's buffers are).
template <bool DUP>
__global__ void __launch_bounds__(32) k_compress_chunks_lz4_direct(const DevTables* __restrict__ T,
        const uint8_t* __restrict__ in, uint64_t n, int chunk_len, int max_clen,
        uint8_t* __restrict__ slots, int slot_stride, uint32_t* __restrict__ file_len, uint32_t* __restrict__ seg_raw) {
    __shared__ __align__(16) uint16_t s_tab[LZ4_TABLE_ENTRIES];
    __shared__ uint8_t s_dup[DUP ? LZ4_DUP_ENTRIES : 1];
    const int lane = threadIdx.x;
    const uint64_t chunk = blockIdx.x;
    const uint64_t start = chunk * (uint64_t)chunk_len;
    const int ulen = (int)min((uint64_t)chunk_len, n - start);
    const uint8_t* src = in + start;
    uint8_t* slot = slots + chunk * (uint64_t)slot_stride;
    if (lane == 0) { slot[0] = (uint8_t)ulen; slot[1] = (uint8_t)(ulen >> 8); slot[2] = (uint8_t)(ulen >> 16); slot[3] = (uint8_t)(ulen >> 24); }
    int clen = 4 + lz4_compress_warp<true>(src, ulen, s_tab, slot + 4, lane, DUP ? s_dup : nullptr);
    if (clen >= max_clen) {                            // flushData :158-177 — store raw when compression did not help enough
        for (int i = lane; i < ulen; i += 32) slot[i] = src[i];
        clen = ulen;
        if (ulen < max_clen) { for (int i = ulen + lane; i < max_clen; i += 32) slot[i] = 0; clen = max_clen; }
    }
    __syncwarp();
    __threadfence_block();
    uint32_t raw = warp_crc32_raw(T, T->crc_adv128, slot, clen, lane);
    uint32_t init = gf2_mulmod(0xFFFFFFFFu, warp_xpow8n(T, (uint32_t)clen, lane));
    uint32_t crc = ~(raw ^ init);
    if (lane == 0) {
        slot[clen] = (uint8_t)(crc >> 24); slot[clen + 1] = (uint8_t)(crc >> 16); slot[clen + 2] = (uint8_t)(crc >> 8); slot[clen + 3] = (uint8_t)crc;
        file_len[chunk] = (uint32_t)clen + 4;
        uint32_t x = raw ^ __byte_perm(crc, 0, 0x0123);
        seg_raw[chunk] = T->crc_t[3][x & 0xff] ^ T->crc_t[2][(x >> 8) & 0xff] ^ T->crc_t[1][(x >> 16) & 0xff] ^ T->crc_t[0][x >> 24];
    }
}

// LZ4 in two passes (lz4_chain.cuh). Pass A: the two nearest earlier same-hash positions of every position, one warp per chunk with the
// hash tables in shared memory and no parse. Pass B: the parse, with one bit per position in shared memory — 2 KiB per 16 KiB chunk
// instead of the 16 KiB table, so residency is set by registers, not by shared memory. ent: one word per byte of the stream.
__global__ void __launch_bounds__(32) k_lz4_chain_build(const uint8_t* __restrict__ in, uint64_t n, int chunk_len, uint32_t* __restrict__ ent) {
    __shared__ __align__(16) uint16_t s_t1[LZ4_TABLE_ENTRIES];
    const uint64_t start = (uint64_t)blockIdx.x * (uint64_t)chunk_len;
    const int ulen = (int)min((uint64_t)chunk_len, n - start);
    lz4_chain_build_warp<true>(in + start, ulen, s_t1, ent + start, threadIdx.x);
}
enum { K5B_WARPS = 4 };
__global__ void __launch_bounds__(32 * K5B_WARPS) k_compress_chunks_lz4_chain(const DevTables* __restrict__ T,
        const uint8_t* __restrict__ in, uint64_t n, int chunk_len, int max_clen, const uint32_t* __restrict__ ent,
        uint8_t* __restrict__ slots, int slot_stride, uint32_t* __restrict__ file_len, uint32_t* __restrict__ seg_raw, uint64_t nchunks) {
    extern __shared__ __align__(16) uint32_t s_bits[];             // K5B_WARPS x ceil(chunk_len / 32) words
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t chunk = (uint64_t)blockIdx.x * K5B_WARPS + wid;
    if (chunk >= nchunks) return;
    const uint64_t start = chunk * (uint64_t)chunk_len;
    const int ulen = (int)min((uint64_t)chunk_len, n - start);
    const uint8_t* src = in + start;
    uint8_t* slot = slots + chunk * (uint64_t)slot_stride;
    if (lane == 0) { slot[0] = (uint8_t)ulen; slot[1] = (uint8_t)(ulen >> 8); slot[2] = (uint8_t)(ulen >> 16); slot[3] = (uint8_t)(ulen >> 24); }
    int clen = 4 + lz4_compress_warp_chain(src, ulen, ent + start, s_bits + (size_t)wid * ((chunk_len + 31) >> 5), slot + 4, lane);
    if (clen >= max_clen) {                            // flushData :158-177 — store raw when compression did not help enough
        for (int i = lane; i < ulen; i += 32) slot[i] = src[i];
        clen = ulen;
        if (ulen < max_clen) { for (int i = ulen + lane; i < max_clen; i += 32) slot[i] = 0; clen = max_clen; }
    }
    __syncwarp();
    __threadfence_block();
    uint32_t raw = warp_crc32_raw(T, T->crc_adv128, slot, clen, lane);
    uint32_t init = gf2_mulmod(0xFFFFFFFFu, warp_xpow8n(T, (uint32_t)clen, lane));
    uint32_t crc = ~(raw ^ init);
    if (lane == 0) {
        slot[clen] = (uint8_t)(crc >> 24); slot[clen + 1] = (uint8_t)(crc >> 16); slot[clen + 2] = (uint8_t)(crc >> 8); slot[clen + 3] = (uint8_t)crc;
        file_len[chunk] = (uint32_t)clen + 4;
        uint32_t x = raw ^ __byte_perm(crc, 0, 0x0123);
        seg_raw[chunk] = T->crc_t[3][x & 0xff] ^ T->crc_t[2][(x >> 8) & 0xff] ^ T->crc_t[1][(x >> 16) & 0xff] ^ T->crc_t[0][x >> 24];
    }
}

// Snappy in two passes (snappy_chain.cuh). dynamic smem of the build pass: one table of table_size u16.
__global__ void __launch_bounds__(32) k_snappy_chain_build(int max_bits, int table_size, const uint8_t* __restrict__ in, uint64_t n, int chunk_len, uint32_t* __restrict__ ent) {
    extern __shared__ __align__(16) uint8_t smem_sc[];               // the table: table_size x u16
    const uint64_t start = (uint64_t)blockIdx.x * (uint64_t)chunk_len;
    const int ulen = (int)min((uint64_t)chunk_len, n - start);
    snappy_chain_build_warp<true>(in + start, ulen, max_bits, (uint16_t*)smem_sc, ent + start, threadIdx.x);
}
__global__ void __launch_bounds__(32 * K5B_WARPS) k_compress_chunks_snappy_chain(const DevTables* __restrict__ T,
        const uint8_t* __restrict__ in, uint64_t n, int chunk_len, int max_clen, const uint32_t* __restrict__ ent,
        uint8_t* __restrict__ slots, int slot_stride, uint32_t* __restrict__ file_len, uint32_t* __restrict__ seg_raw, uint64_t nchunks) {
    extern __shared__ __align__(16) uint32_t s_bits[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t chunk = (uint64_t)blockIdx.x * K5B_WARPS + wid;
    if (chunk >= nchunks) return;
    const uint64_t start = chunk * (uint64_t)chunk_len;
    const int ulen = (int)min((uint64_t)chunk_len, n - start);
    const uint8_t* src = in + start;
    uint8_t* slot = slots + chunk * (uint64_t)slot_stride;
    int clen = snappy_compress_warp_chain(src, ulen, ent + start, s_bits + (size_t)wid * ((chunk_len + 31) >> 5), slot, lane);
    if (clen >= max_clen) {
        for (int i = lane; i < ulen; i += 32) slot[i] = src[i];
        clen = ulen;
        if (ulen < max_clen) { for (int i = ulen + lane; i < max_clen; i += 32) slot[i] = 0; clen = max_clen; }
    }
    __syncwarp();
    __threadfence_block();
    uint32_t raw = warp_crc32_raw(T, T->crc_adv128, slot, clen, lane);
    uint32_t init = gf2_mulmod(0xFFFFFFFFu, warp_xpow8n(T, (uint32_t)clen, lane));
    uint32_t crc = ~(raw ^ init);
    if (lane == 0) {
        slot[clen] = (uint8_t)(crc >> 24); slot[clen + 1] = (uint8_t)(crc >> 16); slot[clen + 2] = (uint8_t)(crc >> 8); slot[clen + 3] = (uint8_t)crc;
        file_len[chunk] = (uint32_t)clen + 4;
        uint32_t x = raw ^ __byte_perm(crc, 0, 0x0123);
        seg_raw[chunk] = T->crc_t[3][x & 0xff] ^ T->crc_t[2][(x >> 8) & 0xff] ^ T->crc_t[1][(x >> 16) & 0xff] ^ T->crc_t[0][x >> 24];
    }
}

// Snappy the same way: only the hash table (32 KiB for 16 KiB chunks, 64 KiB for the 15-bit generation) in shared memory, 6 chunks per SM
// instead of 4. dynamic smem = tab_bytes.
__global__ void __launch_bounds__(32) k_compress_chunks_snappy_direct(const DevTables* __restrict__ T, int max_bits,
        const uint8_t* __restrict__ in, uint64_t n, int chunk_len, int max_clen,
        uint8_t* __restrict__ slots, int slot_stride, uint32_t* __restrict__ file_len, uint32_t* __restrict__ seg_raw) {
    extern __shared__ __align__(16) uint8_t smem_tab[];
    uint16_t* s_tab = (uint16_t*)smem_tab;
    const int lane = threadIdx.x;
    const uint64_t chunk = blockIdx.x;
    const uint64_t start = chunk * (uint64_t)chunk_len;
    const int ulen = (int)min((uint64_t)chunk_len, n - start);
    const uint8_t* src = in + start;
    uint8_t* slot = slots + chunk * (uint64_t)slot_stride;
    int clen = snappy_compress_warp<true>(src, ulen, s_tab, max_bits, slot, lane);
    if (clen >= max_clen) {
        for (int i = lane; i < ulen; i += 32) slot[i] = src[i];
        clen = ulen;
        if (ulen < max_clen) { for (int i = ulen + lane; i < max_clen; i += 32) slot[i] = 0; clen = max_clen; }
    }
    __syncwarp();
    __threadfence_block();
    uint32_t raw = warp_crc32_raw(T, T->crc_adv128, slot, clen, lane);
    uint32_t init = gf2_mulmod(0xFFFFFFFFu, warp_xpow8n(T, (uint32_t)clen, lane));
    uint32_t crc = ~(raw ^ init);
    if (lane == 0) {
        slot[clen] = (uint8_t)(crc >> 24); slot[clen + 1] = (uint8_t)(crc >> 16); slot[clen + 2] = (uint8_t)(crc >> 8); slot[clen + 3] = (uint8_t)crc;
        file_len[chunk] = (uint32_t)clen + 4;
        uint32_t x = raw ^ __byte_perm(crc, 0, 0x0123);
        seg_raw[chunk] = T->crc_t[3][x & 0xff] ^ T->crc_t[2][(x >> 8) & 0xff] ^ T->crc_t[1][(x >> 16) & 0xff] ^ T->crc_t[0][x >> 24];
    }
}

// ---- K5 for chunks of 128 KiB to 1 MiB ---------------------------------------------------------------------------------------------
// A chunk this long does not fit in shared memory: it is read where it lies, as the direct kernels above read theirs. The kernels below
// take every such chunk whatever B200C_K5 says (the switch selects among the kernels of chunks <= 64 KiB), so the output never depends on it.

// the raw-storage rule and the CRC of a finished slot, as the kernels above apply them: stored raw (zero padded to max_clen) when compression
// did not help enough, then the big-endian CRC32 of the bytes as written, the file length and the digest register
__device__ __forceinline__ void k5_finish_slot(const DevTables* __restrict__ T, const uint8_t* src, int ulen, int clen, int max_clen, uint8_t* slot,
                                               uint64_t chunk, uint32_t* __restrict__ file_len, uint32_t* __restrict__ seg_raw, int lane) {
    if (clen >= max_clen) {                            // flushData :158-177
        for (int i = lane; i < ulen; i += 32) slot[i] = src[i];
        clen = ulen;
        if (ulen < max_clen) { for (int i = ulen + lane; i < max_clen; i += 32) slot[i] = 0; clen = max_clen; }
    }
    __syncwarp();
    __threadfence_block();
    uint32_t raw = warp_crc32_raw(T, T->crc_adv128, slot, clen, lane);
    uint32_t init = gf2_mulmod(0xFFFFFFFFu, warp_xpow8n(T, (uint32_t)clen, lane));
    uint32_t crc = ~(raw ^ init);
    if (lane == 0) {
        slot[clen] = (uint8_t)(crc >> 24); slot[clen + 1] = (uint8_t)(crc >> 16); slot[clen + 2] = (uint8_t)(crc >> 8); slot[clen + 3] = (uint8_t)crc;
        file_len[chunk] = (uint32_t)clen + 4;
        uint32_t x = raw ^ __byte_perm(crc, 0, 0x0123);
        seg_raw[chunk] = T->crc_t[3][x & 0xff] ^ T->crc_t[2][(x >> 8) & 0xff] ^ T->crc_t[1][(x >> 16) & 0xff] ^ T->crc_t[0][x >> 24];
    }
}

// LZ4: one warp per chunk in liblz4's byU32 regime (lz4.cuh). A short last chunk below LZ4_64KLIMIT is compressed byU16, as liblz4 does.
// Needs a 4-byte aligned stream start.
__global__ void __launch_bounds__(32) k_compress_chunks_lz4_big(const DevTables* __restrict__ T,
        const uint8_t* __restrict__ in, uint64_t n, int chunk_len, int max_clen,
        uint8_t* __restrict__ slots, int slot_stride, uint32_t* __restrict__ file_len, uint32_t* __restrict__ seg_raw) {
    __shared__ __align__(16) uint32_t s_tab[1 << LZ4_HASHLOG_U32];          // 16 KiB: 4096 x u32, or 8192 x u16 for a short last chunk
    const int lane = threadIdx.x;
    const uint64_t chunk = blockIdx.x;
    const uint64_t start = chunk * (uint64_t)chunk_len;
    const int ulen = (int)min((uint64_t)chunk_len, n - start);
    const uint8_t* src = in + start;
    uint8_t* slot = slots + chunk * (uint64_t)slot_stride;
    if (lane == 0) { slot[0] = (uint8_t)ulen; slot[1] = (uint8_t)(ulen >> 8); slot[2] = (uint8_t)(ulen >> 16); slot[3] = (uint8_t)(ulen >> 24); }
    const int clen = 4 + (ulen >= LZ4_64KLIMIT ? lz4_compress_warp<true, true>(src, ulen, s_tab, slot + 4, lane)
                                               : lz4_compress_warp<true>(src, ulen, (uint16_t*)s_tab, slot + 4, lane));
    k5_finish_slot(T, src, ulen, clen, max_clen, slot, chunk, file_len, seg_raw, lane);
}

// Snappy: snappy::Compress cuts its input into 64 KiB fragments (kBlockSize) and compresses each on its own with a table sized for it, so the
// fragments of a chunk are independent. Pass 1: one warp per fragment (snappy_compress_fragment_warp) into a fragment slot; dynamic smem =
// the table of a 64 KiB fragment. Pass 2: one warp per chunk writes the varint length and the fragments back to back, then the raw rule and CRC.
enum { SNAPPY_BLOCK = 65536 };
__global__ void __launch_bounds__(32) k_snappy_big_fragments(int max_bits, const uint8_t* __restrict__ in, uint64_t n, int chunk_len,
                                                             uint8_t* __restrict__ frag_slots, int frag_stride, uint32_t* __restrict__ frag_len) {
    extern __shared__ __align__(16) uint8_t smem_sf[];
    uint16_t* s_tab = (uint16_t*)smem_sf;
    const int lane = threadIdx.x;
    const uint64_t f = blockIdx.x, fpc = (uint64_t)(chunk_len / SNAPPY_BLOCK);
    const uint64_t start = (f / fpc) * (uint64_t)chunk_len + (f % fpc) * SNAPPY_BLOCK;
    if (start >= n) { if (lane == 0) frag_len[f] = 0; return; }           // past the end of a short last chunk
    const int len = (int)min((uint64_t)SNAPPY_BLOCK, n - start);
    const int tsz = snappy_table_size(len, max_bits);
    for (int i = lane; i < tsz / 2; i += 32) ((uint32_t*)s_tab)[i] = 0;
    __syncwarp();
    const int op = snappy_compress_fragment_warp<true>(in + start, 0, len, s_tab, tsz, max_bits, frag_slots + f * (uint64_t)frag_stride, 0, lane);
    if (lane == 0) frag_len[f] = (uint32_t)op;
}
__global__ void __launch_bounds__(32) k_snappy_big_assemble(const DevTables* __restrict__ T, const uint8_t* __restrict__ in, uint64_t n, int chunk_len, int max_clen,
        const uint8_t* __restrict__ frag_slots, int frag_stride, const uint32_t* __restrict__ frag_len,
        uint8_t* __restrict__ slots, int slot_stride, uint32_t* __restrict__ file_len, uint32_t* __restrict__ seg_raw) {
    const int lane = threadIdx.x;
    const uint64_t chunk = blockIdx.x;
    const uint64_t start = chunk * (uint64_t)chunk_len;
    const int ulen = (int)min((uint64_t)chunk_len, n - start);
    uint8_t* slot = slots + chunk * (uint64_t)slot_stride;
    int op = 0;
    {   uint32_t v = (uint32_t)ulen;
        while (v >= 0x80) { if (lane == 0) slot[op] = (uint8_t)(v | 0x80); v >>= 7; op++; }
        if (lane == 0) slot[op] = (uint8_t)v;
        op++; }
    const uint64_t f0 = chunk * (uint64_t)(chunk_len / SNAPPY_BLOCK);
    for (int k = 0; k * SNAPPY_BLOCK < ulen; k++) {
        const int len = (int)frag_len[f0 + k];
        const uint8_t* s = frag_slots + (f0 + k) * (uint64_t)frag_stride;
        for (int i = lane; i < len; i += 32) slot[op + i] = s[i];
        op += len;
    }
    k5_finish_slot(T, in + start, ulen, op, max_clen, slot, chunk, file_len, seg_raw, lane);
}

// NoopCompressor: the chunk as it is
__global__ void __launch_bounds__(32) k_compress_chunks_noop_big(const DevTables* __restrict__ T, const uint8_t* __restrict__ in, uint64_t n, int chunk_len, int max_clen,
        uint8_t* __restrict__ slots, int slot_stride, uint32_t* __restrict__ file_len, uint32_t* __restrict__ seg_raw) {
    const int lane = threadIdx.x;
    const uint64_t chunk = blockIdx.x;
    const uint64_t start = chunk * (uint64_t)chunk_len;
    const int ulen = (int)min((uint64_t)chunk_len, n - start);
    uint8_t* slot = slots + chunk * (uint64_t)slot_stride;
    for (int i = lane; i < ulen; i += 32) slot[i] = in[start + i];
    k5_finish_slot(T, in + start, ulen, ulen, max_clen, slot, chunk, file_len, seg_raw, lane);
}

// ---- pack: slots -> dense Data.db image --------------------------------------------------------------------------
// one warp per chunk; offs = exclusive scan of file_len
// out_base (optional): device scalar subtracted from the offsets, for an image buffer that holds only a window of the file
__global__ void __launch_bounds__(128) k_pack_chunks(const uint8_t* __restrict__ slots, int slot_stride, const uint32_t* __restrict__ file_len,
                                                     const uint64_t* __restrict__ offs, uint64_t nchunks, uint8_t* __restrict__ out,
                                                     const uint64_t* __restrict__ out_base) {
    uint64_t chunk = (uint64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (chunk >= nchunks) return;
    int lane = threadIdx.x & 31;
    const uint8_t* s = slots + chunk * (uint64_t)slot_stride;
    uint8_t* d = out + (offs[chunk] - (out_base ? *out_base : 0ull));
    int len = (int)file_len[chunk];
    // head bytes until d is 16-byte aligned, then 16-byte stores assembled from two aligned 16-byte loads
    int head = (int)((16 - ((uintptr_t)d & 15)) & 15); if (head > len) head = len;
    if (lane < head) d[lane] = s[lane];
    int body = (len - head) >> 4;
    const uint8_t* sb = s + head; uint8_t* db = d + head;
    int mis = (int)((uintptr_t)sb & 15);
    const uint4* sa = (const uint4*)(sb - mis);
    for (int i = lane; i < body; i += 32) {
        uint4 a = sa[i];
        uint4 r = a;
        if (mis) {
            uint4 b = sa[i + 1];
            uint32_t w[8] = { a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w };
            int ws = mis >> 2, bs = (mis & 3) * 8;
            r.x = __funnelshift_r(w[ws], w[ws + 1], bs); r.y = __funnelshift_r(w[ws + 1], w[ws + 2], bs);
            r.z = __funnelshift_r(w[ws + 2], w[ws + 3], bs); r.w = __funnelshift_r(w[ws + 3], w[ws + 4], bs);
        }
        ((uint4*)db)[i] = r;
    }
    int done = head + (body << 4);
    for (int i = done + lane; i < len; i += 32) d[i] = s[i];
}

// ---- digest: Digest.crc32 from per-chunk registers ---------------------------------------------------------------
// acc[0] ^= seg_raw[i] * x^(8 * bytes after segment i); final value fixed up on the host side of the launch
__global__ void __launch_bounds__(256) k_digest(const DevTables* __restrict__ T, const uint32_t* __restrict__ seg_raw,
                                                const uint64_t* __restrict__ offs /*n+1*/, uint64_t nchunks, uint32_t* __restrict__ acc) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t v = 0;
    if (i < nchunks) {
        uint64_t total = offs[nchunks];
        v = gf2_mulmod(seg_raw[i], gf2_xpow8n(T, total - offs[i + 1]));
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) v ^= __shfl_xor_sync(FULL_MASK, v, d);
    if ((threadIdx.x & 31) == 0 && v) atomicXor(acc, v);
}
__global__ void k_digest_final(const DevTables* __restrict__ T, const uint64_t* __restrict__ offs, uint64_t nchunks, uint32_t* __restrict__ acc) {
    uint64_t total = offs[nchunks];
    acc[1] = ~(acc[0] ^ gf2_mulmod(0xFFFFFFFFu, gf2_xpow8n(T, total)));
}

// ---- uncompressed Data.db + CRC.db: K1 ingest (verify, copy into U) and K5 checksum (copy out, CRC per chunk) -----------------------
// ChecksummedSequentialWriter (S/io/util/ChecksummedSequentialWriter.java) writes Data.db as it is, and CRC.db as the BE i32 chunk size
// followed by one BE i32 CRC32 per chunk (ChecksumWriter.appendDirect, S/io/util/ChecksumWriter.java:62-89). Each chunk is streamed once by
// one block: its warps cut it into contiguous segments of whole 512-byte rows, lane l loads (and stores) the aligned 16-byte words
// l, l + 32, ... of its warp's segment, folds each word with slice-by-4 and advances its register by one row (crc_adv512) per step. The
// lane registers are shifted to the segment's end (xp_lane16) and XOR-reduced, the segments to the chunk's end (x^(8n)).
__device__ __forceinline__ uint32_t crc_step4(const uint32_t (*t)[256], uint32_t x) {
    return t[3][x & 0xff] ^ t[2][(x >> 8) & 0xff] ^ t[1][(x >> 16) & 0xff] ^ t[0][x >> 24];
}
__device__ __forceinline__ void raw_chunks_block(const DevTables* __restrict__ T, const RawArgs& a) {
    __shared__ uint32_t s_crc[4][256], s_adv[4][256], s_xl[32], s_part[RAW_WARPS];
    for (int i = threadIdx.x; i < 1024; i += RAW_THREADS) { s_crc[i >> 8][i & 255] = T->crc_t[i >> 8][i & 255]; s_adv[i >> 8][i & 255] = T->crc_adv512[i >> 8][i & 255]; }
    if (threadIdx.x < 32) s_xl[threadIdx.x] = T->xp_lane16[threadIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (uint64_t chunk = a.chunk0 + blockIdx.x; chunk < a.chunk_end; chunk += gridDim.x) {
        const uint64_t start = chunk * (uint64_t)a.L;
        const uint32_t len = (uint32_t)min((uint64_t)a.L, a.n - start);
        const uint8_t* src = a.src + start; uint8_t* dst = a.dst ? a.dst + start : nullptr;
        // 16-byte words from the first aligned address of the chunk on (a file of an LCS output starts wherever its first partition does);
        // the bytes before it and behind the last whole word go byte by byte below. A destination must share the source's alignment.
        const uint32_t head = min(len, (uint32_t)((16 - ((uintptr_t)src & 15)) & 15));
        const bool vec = !dst || ((((uintptr_t)src) ^ ((uintptr_t)dst)) & 15) == 0;
        const uint32_t nbody = vec ? (len - head) & ~15u : 0;      // bytes taken as 16-byte words
        if (vec) {
            const uint32_t nw = nbody >> 4, rows = (nw + 31) >> 5, rpw = (rows + RAW_WARPS - 1) / RAW_WARPS;
            const uint32_t wb = min(nw, wid * rpw * 32), we = min(nw, (wid + 1) * rpw * 32), sw = we - wb;
            const uint4* s4 = (const uint4*)(src + head) + wb; uint4* d4 = dst ? (uint4*)(dst + head) + wb : nullptr;
            const int pad = (int)((32 - (sw & 31)) & 31), nrow = (int)((sw + pad) >> 5);     // virtual leading zero words: whole rows
            uint32_t u = 0;
#pragma unroll 4
            for (int k = 0; k < nrow; k++) {
                const int idx = k * 32 + lane - pad;
                uint32_t s = 0;
                if (idx >= 0) {
                    const uint4 v = s4[idx];
                    if (d4) d4[idx] = v;
                    s = crc_step4(s_crc, v.x); s = crc_step4(s_crc, s ^ v.y); s = crc_step4(s_crc, s ^ v.z); s = crc_step4(s_crc, s ^ v.w);
                }
                u = crc_adv128(s_adv, u) ^ s;
            }
            uint32_t r = gf2_mulmod(u, s_xl[lane]);
#pragma unroll
            for (int d = 16; d; d >>= 1) r ^= __shfl_xor_sync(FULL_MASK, r, d);
            if (lane == 0) s_part[wid] = (r && nbody > we * 16) ? gf2_mulmod(r, gf2_xpow8n(T, nbody - we * 16)) : r;
        } else {                                                    // source and destination aligned differently: bytes
            if (dst) for (uint32_t i = threadIdx.x; i < len; i += RAW_THREADS) dst[i] = src[i];
            if (wid == 0) { const uint32_t r = warp_crc32_raw(T, T->crc_adv128, src, (int)len, lane); if (lane == 0) s_part[0] = r; }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t raw = s_part[0];
            if (vec) {
                uint32_t body = s_part[0];
                for (int w = 1; w < RAW_WARPS; w++) body ^= s_part[w];
                raw = 0;                                            // register(head || body) = register(head) * x^(8 |body|) ^ register(body)
                for (uint32_t i = 0; i < head; i++) { const uint8_t b = src[i]; raw = s_crc[0][(raw ^ b) & 0xff] ^ (raw >> 8); if (dst) dst[i] = b; }
                if (raw && nbody) raw = gf2_mulmod(raw, gf2_xpow8n(T, nbody));
                raw ^= body;
                for (uint32_t i = head + nbody; i < len; i++) { const uint8_t b = src[i]; raw = s_crc[0][(raw ^ b) & 0xff] ^ (raw >> 8); if (dst) dst[i] = b; }
            }
            const uint32_t crc = ~(raw ^ gf2_mulmod(0xFFFFFFFFu, gf2_xpow8n(T, len)));
            if (a.crc_out) a.crc_out[chunk] = crc;
            if (a.seg_raw) a.seg_raw[chunk] = raw;
            if (a.ends) { a.ends[chunk + 1] = a.ebase + start + len; if (chunk == 0) a.ends[0] = a.ebase; }
            if (a.crc_exp && a.crc_exp[chunk] != (uint64_t)crc) report_chunk_err(a.err, ((uint64_t)a.tag << 40) | chunk, 1);
        }
        __syncthreads();
    }
}
// K1 of an uncompressed input: verify every chunk against CRC.db, copy it into U unless it was copied there from the host
__global__ void __launch_bounds__(RAW_THREADS, 8) k_raw_ingest(const DevTables* __restrict__ T, const RawArgs a) { raw_chunks_block(T, a); }
// K5 of an uncompressed output: the CRC.db entry and digest register of every chunk, the bytes copied out when a destination is given
__global__ void __launch_bounds__(RAW_THREADS, 8) k_raw_checksum(const DevTables* __restrict__ T, const RawArgs a) { raw_chunks_block(T, a); }

// ---- K1: CRC verify + decompress ----------------------------------------------------------------------------------
// One warp per chunk, two chunks per block, NO shared-memory image: literals and matches are written straight to the output
// stream in global memory and match sources are read back from it (a warp may read what its other lanes stored after
// __syncwarp()). Dropping the 16 KiB staging buffer raises residency from 13 to 32 warps per SM, which is what this
// latency-bound, strictly sequential format needs.
// the warp-per-chunk decoder: chunk `chunk` of one file, lanes 0..31 of a warp
__device__ __forceinline__ void decompress_chunk_warp(const DevTables* __restrict__ T, int comp,
        const uint8_t* __restrict__ data, uint64_t data_len, const uint64_t* __restrict__ offs, uint64_t nchunks,
        int chunk_len, int max_clen, uint64_t data_length, uint8_t* out, int verify, ChunkErr* __restrict__ err,
        uint64_t chunk, int tag, const uint8_t* __restrict__ tail, uint64_t tail_off, int lane) {
    const uint64_t off = offs[chunk];
    const uint64_t next = (chunk + 1 < nchunks) ? offs[chunk + 1] : data_len;
    const uint64_t ustart = chunk * (uint64_t)chunk_len;
    if (off + 4 > next || next > data_len || ustart >= data_length || next - off - 4 > (uint64_t)(chunk_max_compressed(comp, chunk_len) + chunk_len)) {
        if (lane == 0) report_chunk_err(err, ((uint64_t)tag << 40) | chunk, 2);
        return;
    }
    const int clen = (int)(next - off - 4);
    const int ulen = (int)min((uint64_t)chunk_len, data_length - ustart);
    const uint8_t* src = k1_src(data, tail, tail_off, off);
    if (verify) {
        uint32_t crc = warp_crc32(T, T->crc_adv128, src, clen, lane);
        uint32_t stored = ((uint32_t)src[clen] << 24) | ((uint32_t)src[clen + 1] << 16) | ((uint32_t)src[clen + 2] << 8) | src[clen + 3];
        if (crc != stored) { if (lane == 0) report_chunk_err(err, ((uint64_t)tag << 40) | chunk, 1); return; }
    }
    uint8_t* dst = out + ustart;
    int got;
    if (clen >= max_clen) {                 // CompressedChunkReader.java:116,219: raw chunk (possibly zero padded at the file end)
        if (clen < ulen) { if (lane == 0) report_chunk_err(err, ((uint64_t)tag << 40) | chunk, 2); return; }
        for (int i = lane; i < ulen; i += 32) dst[i] = src[i];
        got = ulen;
    } else if (comp == COMP_LZ4) {
        int plen = (clen >= 4) ? (int)((uint32_t)src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24)) : -1;
        got = (plen == ulen) ? lz4_decompress_warp(src + 4, clen - 4, dst, ulen, lane) : -1;
    } else if (comp_is_snappy(comp)) {
        got = snappy_decompress_warp(src, clen, dst, ulen, lane);
    } else {
        got = (clen == ulen) ? ulen : -1;
        if (got >= 0) for (int i = lane; i < ulen; i += 32) dst[i] = src[i];
    }
    if (got != ulen && lane == 0) report_chunk_err(err, ((uint64_t)tag << 40) | chunk, 2);
}
__global__ void __launch_bounds__(64) k_decompress_chunks(const DevTables* __restrict__ T, int comp,
        const uint8_t* __restrict__ data, uint64_t data_len, const uint64_t* __restrict__ offs, uint64_t nchunks,
        int chunk_len, int max_clen, uint64_t data_length, uint8_t* out, int verify, ChunkErr* __restrict__ err,
        uint64_t chunk0, uint64_t chunk_end, int tag,         // this launch covers chunks [chunk0, chunk_end) of the file; tag = input number for error reports
        const uint8_t* __restrict__ tail, uint64_t tail_off) {  // (k1_src)
    const int lane = threadIdx.x & 31;
    const uint64_t chunk = chunk0 + (uint64_t)blockIdx.x * 2 + (threadIdx.x >> 5);
    if (chunk >= chunk_end || chunk >= nchunks) return;
    decompress_chunk_warp(T, comp, data, data_len, offs, nchunks, chunk_len, max_clen, data_length, out, verify, err, chunk, tag, tail, tail_off, lane);
}

// chunks above 64 KiB of several inputs in ONE launch, one warp per chunk. Such a chunk is a long chain of dependent steps (a 1 MiB LZ4 chunk
// holds ~10^5 sequences), so a launch lasts as long as its slowest chunk: one launch for all inputs instead of one after the other per input.
__global__ void __launch_bounds__(64) k_decompress_multi_warp(const DevTables* __restrict__ T, const K1Seg* __restrict__ segs, int nseg, uint64_t total,
                                                              int verify, ChunkErr* __restrict__ err) {
    const uint64_t t = (uint64_t)blockIdx.x * 2 + (threadIdx.x >> 5);
    if (t >= total) return;
    int lo = 0, hi = nseg - 1;
    while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (segs[mid].first <= t) lo = mid; else hi = mid - 1; }
    const K1Seg& g = segs[lo];
    const uint64_t chunk = g.chunk0 + (t - g.first);
    if (chunk >= g.nchunks) return;
    decompress_chunk_warp(T, g.comp, g.data, g.data_len, g.offs, g.nchunks, g.chunk_len, g.max_clen, g.data_length, g.out, verify, err, chunk, g.tag,
                          g.tail, g.tail_off, threadIdx.x & 31);
}

// ---- K1, thread-per-chunk variant (LZ4 and stored chunks) -----------------------------------------------------------------
// The warp-per-chunk kernel above has 32 chunks per SM in flight and each of them is a chain of dependent loads; this one has one
// chunk per THREAD (2048 per SM in flight), i.e. it trades coalescing for 64 times the memory-level parallelism. To keep the
// traffic at word granularity the output goes through an 8-byte write-combining register (aligned 64-bit stores only) and all
// sources are read with two aligned 64-bit loads + a funnel shift. CRC32: slice-by-4 with the tables in shared memory.
__device__ __forceinline__ void decompress_chunk_thread(const uint32_t (*s_crc)[256], int comp,
        const uint8_t* __restrict__ data, uint64_t data_len, const uint64_t* __restrict__ offs, uint64_t nchunks,
        int chunk_len, int max_clen, uint64_t data_length, uint8_t* out, int verify, ChunkErr* __restrict__ err, uint64_t chunk, int tag,
        const uint8_t* __restrict__ tail, uint64_t tail_off) {
    const uint64_t off = offs[chunk];
    const uint64_t next = (chunk + 1 < nchunks) ? offs[chunk + 1] : data_len;
    const uint64_t ustart = chunk * (uint64_t)chunk_len;
    const uint64_t ctag = ((uint64_t)tag << 40) | chunk;
    if (off + 4 > next || next > data_len || ustart >= data_length || next - off - 4 > (uint64_t)(chunk_max_compressed(comp, chunk_len) + chunk_len)) { report_chunk_err(err, ctag, 2); return; }
    const int clen = (int)(next - off - 4);
    const int ulen = (int)min((uint64_t)chunk_len, data_length - ustart);
    const uint8_t* src = k1_src(data, tail, tail_off, off);
    if (verify) {
        uint32_t crc = 0xFFFFFFFFu; int i = 0;
        // a thread's chunk is its private stream: fetching it 8 bytes at a time asks for every 32-byte sector four times, with a few thousand
        // other threads' sectors in between, so that the same bytes come from DRAM several times. The body therefore takes whole sectors — two
        // aligned 16-byte loads per step — after a byte-wise run-up to the first 16-byte boundary.
        {
            int head = (int)((16u - (uint32_t)((uintptr_t)src & 15u)) & 15u); if (head > clen) head = clen;
            for (; i < head; i++) crc = s_crc[0][(crc ^ src[i]) & 0xff] ^ (crc >> 8);
            for (; i + 32 <= clen; i += 32) {
                const uint4 a = __ldg((const uint4*)(src + i)), b4 = __ldg((const uint4*)(src + i + 16));
                const uint32_t w[8] = {a.x, a.y, a.z, a.w, b4.x, b4.y, b4.z, b4.w};
#pragma unroll
                for (int k = 0; k < 8; k++) { const uint32_t x = crc ^ w[k]; crc = s_crc[3][x & 0xff] ^ s_crc[2][(x >> 8) & 0xff] ^ s_crc[1][(x >> 16) & 0xff] ^ s_crc[0][x >> 24]; }
            }
        }
        for (; i + 8 <= clen; i += 8) {
            uint64_t v = ld_le64(src + i);
            uint32_t x = crc ^ (uint32_t)v;
            crc = s_crc[3][x & 0xff] ^ s_crc[2][(x >> 8) & 0xff] ^ s_crc[1][(x >> 16) & 0xff] ^ s_crc[0][x >> 24];
            x = crc ^ (uint32_t)(v >> 32);
            crc = s_crc[3][x & 0xff] ^ s_crc[2][(x >> 8) & 0xff] ^ s_crc[1][(x >> 16) & 0xff] ^ s_crc[0][x >> 24];
        }
        for (; i < clen; i++) crc = s_crc[0][(crc ^ src[i]) & 0xff] ^ (crc >> 8);
        crc = ~crc;
        uint32_t stored = ((uint32_t)src[clen] << 24) | ((uint32_t)src[clen + 1] << 16) | ((uint32_t)src[clen + 2] << 8) | src[clen + 3];
        if (crc != stored) { report_chunk_err(err, ctag, 1); return; }
    }
    uint8_t* dst = out + ustart;
    int got;
    if (clen >= max_clen) {                 // stored chunk (possibly zero padded at the file end)
        if (clen < ulen) { report_chunk_err(err, ctag, 2); return; }
        WordSink w{dst, 0, 0ull};
        int i = 0;
        for (; i + 8 <= ulen; i += 8) w.put(ld_le64(src + i), 8);
        if (i < ulen) w.put(low_bytes(ld_le64(src + i), ulen - i), ulen - i);
        w.flush_bytes();
        got = ulen;
    } else {
        int plen = (clen >= 4) ? (int)((uint32_t)src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24)) : -1;
        got = (plen == ulen) ? lz4_decompress_thread(src + 4, clen - 4, dst, ulen) : -1;
    }
    if (got != ulen) report_chunk_err(err, ctag, 2);
}

// threads per block of the two kernels below, their static shared memory (the CRC tables), and the L2 bytes each chunk in flight is
// given (engine.cu: k1_plan). 768: 4 blocks of 128 per SM on an H100 (50 MiB L2, 132 SMs) — the fastest point of the curve measured
// on configs[1] (DESIGN §7: 2 blocks 71 ms, 3: 60, 4: 58, 6: 75; all 12 the registers allow: 138).
enum { K1_THREADS = 128, K1_STATIC_SMEM = 4 * 256 * 4 };
constexpr uint64_t K1_L2_BYTES_PER_CHAIN = 768;

__global__ void __launch_bounds__(K1_THREADS) k_decompress_chunks_thr(const DevTables* __restrict__ T, int comp,
        const uint8_t* __restrict__ data, uint64_t data_len, const uint64_t* __restrict__ offs, uint64_t nchunks,
        int chunk_len, int max_clen, uint64_t data_length, uint8_t* out, int verify, ChunkErr* __restrict__ err,
        uint64_t chunk0, uint64_t chunk_end, int tag, const uint8_t* __restrict__ tail, uint64_t tail_off) {
    __shared__ uint32_t s_crc[4][256];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) s_crc[i >> 8][i & 255] = T->crc_t[i >> 8][i & 255];
    __syncthreads();
    if (chunk_end > nchunks) chunk_end = nchunks;
    for (uint64_t chunk = chunk0 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; chunk < chunk_end; chunk += (uint64_t)gridDim.x * blockDim.x)
        decompress_chunk_thread(s_crc, comp, data, data_len, offs, nchunks, chunk_len, max_clen, data_length, out, verify, err, chunk, tag, tail, tail_off);
}

// the same over chunk ranges of several inputs in ONE launch. Both thread kernels loop over their chunks in launch order; the grid is
// sized by k1_grid (engine.cu) so that the chunks in flight keep their working set in the caches. Here a thread that finishes takes the
// next chunk from a counter (`next`, zeroed by the launch): no thread waits behind a slow chunk's neighbours.
__global__ void __launch_bounds__(K1_THREADS) k_decompress_multi_thr(const DevTables* __restrict__ T, const K1Seg* __restrict__ segs, int nseg, uint64_t total,
                                                              int verify, ChunkErr* __restrict__ err, unsigned long long* __restrict__ next) {
    __shared__ uint32_t s_crc[4][256];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) s_crc[i >> 8][i & 255] = T->crc_t[i >> 8][i & 255];
    __syncthreads();
    const uint64_t G = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t = G + atomicAdd(next, 1ull)) {
        int lo = 0, hi = nseg - 1;
        while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (segs[mid].first <= t) lo = mid; else hi = mid - 1; }
        const K1Seg g = segs[lo];
        const uint64_t chunk = g.chunk0 + (t - g.first);
        if (chunk >= g.nchunks) continue;
        decompress_chunk_thread(s_crc, COMP_LZ4, g.data, g.data_len, g.offs, g.nchunks, g.chunk_len, g.max_clen, g.data_length, g.out, verify, err, chunk, g.tag,
                                g.tail, g.tail_off);
    }
}

// ---- K1 in two passes (lz4_batch.cuh): walk (thread per chunk: validate, record the sequence starts) then copy (warp per chunk, 32 sequences
// per step). Record slots: a block of n bytes has at most (n - 1) / 3 + 1 sequences, so chunk c of a segment owns the u16 slots from
// rec0 + (offs[c] - offs[chunk0]) / 3 + 2 (c - chunk0) on — no scan, no second walk.
enum : uint32_t { K1_SKIP = 0xFFFFFFFFu, K1_BAD = 0xFFFFFFFEu, K1_BAD_OFFS = 0xFFFFFFFDu, K1_RAW = 0xFFFFFFFCu };
struct K1Chunk { const uint8_t* src; uint8_t* dst; int clen, ulen; uint64_t slot, ctag; };
// which chunk thread/warp t of a multi-segment launch owns and where its bytes are; false: nothing to do (K1_SKIP) or bad offsets (reported)
__device__ __forceinline__ uint32_t k1_locate(const K1Seg* __restrict__ segs, int nseg, uint64_t t, K1Chunk& k) {
    int lo = 0, hi = nseg - 1;
    while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (segs[mid].first <= t) lo = mid; else hi = mid - 1; }
    const K1Seg& g = segs[lo];
    const uint64_t chunk = g.chunk0 + (t - g.first);
    if (chunk >= g.nchunks) return K1_SKIP;
    const uint64_t off = g.offs[chunk], next = (chunk + 1 < g.nchunks) ? g.offs[chunk + 1] : g.data_len, off0 = g.offs[g.chunk0];
    const uint64_t ustart = chunk * (uint64_t)g.chunk_len;
    k.ctag = ((uint64_t)g.tag << 40) | chunk;
    if (off + 4 > next || next > g.data_len || ustart >= g.data_length || next - off - 4 > (uint64_t)(chunk_max_compressed(COMP_LZ4, g.chunk_len) + g.chunk_len) ||
        off < off0 || next - off0 > g.rec_span) return K1_BAD_OFFS;
    k.clen = (int)(next - off - 4); k.ulen = (int)min((uint64_t)g.chunk_len, g.data_length - ustart);
    k.src = k1_src(g.data, g.tail, g.tail_off, off); k.dst = g.out + ustart;
    k.slot = g.rec0 + (off - off0) / 3 + 2 * (chunk - g.chunk0);
    return k.clen >= g.max_clen ? K1_RAW : 0u;
}
__global__ void __launch_bounds__(128) k_lz4_walk_multi(const K1Seg* __restrict__ segs, int nseg, uint64_t total, uint16_t* __restrict__ rec,
                                                        uint32_t* __restrict__ nseq, ChunkErr* __restrict__ err) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    K1Chunk k; const uint32_t st = k1_locate(segs, nseg, t, k);
    if (st == K1_SKIP) { nseq[t] = K1_SKIP; return; }
    if (st == K1_BAD_OFFS) { report_chunk_err(err, k.ctag, 2); nseq[t] = K1_BAD_OFFS; return; }
    if (st == K1_RAW) { if (k.clen < k.ulen) { report_chunk_err(err, k.ctag, 2); nseq[t] = K1_BAD; } else nseq[t] = K1_RAW; return; }
    const uint8_t* src = k.src;
    const int plen = (k.clen >= 4) ? (int)((uint32_t)src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24)) : -1;
    const int r = (plen == k.ulen) ? lz4_walk_thread(src + 4, k.clen - 4, k.ulen, rec + k.slot, (k.clen + 4) / 3 + 1) : -1;
    if (r < 0) { report_chunk_err(err, k.ctag, 2); nseq[t] = K1_BAD; } else nseq[t] = (uint32_t)r;
}
enum { K1C_WARPS = 4 };
__global__ void __launch_bounds__(32 * K1C_WARPS) k_lz4_copy_multi(const DevTables* __restrict__ T, const K1Seg* __restrict__ segs, int nseg, uint64_t total,
                                                                   const uint16_t* __restrict__ rec, const uint32_t* __restrict__ nseq, int verify, ChunkErr* __restrict__ err) {
    const int lane = threadIdx.x & 31;
    const uint64_t t = (uint64_t)blockIdx.x * K1C_WARPS + (threadIdx.x >> 5);
    if (t >= total) return;
    const uint32_t ns = nseq[t];
    if (ns == K1_SKIP || ns == K1_BAD_OFFS) return;
    K1Chunk k; (void)k1_locate(segs, nseg, t, k);
    if (verify) {                                      // (a chunk the walk refused still has its CRC looked at: a CRC mismatch is the error reported first)
        const uint32_t crc = warp_crc32(T, T->crc_adv128, k.src, k.clen, lane);
        const uint8_t* s = k.src + k.clen;
        const uint32_t stored = ((uint32_t)s[0] << 24) | ((uint32_t)s[1] << 16) | ((uint32_t)s[2] << 8) | s[3];
        if (crc != stored) { if (lane == 0) report_chunk_err(err, k.ctag, 1); return; }
    }
    if (ns == K1_BAD) return;
    if (ns == K1_RAW) { for (int i = lane; i < k.ulen; i += 32) k.dst[i] = k.src[i]; return; }
    (void)lz4_copy_warp(k.src + 4, k.clen - 4, rec + k.slot, (int)ns, k.dst, lane);
}

} // namespace b200c
