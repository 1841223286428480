// codec_defs.cuh — chunk codec constants shared by the codec kernels (codec.cuh) and the compaction driver (compact.cu).
#pragma once
#include "common.cuh"
#include "k1_tail.cuh"

namespace b200c {

enum { COMP_NONE = 0, COMP_LZ4 = 1, COMP_SNAPPY = 2, COMP_SNAPPY15 = 3 };      // SNAPPY15: hash table of up to 2^15 entries (snappy >= 1.2.0)
// compression disabled: Data.db is the uncompressed stream and the chunk table holds CRC.db's per-chunk CRC32s (include/b200c.h)
enum { COMP_UNCOMPRESSED = 4 };
__host__ __device__ __forceinline__ bool comp_is_snappy(int c) { return c == COMP_SNAPPY || c == COMP_SNAPPY15; }

// chunk lengths: powers of two up to 1 MiB (CompressionParams allows any power of two; tables raise it to 128-512 KiB for scans), up to
// 64 KiB for CRC.db of an uncompressed table (ChecksummedSequentialWriter writes 64 KiB). Chunks above CHUNK_LEN_SMALL take their own K5 kernels.
enum { CHUNK_LEN_SMALL = 65536, CHUNK_LEN_MAX = 1 << 20 };
__host__ __device__ __forceinline__ bool chunk_len_supported(int comp, int chunk_len) {
    return chunk_len > 0 && (chunk_len & (chunk_len - 1)) == 0 && chunk_len <= (comp == COMP_UNCOMPRESSED ? (int)CHUNK_LEN_SMALL : (int)CHUNK_LEN_MAX);
}
__host__ __device__ __forceinline__ int chunk_max_compressed(int comp, int chunk_len) {
    if (comp == COMP_LZ4) return 4 + (chunk_len + chunk_len / 255 + 16);
    if (comp_is_snappy(comp)) return (32 + chunk_len + chunk_len / 6);
    return chunk_len;
}
__host__ __device__ __forceinline__ int chunk_slot_stride(int comp, int chunk_len) {
    int m = chunk_max_compressed(comp, chunk_len); if (m < chunk_len) m = chunk_len;
    return (m + 4 + 16 + 15) & ~15;      // bytes + CRC + read slack, 16-byte aligned
}

struct ChunkErr { unsigned long long first_bad; };   // min over failing chunks of (input << 48 | chunk index << 8 | kind); init ~0

__device__ __forceinline__ void report_chunk_err(ChunkErr* e, uint64_t chunk, int kind) {
    atomicMin(&e->first_bad, ((unsigned long long)chunk << 8) | (unsigned long long)kind);
}

// one input's chunk range [chunk0, chunk0 + count) in a multi-input K1 launch; first = threads of the launch before this segment
struct K1Seg { const uint8_t* data; uint64_t data_len; const uint64_t* offs; uint64_t nchunks; uint64_t data_length; uint8_t* out;
               uint64_t chunk0, count, first; int chunk_len, max_clen, tag, comp;     // comp: read by k_decompress_multi_warp only (the others are LZ4)
               uint64_t rec0, rec_span;         // two-pass LZ4 (lz4_batch.cuh): first record slot of this segment, compressed bytes its slots were sized for
               const uint8_t* tail; uint64_t tail_off; };     // staged copy of the file's bytes from tail_off on (k1_src)

// one launch of the uncompressed-stream kernels (codec.cuh: k_raw_ingest / k_raw_checksum)
enum { RAW_WARPS = 8, RAW_THREADS = 32 * RAW_WARPS };
struct RawArgs {
    const uint8_t* src; uint8_t* dst;       // dst: null = nothing stored (verify in place, checksum only)
    uint64_t n; int L, tag;                 // stream bytes, chunk length, input number of error reports
    uint64_t chunk0, chunk_end;             // chunks [chunk0, chunk_end) of the stream
    const uint64_t* crc_exp;                // K1: CRC.db entries to verify against (kind 1 on a mismatch)
    uint64_t* crc_out;                      // K5: CRC.db entries, zero-extended
    uint32_t* seg_raw;                      // K5: zero-init CRC register of each chunk (k_digest)
    uint64_t* ends; uint64_t ebase;         // K5: ends[c + 1] = ebase + end of chunk c and ends[0] = ebase (k_digest's offsets)
    ChunkErr* err;
};

} // namespace b200c
