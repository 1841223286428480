// codec_defs.cuh — chunk codec constants shared by the codec kernels (codec.cuh) and the compaction driver (compact.cu).
#pragma once
#include "common.cuh"
#include "k1_tail.cuh"

namespace b200c {

enum { COMP_NONE = 0, COMP_LZ4 = 1, COMP_SNAPPY = 2, COMP_SNAPPY15 = 3 };      // SNAPPY15: hash table of up to 2^15 entries (snappy >= 1.2.0)
__host__ __device__ __forceinline__ bool comp_is_snappy(int c) { return c == COMP_SNAPPY || c == COMP_SNAPPY15; }

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
               uint64_t chunk0, count, first; int chunk_len, max_clen, tag, _pad;
               uint64_t rec0, rec_span;         // two-pass LZ4 (lz4_batch.cuh): first record slot of this segment, compressed bytes its slots were sized for
               const uint8_t* tail; uint64_t tail_off; };     // staged copy of the file's bytes from tail_off on (k1_src)

} // namespace b200c
