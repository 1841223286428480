// k1_tail.cuh — where K1 reads a chunk of a device-resident input. Plain C++ for host and device: tests/native/k1_tail_host.cc runs
// K1's per-chunk reads through it on the CPU under AddressSanitizer, over buffers that end exactly at the last byte of the file.
#pragma once
#include <cstdint>
#ifdef __CUDACC__
#define B200C_K1T_HD __host__ __device__ __forceinline__
#else
#define B200C_K1T_HD inline
#endif

namespace b200c {

// K1 reads a caller's device buffer in place, but its decoders fetch whole aligned words (up to 15 bytes past the last byte they use).
// The chunks that start in the last k1_tail_window() bytes of a file are therefore read from a staged copy of that tail, which has
// slack behind it. A chunk that starts earlier and passes K1's size check (record <= max_compressed + chunk_len + 4 bytes) ends more
// than 32 bytes before the end of the file.
B200C_K1T_HD uint64_t k1_tail_window(int max_compressed, int chunk_len) { return (uint64_t)max_compressed + (uint64_t)chunk_len + 4 + 32; }
// where the bytes of a chunk at file offset `off` are read (tail_off = ~0: no staged tail)
B200C_K1T_HD const uint8_t* k1_src(const uint8_t* data, const uint8_t* tail, uint64_t tail_off, uint64_t off) {
    return off >= tail_off ? tail + (off - tail_off) : data + off;
}

} // namespace b200c
