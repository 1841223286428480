// engine.cuh — context, workspace and launch bookkeeping shared by the C-ABI translation units.
#pragma once
#include <cstdio>
#include <cstring>
#include <string>
#include <atomic>
#include <chrono>
#include <vector>
#include "../../include/b200c.h"
#include "common.cuh"

namespace b200c {

enum { WS_SLOTS = 160, WS_K5_ENT = 150, WS_K1_REC = 151, WS_K1_NSEQ = 152, WS_K5_BIGIN = 153, WS_K5_FRAGS = 154, WS_K5_FLEN = 155 };
// (slots 0..15: codec calls, 16..: compact.cu's map, 150: K5's hash-chain entries, 151-152: K1's sequence records, 153-155: K5 of chunks above
//  64 KiB: an aligned copy of a misaligned stream, Snappy's fragment slots and lengths)

struct WsBuf { void* p = nullptr; size_t cap = 0; };

enum { MAX_RANGES = 16 };                // token-range pieces of one b200c_compact call
// slots of b200c_ctx::ev_pool: OutStream piece s uses EV_OUT_PIECE + 2 s (packed) and + 2 s + 1 (copied out); b200c_compact uses
// EV_RANGE + r (piece r's inputs are on the device), EV_INDEX_READY / EV_INDEX_FREE (a piece's Index.db is final / has left IOUT) and
// EV_UOUT_FREE + (r & 1) (the merged stream of an uncompressed host output has left its buffer)
enum { EV_OUT_PIECE = 0, EV_RANGE = 200, EV_INDEX_FREE = 220, EV_INDEX_READY = 221, EV_UOUT_FREE = 230, EV_POOL = 256 };
struct Pinned;

} // namespace b200c

struct b200c_ctx {
    int device = 0;
    int nsm = 0;                                   // SMs of the device: grid-stride kernels launch a fixed number of blocks per SM
    int l2_bytes = 0;                              // L2 cache of the device: sizes K1's chunks in flight (engine.cu: k1_plan)
    int smem_per_sm = 0, smem_reserved_per_block = 0;
    int k1_blocks_per_sm = 1; size_t k1_smem = 0;  // K1 thread kernels: resident blocks per SM and the dynamic shared memory that caps them there
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    b200c::DevTables* d_tables = nullptr;
    b200c::WsBuf ws[b200c::WS_SLOTS];
    b200c::Pinned* h_pinned = nullptr;             // small pinned scratch for scalar read-backs
    std::string err;
    uint64_t launches_call = 0, launches_total = 0;
    double last_ms = 0.0;
    std::atomic<int> cancel{0};
    std::atomic<uint64_t> prog_scanned{0}, prog_total{0};
    std::atomic<int> prog_stage{0}; std::atomic<int> prog_seq{0};
    std::atomic<int> prog_ninputs{0};
    std::atomic<uint64_t> prog_input_pos[B200C_MAX_INPUTS];   // uncompressed bytes of each input consumed so far (b200c_poll_inputs)
    bool timing = false;
    cudaEvent_t ev_stage[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    double stage_ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    int nstages = 0;
    int k4_attr_set = 0, k4s_attr_set = 0;
    cudaStream_t copy_stream = nullptr;            // host->device staging of the inputs, overlapped with K1 input by input
    cudaEvent_t ev_in[64] = {};
    std::vector<cudaEvent_t> ev_marks;             // timed events of the stage clock (grown on demand)
    cudaEvent_t ev_pool[b200c::EV_POOL] = {};      // untimed events (b200c::EV_*)
    cudaStream_t copy_out = nullptr;               // device->host stream of the outputs (the other copy engine)
};

namespace b200c {

#define B200C_CUDA_TRY(ctx, expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) { \
    (ctx)->err = std::string(#expr) + ": " + cudaGetErrorString(_e); return B200C_ECUDA; } } while (0)

#define B200C_LAUNCH(ctx, kernel, grid, block, smem, ...) do { \
    kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__); \
    (ctx)->launches_call++; (ctx)->launches_total++; \
    cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) { \
        (ctx)->err = std::string(#kernel) + " launch: " + cudaGetErrorString(_e); return B200C_ECUDA; } } while (0)

#define B200C_TRY(expr) do { int _rc = (expr); if (_rc != B200C_OK) return _rc; } while (0)

// workspace slot `slot` with at least `bytes` bytes (+64 bytes of readable slack); contents are NOT preserved on growth
inline int ws_get(b200c_ctx* c, int slot, size_t bytes, void** out) {
    WsBuf& b = c->ws[slot];
    size_t need = bytes + 256;
    if (b.cap < need) {
        if (b.p) { cudaStreamSynchronize(c->stream); if (c->copy_stream) cudaStreamSynchronize(c->copy_stream); if (c->copy_out) cudaStreamSynchronize(c->copy_out); cudaFree(b.p); b.p = nullptr; b.cap = 0; }
        size_t cap = need + need / 8;
        cudaError_t e = cudaMalloc(&b.p, cap);
        if (e != cudaSuccess) { cudaGetLastError(); c->err = "cudaMalloc(" + std::to_string(cap) + "): " + cudaGetErrorString(e); b.p = nullptr; return B200C_ENOMEM; }
        b.cap = cap;
    }
    *out = b.p;
    return B200C_OK;
}
template <typename T> inline int ws_typed(b200c_ctx* c, int slot, size_t count, T** out) {
    void* p = nullptr; int rc = ws_get(c, slot, count * sizeof(T), &p); *out = (T*)p; return rc;
}

// workspace slot that keeps its first `used` bytes when it has to grow (whole-file arrays of an OutStream)
template <typename T> inline int ws_grow_keep(b200c_ctx* c, int slot, size_t count, size_t used, T** out) {
    WsBuf& b = c->ws[slot];
    size_t need = count * sizeof(T) + 256;
    if (b.cap < need) {
        cudaStreamSynchronize(c->stream); cudaStreamSynchronize(c->copy_out);
        void* np = nullptr; size_t cap = need * 2;
        cudaError_t e = cudaMalloc(&np, cap);
        if (e != cudaSuccess) { cudaGetLastError(); c->err = "cudaMalloc(" + std::to_string(cap) + "): " + cudaGetErrorString(e); return B200C_ENOMEM; }
        if (b.p && used) cudaMemcpy(np, b.p, std::min(used * sizeof(T), b.cap), cudaMemcpyDeviceToDevice);
        if (b.p) cudaFree(b.p);
        b.p = np; b.cap = cap;
    }
    *out = (T*)b.p;
    return B200C_OK;
}

inline void timing_begin(b200c_ctx* c) { c->launches_call = 0; cudaEventRecord(c->ev0, c->stream); c->timing = true; }
inline int timing_end(b200c_ctx* c) {
    cudaEventRecord(c->ev1, c->stream);
    B200C_CUDA_TRY(c, cudaEventSynchronize(c->ev1));
    float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1); c->last_ms = ms; c->timing = false;
    return B200C_OK;
}

// K5 of one output file fed in pieces (engine.cu)
struct OutStream {
    enum { MAX_PIECES = 96 };
    b200c_ctx* c = nullptr; int comp = 0, L = 0, max_clen = 0, stride = 0, ws_base = 0;
    uint8_t* h_out = nullptr; uint64_t h_cap = 0;           // the caller's Data.db buffer
    uint32_t *file_len = nullptr, *seg_raw = nullptr, *acc = nullptr; uint64_t *d_offs = nullptr, *bases = nullptr;
    uint8_t* img[2] = {nullptr, nullptr}; uint64_t img_cap[2] = {0, 0};
    uint64_t nchunks = 0, ulen = 0, copied = 0; int piece = 0; bool fits = true;
    bool raw = false; uint64_t* ends = nullptr;              // uncompressed output: d_offs holds the CRC.db entries, ends the chunk ends (digest)
};
int out_stream_begin(OutStream& o, b200c_ctx* c, int comp, int chunk_len, int max_clen, uint8_t* h_out, uint64_t h_cap, int ws_base);
int out_stream_append(OutStream& o, const uint8_t* d_in, uint64_t nbytes);
int out_stream_finish(OutStream& o, uint64_t* out_len, uint32_t* digest, uint64_t** d_offs_out);

static_assert(EV_OUT_PIECE + 2 * OutStream::MAX_PIECES <= EV_RANGE && EV_RANGE + MAX_RANGES <= EV_INDEX_FREE &&
              EV_INDEX_FREE < EV_INDEX_READY && EV_INDEX_READY < EV_UOUT_FREE && EV_UOUT_FREE + 2 <= EV_POOL, "ev_pool slots overlap");

// b200c_ctx::h_pinned: every value read back from the device lands in its own member, so no read-back overwrites a value that another
// one still needs
struct Pinned {
    // codec helpers (engine.cu)
    uint64_t packed_len;                                // pack_digest_device: compressed size of the file
    uint32_t digest;                                    // pack_digest_device, raw_digest: Digest.crc32
    uint64_t chunk_err;                                 // b200c_decompress_chunks / b200c_uncompress_chunks: ChunkErr
    // OutStream (engine.cu)
    uint64_t os_end[OutStream::MAX_PIECES];             // file offset behind packed piece s
    uint32_t os_digest;
    // b200c_compact (compact.cu)
    uint64_t cerr, err;                                 // ChunkErr, DevErr
    uint64_t range[2 * B200C_MAX_INPUTS];               // k_input_ranges: partitions [a, b) of every input
    uint64_t scan[B200C_MAX_INPUTS + 1];                // K2: first partition of every input (and the total)
    uint32_t bad[B200C_MAX_INPUTS + 1];                 // K2: inputs whose Summary intervals or speculation did not prove
    uint64_t plan[2 * MAX_RANGES * B200C_MAX_INPUTS];   // k_range_plan: bytes of U every piece reads from every input
    uint64_t nparts, class_end[4];                      // K3: output partitions, ends of the fan-in classes <= 8 / 12 / 16 / 32
    uint64_t scratch_len, iscr_len;                     // K4: scratch bytes for Data.db and Index.db
    uint64_t ntiles, nbig;                              // staged K4: tiles, partitions left to the thread kernels
    uint64_t data_end, index_len, written;              // K4: end of the piece in the file, its Index.db bytes, its written partitions
    uint64_t summary_len;                               // Summary.db entry bytes of the piece
    uint64_t run_stats[3], hist[B200C_MAX_INPUTS], bytes_in_range;   // RunStats, merged_row_counts, bytes in the token range
    uint64_t cut[2], file_end, file_index_len, file_stats[3];       // multi-file output: k_find_cut, end of the file, its Index.db, its RunStats
};
enum { H_PINNED_CAP = 1 << 16 };
static_assert(sizeof(Pinned) <= H_PINNED_CAP, "b200c_ctx::h_pinned");

// device-wide exclusive scan: out[0..n] (n+1 entries, out[n] = total). TIn = uint32_t or uint64_t. scan_slot0: first of 3 ws slots.
template <typename TIn> int exclusive_scan(b200c_ctx* c, const TIn* in, uint64_t n, uint64_t* out, int scan_slot0, int depth = 0);

} // namespace b200c
