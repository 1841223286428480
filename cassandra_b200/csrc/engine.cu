// engine.cu — libb200compact.so: context lifecycle, CRC tables, device scan, and the chunk-codec entry points of
// include/b200c.h (b200c_compress_chunks / b200c_decompress_chunks / ICompressor single-buffer calls).
// No CPU fallback: every compute entry point needs a CUDA device and fails with B200C_ECUDA otherwise.
#include "engine.cuh"
#include <algorithm>
#include "scan.cuh"
#include "codec.cuh"
#include <climits>
#include <vector>

using namespace b200c;

namespace b200c {

enum { WSC_IN = 0, WSC_OUT, WSC_SLOTS, WSC_FILELEN, WSC_SEGRAW, WSC_OFFS, WSC_ACC, WSC_ERR, WSC_CHOFFS, WSC_SCAN0, WSC_SCAN1, WSC_SCAN2 };
int raw_chunks_device(b200c_ctx* c, bool ingest, const RawArgs& a);
static int raw_digest(b200c_ctx* c, const uint32_t* seg_raw, const uint64_t* ends, uint64_t nchunks, uint32_t* acc, uint32_t* digest);

static void build_tables(DevTables* t) {
    for (uint32_t i = 0; i < 256; i++) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (0xEDB88320u ^ (c >> 1)) : (c >> 1);
        t->crc_t[0][i] = c;
    }
    for (uint32_t i = 0; i < 256; i++)
        for (int k = 1; k < 4; k++) t->crc_t[k][i] = (t->crc_t[k - 1][i] >> 8) ^ t->crc_t[0][t->crc_t[k - 1][i] & 0xff];
    // x^(8*2^k)
    uint32_t sq = 0x00800000u;          // x^8, reflected
    for (int k = 0; k < 64; k++) { t->xp_pow2[k] = sq; sq = gf2_mulmod(sq, sq); }
    auto xpow8n = [&](uint64_t n) { uint32_t r = 0x80000000u; for (int k = 0; n; k++, n >>= 1) if (n & 1) r = gf2_mulmod(r, t->xp_pow2[k]); return r; };
    uint32_t x128 = xpow8n(128);
    for (int j = 0; j < 4; j++)
        for (uint32_t b = 0; b < 256; b++) t->crc_adv128[j][b] = gf2_mulmod(b << (8 * j), x128);
    for (int l = 0; l < 32; l++) t->xp_lane[l] = xpow8n(4 * (32 - l));
    uint32_t x512 = xpow8n(512);
    for (int j = 0; j < 4; j++)
        for (uint32_t b = 0; b < 256; b++) t->crc_adv512[j][b] = gf2_mulmod(b << (8 * j), x512);
    for (int l = 0; l < 32; l++) t->xp_lane16[l] = xpow8n(16 * (31 - l));
}

template <typename TIn>
int exclusive_scan(b200c_ctx* c, const TIn* in, uint64_t n, uint64_t* out, int slot, int depth) {
    if (n == 0) { B200C_CUDA_TRY(c, cudaMemsetAsync(out, 0, sizeof(uint64_t), c->stream)); return B200C_OK; }
    uint64_t tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    if (tiles == 1) { B200C_LAUNCH(c, k_scan_down<TIn>, 1, SCAN_THREADS, 0, in, n, (const uint64_t*)nullptr, out, out + n); return B200C_OK; }
    if (depth > 2) { c->err = "scan recursion too deep"; return B200C_EINVAL; }
    uint64_t* sums; B200C_TRY(ws_typed(c, slot + depth, tiles + 1, &sums));
    B200C_LAUNCH(c, k_scan_reduce<TIn>, (unsigned)tiles, SCAN_THREADS, 0, in, n, sums);
    B200C_TRY(exclusive_scan<uint64_t>(c, sums, tiles, sums, slot, depth + 1));
    B200C_LAUNCH(c, k_scan_down<TIn>, (unsigned)tiles, SCAN_THREADS, 0, in, n, (const uint64_t*)sums, out, out + n);
    return B200C_OK;
}
template int exclusive_scan<uint32_t>(b200c_ctx*, const uint32_t*, uint64_t, uint64_t*, int, int);
template int exclusive_scan<uint64_t>(b200c_ctx*, const uint64_t*, uint64_t, uint64_t*, int, int);

// K5 of chunks above 64 KiB (codec.cuh), whatever B200C_K5 says. Their kernels read the chunks in place, 4-byte aligned: a stream that starts
// elsewhere (a file of an LCS output starts where its first partition does) is first copied to an aligned buffer.
static int compress_big_slots_device(b200c_ctx* c, int comp, const uint8_t* d_in, uint64_t n, int chunk_len, int max_clen,
                                     uint8_t* slots, int stride, uint32_t* file_len, uint32_t* seg_raw, uint64_t nchunks) {
    if (((uintptr_t)d_in & 3) != 0) {
        uint8_t* a; B200C_TRY(ws_typed(c, WS_K5_BIGIN, (size_t)n + 64, &a));
        B200C_CUDA_TRY(c, cudaMemcpyAsync(a, d_in, n, cudaMemcpyDeviceToDevice, c->stream));
        d_in = a;
    }
    if (comp == COMP_LZ4) {
        B200C_LAUNCH(c, k_compress_chunks_lz4_big, (unsigned)nchunks, 32, 0, c->d_tables, d_in, n, chunk_len, max_clen, slots, stride, file_len, seg_raw);
    } else if (comp_is_snappy(comp)) {
        const int max_bits = comp == COMP_SNAPPY15 ? 15 : 14, fstride = (snappy_max_compressed_length(SNAPPY_BLOCK) + 15) & ~15;
        const uint64_t nfrag = nchunks * (uint64_t)(chunk_len / SNAPPY_BLOCK);
        uint8_t* frags; uint32_t* flen;
        B200C_TRY(ws_typed(c, WS_K5_FRAGS, nfrag * (uint64_t)fstride + 64, &frags));
        B200C_TRY(ws_typed(c, WS_K5_FLEN, nfrag + 1, &flen));
        B200C_LAUNCH(c, k_snappy_big_fragments, (unsigned)nfrag, 32, (size_t)2 * snappy_table_size(SNAPPY_BLOCK, max_bits), max_bits, d_in, n, chunk_len, frags, fstride, flen);
        B200C_LAUNCH(c, k_snappy_big_assemble, (unsigned)nchunks, 32, 0, c->d_tables, d_in, n, chunk_len, max_clen, (const uint8_t*)frags, fstride, (const uint32_t*)flen,
                     slots, stride, file_len, seg_raw);
    } else {
        B200C_LAUNCH(c, k_compress_chunks_noop_big, (unsigned)nchunks, 32, 0, c->d_tables, d_in, n, chunk_len, max_clen, slots, stride, file_len, seg_raw);
    }
    return B200C_OK;
}

// device-side chunk compression of a resident stream, in two halves so that the LCS writer can compress a window, look at the
// chunk sizes, and only then decide where the file ends:
//   compress_slots_device: every chunk of d_in[0..n) -> its fixed-stride slot (+ CRC), file_len[i] = bytes + 4, seg_raw[i] for the digest
//   pack_digest_device:    first nchunks slots -> dense Data.db image, chunk offsets (nchunks + 1), Digest.crc32
int compress_slots_device(b200c_ctx* c, int comp, const uint8_t* d_in, uint64_t n, int chunk_len, int max_clen,
                          uint8_t* slots, int stride, uint32_t* file_len, uint32_t* seg_raw) {
    uint64_t nchunks = (n + chunk_len - 1) / chunk_len;
    if (!nchunks) return B200C_OK;
    if (chunk_len > CHUNK_LEN_SMALL) return compress_big_slots_device(c, comp, d_in, n, chunk_len, max_clen, slots, stride, file_len, seg_raw, nchunks);
    // B200C_K5: 0 = chunk copy in shared memory, 1 = the chunk read through L1, 3 = two passes (lz4_chain.cuh / snappy_chain.cuh).
    // Unset: what measured fastest on an H100 80GB HBM3 in bench.py's device-resident step — LZ4 mode 1 (K5 on configs[1] at 400 W: 78.5 ms,
    // mode 0: 96.3, two passes: 94.4; the link-building pass is bound by the sector traffic of its random 4-byte reads; with mode 1's reads
    // issued early, at 700 W: 60.3 ms against 78.1), Snappy two passes (configs[2]: 93.5 ms, mode 1: 104.3; its table is 32 KiB, 6 chunks per
    // SM). Mode 2 (mode 1 with a distinct-hash scoreboard in shared memory) measured 66.1 ms against mode 1's 60.3: not the default.
    const int k5_env = []() { const char* e = getenv("B200C_K5"); return e ? atoi(e) : -1; }();
    const int k5_mode = k5_env >= 0 ? k5_env : (comp_is_snappy(comp) ? 3 : 1);
    if (k5_mode == 3 && comp == COMP_LZ4 && ((uintptr_t)d_in & 3) == 0 && (chunk_len & 3) == 0 && chunk_len <= LZ4C_MAX_CHUNK) {
        // two passes (lz4_chain.cuh): same-hash predecessor links for every position, then the parse with one bit per position in shared memory
        uint32_t* ent; B200C_TRY(ws_typed(c, WS_K5_ENT, (size_t)n + 16384, &ent));
        B200C_LAUNCH(c, k_lz4_chain_build, (unsigned)nchunks, 32, 0, d_in, n, chunk_len, ent);
        const size_t smem = (size_t)K5B_WARPS * ((chunk_len + 31) >> 5) * 4;
        B200C_LAUNCH(c, k_compress_chunks_lz4_chain, (unsigned)((nchunks + K5B_WARPS - 1) / K5B_WARPS), 32 * K5B_WARPS, smem, c->d_tables, d_in, n, chunk_len, max_clen, (const uint32_t*)ent,
                     slots, stride, file_len, seg_raw, nchunks);
        return B200C_OK;
    }
    if ((k5_mode == 1 || k5_mode == 2) && comp == COMP_LZ4 && ((uintptr_t)d_in & 3) == 0 && (chunk_len & 3) == 0) {
        if (k5_mode == 2) B200C_LAUNCH(c, k_compress_chunks_lz4_direct<true>, (unsigned)nchunks, 32, 0, c->d_tables, d_in, n, chunk_len, max_clen, slots, stride, file_len, seg_raw);   // + distinct-hash fast path (A/B)
        else B200C_LAUNCH(c, k_compress_chunks_lz4_direct<false>, (unsigned)nchunks, 32, 0, c->d_tables, d_in, n, chunk_len, max_clen, slots, stride, file_len, seg_raw);
        return B200C_OK;
    }
    if (k5_mode == 3 && comp_is_snappy(comp) && ((uintptr_t)d_in & 3) == 0 && (chunk_len & 3) == 0 && chunk_len <= LZ4C_MAX_CHUNK) {
        const int max_bits = comp == COMP_SNAPPY15 ? 15 : 14, tsz = snappy_table_size(chunk_len, max_bits);
        uint32_t* ent; B200C_TRY(ws_typed(c, WS_K5_ENT, (size_t)n + 16384, &ent));
        static bool attr = false; if (!attr) { cudaFuncSetAttribute(k_snappy_chain_build, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 32768); attr = true; }
        B200C_LAUNCH(c, k_snappy_chain_build, (unsigned)nchunks, 32, (size_t)2 * tsz, max_bits, tsz, d_in, n, chunk_len, ent);
        const size_t smem = (size_t)K5B_WARPS * ((chunk_len + 31) >> 5) * 4;
        B200C_LAUNCH(c, k_compress_chunks_snappy_chain, (unsigned)((nchunks + K5B_WARPS - 1) / K5B_WARPS), 32 * K5B_WARPS, smem, c->d_tables, d_in, n, chunk_len, max_clen, (const uint32_t*)ent,
                     slots, stride, file_len, seg_raw, nchunks);
        return B200C_OK;
    }
    int tab_bytes = comp == COMP_SNAPPY15 ? 65536 : (comp == COMP_SNAPPY ? 32768 : 16384);
    if (k5_mode != 0 && comp_is_snappy(comp) && ((uintptr_t)d_in & 3) == 0 && (chunk_len & 3) == 0 && chunk_len <= 65536) {
        // the table a chunk of this length needs (snappy_compress_warp: next power of two >= chunk length, capped by the generation's maximum)
        int need = 512; while (need < 2 * chunk_len && need < tab_bytes) need <<= 1;
        B200C_LAUNCH(c, k_compress_chunks_snappy_direct, (unsigned)nchunks, 32, (size_t)need, c->d_tables, comp == COMP_SNAPPY15 ? 15 : 14, d_in, n, chunk_len, max_clen, slots, stride, file_len, seg_raw);
        return B200C_OK;
    }
    size_t smem = (size_t)tab_bytes + chunk_len + 16;
    B200C_LAUNCH(c, k_compress_chunks, (unsigned)nchunks, 32, smem, c->d_tables, comp, tab_bytes, d_in, n, chunk_len, max_clen, slots, stride, file_len, seg_raw);
    return B200C_OK;
}
int pack_digest_device(b200c_ctx* c, const uint8_t* slots, int stride, const uint32_t* file_len, const uint32_t* seg_raw, uint64_t nchunks,
                       uint8_t* d_out, uint64_t out_cap, uint64_t* d_offs, uint64_t* out_len, uint32_t* digest, int ws_base) {
    if (!nchunks) { *out_len = 0; *digest = 0; B200C_CUDA_TRY(c, cudaMemsetAsync(d_offs, 0, 8, c->stream)); return B200C_OK; }
    uint32_t* acc; B200C_TRY(ws_typed(c, ws_base + WSC_ACC, 4, &acc));
    B200C_CUDA_TRY(c, cudaMemsetAsync(acc, 0, 16, c->stream));
    B200C_TRY(exclusive_scan<uint32_t>(c, file_len, nchunks, d_offs, ws_base + WSC_SCAN0, 0));
    uint64_t* h = &c->h_pinned->packed_len;               // the total size must be known on the host before packing into the caller's buffer
    B200C_CUDA_TRY(c, cudaMemcpyAsync(h, d_offs + nchunks, 8, cudaMemcpyDeviceToHost, c->stream));
    B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    *out_len = h[0];
    if (h[0] > out_cap) { c->err = "output buffer too small"; return B200C_ETOOSMALL; }
    B200C_LAUNCH(c, k_pack_chunks, (unsigned)((nchunks + 3) / 4), 128, 0, slots, stride, file_len, d_offs, nchunks, d_out, (const uint64_t*)nullptr);
    B200C_LAUNCH(c, k_digest, (unsigned)((nchunks + 255) / 256), 256, 0, c->d_tables, seg_raw, d_offs, nchunks, acc);
    B200C_LAUNCH(c, k_digest_final, 1, 1, 0, c->d_tables, d_offs, nchunks, acc);
    uint32_t* h32 = &c->h_pinned->digest;
    B200C_CUDA_TRY(c, cudaMemcpyAsync(h32, acc + 1, 4, cudaMemcpyDeviceToHost, c->stream));
    B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    *digest = h32[0];
    return B200C_OK;
}
int compress_stream_device(b200c_ctx* c, int comp, const uint8_t* d_in, uint64_t n, int chunk_len, int max_clen,
                           uint8_t* d_out, uint64_t out_cap, uint64_t* d_offs /*nchunks+1*/, uint64_t* out_len, uint32_t* digest, int ws_base) {
    uint64_t nchunks = (n + chunk_len - 1) / chunk_len;
    if (nchunks > 0x7fffffffull) { c->err = "too many chunks"; return B200C_EINVAL; }
    int stride = chunk_slot_stride(comp, chunk_len);
    uint8_t* slots = nullptr; uint32_t* file_len = nullptr; uint32_t* seg_raw = nullptr;
    B200C_TRY(ws_typed(c, ws_base + WSC_SLOTS, nchunks * (uint64_t)stride, &slots));
    B200C_TRY(ws_typed(c, ws_base + WSC_FILELEN, nchunks + 1, &file_len));
    B200C_TRY(ws_typed(c, ws_base + WSC_SEGRAW, nchunks + 1, &seg_raw));
    B200C_TRY(compress_slots_device(c, comp, d_in, n, chunk_len, max_clen, slots, stride, file_len, seg_raw));
    return pack_digest_device(c, slots, stride, file_len, seg_raw, nchunks, d_out, out_cap, d_offs, out_len, digest, ws_base);
}

// slice-relative chunk offsets -> absolute offsets in the file image; bases[0] = offset of this slice, bases[1] := offset of the next
__global__ void __launch_bounds__(256) k_offs_add_base(const uint64_t* __restrict__ rel, uint64_t count, uint64_t* __restrict__ bases, uint64_t* __restrict__ offs_abs) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t b = bases[0];
    if (i <= count) offs_abs[i] = b + rel[i];
    if (i == count) bases[1] = b + rel[count];
}

// ---- OutStream: K5 for one output file whose uncompressed stream is handed over in pieces -------------------------------------------
// Every piece is compressed into slots, its chunk sizes are scanned and re-based onto the running file offset (a device scalar, so
// no host round trip sits between the kernels), packed into one of two image buffers and copied to the caller's host buffer on the
// copy stream while the next piece is being produced. The host learns each piece's end offset one piece late (drain).
int out_stream_begin(OutStream& o, b200c_ctx* c, int comp, int chunk_len, int max_clen, uint8_t* h_out, uint64_t h_cap, int ws_base) {
    o = OutStream();
    o.c = c; o.comp = comp; o.L = chunk_len; o.max_clen = max_clen; o.stride = chunk_slot_stride(comp, chunk_len); o.ws_base = ws_base;
    o.raw = comp == COMP_UNCOMPRESSED;
    o.h_out = h_out; o.h_cap = h_out ? h_cap : 0;
    B200C_TRY(ws_typed(c, ws_base + WSC_CHOFFS, (size_t)OutStream::MAX_PIECES + 2, &o.bases));
    B200C_TRY(ws_typed(c, ws_base + WSC_ACC, 4, &o.acc));
    B200C_CUDA_TRY(c, cudaMemsetAsync(o.acc, 0, 16, c->stream));
    B200C_CUDA_TRY(c, cudaMemsetAsync(o.bases, 0, 8, c->stream));
    return B200C_OK;
}

static int out_stream_drain(OutStream& o, int s) {       // piece s is packed once its event fires: hand its bytes to the copy engine
    b200c_ctx* c = o.c;
    uint64_t* h = c->h_pinned->os_end;
    B200C_CUDA_TRY(c, cudaEventSynchronize(c->ev_pool[EV_OUT_PIECE + 2 * s]));
    const uint64_t end = h[s];
    if (end - o.copied > o.img_cap[s & 1]) { c->err = "internal error: compressed piece exceeds its bound"; return B200C_ECUDA; }
    if (end > o.h_cap) o.fits = false;
    if (o.fits && end > o.copied) {
        B200C_CUDA_TRY(c, cudaStreamWaitEvent(c->copy_out, c->ev_pool[EV_OUT_PIECE + 2 * s], 0));
        B200C_CUDA_TRY(c, cudaMemcpyAsync(o.h_out + o.copied, o.img[s & 1], end - o.copied, cudaMemcpyDeviceToHost, c->copy_out));
    }
    B200C_CUDA_TRY(c, cudaEventRecord(c->ev_pool[EV_OUT_PIECE + 2 * s + 1], c->copy_out));
    o.copied = end;
    return B200C_OK;
}

// d_in: the next nbytes of the uncompressed stream, starting on a chunk boundary of the file; every call but the last must pass a
// multiple of the chunk length
int out_stream_append(OutStream& o, const uint8_t* d_in, uint64_t nbytes) {
    b200c_ctx* c = o.c;
    if (!nbytes) return B200C_OK;
    if (o.piece >= OutStream::MAX_PIECES) { c->err = "internal error: too many output pieces"; return B200C_ECUDA; }
    const uint64_t k = (nbytes + o.L - 1) / o.L, a = o.nchunks;
    if (a + k > 0x7fffffffull) { c->err = "too many chunks"; return B200C_EINVAL; }
    if (o.raw) {
        // uncompressed: the CRC.db entries (d_offs) and digest registers of the piece's chunks, and its bytes go to the host straight from the
        // merged stream; the caller keeps that buffer unchanged until the copy has left (compact.cu)
        const int s = o.piece;
        B200C_TRY(ws_grow_keep(c, o.ws_base + WSC_SEGRAW, a + k + 2, a, &o.seg_raw));
        B200C_TRY(ws_grow_keep(c, o.ws_base + WSC_OFFS, a + k + 2, a, &o.d_offs));
        B200C_TRY(ws_grow_keep(c, o.ws_base + WSC_FILELEN, a + k + 2, a + 1, &o.ends));
        RawArgs ra; memset(&ra, 0, sizeof(ra));
        ra.src = d_in; ra.n = nbytes; ra.L = o.L; ra.chunk_end = k; ra.crc_out = o.d_offs + a; ra.seg_raw = o.seg_raw + a; ra.ends = o.ends + a; ra.ebase = o.ulen;
        B200C_TRY(raw_chunks_device(c, false, ra));
        B200C_CUDA_TRY(c, cudaEventRecord(c->ev_pool[EV_OUT_PIECE + 2 * s], c->stream));
        if (o.ulen + nbytes > o.h_cap) o.fits = false;
        if (o.fits) {
            B200C_CUDA_TRY(c, cudaStreamWaitEvent(c->copy_out, c->ev_pool[EV_OUT_PIECE + 2 * s], 0));
            B200C_CUDA_TRY(c, cudaMemcpyAsync(o.h_out + o.ulen, d_in, nbytes, cudaMemcpyDeviceToHost, c->copy_out));
        }
        o.nchunks += k; o.ulen += nbytes; o.copied = o.ulen; o.piece++;
        return B200C_OK;
    }
    uint8_t* slots; uint64_t* rel; const int s = o.piece;
    B200C_TRY(ws_grow_keep(c, o.ws_base + WSC_FILELEN, a + k + 2, a, &o.file_len));
    B200C_TRY(ws_grow_keep(c, o.ws_base + WSC_SEGRAW, a + k + 2, a, &o.seg_raw));
    B200C_TRY(ws_grow_keep(c, o.ws_base + WSC_OFFS, a + k + 2, a + 1, &o.d_offs));
    B200C_TRY(ws_typed(c, o.ws_base + WSC_SLOTS, k * (uint64_t)o.stride, &slots));
    B200C_TRY(ws_typed(c, o.ws_base + WSC_IN, k + 2, &rel));
    B200C_TRY(ws_typed(c, o.ws_base + (s & 1 ? WSC_OUT : WSC_ERR), k * (uint64_t)o.stride + 64, &o.img[s & 1]));
    o.img_cap[s & 1] = k * (uint64_t)o.stride;
    if (s >= 2) B200C_CUDA_TRY(c, cudaStreamWaitEvent(c->stream, c->ev_pool[EV_OUT_PIECE + 2 * (s - 2) + 1], 0));   // the image buffer is free again
    B200C_TRY(compress_slots_device(c, o.comp, d_in, nbytes, o.L, o.max_clen, slots, o.stride, o.file_len + a, o.seg_raw + a));
    B200C_TRY(exclusive_scan<uint32_t>(c, o.file_len + a, k, rel, o.ws_base + WSC_SCAN0, 0));
    B200C_LAUNCH(c, k_offs_add_base, (unsigned)((k + 1 + 255) / 256), 256, 0, rel, k, o.bases + s, o.d_offs + a);
    B200C_LAUNCH(c, k_pack_chunks, (unsigned)((k + 3) / 4), 128, 0, slots, o.stride, o.file_len + a, o.d_offs + a, k, o.img[s & 1], (const uint64_t*)(o.bases + s));
    B200C_CUDA_TRY(c, cudaMemcpyAsync(c->h_pinned->os_end + s, o.bases + s + 1, 8, cudaMemcpyDeviceToHost, c->stream));
    B200C_CUDA_TRY(c, cudaEventRecord(c->ev_pool[EV_OUT_PIECE + 2 * s], c->stream));
    if (s) B200C_TRY(out_stream_drain(o, s - 1));        // after piece s is queued, so the GPU never waits for the host
    o.nchunks += k; o.ulen += nbytes; o.piece++;
    return B200C_OK;
}

// drains the last piece, computes Digest.crc32 and waits for everything; *d_offs_out: the nchunks + 1 chunk offsets (device)
int out_stream_finish(OutStream& o, uint64_t* out_len, uint32_t* digest, uint64_t** d_offs_out) {
    b200c_ctx* c = o.c;
    *out_len = 0; *digest = 0; *d_offs_out = nullptr;
    if (!o.nchunks) return B200C_OK;
    if (o.raw) {
        B200C_TRY(raw_digest(c, o.seg_raw, o.ends, o.nchunks, o.acc, digest));
        B200C_CUDA_TRY(c, cudaStreamSynchronize(c->copy_out));
        *out_len = o.ulen; *d_offs_out = o.d_offs;
        return B200C_OK;
    }
    uint32_t* h32 = &c->h_pinned->os_digest;
    B200C_LAUNCH(c, k_digest, (unsigned)((o.nchunks + 255) / 256), 256, 0, c->d_tables, o.seg_raw, o.d_offs, o.nchunks, o.acc);
    B200C_LAUNCH(c, k_digest_final, 1, 1, 0, c->d_tables, o.d_offs, o.nchunks, o.acc);
    B200C_CUDA_TRY(c, cudaMemcpyAsync(h32, o.acc + 1, 4, cudaMemcpyDeviceToHost, c->stream));
    B200C_TRY(out_stream_drain(o, o.piece - 1));
    B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    B200C_CUDA_TRY(c, cudaStreamSynchronize(c->copy_out));
    *out_len = o.copied; *digest = h32[0]; *d_offs_out = o.d_offs;
    return B200C_OK;
}

// Geometry of the thread-per-chunk K1 kernels. Every chunk in flight is a private chain of dependent loads that touches its compressed
// bytes twice (CRC, decode), its output sectors once per 8-byte store and its own recent output for every match: once the chains in
// flight need more than the caches hold, those bytes come from DRAM again and every dependent load waits longer. So the kernels loop
// over their chunks and a launch keeps L2 size / K1_L2_BYTES_PER_CHAIN of them in flight, in whole blocks per SM (k1_plan, at
// context creation). A grid of that size alone would let the block scheduler stack blocks on some SMs, so each block also asks for
// (unused) dynamic shared memory: exactly that many blocks fill the smallest shared-memory carveout that holds them, and the rest of
// the SM's 256 KB stays L1 for the chains (a carveout sized for the maximum shared memory leaves ~28 KB of L1: K1 then took 80 ms
// instead of 58 on configs[1], DESIGN §7).
static void k1_plan(b200c_ctx* c) {
    static const int carveout_kb[] = {0, 8, 16, 32, 64, 100, 132, 164, 196, 228};      // the shared-memory capacities an sm_90 SM supports
    const int per_sm = (int)std::max<uint64_t>(1, (uint64_t)c->l2_bytes / K1_L2_BYTES_PER_CHAIN / K1_THREADS / (uint64_t)c->nsm);
    const int block = c->smem_reserved_per_block + K1_STATIC_SMEM;
    int carve = c->smem_per_sm;
    for (int kb : carveout_kb) if (kb * 1024 >= per_sm * block) { carve = std::min(kb * 1024, c->smem_per_sm); break; }
    c->k1_blocks_per_sm = per_sm;
    c->k1_smem = (size_t)std::max(0, (carve / per_sm - block) & ~127);
    for (const void* k : {(const void*)k_decompress_multi_thr, (const void*)k_decompress_chunks_thr}) {
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->k1_smem);
        cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, 100 * carve / c->smem_per_sm);
    }
}
static unsigned k1_grid(const b200c_ctx* c, uint64_t nthreads) {
    return (unsigned)std::min<uint64_t>((uint64_t)c->k1_blocks_per_sm * (uint64_t)c->nsm, (nthreads + K1_THREADS - 1) / K1_THREADS);
}

// chunks [chunk0, chunk0 + count) of the file (count = ~0: through the last chunk); chunks from file offset tail_off on are read
// from `tail` (k1_src; tail_off = ~0: none)
int decompress_stream_device(b200c_ctx* c, int comp, const uint8_t* d_data, uint64_t data_len, const uint64_t* d_offs, uint64_t nchunks,
                             int chunk_len, int max_clen, uint64_t data_length, uint8_t* d_out, int verify, ChunkErr* d_err,
                             uint64_t chunk0, uint64_t count, int tag, const uint8_t* tail, uint64_t tail_off) {
    if (chunk0 >= nchunks || count == 0) return B200C_OK;
    const uint64_t end = count > nchunks - chunk0 ? nchunks : chunk0 + count;
    static const int k1_mode = []() { const char* e = getenv("B200C_K1"); return e ? atoi(e) : 1; }();      // 0: warp per chunk, 1: thread per chunk (LZ4)
    // thread per chunk needs tens of thousands of chunks in flight to beat the warp kernel; small launches (token-range pieces of one
    // input) keep the warp mapping unless compact.cu has batched them (decompress_multi_device)
    // chunks above 64 KiB always take the warp kernel: one thread decoding 1 MiB is a chain 16 times longer than the L2 plan of k1_plan assumes
    if (k1_mode == 1 && comp == COMP_LZ4 && (chunk_len & 7) == 0 && chunk_len <= CHUNK_LEN_SMALL && ((uintptr_t)d_out & 7) == 0 && end - chunk0 >= 32768)
        B200C_LAUNCH(c, k_decompress_chunks_thr, k1_grid(c, end - chunk0), K1_THREADS, c->k1_smem, c->d_tables, comp, d_data, data_len, d_offs, nchunks,
                     chunk_len, max_clen, data_length, d_out, verify, d_err, chunk0, end, tag, tail, tail_off);
    else
        B200C_LAUNCH(c, k_decompress_chunks, (unsigned)((end - chunk0 + 1) / 2), 64, 0, c->d_tables, comp, d_data, data_len, d_offs, nchunks,
                     chunk_len, max_clen, data_length, d_out, verify, d_err, chunk0, end, tag, tail, tail_off);
    return B200C_OK;
}

// LZ4 chunk ranges of several inputs in one thread-per-chunk launch (segs: host array, first/_pad filled here)
int decompress_multi_device(b200c_ctx* c, K1Seg* segs, int nseg, int verify, ChunkErr* d_err, int ws_slot) {
    uint64_t total = 0;
    for (int i = 0; i < nseg; i++) { segs[i].first = total; segs[i].count = segs[i].nchunks > segs[i].chunk0 ? std::min(segs[i].count, segs[i].nchunks - segs[i].chunk0) : 0; total += segs[i].count; }
    if (!total) return B200C_OK;
    // B200C_K1=2: two passes (lz4_batch.cuh) — walk: one thread per chunk validates the block and records where its sequences start;
    // copy: one warp per chunk, 32 sequences per step. rec_span (when the caller knows the range's compressed size) sizes the record slots.
    static const int k1_mode = []() { const char* e = getenv("B200C_K1"); return e ? atoi(e) : 1; }();
    uint64_t rec_total = 0;
    for (int i = 0; i < nseg; i++) {
        if (!segs[i].rec_span || segs[i].rec_span > segs[i].data_len) segs[i].rec_span = segs[i].data_len;
        segs[i].rec0 = rec_total; rec_total += segs[i].rec_span / 3 + 2 * segs[i].count + 8;
    }
    K1Seg* d; B200C_TRY(ws_typed(c, ws_slot, (size_t)nseg + 1, &d));
    B200C_CUDA_TRY(c, cudaMemcpyAsync(d, segs, sizeof(K1Seg) * nseg, cudaMemcpyHostToDevice, c->stream));
    if (k1_mode == 2) {
        uint16_t* rec; uint32_t* nseq;
        B200C_TRY(ws_typed(c, WS_K1_REC, (size_t)rec_total + 64, &rec));
        B200C_TRY(ws_typed(c, WS_K1_NSEQ, (size_t)total + 64, &nseq));
        B200C_LAUNCH(c, k_lz4_walk_multi, (unsigned)((total + 127) / 128), 128, 0, d, nseg, total, rec, nseq, d_err);
        // blocks of the copy kernel resident per SM (B200C_K1_COPY_BLOCKS, 4 warps each): every chunk in flight keeps ~30 KB of L2 busy
        static const int copy_blocks = []() { const char* e = getenv("B200C_K1_COPY_BLOCKS"); int v = e ? atoi(e) : 8; return v < 1 ? 1 : (v > 16 ? 16 : v); }();
        static bool attr = false; if (!attr) { cudaFuncSetAttribute(k_lz4_copy_multi, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024); attr = true; }
        const size_t pad = copy_blocks >= 16 ? 0 : (size_t)(220 * 1024) / copy_blocks;
        B200C_LAUNCH(c, k_lz4_copy_multi, (unsigned)((total + K1C_WARPS - 1) / K1C_WARPS), 32 * K1C_WARPS, pad, c->d_tables, (const K1Seg*)d, nseg, total, (const uint16_t*)rec, (const uint32_t*)nseq, verify, d_err);
        return B200C_OK;
    }
    unsigned long long* next = (unsigned long long*)(d + nseg);      // chunk counter of the launch (k_decompress_multi_thr)
    B200C_CUDA_TRY(c, cudaMemsetAsync(next, 0, sizeof(*next), c->stream));
    B200C_LAUNCH(c, k_decompress_multi_thr, k1_grid(c, total), K1_THREADS, c->k1_smem, c->d_tables, d, nseg, total, verify, d_err, next);
    return B200C_OK;
}

// chunk ranges above 64 KiB of several inputs, any compressor, in one warp-per-chunk launch (segs: host array, first filled here)
int decompress_big_device(b200c_ctx* c, K1Seg* segs, int nseg, int verify, ChunkErr* d_err, int ws_slot) {
    uint64_t total = 0;
    for (int i = 0; i < nseg; i++) { segs[i].first = total; segs[i].count = segs[i].nchunks > segs[i].chunk0 ? std::min(segs[i].count, segs[i].nchunks - segs[i].chunk0) : 0; total += segs[i].count; }
    if (!total) return B200C_OK;
    K1Seg* d; B200C_TRY(ws_typed(c, ws_slot, (size_t)nseg, &d));
    B200C_CUDA_TRY(c, cudaMemcpyAsync(d, segs, sizeof(K1Seg) * nseg, cudaMemcpyHostToDevice, c->stream));
    B200C_LAUNCH(c, k_decompress_multi_warp, (unsigned)((total + 1) / 2), 64, 0, c->d_tables, (const K1Seg*)d, nseg, total, verify, d_err);
    return B200C_OK;
}

// uncompressed streams: chunks [a.chunk0, a.chunk_end), one block per chunk, eight blocks per SM looping over them
int raw_chunks_device(b200c_ctx* c, bool ingest, const RawArgs& a) {
    if (a.chunk_end <= a.chunk0) return B200C_OK;
    const unsigned grid = (unsigned)std::min<uint64_t>(a.chunk_end - a.chunk0, (uint64_t)c->nsm * 8);
    if (ingest) B200C_LAUNCH(c, k_raw_ingest, grid, RAW_THREADS, 0, c->d_tables, a);
    else B200C_LAUNCH(c, k_raw_checksum, grid, RAW_THREADS, 0, c->d_tables, a);
    return B200C_OK;
}
static int raw_digest(b200c_ctx* c, const uint32_t* seg_raw, const uint64_t* ends, uint64_t nchunks, uint32_t* acc, uint32_t* digest) {
    B200C_LAUNCH(c, k_digest, (unsigned)((nchunks + 255) / 256), 256, 0, c->d_tables, seg_raw, ends, nchunks, acc);
    B200C_LAUNCH(c, k_digest_final, 1, 1, 0, c->d_tables, ends, nchunks, acc);
    uint32_t* h32 = &c->h_pinned->digest;
    B200C_CUDA_TRY(c, cudaMemcpyAsync(h32, acc + 1, 4, cudaMemcpyDeviceToHost, c->stream));
    B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    *digest = h32[0];
    return B200C_OK;
}
// ChecksummedSequentialWriter over a resident stream: d_out (optional) receives the bytes, d_crc[0..nchunks) the CRC.db entries, *digest
// Digest.crc32 of the bytes alone
int raw_stream_device(b200c_ctx* c, const uint8_t* d_in, uint64_t n, int chunk_len, uint8_t* d_out, uint64_t* d_crc, uint32_t* digest, int ws_base) {
    const uint64_t nchunks = (n + chunk_len - 1) / chunk_len;
    *digest = 0;
    if (!nchunks) return B200C_OK;
    uint32_t *seg_raw, *acc; uint64_t* ends;
    B200C_TRY(ws_typed(c, ws_base + WSC_SEGRAW, nchunks + 1, &seg_raw));
    B200C_TRY(ws_typed(c, ws_base + WSC_SCAN1, nchunks + 2, &ends));
    B200C_TRY(ws_typed(c, ws_base + WSC_ACC, 4, &acc));
    B200C_CUDA_TRY(c, cudaMemsetAsync(acc, 0, 16, c->stream));
    RawArgs a; memset(&a, 0, sizeof(a));
    a.src = d_in; a.dst = d_out; a.n = n; a.L = chunk_len; a.chunk_end = nchunks; a.crc_out = d_crc; a.seg_raw = seg_raw; a.ends = ends;
    B200C_TRY(raw_chunks_device(c, false, a));
    return raw_digest(c, seg_raw, ends, nchunks, acc, digest);
}

} // namespace b200c

// ---------------------------------------------------------------------------------------------------------------------
extern "C" {

int b200c_abi_version(void) { return B200C_ABI_VERSION; }

int b200c_device_count(void) {
    int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; } return n;
}

b200c_ctx* b200c_create(int device, size_t workspace_bytes) {
    int n = b200c_device_count();
    if (device < 0 || device >= n) return nullptr;       // no device => no context: the product path has no CPU fallback
    if (cudaSetDevice(device) != cudaSuccess) return nullptr;
    b200c_ctx* c = new b200c_ctx();
    c->device = device;
    if (cudaDeviceGetAttribute(&c->nsm, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || c->nsm <= 0) { delete c; return nullptr; }
    if (cudaDeviceGetAttribute(&c->l2_bytes, cudaDevAttrL2CacheSize, device) != cudaSuccess || c->l2_bytes <= 0) { delete c; return nullptr; }
    if (cudaDeviceGetAttribute(&c->smem_per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, device) != cudaSuccess ||
        cudaDeviceGetAttribute(&c->smem_reserved_per_block, cudaDevAttrReservedSharedMemoryPerBlock, device) != cudaSuccess) { delete c; return nullptr; }
    if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) { delete c; return nullptr; }
    cudaEventCreate(&c->ev0); cudaEventCreate(&c->ev1);
    for (auto& e : c->ev_stage) cudaEventCreate(&e);
    cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking);
    for (auto& e : c->ev_in) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    for (auto& e : c->ev_pool) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    cudaStreamCreateWithFlags(&c->copy_out, cudaStreamNonBlocking);
    DevTables* h = new DevTables(); build_tables(h);
    if (cudaMalloc(&c->d_tables, sizeof(DevTables)) != cudaSuccess) { delete h; delete c; return nullptr; }
    cudaMemcpy(c->d_tables, h, sizeof(DevTables), cudaMemcpyHostToDevice);
    delete h;
    if (cudaMallocHost((void**)&c->h_pinned, H_PINNED_CAP) != cudaSuccess) { cudaFree(c->d_tables); delete c; return nullptr; }
    cudaFuncSetAttribute(k_compress_chunks, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536 + 65536 + 16);
    cudaFuncSetAttribute(k_compress_chunks_snappy_direct, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536);
    cudaFuncSetAttribute(k_snappy_big_fragments, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536);     // the 2^15 table of a 64 KiB fragment
    k1_plan(c);
    (void)workspace_bytes;
    return c;
}

void b200c_destroy(b200c_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    for (auto& b : c->ws) if (b.p) cudaFree(b.p);
    if (c->d_tables) cudaFree(c->d_tables);
    if (c->h_pinned) cudaFreeHost(c->h_pinned);
    cudaEventDestroy(c->ev0); cudaEventDestroy(c->ev1);
    for (auto& e : c->ev_stage) cudaEventDestroy(e);
    for (auto& e : c->ev_in) cudaEventDestroy(e);
    for (auto& e : c->ev_pool) cudaEventDestroy(e);
    for (auto& e : c->ev_marks) cudaEventDestroy(e);
    if (c->copy_out) cudaStreamDestroy(c->copy_out);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    cudaStreamDestroy(c->stream);
    delete c;
}

const char* b200c_last_error(b200c_ctx* c) { return c ? c->err.c_str() : "no context (no CUDA device?)"; }

int b200c_host_register(void* p, size_t n) { cudaError_t e = cudaHostRegister(p, n, cudaHostRegisterDefault); if (e != cudaSuccess) { cudaGetLastError(); return B200C_ECUDA; } return B200C_OK; }
int b200c_host_unregister(void* p) { cudaError_t e = cudaHostUnregister(p); if (e != cudaSuccess) { cudaGetLastError(); return B200C_ECUDA; } return B200C_OK; }

int b200c_dev_alloc(b200c_ctx* c, size_t n, void** dptr) {
    if (!c || !dptr) return B200C_EINVAL;
    cudaSetDevice(c->device);
    B200C_CUDA_TRY(c, cudaMalloc(dptr, n + 256));
    return B200C_OK;
}
int b200c_dev_free(b200c_ctx* c, void* dptr) { if (!c) return B200C_EINVAL; cudaSetDevice(c->device); B200C_CUDA_TRY(c, cudaFree(dptr)); return B200C_OK; }
int b200c_memcpy_h2d(b200c_ctx* c, void* d, const void* s, size_t n) {
    if (!c) return B200C_EINVAL;
    B200C_CUDA_TRY(c, cudaMemcpyAsync(d, s, n, cudaMemcpyHostToDevice, c->stream));
    B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream)); return B200C_OK;
}
int b200c_memcpy_d2h(b200c_ctx* c, void* d, const void* s, size_t n) {
    if (!c) return B200C_EINVAL;
    B200C_CUDA_TRY(c, cudaMemcpyAsync(d, s, n, cudaMemcpyDeviceToHost, c->stream));
    B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream)); return B200C_OK;
}
int b200c_sync(b200c_ctx* c) { if (!c) return B200C_EINVAL; B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream)); return B200C_OK; }
double b200c_last_kernel_ms(b200c_ctx* c) { return c ? c->last_ms : 0.0; }
uint64_t b200c_last_kernel_launches(b200c_ctx* c) { return c ? c->launches_call : 0; }
uint64_t b200c_total_kernel_launches(b200c_ctx* c) { return c ? c->launches_total : 0; }
int b200c_last_stage_ms(b200c_ctx* c, double* out, int n) {
    if (!c || !out) return 0;
    int k = c->nstages < n ? c->nstages : n;
    for (int i = 0; i < k; i++) out[i] = c->stage_ms[i];
    return k;
}

uint64_t b200c_chunk_count(uint64_t n, int chunk_len) { return chunk_len > 0 ? (n + chunk_len - 1) / chunk_len : 0; }
uint64_t b200c_compress_bound(int comp, uint64_t n, int chunk_len) {
    if (comp == COMP_UNCOMPRESSED) return n;             // Data.db is the stream itself
    uint64_t nch = b200c_chunk_count(n, chunk_len);
    int m = chunk_max_compressed(comp, chunk_len); if (m < chunk_len) m = chunk_len;
    return nch * ((uint64_t)m + 4) + 64;
}
int b200c_initial_compressed_buffer_length(int comp, int chunk_len) { return chunk_max_compressed(comp, chunk_len); }

static int check_codec_args(b200c_ctx* c, int comp, int chunk_len) {
    if (!c) return B200C_EINVAL;
    if (comp != COMP_LZ4 && !comp_is_snappy(comp) && comp != COMP_NONE && comp != COMP_UNCOMPRESSED) { c->err = "unknown compressor"; return B200C_EINVAL; }
    if (!chunk_len_supported(comp, chunk_len)) { c->err = comp == COMP_UNCOMPRESSED ? "CRC.db chunk_len must be a power of two <= 64 KiB" : "chunk_len must be a power of two <= 1 MiB"; return B200C_EUNSUPPORTED; }
    return B200C_OK;
}

int b200c_compress_chunks(b200c_ctx* c, int comp, const uint8_t* in, uint64_t n, int chunk_len, int max_clen,
                          uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* chunk_offsets, uint32_t* digest, int flags) {
    B200C_TRY(check_codec_args(c, comp, chunk_len));
    if ((!in && n) || !out || !out_len || !digest) { c->err = "null argument"; return B200C_EINVAL; }
    cudaSetDevice(c->device);
    const bool dev = flags & B200C_FLAG_DEVICE_PTRS;
    uint64_t nchunks = b200c_chunk_count(n, chunk_len);
    const uint8_t* d_in = in; uint8_t* d_out = out; uint64_t* d_offs;
    if (!dev) {
        uint8_t* p; B200C_TRY(ws_typed(c, WSC_IN, n + 64, &p));
        B200C_CUDA_TRY(c, cudaMemcpyAsync(p, in, n, cudaMemcpyHostToDevice, c->stream)); d_in = p;
        B200C_TRY(ws_typed(c, WSC_OUT, out_cap, &d_out));
    }
    if (dev && chunk_offsets) d_offs = chunk_offsets;     // caller provides nchunks+1 entries on the device
    else B200C_TRY(ws_typed(c, WSC_OFFS, nchunks + 1, &d_offs));
    if (comp == COMP_UNCOMPRESSED) {
        // ChecksummedSequentialWriter: Data.db = the stream, chunk_offsets[0..nchunks) = the CRC.db entries, digest over the bytes alone
        if (out_cap < n) { *out_len = n; c->err = "output buffer too small"; return B200C_ETOOSMALL; }
        timing_begin(c);
        int rc = raw_stream_device(c, d_in, n, chunk_len, dev ? d_out : nullptr, d_offs, digest, 0);
        int rc2 = timing_end(c);
        if (rc != B200C_OK) return rc;
        if (rc2 != B200C_OK) return rc2;
        *out_len = n;
        if (!dev) {
            if (n) B200C_CUDA_TRY(c, cudaMemcpyAsync(out, d_in, n, cudaMemcpyDeviceToHost, c->stream));
            if (chunk_offsets && nchunks) B200C_CUDA_TRY(c, cudaMemcpyAsync(chunk_offsets, d_offs, nchunks * 8, cudaMemcpyDeviceToHost, c->stream));
            B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
        }
        return B200C_OK;
    }
    timing_begin(c);
    int rc = compress_stream_device(c, comp, d_in, n, chunk_len, max_clen, d_out, out_cap, d_offs, out_len, digest, 0);
    int rc2 = timing_end(c);
    if (rc != B200C_OK) return rc;
    if (rc2 != B200C_OK) return rc2;
    if (!dev) {
        B200C_CUDA_TRY(c, cudaMemcpyAsync(out, d_out, *out_len, cudaMemcpyDeviceToHost, c->stream));
        if (chunk_offsets && nchunks) B200C_CUDA_TRY(c, cudaMemcpyAsync(chunk_offsets, d_offs, nchunks * 8, cudaMemcpyDeviceToHost, c->stream));
        B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    }
    return B200C_OK;
}

int b200c_decompress_chunks(b200c_ctx* c, int comp, const uint8_t* data, uint64_t data_len, const uint64_t* chunk_offsets, uint64_t nchunks,
                            int chunk_len, int max_clen, uint64_t data_length, uint8_t* out, int verify_crc, b200c_corruption* where, int flags) {
    B200C_TRY(check_codec_args(c, comp, chunk_len));
    if ((!data && data_len) || (!chunk_offsets && nchunks) || (!out && data_length)) { c->err = "null argument"; return B200C_EINVAL; }
    if (nchunks != b200c_chunk_count(data_length, chunk_len)) { c->err = "chunk count does not match data_length"; return B200C_EINVAL; }
    if (comp == COMP_UNCOMPRESSED && data_len != data_length) { c->err = "uncompressed Data.db: data_length must equal data_len"; return B200C_EINVAL; }
    cudaSetDevice(c->device);
    const bool dev = flags & B200C_FLAG_DEVICE_PTRS;
    if (comp == COMP_UNCOMPRESSED) {
        // every chunk checked against its CRC.db entry (chunk_offsets) and copied out; host buffers are verified where they were staged
        const uint8_t* d_data = data; const uint64_t* d_crc = chunk_offsets;
        if (!dev) {
            uint8_t* p; B200C_TRY(ws_typed(c, WSC_IN, data_len + 64, &p));
            if (data_len) B200C_CUDA_TRY(c, cudaMemcpyAsync(p, data, data_len, cudaMemcpyHostToDevice, c->stream));
            d_data = p;
            uint64_t* po; B200C_TRY(ws_typed(c, WSC_CHOFFS, nchunks + 1, &po));
            if (nchunks) B200C_CUDA_TRY(c, cudaMemcpyAsync(po, chunk_offsets, nchunks * 8, cudaMemcpyHostToDevice, c->stream));
            d_crc = po;
        }
        ChunkErr* d_err; B200C_TRY(ws_typed(c, WSC_ERR, 1, &d_err));
        B200C_CUDA_TRY(c, cudaMemsetAsync(d_err, 0xFF, sizeof(ChunkErr), c->stream));
        RawArgs a; memset(&a, 0, sizeof(a));
        a.src = d_data; a.dst = dev ? out : nullptr; a.n = data_len; a.L = chunk_len; a.chunk_end = nchunks; a.crc_exp = verify_crc ? d_crc : nullptr; a.err = d_err;
        timing_begin(c);
        int rc = raw_chunks_device(c, true, a);
        int rc2 = timing_end(c);
        if (rc != B200C_OK) return rc;
        if (rc2 != B200C_OK) return rc2;
        ChunkErr* h = (ChunkErr*)&c->h_pinned->chunk_err;
        B200C_CUDA_TRY(c, cudaMemcpyAsync(h, d_err, sizeof(ChunkErr), cudaMemcpyDeviceToHost, c->stream));
        B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
        if (h->first_bad != ~0ull) {
            const uint64_t chunk = (h->first_bad >> 8) & 0xFFFFFFFFFFull;
            if (where) { where->input = 0; where->kind = 1; where->chunk = chunk; where->offset = chunk * (uint64_t)chunk_len; }
            c->err = "chunk CRC mismatch at chunk " + std::to_string(chunk);
            return B200C_ECORRUPT;
        }
        if (!dev && data_len) {
            B200C_CUDA_TRY(c, cudaMemcpyAsync(out, d_data, data_len, cudaMemcpyDeviceToHost, c->stream));
            B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
        }
        return B200C_OK;
    }
    const uint8_t* d_data = data; const uint64_t* d_offs = chunk_offsets; uint8_t* d_out = out;
    if (!dev) {
        uint8_t* p; B200C_TRY(ws_typed(c, WSC_IN, data_len + 64, &p));
        B200C_CUDA_TRY(c, cudaMemcpyAsync(p, data, data_len, cudaMemcpyHostToDevice, c->stream)); d_data = p;
        uint64_t* po; B200C_TRY(ws_typed(c, WSC_CHOFFS, nchunks + 1, &po));
        B200C_CUDA_TRY(c, cudaMemcpyAsync(po, chunk_offsets, nchunks * 8, cudaMemcpyHostToDevice, c->stream)); d_offs = po;
        B200C_TRY(ws_typed(c, WSC_OUT, data_length + 64, &d_out));
    }
    ChunkErr* d_err; B200C_TRY(ws_typed(c, WSC_ERR, 1, &d_err));
    B200C_CUDA_TRY(c, cudaMemsetAsync(d_err, 0xFF, sizeof(ChunkErr), c->stream));
    timing_begin(c);
    int rc = decompress_stream_device(c, comp, d_data, data_len, d_offs, nchunks, chunk_len, max_clen, data_length, d_out, verify_crc, d_err, 0, ~0ull, 0, nullptr, ~0ull);
    int rc2 = timing_end(c);
    if (rc != B200C_OK) return rc;
    if (rc2 != B200C_OK) return rc2;
    ChunkErr* h = (ChunkErr*)&c->h_pinned->chunk_err;
    B200C_CUDA_TRY(c, cudaMemcpyAsync(h, d_err, sizeof(ChunkErr), cudaMemcpyDeviceToHost, c->stream));
    B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (h->first_bad != ~0ull) {
        uint64_t chunk = (h->first_bad >> 8) & 0xFFFFFFFFFFull; int kind = (int)(h->first_bad & 0xff);
        if (where) { where->input = 0; where->kind = kind; where->chunk = chunk; where->offset = 0; }
        c->err = std::string(kind == 1 ? "chunk CRC mismatch" : "malformed compressed chunk") + " at chunk " + std::to_string(chunk);
        return B200C_ECORRUPT;
    }
    if (!dev && data_length) {
        B200C_CUDA_TRY(c, cudaMemcpyAsync(out, d_out, data_length, cudaMemcpyDeviceToHost, c->stream));
        B200C_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    }
    return B200C_OK;
}

// ICompressor.compress: one buffer in, compressor output (no CRC) out.
int b200c_compress(b200c_ctx* c, int comp, const uint8_t* in, int n, uint8_t* out, int out_cap) {
    if (!c || n < 0 || !out) return B200C_EINVAL;
    if (comp == COMP_UNCOMPRESSED) { c->err = "compression disabled is not an ICompressor"; return B200C_EINVAL; }
    if (n > CHUNK_LEN_MAX) { c->err = "single-buffer compress is limited to 1 MiB"; return B200C_EUNSUPPORTED; }
    int chunk_len = 1; while (chunk_len < n) chunk_len <<= 1;
    if (n == 0) {   // degenerate: LZ4 of nothing = length prefix + one empty-literal token; Snappy = varint 0
        if (comp == COMP_LZ4) { if (out_cap < 5) return B200C_ETOOSMALL; memset(out, 0, 5); return 5; }
        if (comp_is_snappy(comp)) { if (out_cap < 1) return B200C_ETOOSMALL; out[0] = 0; return 1; }
        return 0;
    }
    std::vector<uint8_t> tmp(b200c_compress_bound(comp, n, chunk_len));
    uint64_t out_len = 0, off = 0; uint32_t dig = 0;
    int rc = b200c_compress_chunks(c, comp, in, (uint64_t)n, chunk_len, INT_MAX, tmp.data(), tmp.size(), &out_len, &off, &dig, 0);
    if (rc != B200C_OK) return rc;
    int clen = (int)out_len - 4;
    if (clen > out_cap) { c->err = "output buffer too small"; return B200C_ETOOSMALL; }
    memcpy(out, tmp.data(), clen);
    return clen;
}

// ICompressor.uncompress: compressor output in, plain bytes out; returns the decoded length.
int b200c_uncompress(b200c_ctx* c, int comp, const uint8_t* in, int n, uint8_t* out, int out_cap) {
    if (!c || !in || n <= 0 || out_cap < 0) return B200C_EINVAL;
    if (comp == COMP_UNCOMPRESSED) { c->err = "compression disabled is not an ICompressor"; return B200C_EINVAL; }
    int ulen;
    if (comp == COMP_LZ4) { if (n < 4) { c->err = "truncated"; return B200C_ECORRUPT; } ulen = (int)((uint32_t)in[0] | ((uint32_t)in[1] << 8) | ((uint32_t)in[2] << 16) | ((uint32_t)in[3] << 24)); }
    else if (comp_is_snappy(comp)) { uint32_t v = 0; int sh = 0, i = 0; bool ok = false; for (; i < n && i < 5; i++) { v |= (uint32_t)(in[i] & 0x7f) << sh; if (!(in[i] & 0x80)) { ok = true; break; } sh += 7; } if (!ok) { c->err = "bad varint"; return B200C_ECORRUPT; } ulen = (int)v; }
    else ulen = n;
    if (ulen < 0 || ulen > CHUNK_LEN_MAX) { c->err = "single-buffer uncompress is limited to 1 MiB"; return B200C_ECORRUPT; }
    if (ulen > out_cap) { c->err = "output buffer too small"; return B200C_ETOOSMALL; }
    if (ulen == 0) return 0;
    int chunk_len = 1; while (chunk_len < ulen) chunk_len <<= 1;
    std::vector<uint8_t> img(n + 4); memcpy(img.data(), in, n); memset(img.data() + n, 0, 4);
    uint64_t off = 0;
    int rc = b200c_decompress_chunks(c, comp, img.data(), img.size(), &off, 1, chunk_len, INT_MAX, (uint64_t)ulen, out, 0, nullptr, 0);
    if (rc != B200C_OK) return rc;
    return ulen;
}

} // extern "C"
