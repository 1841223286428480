"""Times configs[1]'s compaction with its inputs and output stored at 64 KiB, 256 KiB and 1 MiB chunks and prints one JSON line per chunk length.

The inputs are bench.py's configs[1] streams (bench.make_inputs), each compressed on the GPU at every chunk length (b200c_compress_chunks, LZ4).
For each length the compaction writes its output at the same length and is timed as bench.py times it: `value` with inputs and outputs resident
in device memory, `e2e` with host buffers. Each line reports the stage clock (b200c_last_stage_ms: K1 decompress + verify, K5 compress + CRC +
pack) and the card's name and power limit, read in the same run.

Every run is checked without a CPU oracle: its Data.db decompressed on the GPU must equal the 64 KiB run's (SHA-256 of the streams), its
Index.db must be identical, and every chunk's CRC32 and the digest are recomputed with zlib.

  python scripts/bench_chunk_length.py --steps 3 --warmup 1 [--mib 512]
"""
import argparse, ctypes as C, hashlib, json, os, subprocess, sys, time, zlib
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench

LENGTHS = (64 << 10, 256 << 10, 1 << 20)
NAMES = ["K1_decompress_verify", "K2_index", "K3_merge", "K4_size", "K4_emit", "K5_compress_crc_pack"]

def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1])}
    except Exception as e:
        return {"error": str(e)[:80]}

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3); ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--mib", type=float, default=None, help="uncompressed MiB per input (default: configs[1]'s 512)")
    args = ap.parse_args()
    import numpy as np, torch
    from cassandra_b200 import native
    wl = dict(bench.WORKLOADS["cfg1"])
    if args.mib: wl["mib"] = args.mib
    L = native.lib(); ctx = native.Context(0); LZ4 = native.COMP_LZ4
    threads = len(os.sched_getaffinity(0))

    def compress(stream, chunk_len):
        n = len(stream); cap = L.b200c_compress_bound(LZ4, n, chunk_len); nch = L.b200c_chunk_count(n, chunk_len)
        out = np.empty(cap, dtype=np.uint8); offs = np.zeros(max(nch, 1), dtype=np.uint64); out_len = C.c_uint64(); dig = C.c_uint32()
        ctx.check(L.b200c_compress_chunks(ctx.handle, LZ4, stream.ctypes.data, n, chunk_len, native.INT32_MAX, out.ctypes.data, cap, C.byref(out_len), offs.ctypes.data, C.byref(dig), 0))
        return out[:out_len.value], offs[:nch]
    streams = []
    def keep(stream):
        streams.append(stream)                                 # the uncompressed stream, compressed again at each length below
        return compress(stream, LENGTHS[0])
    t0 = time.time()
    tabs = bench.make_inputs(wl, keep, threads)
    u_in = sum(t.compression.data_length for t in tabs); i_in = sum(t.hold[1].numel() for t in tabs)
    bench.log("inputs ready: %.2f GB in %.0fs" % (u_in / 1e9, time.time() - t0))

    def timed(m, bufs, dev, steps):
        torch.cuda.synchronize(); t = time.perf_counter(); stages = [0.0] * 6; last = None
        for _ in range(steps):
            last = bufs.result()
            ctx.check(L.b200c_compact(ctx.handle, C.byref(m), C.byref(last), 1 if dev else 0), last.corruption)
            for i, v in enumerate(ctx.last_stage_ms()): stages[i] += v
        torch.cuda.synchronize()
        return (time.perf_counter() - t) / steps, [s / steps for s in stages], last

    def stored_at(chunk_len):
        if chunk_len != LENGTHS[0]:
            for t, s in zip(tabs, streams):
                image, offs = compress(s, chunk_len)
                t.hold = (torch.from_numpy(image).pin_memory(), t.hold[1], torch.from_numpy(offs.view(np.int64)).pin_memory()); t.nchunks = len(offs)
    def manifest(chunk_len, device_copies=None):
        m = bench.build_manifest(tabs, wl, device_copies)
        for k in range(m.ninputs): m.inputs[k].chunk_len = chunk_len
        m.out_chunk_len = chunk_len
        return m

    base = None
    for chunk_len in LENGTHS:
        stored_at(chunk_len)
        c_in = sum(t.hold[0].numel() for t in tabs)
        cap_d = L.b200c_compress_bound(LZ4, u_in, chunk_len); cap_i = i_in + (1 << 20); cap_c = u_in // chunk_len + 16
        line = {"workload": wl["name"] + ", inputs and output at %d KiB chunks" % (chunk_len >> 10), "chunk_len": chunk_len, "u_in_bytes": u_in,
                "c_in_bytes": c_in, "card": card()}
        # ---- e2e: host buffers ----
        ho = bench.OutBufs(1, cap_d, cap_i, cap_c, device=False); m_host = manifest(chunk_len)
        for _ in range(args.warmup): timed(m_host, ho, False, 1)
        dt, st, res = timed(m_host, ho, False, args.steps)
        files = ho.files(res); data, index, offs, digest = files[0][0], files[0][1], files[0][2], files[0][3]
        line["e2e"] = {"ms_per_step": round(dt * 1e3, 2), "MB_per_s": round(u_in / dt / 1e6, 1), "stage_ms": {n: round(s, 2) for n, s in zip(NAMES, st)}}
        # ---- checks: the stream against the 64 KiB run's, Index.db, every chunk CRC and the digest recomputed ----
        ulen = int(res.outputs[0].data_length)
        back = ctx.decompress_chunks(LZ4, data, offs, ulen, chunk_len)
        sha = hashlib.sha256(back).hexdigest(); del back
        mv = memoryview(data); starts = offs.tolist(); ends = starts[1:] + [len(data)]
        crc_ok = all(zlib.crc32(mv[a:b - 4]) == int.from_bytes(mv[b - 4:b], "big") for a, b in zip(starts, ends))
        if base is None: base = (sha, index.copy(), ulen)
        checks = {"stream_equals_64k_run": sha == base[0] and ulen == base[2], "index_identical": bool(np.array_equal(index, base[1])),
                  "chunk_crcs_recomputed": crc_ok, "digest_recomputed": digest == zlib.crc32(mv), "chunks": len(offs) == (ulen + chunk_len - 1) // chunk_len}
        # ---- value: inputs and outputs in device memory ----
        dev_in = [(t.hold[0].cuda(), t.hold[1].cuda(), t.hold[2].cuda(), t.summary.cuda()) for t in tabs]
        m_dev = manifest(chunk_len, [(a.data_ptr(), b.data_ptr(), c.data_ptr(), d.data_ptr()) for a, b, c, d in dev_in])
        do = bench.OutBufs(1, cap_d, cap_i, cap_c, device=True)
        for _ in range(args.warmup): timed(m_dev, do, True, 1)
        dt, st, res = timed(m_dev, do, True, args.steps)
        checks["value_output_equals_e2e"] = bench.same_files(do.files(res), files) is None
        line["value"] = {"ms_per_step": round(dt * 1e3, 2), "MB_per_s": round(u_in / dt / 1e6, 1), "stage_ms": {n: round(s, 2) for n, s in zip(NAMES, st)}}
        line["verified"] = all(checks.values()); line["checks"] = checks
        line["card_after"] = card()
        print(json.dumps(line), flush=True)
        del dev_in, do, ho, files, data, mv
        torch.cuda.empty_cache()
    ctx.close()

if __name__ == "__main__":
    main()
