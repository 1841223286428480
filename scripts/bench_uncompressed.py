"""Times compactions of tables whose compression is disabled (Data.db + CRC.db) on bench.py's configs[1] shape and prints one JSON line.

The inputs are configs[1]'s streams (bench.make_inputs) stored uncompressed, their CRC.db tables written by
b200c_compress_chunks(B200C_COMP_UNCOMPRESSED). Steps are timed as bench.py times them: `value` with inputs and outputs resident in device
memory, `e2e` with host buffers. Each reports the stage clock (b200c_last_stage_ms) and, for K1 (copy + verify) and K5 (copy + CRC),
the data-sheet bandwidth floor of the stage, 2 x bytes / 3.35 TB/s (read and write). The floors are bounds, not measurements.

Verification needs no CPU oracle: the same compaction with LZ4 output is run once, its Data.db decompressed on the GPU must equal the
uncompressed output's Data.db and its Index.db must be identical; the output's CRC.db entries and digest are recomputed with zlib.

  python scripts/bench_uncompressed.py --steps 5 --warmup 3 [--mib 512]
"""
import argparse, ctypes as C, json, os, subprocess, sys, time, zlib
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench

HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet
CRC_CHUNK = 65536                    # CRC.db chunk size a compaction writer uses (SequentialWriterOption default buffer)

def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1])}
    except Exception as e:
        return {"error": str(e)[:80]}

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mib", type=float, default=None, help="uncompressed MiB per input (default: configs[1]'s 512)")
    args = ap.parse_args()
    import numpy as np, torch
    from cassandra_b200 import native
    wl = dict(bench.WORKLOADS["cfg1"])
    if args.mib: wl["mib"] = args.mib
    L = native.lib(); ctx = native.Context(0); UNC = native.COMP_UNCOMPRESSED
    threads = len(os.sched_getaffinity(0))

    def store_uncompressed(stream):          # ChecksummedSequentialWriter on the GPU: Data.db = the stream, CRC.db entries
        n = len(stream); nch = L.b200c_chunk_count(n, CRC_CHUNK)
        crcs = np.zeros(max(nch, 1), dtype=np.uint64); out = np.empty(max(n, 1), dtype=np.uint8); out_len = C.c_uint64(); dig = C.c_uint32()
        ctx.check(L.b200c_compress_chunks(ctx.handle, UNC, stream.ctypes.data, n, CRC_CHUNK, 0, out.ctypes.data, n, C.byref(out_len), crcs.ctypes.data, C.byref(dig), 0))
        return out[:n], crcs[:nch]
    t0 = time.time()
    tabs = bench.make_inputs(wl, store_uncompressed, threads)
    u_in = sum(t.compression.data_length for t in tabs); i_in = sum(t.hold[1].numel() for t in tabs)
    bench.log("uncompressed inputs ready: %.2f GB in %.0fs" % (u_in / 1e9, time.time() - t0))

    def manifest(out_comp, device_copies=None):
        m = bench.build_manifest(tabs, wl, device_copies)
        for k in range(m.ninputs):
            m.inputs[k].compressor = UNC; m.inputs[k].chunk_len = CRC_CHUNK; m.inputs[k].data_length = m.inputs[k].data_len
        m.out_compressor = out_comp
        if out_comp == UNC: m.out_chunk_len = CRC_CHUNK
        return m
    cap_d = u_in + (64 << 20); cap_i = i_in + (1 << 20); cap_c = u_in // 16384 + 16

    def timed(m, bufs, dev, steps):
        torch.cuda.synchronize(); t = time.perf_counter(); stages = [0.0] * 6; last = None
        for _ in range(steps):
            last = bufs.result()
            ctx.check(L.b200c_compact(ctx.handle, C.byref(m), C.byref(last), 1 if dev else 0), last.corruption)
            for i, v in enumerate(ctx.last_stage_ms()): stages[i] += v
        torch.cuda.synchronize()
        return (time.perf_counter() - t) / steps, [s / steps for s in stages], last

    names = ["K1_ingest_verify", "K2_index", "K3_merge", "K4_size", "K4_emit", "K5_checksum"]
    line = {"workload": wl["name"] + ", stored uncompressed (CRC.db chunk 64 KiB), uncompressed output", "u_in_bytes": u_in, "card": card()}

    # ---- e2e: host buffers ----
    m_host = manifest(UNC); ho = bench.OutBufs(1, cap_d, cap_i, cap_c, device=False)
    for _ in range(args.warmup): timed(m_host, ho, False, 1)
    dt, st, res = timed(m_host, ho, False, args.steps)
    files = ho.files(res); u_out = int(res.outputs[0].data_length)
    line["e2e"] = {"ms_per_step": round(dt * 1e3, 2), "MB_per_s": round(u_in / dt / 1e6, 1), "stage_ms": {n: round(s, 2) for n, s in zip(names, st)}}

    # ---- verification: the LZ4-output run decompressed on the GPU, Index.db, CRC.db recomputed ----
    data, index, crcs, digest = files[0][0], files[0][1], files[0][2], files[0][3]
    lo = bench.OutBufs(1, L.b200c_compress_bound(native.COMP_LZ4, u_in, 16384), cap_i, cap_c, device=False)
    _, _, r2 = timed(manifest(native.COMP_LZ4), lo, False, 1)
    lz4 = lo.files(r2)[0]
    back = ctx.decompress_chunks(native.COMP_LZ4, lz4[0], lz4[2], int(r2.outputs[0].data_length), 16384)
    want_crcs = np.asarray([zlib.crc32(memoryview(data)[i:i + CRC_CHUNK]) for i in range(0, len(data), CRC_CHUNK)], dtype=np.uint64)
    checks = {"data_equals_lz4_output_decompressed": bool(len(back) == len(data) and np.array_equal(np.frombuffer(back, dtype=np.uint8), data)),
              "index_identical": bool(np.array_equal(index, lz4[1])),
              "crc_table_recomputed": bool(np.array_equal(crcs, want_crcs)), "digest_recomputed": digest == zlib.crc32(memoryview(data)),
              "short_last_chunk": len(data) % CRC_CHUNK != 0}
    del back, lz4, lo
    line["verified"] = all(checks.values()); line["checks"] = checks

    # ---- value: inputs and outputs in device memory ----
    dev_in = [(t.hold[0].cuda(), t.hold[1].cuda(), t.hold[2].cuda(), t.summary.cuda()) for t in tabs]
    m_dev = manifest(UNC, [(a.data_ptr(), b.data_ptr(), c.data_ptr(), d.data_ptr()) for a, b, c, d in dev_in])
    do = bench.OutBufs(1, cap_d, cap_i, cap_c, device=True)
    for _ in range(args.warmup): timed(m_dev, do, True, 1)
    dt, st, res = timed(m_dev, do, True, args.steps)
    dfiles = do.files(res)
    line["value"] = {"ms_per_step": round(dt * 1e3, 2), "MB_per_s": round(u_in / dt / 1e6, 1), "stage_ms": {n: round(s, 2) for n, s in zip(names, st)}}
    line["value_output_equals_e2e"] = bool(bench.same_files(dfiles, files) is None)
    free_b, total_b = torch.cuda.mem_get_info(0)
    line["device_memory_in_use_gb"] = round((total_b - free_b) / 1e9, 1)
    line["floors_ms"] = {"K1": round(2 * u_in / HBM_BYTES_PER_S * 1e3, 2), "K5": round(2 * u_out / HBM_BYTES_PER_S * 1e3, 2), "basis": "2 x bytes / 3.35 TB/s (H100 SXM data sheet)"}
    line["card_after"] = card()
    print(json.dumps(line), flush=True)
    ctx.close()

if __name__ == "__main__":
    main()
