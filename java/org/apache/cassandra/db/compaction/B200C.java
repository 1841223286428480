/*
 * JNI surface of include/b200c.h (libb200compact.so), bound by java/b200c_jni.c.
 *
 * Not compiled in the build image (no JDK there); compile-checked where a JDK 11/17 and the Cassandra jars exist:
 *   javac -cp "$CASSANDRA_HOME/build/classes/main:$CASSANDRA_HOME/lib/*" -d build/java $(find java -name '*.java')
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude java/b200c_jni.c -Lcassandra_b200 -lb200compact -o libb200compact_jni.so
 *
 * Every method takes raw addresses of DirectByteBuffers (or of mmapped component files) and lengths; nothing here touches a Java
 * object on the hot path. One context per CompactionExecutor thread: the library is re-entrant per context.
 */
package org.apache.cassandra.db.compaction;

import java.nio.ByteBuffer;
import java.nio.ByteOrder;

public final class B200C
{
    static { System.loadLibrary("b200compact_jni"); }

    private B200C() {}

    // ---- return codes of b200c.h --------------------------------------------------------------------------------------------
    public static final int OK = 0, EINVAL = -1, ECUDA = -2, ECORRUPT = -3, ECANCELLED = -4, EUNSUPPORTED = -5, ENOMEM = -6, ETOOSMALL = -7;
    public static final int COMP_NONE = 0, COMP_LZ4 = 1, COMP_SNAPPY = 2, COMP_UNCOMPRESSED = 4;      // 4: compression disabled, Data.db + CRC.db
    public static final int PARTITIONER_MURMUR3 = 0, PARTITIONER_BYTE_ORDERED = 1;
    public static final int TYPE_BYTES = 0, TYPE_FIXED_SIGNED = 1, TYPE_FIXED_BYTES = 2, TYPE_VAR_SIGNED = 3, TYPE_TIMEUUID = 4, TYPE_COUNTER = 5;
    public static final int MAX_COMPLEX_COLUMNS = 8;       // multi-cell (map / set / list) columns per table, B200C_MAX_COMPLEX_COLUMNS
    public static final int ABI_VERSION = 2;
    public static final int MAX_CLUSTERING = 8, MAX_COLUMNS = 64, MAX_INPUTS = 64, MAX_STATIC_COLUMNS = 16;
    public static final int MAX_CHUNK_LENGTH = 1 << 20;      // compression chunk_length_in_kb up to 1024 (CRC.db chunks of uncompressed tables: 64 KiB)

    // ---- lifecycle ----------------------------------------------------------------------------------------------------------
    public static native int    abiVersion();                                       // b200c_abi_version
    public static native int    deviceCount();                                      // b200c_device_count
    public static native long   create(int device, long workspaceBytes);            // b200c_create  (0 = no CUDA device: there is no CPU fallback)
    public static native void   destroy(long ctx);                                  // b200c_destroy
    public static native String lastError(long ctx);                                // b200c_last_error
    public static native int    hostRegister(long address, long length);            // b200c_host_register (pin DirectByteBuffers / mmaps once)
    public static native int    hostUnregister(long address);                       // b200c_host_unregister

    // ---- compaction ---------------------------------------------------------------------------------------------------------
    /** manifestAddress / resultAddress: DirectByteBuffers laid out as b200c_manifest / b200c_result (native order; see {@link Layout}) */
    public static native int    compact(long ctx, long manifestAddress, long resultAddress, int flags);   // b200c_compact
    public static native int    poll(long ctx, long progressAddress);                // b200c_poll        -> CompactionInfo.Holder
    public static native int    pollInputs(long ctx, long positionsAddress, int n);  // b200c_poll_inputs -> ISSTableScanner.getCurrentPosition
    public static native void   cancel(long ctx);                                    // b200c_cancel      <- isStopRequested()
    public static native void   cancelReset(long ctx);                               // b200c_cancel_reset (when a new task is bound to the context)
    public static native long   token(int partitioner, long keyAddress, int keyLength);   // b200c_token

    // ---- chunk codec (CompressedSequentialWriter / CompressedChunkReader data plane, batched) ---------------------------------
    public static native long   compressBound(int compressor, long n, int chunkLength);
    public static native int    compressChunks(long ctx, int compressor, long in, long n, int chunkLength, int maxCompressedLength,
                                               long out, long outCap, long outLenAddress, long offsetsAddress, long digestAddress, int flags);
    public static native int    decompressChunks(long ctx, int compressor, long data, long dataLength, long offsetsAddress, long nChunks, int chunkLength,
                                                 int maxCompressedLength, long uncompressedLength, long out, int verifyCrc, long whereAddress, int flags);
    // ---- ICompressor single-buffer contract -----------------------------------------------------------------------------------
    public static native int    initialCompressedBufferLength(int compressor, int chunkLength);
    public static native int    compress(long ctx, int compressor, long in, int n, long out, int outCap);
    public static native int    uncompress(long ctx, int compressor, long in, int n, long out, int outCap);

    /**
     * sizeof / offsetof of the C structs, asked from the native side once (java/b200c_jni.c: layout()) so that this class can never
     * drift from include/b200c.h. Order of the returned array: see b200c_jni.c.
     */
    public static native int[]  layout();

    /** address of a direct buffer's first byte (GetDirectBufferAddress) */
    public static native long   address(ByteBuffer direct);

    /** One context per thread, created lazily, destroyed with the thread. */
    private static final ThreadLocal<long[]> CONTEXT = ThreadLocal.withInitial(() -> new long[]{ 0L });

    public static long context()
    {
        long[] c = CONTEXT.get();
        if (c[0] == 0L)
        {
            int device = Integer.getInteger("cassandra.b200c.device", 0);
            c[0] = create(device, 0L);
            if (c[0] == 0L)
                throw new IllegalStateException("b200c_create failed: no CUDA device " + device + " (the GPU engine has no CPU fallback)");
        }
        return c[0];
    }

    public static ByteBuffer struct(int bytes)
    {
        return ByteBuffer.allocateDirect(bytes).order(ByteOrder.nativeOrder());
    }

    /** struct layouts of b200c.h as (offset) constants resolved at class-initialisation time */
    public static final class Layout
    {
        private static final int[] L = layout();
        private static int k = 0;
        private static int next() { return L[k++]; }
        // sizes
        public static final int SIZEOF_INPUT = next(), SIZEOF_MANIFEST = next(), SIZEOF_OUTPUT = next(), SIZEOF_RESULT = next(), SIZEOF_PROGRESS = next(),
                                SIZEOF_STATS = next(), SIZEOF_CORRUPTION = next();
        // b200c_input
        public static final int IN_DATA = next(), IN_DATA_LEN = next(), IN_INDEX = next(), IN_INDEX_LEN = next(), IN_CHUNK_OFFSETS = next(), IN_NCHUNKS = next(),
                                IN_DATA_LENGTH = next(), IN_COMPRESSOR = next(), IN_CHUNK_LEN = next(), IN_MAX_COMPRESSED_LEN = next(), IN_NCOLUMNS = next(),
                                IN_COLUMN_MAP = next(), IN_HEADER_STATS = next(), IN_LEVEL = next(), IN_SUMMARY_POSITIONS = next(), IN_NSUMMARY = next(),
                                IN_NSTATIC_COLUMNS = next(), IN_STATIC_COLUMN_MAP = next();
        // b200c_manifest
        public static final int M_ABI_VERSION = next(), M_NINPUTS = next(), M_INPUTS = next(), M_NCLUSTERING = next(), M_CLUSTERING = next(), M_NCOLUMNS = next(),
                                M_COLUMNS = next(), M_NSTATIC_COLUMNS = next(), M_OUT_STATS = next(), M_OUT_COMPRESSOR = next(), M_OUT_CHUNK_LEN = next(),
                                M_OUT_MAX_COMPRESSED_LEN = next(), M_COLUMN_INDEX_SIZE = next(), M_NOW_IN_SEC = next(), M_GC_BEFORE = next(),
                                M_PURGE_MAX_TIMESTAMP = next(), M_TOMBSTONE_OPTION = next(), M_ENFORCE_STRICT_LIVENESS = next(), M_TOKEN_LO = next(),
                                M_TOKEN_HI = next(), M_MAX_SSTABLE_BYTES = next(), M_PARTITIONER = next(), M_NPURGE_RANGES = next(), M_PURGE_RANGE_HI = next(),
                                M_PURGE_RANGE_MAX_TS = next(), M_BLOOM_HASH_COUNT = next(), M_MIN_INDEX_INTERVAL = next(), M_BLOOM_WORDS = next(), M_STATIC_COLUMNS = next();
        // b200c_output
        public static final int O_DATA = next(), O_DATA_CAP = next(), O_DATA_LEN = next(), O_INDEX = next(), O_INDEX_CAP = next(), O_INDEX_LEN = next(),
                                O_CHUNK_OFFSETS = next(), O_CHUNK_CAP = next(), O_NCHUNKS = next(), O_DATA_LENGTH = next(), O_DIGEST = next(), O_PARTITIONS = next(),
                                O_ROWS = next(), O_KEY_BUF = next(), O_KEY_CAP = next(), O_FIRST_KEY_LEN = next(), O_LAST_KEY_LEN = next(), O_FILTER = next(),
                                O_FILTER_CAP = next(), O_FILTER_LEN = next(), O_SUMMARY = next(), O_SUMMARY_CAP = next(), O_SUMMARY_LEN = next(), O_STATS = next();
        // b200c_result
        public static final int R_NOUTPUTS_CAP = next(), R_NOUTPUTS = next(), R_OUTPUTS = next(), R_BYTES_READ = next(), R_BYTES_IN_RANGE = next(), R_BYTES_WRITTEN = next(),
                                R_TOTAL_SOURCE_ROWS = next(), R_INPUT_PARTITIONS = next(), R_MERGED_ROW_COUNTS = next(), R_REQUIRED_DATA_CAP = next(),
                                R_REQUIRED_INDEX_CAP = next(), R_REQUIRED_CHUNK_CAP = next(), R_CORRUPTION = next(), R_KERNEL_MS = next(), R_TOTAL_MS = next();
        // b200c_sstable_stats
        public static final int S_MIN_TIMESTAMP = next(), S_MAX_TIMESTAMP = next(), S_MIN_LDT = next(), S_MAX_LDT = next(), S_MIN_TTL = next(), S_MAX_TTL = next(),
                                S_TOTAL_ROWS = next(), S_TOTAL_COLUMNS_SET = next(), S_TOTAL_CELLS = next(), S_TOTAL_TOMBSTONES = next(), S_HAS_PARTITION_DELETIONS = next(),
                                S_TDROP_OVERFLOW = next(), S_PARTITION_SIZE_HIST = next(), S_CELLS_HIST = next(), S_NTDROP = next(), S_HAS_LEGACY_COUNTER_SHARDS = next(), S_TDROP_POINT = next(),
                                S_TDROP_COUNT = next(), S_HLL_REGISTERS = next();
        // b200c_corruption, b200c_encoding_stats, b200c_column are {i32 input, i32 kind, u64 chunk, u64 offset} / {i64, i64, i32, pad} / {i32, i32}
        private Layout() {}
    }
}
