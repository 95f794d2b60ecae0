package io.aiven.kafka.tieredstorage.transform.gpu;

import java.nio.ByteBuffer;

/** Native entry points of libtsgpu (see include/tsgpu.h and jni/tsgpu_jni.c). */
public final class TsGpu {
    public static final int FLAG_ZSTD = 1;
    public static final int FLAG_AES = 2;
    // flags pass through to the C-ABI unchanged: TSGPU_FLAG_ZSTD_CHECKSUM (16, include/tsgpu.h) ends every zstd frame with its
    // Content_Checksum; TSGPU_ZSTD_CHECKSUM=1 in the broker's environment turns it on without a change here
    /** Check every record batch of the segment (length, magic, CRC) on the GPU before it is uploaded; needs FLAG_ZSTD or
     *  FLAG_AES.  A damaged batch fails the call with a RuntimeException, so Kafka keeps the local segment and retries the
     *  copy.  Segments that arrive in windows carry the state from one window to the next in a {@link RecordsCursor}. */
    public static final int FLAG_VALIDATE_RECORDS = 32;
    /** RewriteCursor only, with FLAG_ZSTD on both sides: seal the kept frames with their Content_Checksum (with 16,
     *  TSGPU_FLAG_ZSTD_CHECKSUM) or re-encode them in dense mode when that is smaller (with 4, TSGPU_FLAG_ZSTD_DENSE); every new
     *  chunk is then read back on the GPU before it leaves.  Every other call refuses it. */
    public static final int FLAG_REFRAME = 64;
    public static final int IV_SIZE = 12;

    static {
        System.loadLibrary("tsgpu_jni");
    }

    private TsGpu() {
    }

    public static native long create(int[] devices, int maxChunkBytes, int maxBatch);

    public static native void destroy(long ctx);

    public static native ByteBuffer allocPinned(long bytes);

    public static native void freePinned(ByteBuffer buffer);

    public static native long transformBound(int flags, long srcLen, int chunkSize);

    public static native int transform(long ctx, int flags, ByteBuffer src, long srcLen, int chunkSize,
                                       byte[] key, byte[] aad, byte[] ivs, ByteBuffer dst, int[] transformedSizes);

    public static native void detransform(long ctx, int flags, ByteBuffer src, long srcLen, int[] transformedSizes,
                                          byte[] key, byte[] aad, ByteBuffer dst, int[] originalSizes);
}
