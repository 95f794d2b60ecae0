package io.aiven.kafka.tieredstorage.transform.gpu;

import java.nio.ByteBuffer;

/**
 * The state of ONE stored .log object while it is rewritten on the GPU in windows of chunks (tsgpu_rewrite_cursor of
 * include/tsgpu.h): the check of the old object (chunks and bytes so far, the running CRC-32C of the old object and of the decoded
 * segment, the record validation state) and the new object's open upload part.  Each window goes through tsgpu_rewrite_object,
 * which checks it as CheckCursor does and transforms it under the new key and flags without copying any plaintext back; the
 * window's new chunks land in dst with the CRC-32C of every upload part they complete.  After the last window,
 * sourceCrc32c() is compared with the store's checksum of the old object, segmentCrc32c() with the segment CRC recorded earlier,
 * and objectCrc32c() completes the upload (S3 FULL_OBJECT, GCS crc32c).  A failed window throws RuntimeException
 * (IllegalArgumentException for arguments, among them an old chunk's IV reused under the same key) with the library's message,
 * and the cursor is then spent.
 */
public final class RewriteCursor {
    public static final int SIZE = 192;
    private final ByteBuffer state = ByteBuffer.allocateDirect(SIZE);    // zeros: the start of an object
    private final int[] crcs = new int[3];
    private final int[] nParts = new int[1];
    private boolean ended = false;

    /**
     * One window: old transformed chunks transformedSizes back to back in src.  fromFlags are the old manifest's (TsGpu.FLAG_ZSTD,
     * TsGpu.FLAG_AES), plus TsGpu.FLAG_VALIDATE_RECORDS; toFlags the new object's (FLAG_ZSTD and/or FLAG_AES, plus FLAG_VERIFY).
     * toIvs holds 12 bytes per chunk of the window when toFlags has FLAG_AES.  newTransformedSizes receives one size per chunk,
     * partCrcs the CRC-32C of the parts the window completes; returns their count.
     */
    public int rewrite(final long ctx, final int fromFlags, final ByteBuffer src, final long srcLen, final int[] transformedSizes,
                       final int originalChunkSize, final long originalFileSize, final byte[] fromKey, final byte[] fromAad,
                       final int toFlags, final byte[] toKey, final byte[] toAad, final byte[] toIvs, final ByteBuffer dst,
                       final long dstCap, final int[] newTransformedSizes, final long partSize, final int[] partCrcs,
                       final boolean objectEndsHere) {
        if (ended) {
            throw new IllegalStateException("the object's last window has already been rewritten");
        }
        rewriteObject(ctx, fromFlags, src, srcLen, transformedSizes, originalChunkSize, originalFileSize, fromKey, fromAad,
            toFlags, toKey, toAad, toIvs, dst, dstCap, newTransformedSizes, partSize, partCrcs, nParts, state, objectEndsHere, crcs);
        ended = objectEndsHere;
        return nParts[0];
    }

    /** The CRC-32C of the old object, once the last window is rewritten. */
    public int sourceCrc32c() {
        return crc(0);
    }

    /** The CRC-32C of the new object, once the last window is rewritten. */
    public int objectCrc32c() {
        return crc(1);
    }

    /** The CRC-32C of the decoded segment, once the last window is rewritten. */
    public int segmentCrc32c() {
        return crc(2);
    }

    private int crc(final int k) {
        if (!ended) {
            throw new IllegalStateException("the object's last window has not been rewritten yet");
        }
        return crcs[k];
    }

    static {
        System.loadLibrary("tsgpu_jni");
    }

    public static native void rewriteObject(long ctx, int fromFlags, ByteBuffer src, long srcLen, int[] transformedSizes,
                                            int originalChunkSize, long originalFileSize, byte[] fromKey, byte[] fromAad,
                                            int toFlags, byte[] toKey, byte[] toAad, byte[] toIvs, ByteBuffer dst, long dstCap,
                                            int[] newTransformedSizes, long partSize, int[] partCrcs, int[] nPartsOut,
                                            ByteBuffer cursor, boolean objectEndsHere, int[] crcsOut);
}
