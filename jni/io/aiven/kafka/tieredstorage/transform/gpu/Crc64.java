package io.aiven.kafka.tieredstorage.transform.gpu;

import java.nio.ByteBuffer;

/**
 * The CRC-64/NVME twins of PartsCursor.transformParts, CheckCursor.checkObject and RewriteCursor.rewriteObject
 * (tsgpu_transform_parts_crc64, tsgpu_check_object_crc64, tsgpu_rewrite_object_crc64 of include/tsgpu.h).  Each takes its twin's
 * arguments and writes the same bytes; the 64-bit checksums come back in direct ByteBuffers, 8 bytes per word in
 * ByteOrder.nativeOrder().  Callers use them through PartsCursor, CheckCursor and RewriteCursor constructed with crc64 = true.
 * CRC-64/NVME is what S3 takes as CRC64NVME (part and FULL_OBJECT checksums) and, unverified, Azure as x-ms-content-crc64.
 */
public final class Crc64 {
    private Crc64() {
    }

    static {
        System.loadLibrary("tsgpu_jni");
    }

    /** partCrc64: capacity / 8 is part_cap; nPartsOut[0] receives the count, objectCrc64Out the object's CRC at the end. */
    public static native int transformParts(long ctx, int flags, ByteBuffer src, long srcLen, int chunkSize, byte[] key, byte[] aad,
                                            byte[] ivs, ByteBuffer dst, int[] transformedSizes, ByteBuffer recordsCursor,
                                            boolean segmentEndsHere, long partSize, ByteBuffer partsCursor, ByteBuffer partCrc64,
                                            int[] nPartsOut, ByteBuffer objectCrc64Out);

    /** crcsOut (16 bytes): the object's and the decoded segment's CRC on the object's last window. */
    public static native void checkObject(long ctx, int flags, ByteBuffer src, long srcLen, int[] transformedSizes,
                                          int originalChunkSize, long originalFileSize, byte[] key, byte[] aad, ByteBuffer cursor,
                                          boolean objectEndsHere, ByteBuffer crcsOut);

    /** partCrc64: capacity / 8 is part_cap; crcsOut (24 bytes): the old object's, the new object's and the segment's CRC. */
    public static native void rewriteObject(long ctx, int fromFlags, ByteBuffer src, long srcLen, int[] transformedSizes,
                                            int originalChunkSize, long originalFileSize, byte[] fromKey, byte[] fromAad,
                                            int toFlags, byte[] toKey, byte[] toAad, byte[] toIvs, ByteBuffer dst, long dstCap,
                                            int[] newTransformedSizes, long partSize, ByteBuffer partCrc64, int[] nPartsOut,
                                            ByteBuffer cursor, boolean objectEndsHere, ByteBuffer crcsOut);
}
