package io.aiven.kafka.tieredstorage.transform.gpu;

import java.nio.ByteBuffer;
import java.nio.ByteOrder;

/**
 * The state of ONE stored .log object while it is rewritten on the GPU in windows of chunks (tsgpu_rewrite_cursor of
 * include/tsgpu.h): the check of the old object (chunks and bytes so far, the running CRC-32C of the old object and of the decoded
 * segment, the record validation state) and the new object's open upload part.  Each window goes through tsgpu_rewrite_object,
 * which checks it as CheckCursor does and transforms it under the new key and flags without copying any plaintext back; the
 * window's new chunks land in dst with the CRC-32C of every upload part they complete.  After the last window,
 * sourceCrc32c() is compared with the store's checksum of the old object, segmentCrc32c() with the segment CRC recorded earlier,
 * and objectCrc32c() completes the upload (S3 FULL_OBJECT, GCS crc32c).  A failed window throws RuntimeException
 * (IllegalArgumentException for arguments, among them an old chunk's IV reused under the same key) with the library's message,
 * and the cursor is then spent.  Constructed with crc64 = true, the windows go through tsgpu_rewrite_object_crc64
 * (Crc64.rewriteObject): {@link #rewrite64} returns the parts' CRC-64/NVME, and sourceCrc64 / objectCrc64 / segmentCrc64 the
 * object words.
 */
public final class RewriteCursor {
    public static final int SIZE = 192;
    private final ByteBuffer state = ByteBuffer.allocateDirect(SIZE);    // zeros: the start of an object
    private final int[] crcs = new int[3];
    private final int[] nParts = new int[1];
    private boolean ended = false;
    private final ByteBuffer crcs64;                                       // null for CRC-32C

    public RewriteCursor() {
        this(false);
    }

    /** crc64: CRC-64/NVME part, source, object and segment checksums instead of CRC-32C; one cursor carries one width. */
    public RewriteCursor(final boolean crc64) {
        crcs64 = crc64 ? ByteBuffer.allocateDirect(24).order(ByteOrder.nativeOrder()) : null;
    }

    /**
     * One window: old transformed chunks transformedSizes back to back in src.  fromFlags are the old manifest's (TsGpu.FLAG_ZSTD,
     * TsGpu.FLAG_AES), plus TsGpu.FLAG_VALIDATE_RECORDS; toFlags the new object's (FLAG_ZSTD and/or FLAG_AES, plus FLAG_VERIFY).
     * When both have FLAG_ZSTD, TsGpu.FLAG_REFRAME with 16 (checksum) and/or 4 (dense) in toFlags seals the old frames with their
     * Content_Checksum or re-encodes them when that makes them smaller: each new chunk is then up to 4 bytes longer than its old
     * frame, so dst needs 4 more bytes per chunk.  Set FLAG_VALIDATE_RECORDS in fromFlags when sealing.
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
        if (crcs64 != null) {
            throw new IllegalStateException("this cursor computes CRC-64/NVME: call rewrite64");
        }
        rewriteObject(ctx, fromFlags, src, srcLen, transformedSizes, originalChunkSize, originalFileSize, fromKey, fromAad,
            toFlags, toKey, toAad, toIvs, dst, dstCap, newTransformedSizes, partSize, partCrcs, nParts, state, objectEndsHere, crcs);
        ended = objectEndsHere;
        return nParts[0];
    }

    /**
     * {@link #rewrite} for a crc64 cursor: partCrc64 receives the CRC-64/NVME of the parts the window completes (its length is
     * part_cap); returns their count.
     */
    public int rewrite64(final long ctx, final int fromFlags, final ByteBuffer src, final long srcLen, final int[] transformedSizes,
                         final int originalChunkSize, final long originalFileSize, final byte[] fromKey, final byte[] fromAad,
                         final int toFlags, final byte[] toKey, final byte[] toAad, final byte[] toIvs, final ByteBuffer dst,
                         final long dstCap, final int[] newTransformedSizes, final long partSize, final long[] partCrc64,
                         final boolean objectEndsHere) {
        if (crcs64 == null) {
            throw new IllegalStateException("this cursor computes CRC-32C: construct it with crc64 = true");
        }
        if (ended) {
            throw new IllegalStateException("the object's last window has already been rewritten");
        }
        final ByteBuffer out = ByteBuffer.allocateDirect(8 * partCrc64.length).order(ByteOrder.nativeOrder());
        Crc64.rewriteObject(ctx, fromFlags, src, srcLen, transformedSizes, originalChunkSize, originalFileSize, fromKey, fromAad,
            toFlags, toKey, toAad, toIvs, dst, dstCap, newTransformedSizes, partSize, out, nParts, state, objectEndsHere, crcs64);
        for (int i = 0; i < nParts[0]; i++) {
            partCrc64[i] = out.getLong(8 * i);
        }
        ended = objectEndsHere;
        return nParts[0];
    }

    /** The CRC-64/NVME of the old object of a crc64 cursor, once the last window is rewritten. */
    public long sourceCrc64() {
        return crc64(0);
    }

    /** The CRC-64/NVME of the new object of a crc64 cursor, once the last window is rewritten. */
    public long objectCrc64() {
        return crc64(1);
    }

    /** The CRC-64/NVME of the decoded segment of a crc64 cursor, once the last window is rewritten. */
    public long segmentCrc64() {
        return crc64(2);
    }

    private long crc64(final int k) {
        if (crcs64 == null) {
            throw new IllegalStateException("this cursor computes CRC-32C: construct it with crc64 = true");
        }
        if (!ended) {
            throw new IllegalStateException("the object's last window has not been rewritten yet");
        }
        return crcs64.getLong(8 * k);
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
