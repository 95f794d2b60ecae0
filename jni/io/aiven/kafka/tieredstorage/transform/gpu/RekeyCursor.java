package io.aiven.kafka.tieredstorage.transform.gpu;

import java.nio.ByteBuffer;
import java.nio.ByteOrder;

/**
 * The state of ONE stored object (a segment's .log object, or its .indexes object) while its AES-GCM chunks are re-encrypted under
 * a new data key on the GPU in windows of chunks (tsgpu_rekey_cursor of include/tsgpu.h): the chunk count, the running CRC-32C of
 * the old object and the new object's open upload part.  Each window goes through tsgpu_rekey_object, which checks every old tag
 * and writes every chunk under the new key and IV with nothing decoded: the window's new chunks land in dst, each the size of its
 * old chunk, with the CRC-32C of every upload part they complete.  After the last window, sourceCrc32c() is compared with the
 * store's checksum of the old object and objectCrc32c() completes the upload (S3 FULL_OBJECT, GCS crc32c).  The chunk index and
 * SegmentIndexesV1 do not change; only the manifest's encryption metadata does.  A failed window throws RuntimeException
 * (IllegalArgumentException for arguments, among them an old chunk's IV reused under the same key) with the library's message,
 * and the cursor is then spent.  Constructed with crc64 = true, the windows go through tsgpu_rekey_object_crc64:
 * {@link #rekey64} returns the parts' CRC-64/NVME, and sourceCrc64 / objectCrc64 the object words.
 */
public final class RekeyCursor {
    public static final int SIZE = 64;
    private final ByteBuffer state = ByteBuffer.allocateDirect(SIZE);    // zeros: the start of an object
    private final int[] crcs = new int[2];
    private final int[] nParts = new int[1];
    private boolean ended = false;
    private final ByteBuffer crcs64;                                       // null for CRC-32C

    public RekeyCursor() {
        this(false);
    }

    /** crc64: CRC-64/NVME part, source and object checksums instead of CRC-32C; one cursor carries one width. */
    public RekeyCursor(final boolean crc64) {
        crcs64 = crc64 ? ByteBuffer.allocateDirect(16).order(ByteOrder.nativeOrder()) : null;
    }

    /**
     * One window: old chunks (IV || CT || TAG) transformedSizes back to back in src.  flags: 0 or TsGpu.FLAG_VERIFY.  toIvs holds
     * 12 bytes per chunk of the window (an empty chunk takes none; its 12 bytes are not read).  dst receives exactly the window's
     * bytes; partCrcs the CRC-32C of the parts the window completes (its length is part_cap); returns their count.
     */
    public int rekey(final long ctx, final int flags, final ByteBuffer src, final long srcLen, final int[] transformedSizes,
                     final byte[] fromKey, final byte[] fromAad, final byte[] toKey, final byte[] toAad, final byte[] toIvs,
                     final ByteBuffer dst, final long dstCap, final long partSize, final int[] partCrcs, final boolean objectEndsHere) {
        if (ended) {
            throw new IllegalStateException("the object's last window has already been rekeyed");
        }
        if (crcs64 != null) {
            throw new IllegalStateException("this cursor computes CRC-64/NVME: call rekey64");
        }
        rekeyObject(ctx, flags, src, srcLen, transformedSizes, fromKey, fromAad, toKey, toAad, toIvs, dst, dstCap, partSize,
            partCrcs, nParts, state, objectEndsHere, crcs);
        ended = objectEndsHere;
        return nParts[0];
    }

    /**
     * {@link #rekey} for a crc64 cursor: partCrc64 receives the CRC-64/NVME of the parts the window completes (its length is
     * part_cap); returns their count.
     */
    public int rekey64(final long ctx, final int flags, final ByteBuffer src, final long srcLen, final int[] transformedSizes,
                       final byte[] fromKey, final byte[] fromAad, final byte[] toKey, final byte[] toAad, final byte[] toIvs,
                       final ByteBuffer dst, final long dstCap, final long partSize, final long[] partCrc64,
                       final boolean objectEndsHere) {
        if (crcs64 == null) {
            throw new IllegalStateException("this cursor computes CRC-32C: construct it with crc64 = true");
        }
        if (ended) {
            throw new IllegalStateException("the object's last window has already been rekeyed");
        }
        final ByteBuffer out = ByteBuffer.allocateDirect(8 * partCrc64.length).order(ByteOrder.nativeOrder());
        rekeyObjectCrc64(ctx, flags, src, srcLen, transformedSizes, fromKey, fromAad, toKey, toAad, toIvs, dst, dstCap, partSize,
            out, nParts, state, objectEndsHere, crcs64);
        for (int i = 0; i < nParts[0]; i++) {
            partCrc64[i] = out.getLong(8 * i);
        }
        ended = objectEndsHere;
        return nParts[0];
    }

    /** The CRC-64/NVME of the old object of a crc64 cursor, once the last window is rekeyed. */
    public long sourceCrc64() {
        return crc64(0);
    }

    /** The CRC-64/NVME of the new object of a crc64 cursor, once the last window is rekeyed. */
    public long objectCrc64() {
        return crc64(1);
    }

    private long crc64(final int k) {
        if (crcs64 == null) {
            throw new IllegalStateException("this cursor computes CRC-32C: construct it with crc64 = true");
        }
        if (!ended) {
            throw new IllegalStateException("the object's last window has not been rekeyed yet");
        }
        return crcs64.getLong(8 * k);
    }

    /** The CRC-32C of the old object, once the last window is rekeyed. */
    public int sourceCrc32c() {
        return crc(0);
    }

    /** The CRC-32C of the new object, once the last window is rekeyed. */
    public int objectCrc32c() {
        return crc(1);
    }

    private int crc(final int k) {
        if (crcs64 != null) {
            throw new IllegalStateException("this cursor computes CRC-64/NVME: call sourceCrc64 / objectCrc64");
        }
        if (!ended) {
            throw new IllegalStateException("the object's last window has not been rekeyed yet");
        }
        return crcs[k];
    }

    static {
        System.loadLibrary("tsgpu_jni");
    }

    public static native void rekeyObject(long ctx, int flags, ByteBuffer src, long srcLen, int[] transformedSizes, byte[] fromKey,
                                          byte[] fromAad, byte[] toKey, byte[] toAad, byte[] toIvs, ByteBuffer dst, long dstCap,
                                          long partSize, int[] partCrcs, int[] nPartsOut, ByteBuffer cursor, boolean objectEndsHere,
                                          int[] crcsOut);

    public static native void rekeyObjectCrc64(long ctx, int flags, ByteBuffer src, long srcLen, int[] transformedSizes,
                                               byte[] fromKey, byte[] fromAad, byte[] toKey, byte[] toAad, byte[] toIvs,
                                               ByteBuffer dst, long dstCap, long partSize, ByteBuffer partCrc64, int[] nPartsOut,
                                               ByteBuffer cursor, boolean objectEndsHere, ByteBuffer crcsOut);
}
