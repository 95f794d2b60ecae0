package io.aiven.kafka.tieredstorage.transform.gpu;

import java.nio.ByteBuffer;
import java.nio.ByteOrder;

/**
 * The state of ONE stored unencrypted object (a segment's .log object, or its .indexes object) while its chunks are encrypted on
 * the GPU in windows of chunks (tsgpu_encrypt_cursor of include/tsgpu.h): the chunk count, the running CRC-32C of the old object
 * and the new object's open upload part.  Each window goes through tsgpu_encrypt_object, which encrypts every chunk as it is, frame
 * or plain chunk, with nothing decoded: the window's new chunks (IV || CT || TAG, 28 bytes longer; an empty chunk stays empty)
 * land in dst with their sizes in newSizes, and the CRC-32C of every upload part they complete is returned.  A .log object's
 * chunks are checked against its chunk index (originalChunkSize, originalFileSize), and with FLAG_ZSTD every frame's header and
 * block walk; an .indexes object passes originalChunkSize 0.  After the last window, sourceCrc32c() is compared with the store's
 * checksum of the old object and objectCrc32c() completes the upload (S3 FULL_OBJECT, GCS crc32c).  A failed window throws
 * RuntimeException (IllegalArgumentException for arguments, among them a reused IV) with the library's message, and the cursor is
 * then spent.  Constructed with crc64 = true, the windows go through tsgpu_encrypt_object_crc64: {@link #encrypt64} returns the
 * parts' CRC-64/NVME, and sourceCrc64 / objectCrc64 the object words.
 */
public final class EncryptCursor {
    public static final int SIZE = 64;
    private final ByteBuffer state = ByteBuffer.allocateDirect(SIZE);    // zeros: the start of an object
    private final int[] crcs = new int[2];
    private final int[] nParts = new int[1];
    private boolean ended = false;
    private final ByteBuffer crcs64;                                       // null for CRC-32C

    public EncryptCursor() {
        this(false);
    }

    /** crc64: CRC-64/NVME part, source and object checksums instead of CRC-32C; one cursor carries one width. */
    public EncryptCursor(final boolean crc64) {
        crcs64 = crc64 ? ByteBuffer.allocateDirect(16).order(ByteOrder.nativeOrder()) : null;
    }

    /**
     * One window: chunks of chunkSizes back to back in src.  flags: TsGpu.FLAG_ZSTD for a compressed object, TsGpu.FLAG_VERIFY.
     * ivs holds 12 bytes per chunk of the window (an empty chunk takes none; its 12 bytes are not read).  dst receives exactly the
     * window's new bytes, newSizes (one int per chunk) their sizes; partCrcs the CRC-32C of the parts the window completes (its
     * length is part_cap); returns their count.
     */
    public int encrypt(final long ctx, final int flags, final ByteBuffer src, final long srcLen, final int[] chunkSizes,
                       final int originalChunkSize, final long originalFileSize, final byte[] key, final byte[] aad,
                       final byte[] ivs, final ByteBuffer dst, final long dstCap, final int[] newSizes, final long partSize,
                       final int[] partCrcs, final boolean objectEndsHere) {
        if (ended) {
            throw new IllegalStateException("the object's last window has already been encrypted");
        }
        if (crcs64 != null) {
            throw new IllegalStateException("this cursor computes CRC-64/NVME: call encrypt64");
        }
        encryptObject(ctx, flags, src, srcLen, chunkSizes, originalChunkSize, originalFileSize, key, aad, ivs, dst, dstCap,
            newSizes, partSize, partCrcs, nParts, state, objectEndsHere, crcs);
        ended = objectEndsHere;
        return nParts[0];
    }

    /**
     * {@link #encrypt} for a crc64 cursor: partCrc64 receives the CRC-64/NVME of the parts the window completes (its length is
     * part_cap); returns their count.
     */
    public int encrypt64(final long ctx, final int flags, final ByteBuffer src, final long srcLen, final int[] chunkSizes,
                         final int originalChunkSize, final long originalFileSize, final byte[] key, final byte[] aad,
                         final byte[] ivs, final ByteBuffer dst, final long dstCap, final int[] newSizes, final long partSize,
                         final long[] partCrc64, final boolean objectEndsHere) {
        if (crcs64 == null) {
            throw new IllegalStateException("this cursor computes CRC-32C: construct it with crc64 = true");
        }
        if (ended) {
            throw new IllegalStateException("the object's last window has already been encrypted");
        }
        final ByteBuffer out = ByteBuffer.allocateDirect(8 * partCrc64.length).order(ByteOrder.nativeOrder());
        encryptObjectCrc64(ctx, flags, src, srcLen, chunkSizes, originalChunkSize, originalFileSize, key, aad, ivs, dst, dstCap,
            newSizes, partSize, out, nParts, state, objectEndsHere, crcs64);
        for (int i = 0; i < nParts[0]; i++) {
            partCrc64[i] = out.getLong(8 * i);
        }
        ended = objectEndsHere;
        return nParts[0];
    }

    /** The CRC-64/NVME of the old object of a crc64 cursor, once the last window is encrypted. */
    public long sourceCrc64() {
        return crc64(0);
    }

    /** The CRC-64/NVME of the new object of a crc64 cursor, once the last window is encrypted. */
    public long objectCrc64() {
        return crc64(1);
    }

    private long crc64(final int k) {
        if (crcs64 == null) {
            throw new IllegalStateException("this cursor computes CRC-32C: construct it with crc64 = true");
        }
        if (!ended) {
            throw new IllegalStateException("the object's last window has not been encrypted yet");
        }
        return crcs64.getLong(8 * k);
    }

    /** The CRC-32C of the old object, once the last window is encrypted. */
    public int sourceCrc32c() {
        return crc(0);
    }

    /** The CRC-32C of the new object, once the last window is encrypted. */
    public int objectCrc32c() {
        return crc(1);
    }

    private int crc(final int k) {
        if (crcs64 != null) {
            throw new IllegalStateException("this cursor computes CRC-64/NVME: call sourceCrc64 / objectCrc64");
        }
        if (!ended) {
            throw new IllegalStateException("the object's last window has not been encrypted yet");
        }
        return crcs[k];
    }

    static {
        System.loadLibrary("tsgpu_jni");
    }

    public static native void encryptObject(long ctx, int flags, ByteBuffer src, long srcLen, int[] chunkSizes,
                                            int originalChunkSize, long originalFileSize, byte[] key, byte[] aad, byte[] ivs,
                                            ByteBuffer dst, long dstCap, int[] newSizes, long partSize, int[] partCrcs,
                                            int[] nPartsOut, ByteBuffer cursor, boolean objectEndsHere, int[] crcsOut);

    public static native void encryptObjectCrc64(long ctx, int flags, ByteBuffer src, long srcLen, int[] chunkSizes,
                                                 int originalChunkSize, long originalFileSize, byte[] key, byte[] aad, byte[] ivs,
                                                 ByteBuffer dst, long dstCap, int[] newSizes, long partSize, ByteBuffer partCrc64,
                                                 int[] nPartsOut, ByteBuffer cursor, boolean objectEndsHere, ByteBuffer crcsOut);
}
