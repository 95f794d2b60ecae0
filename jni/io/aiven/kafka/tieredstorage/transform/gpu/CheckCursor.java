package io.aiven.kafka.tieredstorage.transform.gpu;

import java.nio.ByteBuffer;
import java.nio.ByteOrder;

/**
 * The state of ONE stored .log object while it is checked on the GPU in windows of chunks (tsgpu_check_cursor of
 * include/tsgpu.h): chunks and bytes so far, the running CRC-32C of the object and of the decoded segment, and the record
 * validation state of an entry that crosses a window.  Each window goes through tsgpu_check_object, which decrypts, decodes and
 * checks it against the manifest's chunk index without copying any plaintext back.  After the last window, objectCrc32c() is
 * compared with the object store's checksum (S3 FULL_OBJECT, GCS crc32c, or the one recorded at upload) and segmentCrc32c() with
 * the local segment file before it is deleted.  A failed window throws RuntimeException (IllegalArgumentException for arguments)
 * with the library's message, and the cursor is then spent.  Constructed with crc64 = true, the
 * windows go through tsgpu_check_object_crc64 (Crc64.checkObject) and objectCrc64 / segmentCrc64 give CRC-64/NVME (S3's
 * CRC64NVME full-object checksum).
 */
public final class CheckCursor {
    public static final int SIZE = 128;
    private final ByteBuffer state = ByteBuffer.allocateDirect(SIZE);    // zeros: the start of an object
    private final int[] crcs = new int[2];
    private boolean ended = false;
    private final ByteBuffer crcs64;                                       // null for CRC-32C

    public CheckCursor() {
        this(false);
    }

    /** crc64: CRC-64/NVME object and segment checksums instead of CRC-32C; one cursor carries one width. */
    public CheckCursor(final boolean crc64) {
        crcs64 = crc64 ? ByteBuffer.allocateDirect(16).order(ByteOrder.nativeOrder()) : null;
    }

    /**
     * One window: transformed chunks transformedSizes back to back in src.  flags are the manifest's (TsGpu.FLAG_ZSTD,
     * TsGpu.FLAG_AES), plus TsGpu.FLAG_VALIDATE_RECORDS to check every record batch; key and aad are null without encryption.
     */
    public void check(final long ctx, final int flags, final ByteBuffer src, final long srcLen, final int[] transformedSizes,
                      final int originalChunkSize, final long originalFileSize, final byte[] key, final byte[] aad,
                      final boolean objectEndsHere) {
        if (ended) {
            throw new IllegalStateException("the object's last window has already been checked");
        }
        if (crcs64 != null) {
            Crc64.checkObject(ctx, flags, src, srcLen, transformedSizes, originalChunkSize, originalFileSize, key, aad, state,
                objectEndsHere, crcs64);
        } else {
            checkObject(ctx, flags, src, srcLen, transformedSizes, originalChunkSize, originalFileSize, key, aad, state,
                objectEndsHere, crcs);
        }
        ended = objectEndsHere;
    }

    /** The CRC-32C of the whole object, once its last window is checked. */
    public int objectCrc32c() {
        if (!ended) {
            throw new IllegalStateException("the object's last window has not been checked yet");
        }
        return crcs[0];
    }

    /** The CRC-32C of the decoded segment, once the object's last window is checked. */
    public int segmentCrc32c() {
        if (!ended) {
            throw new IllegalStateException("the object's last window has not been checked yet");
        }
        return crcs[1];
    }

    /** The CRC-64/NVME of the whole object of a crc64 cursor, once its last window is checked. */
    public long objectCrc64() {
        return crc64(0);
    }

    /** The CRC-64/NVME of the decoded segment of a crc64 cursor, once the object's last window is checked. */
    public long segmentCrc64() {
        return crc64(1);
    }

    private long crc64(final int k) {
        if (crcs64 == null) {
            throw new IllegalStateException("this cursor computes CRC-32C: construct it with crc64 = true");
        }
        if (!ended) {
            throw new IllegalStateException("the object's last window has not been checked yet");
        }
        return crcs64.getLong(8 * k);
    }

    static {
        System.loadLibrary("tsgpu_jni");
    }

    public static native void checkObject(long ctx, int flags, ByteBuffer src, long srcLen, int[] transformedSizes,
                                          int originalChunkSize, long originalFileSize, byte[] key, byte[] aad, ByteBuffer cursor,
                                          boolean objectEndsHere, int[] crcsOut);
}
