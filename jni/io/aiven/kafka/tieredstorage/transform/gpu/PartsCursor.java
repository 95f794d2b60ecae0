package io.aiven.kafka.tieredstorage.transform.gpu;

import java.nio.ByteBuffer;
import java.nio.ByteOrder;

/**
 * The upload-part checksum state of ONE object between the windows it is transformed in (tsgpu_parts_cursor of
 * include/tsgpu.h): part k is bytes [k * partSize, (k + 1) * partSize) of the transformed object, and a part may start in one
 * window and end in a later one.  Each window goes through tsgpu_transform_parts, which hashes the bytes it copies out on the
 * GPU; the CRC-32C of every part the window completes is kept here, and on the last window the CRC-32C of the whole object.
 * A storage backend sends them with the parts (S3 x-amz-checksum-crc32c, GCS crc32c), so the object store refuses a part
 * that changed after it left the GPU.  Constructed with crc64 = true, the windows go through tsgpu_transform_parts_crc64
 * (Crc64.transformParts) instead and partCrc64 / objectCrc64 give CRC-64/NVME (S3 CRC64NVME, Azure x-ms-content-crc64).
 */
public final class PartsCursor {
    public static final int SIZE = 32;
    private final ByteBuffer state = ByteBuffer.allocateDirect(SIZE);    // zeros: the start of an object
    private final long partSize;
    private int[] crcs = new int[16];
    private int parts = 0;
    private Integer objectCrc32c = null;
    private final boolean crc64;
    private long[] crcs64 = new long[16];
    private Long objectCrc64 = null;

    public PartsCursor(final long partSize) {
        this(partSize, false);
    }

    /** crc64: CRC-64/NVME part and object checksums instead of CRC-32C; one cursor carries one width. */
    public PartsCursor(final long partSize, final boolean crc64) {
        if (partSize < 1) {
            throw new IllegalArgumentException("partSize must be positive, " + partSize + " given");
        }
        this.partSize = partSize;
        this.crc64 = crc64;
    }

    /** One window of the segment, as {@link RecordsCursor#transform} (the record cursor is shared); returns the number of chunks. */
    public int transform(final long ctx, final int flags, final ByteBuffer src, final long srcLen, final int chunkSize,
                         final byte[] key, final byte[] aad, final byte[] ivs, final ByteBuffer dst, final int[] transformedSizes,
                         final RecordsCursor records, final boolean segmentEndsHere) {
        // the open part carried in is shorter than partSize: this is at least the bound include/tsgpu.h gives for part_cap
        final long bound = srcLen > 0 ? TsGpu.transformBound(flags, srcLen, chunkSize) : 0;
        final int cap = (int) Math.min(Integer.MAX_VALUE - 8, (partSize - 1 + bound) / partSize + 1);
        if (crc64) {
            return transform64(ctx, flags, src, srcLen, chunkSize, key, aad, ivs, dst, transformedSizes, records, segmentEndsHere, cap);
        }
        final int[] out = new int[cap];
        final int[] counts = new int[2];
        final int n = transformParts(ctx, flags, src, srcLen, chunkSize, key, aad, ivs, dst, transformedSizes, records.buffer(),
            segmentEndsHere, partSize, state, out, counts);
        if (parts + counts[0] > crcs.length) {
            crcs = java.util.Arrays.copyOf(crcs, Math.max(2 * crcs.length, parts + counts[0]));
        }
        System.arraycopy(out, 0, crcs, parts, counts[0]);
        parts += counts[0];
        if (segmentEndsHere) {
            objectCrc32c = counts[1];
        }
        return n;
    }

    private int transform64(final long ctx, final int flags, final ByteBuffer src, final long srcLen, final int chunkSize,
                            final byte[] key, final byte[] aad, final byte[] ivs, final ByteBuffer dst, final int[] transformedSizes,
                            final RecordsCursor records, final boolean segmentEndsHere, final int cap) {
        final ByteBuffer out = ByteBuffer.allocateDirect(8 * cap).order(ByteOrder.nativeOrder());
        final ByteBuffer obj = ByteBuffer.allocateDirect(8).order(ByteOrder.nativeOrder());
        final int[] count = new int[1];
        final int n = Crc64.transformParts(ctx, flags, src, srcLen, chunkSize, key, aad, ivs, dst, transformedSizes,
            records.buffer(), segmentEndsHere, partSize, state, out, count, obj);
        if (parts + count[0] > crcs64.length) {
            crcs64 = java.util.Arrays.copyOf(crcs64, Math.max(2 * crcs64.length, parts + count[0]));
        }
        for (int i = 0; i < count[0]; i++) {
            crcs64[parts + i] = out.getLong(8 * i);
        }
        parts += count[0];
        if (segmentEndsHere) {
            objectCrc64 = obj.getLong(0);
        }
        return n;
    }

    /** The CRC-64/NVME of part partNumber (1-based) of a crc64 cursor, once the window that ends it is transformed. */
    public long partCrc64(final int partNumber) {
        if (!crc64) {
            throw new IllegalStateException("this cursor computes CRC-32C: construct it with crc64 = true");
        }
        if (partNumber < 1 || partNumber > parts) {
            throw new IllegalStateException("part " + partNumber + " has not been transformed yet (" + parts + " are)");
        }
        return crcs64[partNumber - 1];
    }

    /** The CRC-64/NVME of the whole object of a crc64 cursor, once its last window is transformed. */
    public long objectCrc64() {
        if (objectCrc64 == null) {
            throw new IllegalStateException(crc64 ? "the object's last window has not been transformed yet"
                : "this cursor computes CRC-32C: construct it with crc64 = true");
        }
        return objectCrc64;
    }

    /** The CRC-32C of part partNumber (1-based, as UploadPart numbers parts), once the window that ends it is transformed. */
    public int partCrc32c(final int partNumber) {
        if (partNumber < 1 || partNumber > parts) {
            throw new IllegalStateException("part " + partNumber + " has not been transformed yet (" + parts + " are)");
        }
        return crcs[partNumber - 1];
    }

    /** The CRC-32C of the whole object, once its last window is transformed. */
    public int objectCrc32c() {
        if (objectCrc32c == null) {
            throw new IllegalStateException("the object's last window has not been transformed yet");
        }
        return objectCrc32c;
    }

    static {
        System.loadLibrary("tsgpu_jni");
    }

    public static native int transformParts(long ctx, int flags, ByteBuffer src, long srcLen, int chunkSize, byte[] key, byte[] aad,
                                            byte[] ivs, ByteBuffer dst, int[] transformedSizes, ByteBuffer recordsCursor,
                                            boolean segmentEndsHere, long partSize, ByteBuffer partsCursor, int[] partCrc32c,
                                            int[] partsOut);
}
