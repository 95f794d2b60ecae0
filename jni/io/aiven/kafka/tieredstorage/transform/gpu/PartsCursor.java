package io.aiven.kafka.tieredstorage.transform.gpu;

import java.nio.ByteBuffer;

/**
 * The upload-part checksum state of ONE object between the windows it is transformed in (tsgpu_parts_cursor of
 * include/tsgpu.h): part k is bytes [k * partSize, (k + 1) * partSize) of the transformed object, and a part may start in one
 * window and end in a later one.  Each window goes through tsgpu_transform_parts, which hashes the bytes it copies out on the
 * GPU; the CRC-32C of every part the window completes is kept here, and on the last window the CRC-32C of the whole object.
 * A storage backend sends them with the parts (S3 x-amz-checksum-crc32c, GCS crc32c), so the object store refuses a part
 * that changed after it left the GPU.
 */
public final class PartsCursor {
    public static final int SIZE = 32;
    private final ByteBuffer state = ByteBuffer.allocateDirect(SIZE);    // zeros: the start of an object
    private final long partSize;
    private int[] crcs = new int[16];
    private int parts = 0;
    private Integer objectCrc32c = null;

    public PartsCursor(final long partSize) {
        if (partSize < 1) {
            throw new IllegalArgumentException("partSize must be positive, " + partSize + " given");
        }
        this.partSize = partSize;
    }

    /** One window of the segment, as {@link RecordsCursor#transform} (the record cursor is shared); returns the number of chunks. */
    public int transform(final long ctx, final int flags, final ByteBuffer src, final long srcLen, final int chunkSize,
                         final byte[] key, final byte[] aad, final byte[] ivs, final ByteBuffer dst, final int[] transformedSizes,
                         final RecordsCursor records, final boolean segmentEndsHere) {
        // the open part carried in is shorter than partSize: this is at least the bound include/tsgpu.h gives for part_cap
        final long bound = srcLen > 0 ? TsGpu.transformBound(flags, srcLen, chunkSize) : 0;
        final int cap = (int) Math.min(Integer.MAX_VALUE - 8, (partSize - 1 + bound) / partSize + 1);
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
