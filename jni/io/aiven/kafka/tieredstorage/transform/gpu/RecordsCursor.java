package io.aiven.kafka.tieredstorage.transform.gpu;

import java.nio.ByteBuffer;

/**
 * The record-validation state of ONE segment between the windows it is transformed in (tsgpu_records_cursor of
 * include/tsgpu.h): a record batch may start in one window and end in a later one.  A new cursor is the start of a
 * segment; {@link #transform} continues where the previous window ended and updates the cursor.  Validation runs when the
 * flags carry {@link TsGpu#FLAG_VALIDATE_RECORDS}, or when TSGPU_VALIDATE_RECORDS=1 is set in the broker's environment;
 * otherwise the cursor is not used and the call is TsGpu.transform.
 */
public final class RecordsCursor {
    public static final int SIZE = 64;
    private final ByteBuffer state = ByteBuffer.allocateDirect(SIZE);    // zeros: the start of a segment

    /** One window of the segment; segmentEndsHere on its last (short or empty) window.  Returns the number of chunks. */
    public int transform(final long ctx, final int flags, final ByteBuffer src, final long srcLen, final int chunkSize,
                         final byte[] key, final byte[] aad, final byte[] ivs, final ByteBuffer dst, final int[] transformedSizes,
                         final boolean segmentEndsHere) {
        return transformCursor(ctx, flags, src, srcLen, chunkSize, key, aad, ivs, dst, transformedSizes, state, segmentEndsHere);
    }

    /** The cursor's direct buffer, for PartsCursor.transformParts, which continues the same segment. */
    ByteBuffer buffer() {
        return state;
    }

    static {
        System.loadLibrary("tsgpu_jni");
    }

    public static native int transformCursor(long ctx, int flags, ByteBuffer src, long srcLen, int chunkSize, byte[] key, byte[] aad,
                                             byte[] ivs, ByteBuffer dst, int[] transformedSizes, ByteBuffer cursor,
                                             boolean segmentEndsHere);
}
