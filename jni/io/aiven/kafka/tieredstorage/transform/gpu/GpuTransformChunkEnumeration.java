package io.aiven.kafka.tieredstorage.transform.gpu;

import java.io.IOException;
import java.io.InputStream;
import java.nio.ByteBuffer;
import java.nio.channels.Channels;
import java.nio.channels.ReadableByteChannel;
import java.security.SecureRandom;
import java.util.ArrayDeque;
import java.util.NoSuchElementException;

import io.aiven.kafka.tieredstorage.security.DataKeyAndAAD;
import io.aiven.kafka.tieredstorage.transform.TransformChunkEnumeration;

/**
 * Drop-in for the chain Base -> [Compression] -> [Encryption] built by RemoteStorageManager.transformation
 * (RemoteStorageManager.java:434-453): reads a batch of original chunks from the segment stream, transforms the
 * whole batch on the GPU with one native call and serves one byte[] per nextElement(), so TransformFinisher,
 * the ChunkIndex builders and the storage backends are unchanged.
 *
 * <p>The segment stream is read straight into a pinned direct buffer (no byte[] bounce in front of the H2D copy).
 * The two pinned staging buffers come from a per-context {@link PinnedPool} and go back to it when the stream is
 * exhausted, on {@link #close()}, or — as a last resort — when the enumeration is garbage collected.
 *
 * <p>One enumeration is one segment, so it keeps one {@link RecordsCursor} across its windows and marks the last (short
 * or empty) window: with record validation on (the validateRecords argument, or TSGPU_VALIDATE_RECORDS=1 in the
 * environment) a record batch that crosses a window is checked whole, and a segment that ends inside a batch fails.
 *
 * <p>With a partSize, every window also goes through tsgpu_transform_parts, which hashes the bytes it copies out on the GPU:
 * {@link #partCrc32c(int)} and {@link #objectCrc32c()} then give the CRC-32C of each upload part of the object and of the whole
 * object, for the storage backend to send with the parts (INTEGRATION.md).
 */
public class GpuTransformChunkEnumeration implements TransformChunkEnumeration, AutoCloseable {
    private final long ctx;
    private final InputStream inputStream;
    private final ReadableByteChannel channel;
    private final int originalChunkSize;
    private final int flags;
    private final DataKeyAndAAD keyAndAad;   // null when encryption is off
    private final int batchChunks;
    private final RecordsCursor records = new RecordsCursor();
    private final PartsCursor parts;                  // null without part checksums
    private final SecureRandom random = new SecureRandom();
    private final ArrayDeque<byte[]> ready = new ArrayDeque<>();
    private final PinnedPool pool;
    private PinnedPool.Lease src;
    private PinnedPool.Lease dst;
    private boolean eof = false;

    public GpuTransformChunkEnumeration(final long ctx, final PinnedPool pool, final InputStream inputStream,
                                        final int originalChunkSize, final boolean compression,
                                        final DataKeyAndAAD keyAndAad, final int batchChunks) {
        this(ctx, pool, inputStream, originalChunkSize, compression, keyAndAad, batchChunks, false);
    }

    public GpuTransformChunkEnumeration(final long ctx, final PinnedPool pool, final InputStream inputStream,
                                        final int originalChunkSize, final boolean compression,
                                        final DataKeyAndAAD keyAndAad, final int batchChunks, final boolean validateRecords) {
        this(ctx, pool, inputStream, originalChunkSize, compression, keyAndAad, batchChunks, validateRecords, 0);
    }

    /** validateRecords: check every record batch of the segment on the GPU (TsGpu.FLAG_VALIDATE_RECORDS); it applies when the
     *  segment is compressed or encrypted, otherwise the bytes are copied on the host and never reach the GPU.
     *  partSize: the storage backend's multipart part size; above 0 the CRC-32C of every part is computed on the GPU
     *  ({@link #partCrc32c(int)}), which needs compression or encryption for the same reason.  0 turns it off. */
    public GpuTransformChunkEnumeration(final long ctx, final PinnedPool pool, final InputStream inputStream,
                                        final int originalChunkSize, final boolean compression,
                                        final DataKeyAndAAD keyAndAad, final int batchChunks, final boolean validateRecords,
                                        final long partSize) {
        this(ctx, pool, inputStream, originalChunkSize, compression, keyAndAad, batchChunks, validateRecords, partSize, false);
    }

    /** crc64Parts: with a partSize, the CRC-64/NVME of every part and of the object ({@link #partCrc64(int)},
     *  {@link #objectCrc64()}; S3 CRC64NVME, Azure x-ms-content-crc64) instead of CRC-32C. */
    public GpuTransformChunkEnumeration(final long ctx, final PinnedPool pool, final InputStream inputStream,
                                        final int originalChunkSize, final boolean compression,
                                        final DataKeyAndAAD keyAndAad, final int batchChunks, final boolean validateRecords,
                                        final long partSize, final boolean crc64Parts) {
        if (inputStream == null) {
            throw new NullPointerException("inputStream cannot be null");
        }
        if (originalChunkSize < 0) {
            throw new IllegalArgumentException(
                "originalChunkSize must be non-negative, " + originalChunkSize + " given");   // BaseTransformChunkEnumeration.java:45-48
        }
        this.ctx = ctx;
        this.pool = pool;
        this.inputStream = inputStream;
        this.channel = Channels.newChannel(inputStream);
        this.originalChunkSize = originalChunkSize;
        final int transforms = (compression ? TsGpu.FLAG_ZSTD : 0) | (keyAndAad != null ? TsGpu.FLAG_AES : 0);
        this.flags = transforms | (validateRecords && transforms != 0 ? TsGpu.FLAG_VALIDATE_RECORDS : 0);
        if (partSize < 0 || (partSize > 0 && transforms == 0)) {
            throw new IllegalArgumentException("partSize must be 0, or positive with compression or encryption; " + partSize + " given");
        }
        this.parts = partSize <= 0 ? null : crc64Parts ? new PartsCursor(partSize, true) : new PartsCursor(partSize);
        this.keyAndAad = keyAndAad;
        this.batchChunks = batchChunks;
        if (originalChunkSize > 0) {
            final long batchBytes = (long) batchChunks * originalChunkSize;
            this.src = pool.lease(batchBytes);
            this.dst = pool.lease(TsGpu.transformBound(flags, batchBytes, originalChunkSize));
        }   // chunking disabled (size 0, BaseTransformChunkEnumeration.java:37-39): the buffers are sized once the stream has been read
    }

    @Override
    public int originalChunkSize() {
        return originalChunkSize;
    }

    @Override
    public Integer transformedChunkSize() {
        // Same arithmetic as the decorators: variable with compression, +28 with encryption only.
        if ((flags & TsGpu.FLAG_ZSTD) != 0) {
            return null;
        }
        return (flags & TsGpu.FLAG_AES) != 0 ? originalChunkSize + 28 : originalChunkSize;
    }

    /** The CRC-32C of upload part partNumber (1-based), valid once the window that ends that part has been transformed. */
    public int partCrc32c(final int partNumber) {
        if (parts == null) {
            throw new IllegalStateException("part checksums were not requested (partSize 0)");
        }
        return parts.partCrc32c(partNumber);
    }

    /** The CRC-32C of the whole object (S3 FULL_OBJECT, GCS crc32c), valid after the last window. */
    public int objectCrc32c() {
        if (parts == null) {
            throw new IllegalStateException("part checksums were not requested (partSize 0)");
        }
        return parts.objectCrc32c();
    }

    /** The CRC-64/NVME of upload part partNumber (1-based) with crc64Parts, valid once the window that ends it is transformed. */
    public long partCrc64(final int partNumber) {
        if (parts == null) {
            throw new IllegalStateException("part checksums were not requested (partSize 0)");
        }
        return parts.partCrc64(partNumber);
    }

    /** The CRC-64/NVME of the whole object (S3 FULL_OBJECT CRC64NVME) with crc64Parts, valid after the last window. */
    public long objectCrc64() {
        if (parts == null) {
            throw new IllegalStateException("part checksums were not requested (partSize 0)");
        }
        return parts.objectCrc64();
    }

    @Override
    public boolean hasMoreElements() {
        fill();
        return !ready.isEmpty();
    }

    @Override
    public byte[] nextElement() {
        fill();
        if (ready.isEmpty()) {
            throw new NoSuchElementException();
        }
        return ready.poll();
    }

    private void fill() {
        if (!ready.isEmpty() || eof) {
            return;
        }
        if (originalChunkSize == 0) {
            fillUnchunked();
            return;
        }
        try {
            final ByteBuffer in = src.buffer();
            in.clear();
            in.limit((int) Math.min(in.capacity(), (long) batchChunks * originalChunkSize));
            while (in.hasRemaining()) {                 // the stream lands directly in pinned memory
                if (channel.read(in) < 0) {
                    eof = true;
                    break;
                }
            }
            final long total = in.position();
            if (total == 0) {                            // the segment ended with the previous, full window
                if (parts == null) records.transform(ctx, flags, in, 0, originalChunkSize,
                    keyAndAad == null ? null : keyAndAad.dataKey.getEncoded(), keyAndAad == null ? null : keyAndAad.aad,
                    new byte[TsGpu.IV_SIZE], dst.buffer(), new int[0], true);
                else parts.transform(ctx, flags, in, 0, originalChunkSize,       // ... which also ends the last part
                    keyAndAad == null ? null : keyAndAad.dataKey.getEncoded(), keyAndAad == null ? null : keyAndAad.aad,
                    new byte[TsGpu.IV_SIZE], dst.buffer(), new int[0], records, true);
                release();
                return;
            }
            final int chunks = (int) ((total + originalChunkSize - 1) / originalChunkSize);
            if (total < (long) batchChunks * originalChunkSize) {
                eof = true;                              // a short batch ends the segment (BaseTransformChunkEnumeration:61-93)
            }
            final byte[] ivs = new byte[chunks * TsGpu.IV_SIZE];
            random.nextBytes(ivs);
            final int[] sizes = new int[chunks];
            final ByteBuffer out = dst.buffer();
            final int n = parts != null                 // with part checksums the window also hashes what it copies out
                ? parts.transform(ctx, flags, in, total, originalChunkSize,
                    keyAndAad == null ? null : keyAndAad.dataKey.getEncoded(), keyAndAad == null ? null : keyAndAad.aad,
                    ivs, out, sizes, records, eof)
                : records.transform(ctx, flags, in, total, originalChunkSize,
                    keyAndAad == null ? null : keyAndAad.dataKey.getEncoded(), keyAndAad == null ? null : keyAndAad.aad,
                    ivs, out, sizes, eof);
            out.clear();
            for (int i = 0; i < n; i++) {
                final byte[] chunk = new byte[sizes[i]];
                out.get(chunk);
                ready.add(chunk);
            }
            if (eof) {
                release();
            }
        } catch (final IOException e) {
            release();
            throw new RuntimeException(e);
        } catch (final RuntimeException e) {
            release();
            throw e;
        }
    }

    /** Chunking disabled: the whole stream is ONE chunk (readAllBytes in the reference, BaseTransformChunkEnumeration.java:84-88);
     *  an empty stream yields no element. */
    private void fillUnchunked() {
        eof = true;
        try {
            final byte[] all = inputStream.readAllBytes();
            if (all.length == 0) {
                if (parts != null) {                     // an empty object: no part, CRC 0
                    parts.transform(ctx, flags, ByteBuffer.allocateDirect(1), 0, 0,
                        keyAndAad == null ? null : keyAndAad.dataKey.getEncoded(), keyAndAad == null ? null : keyAndAad.aad,
                        new byte[TsGpu.IV_SIZE], ByteBuffer.allocateDirect(1), new int[0], records, true);
                }
                return;
            }
            src = pool.lease(all.length);
            dst = pool.lease(TsGpu.transformBound(flags, all.length, 0));
            final ByteBuffer in = src.buffer();
            in.clear();
            in.put(all);
            final byte[] ivs = new byte[TsGpu.IV_SIZE];
            random.nextBytes(ivs);
            final int[] sizes = new int[1];
            final ByteBuffer out = dst.buffer();
            final int n = parts != null
                ? parts.transform(ctx, flags, in, all.length, 0,
                    keyAndAad == null ? null : keyAndAad.dataKey.getEncoded(), keyAndAad == null ? null : keyAndAad.aad,
                    ivs, out, sizes, records, true)
                : records.transform(ctx, flags, in, all.length, 0,
                    keyAndAad == null ? null : keyAndAad.dataKey.getEncoded(), keyAndAad == null ? null : keyAndAad.aad,
                    ivs, out, sizes, true);
            out.clear();
            for (int i = 0; i < n; i++) {
                final byte[] chunk = new byte[sizes[i]];
                out.get(chunk);
                ready.add(chunk);
            }
        } catch (final IOException e) {
            throw new RuntimeException(e);
        } finally {
            release();
        }
    }

    private void release() {
        if (src != null) {
            src.close();
            src = null;
        }
        if (dst != null) {
            dst.close();
            dst = null;
        }
    }

    /** Returns the pinned staging buffers to the pool.  Idempotent; also called when the stream is exhausted. */
    @Override
    public void close() {
        eof = true;
        ready.clear();
        release();
    }
}
