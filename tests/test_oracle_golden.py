"""Pins the CPU oracle on every golden vector / exact expectation the reference's own tests hold for the
hot path (SURVEY.md §8c).  Citations: core/T = <reference>/core/src/test/java/io/aiven/kafka/tieredstorage."""
import base64

import numpy as np
import pytest

from oracle import oracle as ora

# core/T/manifest/index/ChunkIndexSerializationTest.java:39-74
ENCODED_CHUNKS = "KLUv/SAPeQAAAAAAAwAAAAoBAAoAAAAe"
FIXED_JSON = ('{"type":"fixed","originalChunkSize":100,"originalFileSize":250,'
              '"transformedChunkSize":110,"finalTransformedChunkSize":30}')
VARIABLE_JSON = ('{"type":"variable","originalChunkSize":100,"originalFileSize":250,'
                 '"transformedChunks":"' + ENCODED_CHUNKS + '"}')


def test_encoded_chunks_golden_vector():
    # codec bytes 00000003 0000000a 01 00 0a 0000001e, then zstd(contentSize) then Base64
    assert ora.codec_encode([10, 20, 30]) == bytes.fromhex("000000030000000a01000a0000001e")
    assert ora.transformed_chunks_serialize([10, 20, 30]) == ENCODED_CHUNKS
    assert ora.transformed_chunks_deserialize(ENCODED_CHUNKS) == [10, 20, 30]
    frame = base64.b64decode(ENCODED_CHUNKS)
    assert frame[:4] == bytes.fromhex("28b52ffd") and frame[4] == 0x20 and frame[5] == 15
    assert ora.zstd_content_size(frame) == 15


def test_chunk_index_json_golden():
    assert ora.ChunkIndex.fixed(100, 250, 110, 30).to_json() == FIXED_JSON
    assert ora.ChunkIndex.variable(100, 250, [10, 20, 30]).to_json() == VARIABLE_JSON


def test_chunk_index_materialized_chunks():
    # ChunkIndexSerializationTest.java:93-97, :118-122
    assert ora.ChunkIndex.fixed(100, 250, 110, 30).chunks() == [
        (0, 0, 100, 0, 110), (1, 100, 100, 110, 110), (2, 200, 50, 220, 30)]
    assert ora.ChunkIndex.variable(100, 250, [10, 20, 30]).chunks() == [
        (0, 0, 100, 0, 10), (1, 100, 100, 10, 20), (2, 200, 50, 30, 30)]


# core/T/manifest/index/serde/ChunkSizesBinaryCodecTest.java:34-118
INT_MAX = 2**31 - 1


@pytest.mark.parametrize("values,bpv", [
    ([0, 1000, 2, 44002, 369], 2),
    ([INT_MAX, INT_MAX - 1, INT_MAX - 2, 10], 1),
    ([INT_MAX // 2, INT_MAX // 2 - 1, INT_MAX // 2 - 2, 10], 1),
    ([1, 2, 3, INT_MAX], 1),
    ([1, 0xFF + 10, 0xFF + 20, 0xFF + 30, INT_MAX], 2),
    ([1, 0xFFFF + 10, 0xFFFF + 20, 0xFFFF + 30, INT_MAX], 3),
    ([1, 0xFFFFFF + 10, 0xFFFFFF + 20, 0xFFFFFF + 30, INT_MAX], 4),
    (list(range(0, INT_MAX - 2000, 1000))[:200000], 4),
    (list(range(0, INT_MAX - 2000, 1000))[:200000][::-1], 4),
])
def test_codec_multiple_values(values, bpv):
    enc = ora.codec_encode(values)
    assert len(enc) == 4 + 4 + 1 + (len(values) - 1) * bpv + 4
    assert int.from_bytes(enc[:4], "big") == len(values)
    assert enc[8] == bpv
    assert ora.codec_decode(enc) == values


@pytest.mark.parametrize("values", [[], [213], [INT_MAX]])
def test_codec_small(values):
    assert ora.codec_decode(ora.codec_encode(values)) == values


@pytest.mark.parametrize("values", [[-1], [-1, 2, 3], [1, -2, 3], [1, 2, -3]])
def test_codec_negative(values):
    with pytest.raises(ora.OracleError, match="Values cannot be negative"):
        ora.codec_encode(values)


# core/T/manifest/index/ChunkIndexBuilderCommonTest.java:37-127 (both builder kinds)
@pytest.mark.parametrize("tcs", [None, 110])
def test_builder_state_machine(tcs):
    def mk(ocs=100, ofs=250):
        return ora.ChunkIndexBuilder(ocs, ofs, tcs)
    with pytest.raises(ora.OracleError, match="Original chunk size must be non-negative, -1 given"):
        mk(ocs=-1)
    with pytest.raises(ora.OracleError, match="Original file size must be non-negative, -1 given"):
        mk(ofs=-1)
    b = mk()
    with pytest.raises(ora.OracleError, match="Transformed chunk size must be non-negative, -1 given"):
        b.add_chunk(-1)
    b.add_chunk(110)
    b.add_chunk(110)
    with pytest.raises(ora.OracleError, match="This must be final chunk. Call `finish` instead."):
        b.add_chunk(110)
    b.finish(30)
    with pytest.raises(ora.OracleError, match="Cannot add chunk to already finished index"):
        b.add_chunk(110)
    with pytest.raises(ora.OracleError, match="Cannot finish already finished index"):
        b.finish(30)
    b = mk()
    b.add_chunk(110)
    with pytest.raises(ora.OracleError, match="This cannot be final chunk: not enough chunks to cover original file"):
        b.finish(30)
    # empty file: finish(0) gives the single zero chunk; every lookup is null
    idx = mk(ofs=0).finish(0)
    assert idx.chunks() == [(0, 0, 0, 0, 0)]
    assert idx.find_chunk_for_original_offset(0) is None
    # beyond EOF => null
    b = mk()
    b.add_chunk(110); b.add_chunk(110)
    idx = b.finish(30)
    assert idx.find_chunk_for_original_offset(250) is None
    assert idx.find_chunk_for_original_offset(249) is not None
    with pytest.raises(ora.OracleError, match="Offset must be non-negative, -1 given"):
        idx.find_chunk_for_original_offset(-1)


def test_fixed_builder_rejects_wrong_size():
    # core/T/manifest/index/FixedSizeChunkIndexBuilderTest.java:35-53
    b = ora.ChunkIndexBuilder(100, 250, 110)
    with pytest.raises(ora.OracleError, match="Non-final chunk must be of size 110, but 109 given"):
        b.add_chunk(109)


def test_three_chunks_fixed_and_every_offset():
    # FixedSizeChunkIndexBuilderTest.java:55-88
    b = ora.ChunkIndexBuilder(100, 250, 110)
    b.add_chunk(110); b.add_chunk(110)
    idx = b.finish(30)
    assert idx.chunks() == [(0, 0, 100, 0, 110), (1, 100, 100, 110, 110), (2, 200, 50, 220, 30)]
    for off in range(250):
        want = idx.chunks()[off // 100]
        assert idx.find_chunk_for_original_offset(off) == want


def test_three_chunks_variable_and_every_offset():
    # VariableSizeChunkIndexBuilderTest.java:45-81
    b = ora.ChunkIndexBuilder(100, 250, None)
    b.add_chunk(10); b.add_chunk(20)
    idx = b.finish(30)
    assert idx.chunks() == [(0, 0, 100, 0, 10), (1, 100, 100, 10, 20), (2, 200, 50, 30, 30)]
    for off in range(250):
        assert idx.find_chunk_for_original_offset(off) == idx.chunks()[off // 100]


def test_finisher_index_from_sizes():
    # core/T/transform/TransformFinisherTest.java:97-125: chunks {0,1,2},{3,4,5},{6}
    for tcs in (3, None):
        b = ora.ChunkIndexBuilder(3, 7, tcs)
        b.add_chunk(3); b.add_chunk(3)
        assert b.finish(1).chunks() == [(0, 0, 3, 0, 3), (1, 3, 3, 3, 3), (2, 6, 1, 6, 1)]


def test_fetch_plan_matches_fetch_chunk_enumeration():
    # core/T/fetch/FetchChunkEnumerationTest.java:105-145: chunk size 10, content "0123456789" per chunk
    idx = ora.ChunkIndex.fixed(10, 30, 10, 10)
    assert idx.fetch_plan(2, 4) == [(0, 2, 3)]                        # "234"
    assert idx.fetch_plan(5, 24) == [(0, 5, 5), (1, 0, 10), (2, 0, 5)]  # "56789" "0123456789" "01234"
    assert idx.fetch_plan(25, 1000) == [(2, 5, 5)]                    # end beyond EOF => last chunk, bounded by data
    with pytest.raises(ora.OracleError, match="Invalid start position 30"):
        idx.fetch_plan(30, 31)


# ---- AES-256-GCM: the GCM spec (McGrew/Viega) AES-256 test cases 13-16 pin both the OpenSSL stand-in and
# the plain-C SP 800-38D restatement
K0 = bytes(32)
K1 = bytes.fromhex("feffe9928665731c6d6a8f9467308308feffe9928665731c6d6a8f9467308308")
P15 = bytes.fromhex("d9313225f88406e5a55909c5aff5269a86a7a9531534f7da2e4c303d8a318a72"
                    "1c3c0c95956809532fcf0e2449a6b525b16aedf5aa0de657ba637b391aafd255")
C15 = bytes.fromhex("522dc1f099567d07f47f37a32a84427d643a8cdcbfe5c0c97598a2bd2555d1aa"
                    "8cb08e48590dbb3da7b08b1056828838c5f61e6393ba7a0abcc9f662898015ad")
IV1 = bytes.fromhex("cafebabefacedbaddecaf888")
A16 = bytes.fromhex("feedfacedeadbeeffeedfacedeadbeefabaddad2")
GCM_KATS = [
    (K0, bytes(12), b"", b"", b"", "530f8afbc74536b9a963b4f1c4cb738b"),
    (K0, bytes(12), b"", bytes(16), bytes.fromhex("cea7403d4d606b6e074ec5d3baf39d18"), "d0d1c8a799996bf0265b98b5d48ab919"),
    (K1, IV1, b"", P15, C15, "b094dac5d93471bdec1a502270e3cc6c"),
    (K1, IV1, A16, P15[:60], C15[:60], "76fc6ece0f4e1768cddf8853bb2d551b"),
]


@pytest.mark.parametrize("key,iv,aad,pt,ct,tag", GCM_KATS)
def test_aes256_gcm_kats(key, iv, aad, pt, ct, tag):
    out = ora.aesgcm_encrypt_chunk(key, iv, aad, pt)
    assert out == iv + ct + bytes.fromhex(tag)                      # IV || CT || TAG layout
    assert ora.aesgcm_plain_encrypt(key, iv, aad, pt) == (ct, bytes.fromhex(tag))
    assert ora.aesgcm_decrypt_chunk(key, aad, out) == pt
    bad = bytearray(out); bad[-1] ^= 1
    with pytest.raises(ora.OracleError) as e:
        ora.aesgcm_decrypt_chunk(key, aad, bytes(bad))
    assert e.value.code == ora.E_AUTH


def test_aes256_block_fips197():
    # FIPS-197 appendix C.3
    key = bytes(range(32))
    assert ora.aes256_encrypt_block(key, bytes.fromhex("00112233445566778899aabbccddeeff")) == \
        bytes.fromhex("8ea2b7ca516745bfeafc49904b496089")


def test_plain_gcm_matches_openssl_on_random():
    rng = np.random.default_rng(7)
    for n in [0, 1, 15, 16, 17, 31, 32, 33, 1000, 4097]:
        key = rng.bytes(32); iv = rng.bytes(12); aad = rng.bytes(32); pt = rng.bytes(n)
        out = ora.aesgcm_encrypt_chunk(key, iv, aad, pt)
        ct, tag = ora.aesgcm_plain_encrypt(key, iv, aad, pt)
        assert out == iv + ct + tag


# ---- chains: TransformsEndToEndTest.java:44-116 grid on the oracle itself (round trip)
@pytest.mark.parametrize("flags", [0, ora.FLAG_AES, ora.FLAG_ZSTD, ora.FLAG_ZSTD | ora.FLAG_AES])
@pytest.mark.parametrize("chunk_size", [0, 1, 2, 3, 5, 13, 1024, 2048, 5123, 181200 - 1, 181200 * 2])
def test_oracle_round_trip_grid(flags, chunk_size):
    n = 181200                       # reference uses 1,812,004 random bytes; a tenth keeps chunk_size=1 quick
    if chunk_size in (1, 2, 3, 5) and flags:
        n = 4000
    rng = np.random.default_rng(1234)
    src = rng.integers(0, 256, n, dtype=np.uint8)
    key, aad = rng.bytes(32), rng.bytes(32)
    nch = (n + chunk_size - 1) // chunk_size if chunk_size else 1
    ivs = rng.bytes(12 * nch)
    t, sizes = ora.transform_segment(flags, src, chunk_size, key, aad, ivs)
    assert len(sizes) == nch
    if flags == ora.FLAG_AES:
        cs = chunk_size if chunk_size else n
        assert all(s == min(cs, n - i * cs) + 28 for i, s in enumerate(sizes))
    back, osz = ora.detransform_chunks(flags, t, sizes, n, key, aad)
    assert np.array_equal(back, src)
