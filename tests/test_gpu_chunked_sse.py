"""Streaming-signed bodies of encrypted buckets on the device (mec_encode_chunked_sse): part files byte-equal to mec_encode_sse of the
de-framed plaintext at every length class, aws-chunk size and pipeline-chunk cut; the data shards open with an independent AES-GCM
and through mec_decode_sse; every damaged body gets the same code as from mec_encode_chunked and the serial reader of
tests/sigv4_ref.py; "checksums" equals the host CRCs of the plaintext; and no key material is left in the codec."""
import numpy as np
import pytest

import dare_ref as dref
import minio_b200 as mb
import sigv4_ref as ref
from test_gpu_chunked import TRAILER, tamper_cases, trailer_cases

pytestmark = pytest.mark.gpu

KiB, MiB = 1 << 10, 1 << 20
PKG, EPKG = dref.PKG, dref.EPKG
KEY = ref.signing_key("wJalrXUtnFEMI/K7MDENG/bPxRfiCYEXAMPLEKEY")
SEED = b"4f232c4386841ef735655705268965c44a0e4690baa4adea153f7db9fa80a0a9"
SCOPE = ref.scope_of()
SSE_KEY, NONCE = bytes(range(32)), bytes.fromhex("0123456789abcdeffedcba98")


def rnd(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def plain_len(enc):
    """the plaintext length whose DARE stream is `enc` bytes long (None: no stream is)"""
    q, r = divmod(enc, EPKG)
    if r == 0:
        return q * PKG
    return q * PKG + r - 32 if r > 32 else None


def lengths():
    out = {0, 1}
    for n in (1, 2, 16):
        out |= {n * PKG - 1, n * PKG, n * PKG + 1}
    for b in (1, 2, 3):  # ciphertext at erasure-block boundaries +- 1
        out |= {d for d in (plain_len(b * MiB - 1), plain_len(b * MiB), plain_len(b * MiB + 1)) if d is not None}
    return sorted(out)


def sizes_of(D, csize):
    return [min(csize, D - o) for o in range(0, D, csize)]


def same(got, want):
    return len(got) == len(want) and all((a is None and b is None) or np.array_equal(a, b) for a, b in zip(got, want))


@pytest.mark.parametrize("k,m", [(4, 2), (12, 4), (8, 8)])
def test_matches_encode_sse(oracle, k, m):
    """part files == mec_encode_sse of the plaintext; checksums == host CRCs; counters advance as the parent calls advance them"""
    c = mb.Codec(k, m, MiB)
    c.set_option("checksums", 7)
    for i, D in enumerate(lengths()):
        data = rnd(D, 100 * k + i)
        c.set_option("chunk_blocks", 0)
        s0 = c.stat("dare_sealed")
        want = c.encode_sse(data, SSE_KEY, NONCE)
        sealed = c.stat("dare_sealed") - s0
        for j, csize in enumerate((8 * KiB, 64 * KiB, 65537, MiB)):
            tr = TRAILER if (i + j) % 2 else None
            body = ref.build(data, sizes_of(D, csize), KEY, SEED, trailer=tr).data
            for cb in (0, 1, 2):
                c.set_option("chunk_blocks", cb)
                r0, s1 = c.stat("sigv4_chunks"), c.stat("dare_sealed")
                if tr is None:
                    got = c.encode_chunked_sse(body, D, KEY, SEED, ref.DATE, SCOPE, SSE_KEY, NONCE)
                else:
                    got, val = c.encode_chunked_sse(body, D, KEY, SEED, ref.DATE, SCOPE, SSE_KEY, NONCE, trailer=True)
                    assert val == tr + b"\n"
                assert same(got, want), (k, m, D, csize, cb)
                assert c.last_checksums() == (oracle.crcs(data), D), (D, csize, cb)
                assert c.stat("sigv4_chunks") - r0 == len(sizes_of(D, csize)) + 1 + (tr is not None)
                if cb == 0:
                    assert c.stat("dare_sealed") - s1 == sealed
                assert c.stat("sigv4_key_bytes") == 0
    c.close()


def test_offline_writers_down_to_quorum():
    k, m = 12, 4
    c = mb.Codec(k, m, MiB)
    c.set_option("chunk_blocks", 1)
    D = 3 * MiB + 12345
    data = rnd(D, 7)
    body = ref.build(data, sizes_of(D, 64 * KiB), KEY, SEED).data
    for off in (0, 1, m):
        online = [i >= off for i in range(k + m)]
        want = c.encode_sse(data, SSE_KEY, NONCE, online=online, write_quorum=k)
        got = c.encode_chunked_sse(body, D, KEY, SEED, ref.DATE, SCOPE, SSE_KEY, NONCE, online=online, write_quorum=k)
        assert same(got, want) and sum(f is None for f in got) == off
    online = [i > m for i in range(k + m)]
    with pytest.raises(mb.MecError) as ei:
        c.encode_chunked_sse(body, D, KEY, SEED, ref.DATE, SCOPE, SSE_KEY, NONCE, online=online, write_quorum=k)
    assert ei.value.code == -11
    c.close()


@pytest.mark.parametrize("D,csize,cb", [(5 * MiB + 333, 64 * KiB, 1), (2 * MiB, 65537, 0), (65536, 8 * KiB, 1)])
def test_opens_independently(oracle, D, csize, cb):
    """the data shards hold a DARE stream that AES-GCM (`cryptography`) opens to the payload; mec_decode_sse reads it back"""
    pytest.importorskip("cryptography")
    k, m = 12, 4
    c = mb.Codec(k, m, MiB)
    c.set_option("chunk_blocks", cb)
    data = rnd(D, D)
    body = ref.build(data, sizes_of(D, csize), KEY, SEED).data
    files = c.encode_chunked_sse(body, D, KEY, SEED, ref.DATE, SCOPE, SSE_KEY, NONCE)
    E = dref.encrypted_size(D)
    rc, ct, _ = oracle.erasure_decode(k, m, MiB, oracle.HIGHWAYHASH256S, files, [1] * (k + m), 0, E, E)
    assert rc >= 0
    assert dref.open_stream(SSE_KEY, ct.tobytes()) == data.tobytes()
    out, hint = c.decode_sse([None] * m + files[m:], 0, D, E, SSE_KEY)
    assert np.array_equal(out, data) and hint == 0
    c.close()


@pytest.fixture(scope="module")
def codec():
    c = mb.Codec(4, 2, 1 << 16)
    yield c
    c.close()


def _code(fn):
    try:
        fn()
    except mb.MecError as e:
        return e.code
    return ref.OK


@pytest.mark.parametrize("case", tamper_cases(), ids=lambda x: x[0])
def test_tampered_same_verdict(codec, case):
    name, body, D, _ = case
    want = ref.read(body, D, KEY, SEED)[0]
    assert want != ref.OK
    assert _code(lambda: codec.encode_chunked(body, D, KEY, SEED, ref.DATE, SCOPE)) == want, name
    assert _code(lambda: codec.encode_chunked_sse(body, D, KEY, SEED, ref.DATE, SCOPE, SSE_KEY, NONCE)) == want, name
    assert codec.stat("sigv4_key_bytes") == 0


@pytest.mark.parametrize("case", trailer_cases(), ids=lambda x: x[0])
def test_trailer_same_verdict(codec, case):
    name, body, D, _ = case
    want, out, val = ref.read(body, D, KEY, SEED, trailer=True)
    if want == ref.OK:
        files, got = codec.encode_chunked_sse(body, D, KEY, SEED, ref.DATE, SCOPE, SSE_KEY, NONCE, trailer=True)
        assert got == val
        assert same(files, codec.encode_sse(np.frombuffer(out, dtype=np.uint8), SSE_KEY, NONCE))
    else:
        assert _code(lambda: codec.encode_chunked(body, D, KEY, SEED, ref.DATE, SCOPE, trailer=True)) == want, name
        assert _code(lambda: codec.encode_chunked_sse(body, D, KEY, SEED, ref.DATE, SCOPE, SSE_KEY, NONCE, trailer=True)) == want, name
    assert codec.stat("sigv4_key_bytes") == 0


def test_wrong_credentials(codec):
    data = rnd(70000, 3)
    body = ref.build(data, [1000, 69000], KEY, SEED).data
    for args in ((ref.signing_key("other"), SEED, ref.DATE, SCOPE), (KEY, SEED[:-1] + b"0", ref.DATE, SCOPE),
                 (KEY, SEED, "20130524T000001Z", SCOPE), (KEY, SEED, ref.DATE, ref.scope_of(region="eu-west-1"))):
        assert ref.read(body, data.size, args[0], args[1], args[2], args[3])[0] == ref.SIGNATURE_MISMATCH
        assert _code(lambda: codec.encode_chunked_sse(body, data.size, *args, SSE_KEY, NONCE)) == ref.SIGNATURE_MISMATCH
        assert codec.stat("sigv4_key_bytes") == 0
    # a wrong SSE key is no signature matter: the call succeeds and the stream opens only with the key it was given
    other = bytes(32)
    files = codec.encode_chunked_sse(body, data.size, KEY, SEED, ref.DATE, SCOPE, other, NONCE)
    assert same(files, codec.encode_sse(data, other, NONCE))


def test_stops_at_the_first_failure(codec):
    """a signature failure in the last pipeline chunk of a many-chunk call: every row is still verified exactly once"""
    codec.set_option("chunk_blocks", 1)
    try:
        D = 4 * (1 << 16) + 100
        data = rnd(D, 9)
        sizes = sizes_of(D, 8 * KiB)
        b = ref.build(data, sizes, KEY, SEED)
        bad = bytearray(b.data)
        bad[b.chunks[-2]["payload"][0]] ^= 1
        r0 = codec.stat("sigv4_chunks")
        assert _code(lambda: codec.encode_chunked_sse(bytes(bad), D, KEY, SEED, ref.DATE, SCOPE, SSE_KEY, NONCE)) == ref.SIGNATURE_MISMATCH
        assert codec.stat("sigv4_chunks") - r0 == len(sizes) + 1
        r0 = codec.stat("sigv4_chunks")
        files = codec.encode_chunked_sse(b.data, D, KEY, SEED, ref.DATE, SCOPE, SSE_KEY, NONCE)
        assert codec.stat("sigv4_chunks") - r0 == len(sizes) + 1
        codec.set_option("chunk_blocks", 0)
        assert same(files, codec.encode_sse(data, SSE_KEY, NONCE))
    finally:
        codec.set_option("chunk_blocks", 0)
