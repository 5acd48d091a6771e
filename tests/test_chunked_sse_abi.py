"""CPU-side checks of mec_encode_chunked_sse (streaming-signed bodies of encrypted buckets): the binding's signature, and every
refusal in its order before any device work: mec_encode_chunked's argument checks plus a NULL SSE key or nonce, a decoded length no
DARE stream holds, the write quorum, and an error in the first chunk's header, which no signature precedes."""
import ctypes as C

import numpy as np
import pytest

import sigv4_ref as ref

INVALID_ARGUMENT, WRITE_QUORUM = -12, -11
KEY = ref.signing_key("wJalrXUtnFEMI/K7MDENG/bPxRfiCYEXAMPLEKEY")
SEED = b"4f232c4386841ef735655705268965c44a0e4690baa4adea153f7db9fa80a0a9"
SCOPE = ref.scope_of()
SSE_KEY, NONCE = bytes(range(32)), bytes.fromhex("0123456789abcdeffedcba98")
DARE_MAX = (1 << 32) * 65536  # plaintext bytes of 2^32 packages


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


def _call(mb, codec, body, D, key=KEY, seed=SEED, date=ref.DATE, scope=SCOPE, trailer=0, sse_key=SSE_KEY, nonce=NONCE, files=None,
          wq=0, tcap=0, tlen=True):
    L = mb.lib()
    b = np.frombuffer(bytes(body), dtype=np.uint8) if body is not None else None
    fa = (C.c_void_p * 16)(*([1] * 16)) if files is None else files  # never dereferenced: every call below stops first
    n = C.c_int64(-5)
    rc = L.mec_encode_chunked_sse(codec, None if b is None or not b.size else b.ctypes.data, 0 if b is None else b.size, D, key, seed,
                                  None if date is None else date.encode(), None if scope is None else scope.encode(), trailer,
                                  sse_key, nonce, fa, wq, None, tcap, C.byref(n) if tlen else None)
    return rc, n.value


def test_binding_signature(mb):
    f = mb.lib().mec_encode_chunked_sse
    assert f.restype == C.c_int64 and len(f.argtypes) == 16


def test_refusals_in_order(mb):
    c = mb.Codec(12, 4)
    good = bytes(ref.build(b"x" * 10, [10], KEY, SEED).data)
    assert _call(mb, None, good, 10)[0] == INVALID_ARGUMENT
    for kw in ({"key": None}, {"seed": None}, {"date": None}, {"scope": None}, {"sse_key": None}, {"nonce": None}):
        assert _call(mb, c.h, good, 10, **kw)[0] == INVALID_ARGUMENT, kw
    assert _call(mb, c.h, good, -1)[0] == INVALID_ARGUMENT
    assert _call(mb, c.h, good, DARE_MAX + 1)[0] == INVALID_ARGUMENT
    L = mb.lib()
    fa = (C.c_void_p * 16)(*([1] * 16))
    assert L.mec_encode_chunked_sse(c.h, None, 5, 10, KEY, SEED, b"d", b"s", 0, SSE_KEY, NONCE, fa, 0, None, 0, None) == INVALID_ARGUMENT
    assert L.mec_encode_chunked_sse(c.h, good, -1, 10, KEY, SEED, b"d", b"s", 0, SSE_KEY, NONCE, fa, 0, None, 0, None) == INVALID_ARGUMENT
    assert L.mec_encode_chunked_sse(c.h, good, len(good), 10, KEY, SEED, b"d", b"s", 0, SSE_KEY, NONCE, None, 0, None, 0,
                                    None) == INVALID_ARGUMENT
    for seed in (SEED.upper(), SEED[:63] + b"g", b"z" * 64, SEED[:63] + b"\0"):
        assert _call(mb, c.h, good, 10, seed=seed)[0] == INVALID_ARGUMENT, seed
    assert _call(mb, c.h, good, 10, scope="s" * 239)[0] == INVALID_ARGUMENT
    assert _call(mb, c.h, good, 10, trailer=1, tlen=False)[0] == INVALID_ARGUMENT
    assert _call(mb, c.h, good, 10, trailer=1, tcap=8)[0] == INVALID_ARGUMENT
    assert _call(mb, c.h, good, 10, trailer=1, tcap=-1)[0] == INVALID_ARGUMENT
    # an argument error wins over the write quorum, which wins over the body
    off = (C.c_void_p * 16)(*([None] * 8 + [1] * 8))
    assert _call(mb, c.h, good, 10, nonce=None, files=off, wq=9)[0] == INVALID_ARGUMENT
    assert _call(mb, c.h, good, 10, seed=SEED.upper(), files=off, wq=9)[0] == INVALID_ARGUMENT
    assert _call(mb, c.h, b"zz", 10, files=off, wq=9)[0] == WRITE_QUORUM
    assert _call(mb, c.h, b"zz", 10, files=off, wq=8)[0] == ref.MALFORMED_ENCODING
    assert c.stat("launches") == 0 and c.stat("sigv4_chunks") == 0 and c.stat("dare_sealed") == 0
    c.close()


FIRST_HEADER = [
    (b"", ref.INCOMPLETE_BODY),
    (b"1g;", ref.MALFORMED_ENCODING),
    (b"1000001;", ref.CHUNK_TOO_BIG),
    (b"10;chunk-signaturE=" + b"0" * 64 + b"\r\n", ref.MALFORMED_ENCODING),
    (b"10;chunk-signature=" + b"0" * 64 + b"\r", ref.INCOMPLETE_BODY),
    (b"10;chunk-signature=" + b"0" * 64 + b"\r\n" + b"x" * 15, ref.INCOMPLETE_BODY),
]


@pytest.mark.parametrize("body,code", FIRST_HEADER)
def test_first_header_errors_need_no_device(mb, body, code):
    """the same code as mec_encode_chunked and the serial reader, at once"""
    assert ref.read(body, 16, KEY, SEED)[0] == code
    c = mb.Codec(12, 4)
    assert _call(mb, c.h, body, 16)[0] == code
    assert mb.lib().mec_encode_chunked(c.h, body if body else None, len(body), 16, KEY, SEED, ref.DATE.encode(), SCOPE.encode(), 0,
                                       (C.c_void_p * 16)(*([1] * 16)), 0, None, 0, None) == code
    assert c.stat("launches") == 0 and c.stat("sigv4_chunks") == 0 and c.stat("dare_sealed") == 0
    with pytest.raises(mb.MecError) as ei:
        c.encode_chunked_sse(body, 16, KEY, SEED, ref.DATE, SCOPE, SSE_KEY, NONCE)
    assert ei.value.code == code
    c.close()


def test_wrapper_refuses_bad_key_sizes(mb):
    c = mb.Codec(4, 2)
    good = bytes(ref.build(b"x" * 10, [10], KEY, SEED).data)
    for sse_key, nonce in ((SSE_KEY[:31], NONCE), (SSE_KEY, NONCE + b"\0")):
        with pytest.raises(ValueError):
            c.encode_chunked_sse(good, 10, KEY, SEED, ref.DATE, SCOPE, sse_key, nonce)
    c.close()
