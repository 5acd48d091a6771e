"""CPU-side checks of mec_batcher_encode_sse / mec_batcher_decode_sse, server-side encryption through the cross-request coalescer: the
symbols are exported with the header's signatures, which are the single-codec calls' with the batcher in place of the codec, every
refusal that needs no batcher is made with MEC_ERR_INVALID_ARGUMENT (*heal_hint cleared, dst untouched), and the Python wrappers
raise MecError with that code.  The refusals that need a live batcher are checked in tests/test_gpu_batcher_sse.py."""
import ctypes as C

import numpy as np
import pytest

from test_batcher_mixed_bitrot_abi import header_params
from test_sse_abi import proto

MiB = 1 << 20
INVALID = -12
NAMES = {"mec_batcher_encode_sse": "mec_encode_sse", "mec_batcher_decode_sse": "mec_decode_sse"}


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


@pytest.mark.parametrize("name", sorted(NAMES))
def test_signature_matches_header(mb, name):
    ret, kinds = proto(name)
    fn = getattr(mb.lib(), name)
    assert fn.restype is (C.c_int64 if ret == "int64_t" else C.c_int)
    assert ["int64" if a is C.c_int64 else "int" if a is C.c_int else "pointer" for a in fn.argtypes] == kinds


@pytest.mark.parametrize("name", sorted(NAMES))
def test_batcher_call_follows_codec_call(mb, name):
    r1, p1 = header_params(NAMES[name])
    r2, p2 = header_params(name)
    assert r1 == r2 and p1[1:] == p2[1:] and p1[0] == "mec_codec*" and p2[0] == "mec_batcher*"


def test_exported(mb):
    import subprocess
    out = subprocess.run(["nm", "-D", "--defined-only", mb.lib_path()], capture_output=True, text=True, check=True).stdout
    syms = {ln.split()[-1] for ln in out.splitlines() if ln.strip()}
    assert set(NAMES) <= syms


def test_encode_refusals(mb):
    L = mb.lib()
    key, nonce, src = np.zeros(32, np.uint8), np.zeros(12, np.uint8), np.zeros(10, np.uint8)
    files = [np.zeros(64, np.uint8) for _ in range(16)]
    ptrs = (C.c_void_p * 16)(*[f.ctypes.data for f in files])
    for args in [(None, src.ctypes.data, 10, key.ctypes.data, nonce.ctypes.data, ptrs, 0),       # NULL batcher
                 (None, src.ctypes.data, 10, None, nonce.ctypes.data, ptrs, 0),                  # and NULL key
                 (None, src.ctypes.data, 10, key.ctypes.data, None, ptrs, 0),                    # NULL nonce
                 (None, None, 10, key.ctypes.data, nonce.ctypes.data, ptrs, 0),                  # NULL src
                 (None, src.ctypes.data, 10, key.ctypes.data, nonce.ctypes.data, None, 0),       # NULL files
                 (None, src.ctypes.data, -1, key.ctypes.data, nonce.ctypes.data, ptrs, 0),       # negative len
                 (None, None, 0, key.ctypes.data, nonce.ctypes.data, ptrs, 0),                   # len == 0 without a batcher
                 (None, src.ctypes.data, 10, key.ctypes.data, nonce.ctypes.data, ptrs, 17)]:     # quorum without a batcher
        assert L.mec_batcher_encode_sse(*args) == INVALID
    assert not any(f.any() for f in files)


def test_decode_refusals(mb):
    L = mb.lib()
    key = np.zeros(32, np.uint8)
    files = [np.zeros(64, np.uint8) for _ in range(16)]
    ptrs = (C.c_void_p * 16)(*[f.ctypes.data for f in files])
    dst = np.full(16, 0x5A, np.uint8)
    hint = C.c_int(5)
    for args in [(ptrs, 0, 1, 33, key.ctypes.data, dst.ctypes.data),    # NULL batcher
                 (None, 0, 1, 33, key.ctypes.data, dst.ctypes.data),    # NULL files
                 (ptrs, 0, 1, 33, None, dst.ctypes.data),               # NULL key
                 (ptrs, 0, 1, 33, key.ctypes.data, None),               # NULL dst
                 (ptrs, -1, 1, 33, key.ctypes.data, dst.ctypes.data),   # negative offset
                 (ptrs, 0, -1, 33, key.ctypes.data, dst.ctypes.data),   # negative length
                 (ptrs, 0, 1, -1, key.ctypes.data, dst.ctypes.data),    # negative stored size
                 (ptrs, 0, 1, 20, key.ctypes.data, dst.ctypes.data),    # no DARE size, but no batcher either
                 (ptrs, 0, 0, 33, key.ctypes.data, dst.ctypes.data)]:   # length == 0 without a batcher
        hint.value = 5
        assert L.mec_batcher_decode_sse(None, args[0], None, *args[1:], C.byref(hint)) == INVALID
        assert hint.value == 0
    assert L.mec_batcher_decode_sse(None, ptrs, None, 0, 1, 33, key.ctypes.data, dst.ctypes.data, None) == INVALID  # no heal_hint
    assert (dst == 0x5A).all()


@pytest.fixture
def closed_batcher(mb):
    """a Batcher whose handle is NULL (as after close()): every call reaches the library's NULL-batcher refusal"""
    bat = object.__new__(mb.Batcher)
    bat.h, bat.k, bat.m, bat.n, bat.block_size = None, 12, 4, 16, MiB
    bat._sizes, bat._dst_sizes = mb.Codec(12, 4, MiB), None
    yield bat
    bat._sizes.close()


def test_wrappers_raise(mb, closed_batcher):
    key, nonce = np.zeros(32, np.uint8), np.zeros(12, np.uint8)
    with pytest.raises(mb.MecError) as e:
        closed_batcher.encode_sse(np.zeros(10, np.uint8), key, nonce)
    assert e.value.code == INVALID
    with pytest.raises(mb.MecError) as e:
        closed_batcher.decode_sse([np.zeros(64, np.uint8)] * 16, 0, 1, 33, key)
    assert e.value.code == INVALID
    with pytest.raises(ValueError):
        closed_batcher.encode_sse(np.zeros(10, np.uint8), key[:16], nonce)
    with pytest.raises(ValueError):
        closed_batcher.decode_sse([None] * 16, 0, 1, 33, key[:5])
