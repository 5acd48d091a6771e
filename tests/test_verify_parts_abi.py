"""CPU-side checks of mec_bitrot_verify_parts and mec_batcher_verify (VerifyFile in one call, on a codec and through the coalescer):
the symbols are exported with the header's signatures, both take the same arguments but for the handle, a NULL codec or batcher is
refused first with MEC_ERR_INVALID_ARGUMENT and results[] untouched, the refusals that need no device leave results[] untouched too,
and the Python wrappers raise MecError with that code."""
import ctypes as C

import numpy as np
import pytest

from test_batcher_mixed_bitrot_abi import capi_kind, ctype_of, header_params

MiB = 1 << 20
INVALID, FILE_CORRUPT = -12, -7
SHA256, HIGHWAYHASH256, HIGHWAYHASH256S, BLAKE2B512 = 1, 2, 3, 4


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


@pytest.mark.parametrize("name", ["mec_bitrot_verify_parts", "mec_batcher_verify"])
def test_signature_matches_header(mb, name):
    ret, params = header_params(name)
    fn = getattr(mb.lib(), name)
    assert ret == "int" and fn.restype is C.c_int
    assert [capi_kind(a) for a in fn.argtypes] == [ctype_of(p) for p in params]


def test_batcher_call_follows_codec_call(mb):
    r1, p1 = header_params("mec_bitrot_verify_parts")
    r2, p2 = header_params("mec_batcher_verify")
    assert r1 == r2 and p1[1:] == p2[1:] and p1[0] == "mec_codec*" and p2[0] == "mec_batcher*"


def raw(mb, fn, h, n=3, algos=True, files=True, file_lens=True, part_lens=True, sums=True, results=True, algo=SHA256):
    """-> (return code, results[] pre-filled with 99)"""
    al = (C.c_int32 * 3)(algo, HIGHWAYHASH256S, algo)
    f = [np.zeros(64, dtype=np.uint8) for _ in range(3)]
    fl = (C.c_int64 * 3)(64, 64, 64)
    pl = (C.c_int64 * 3)(64, 32, 64)
    sm = np.zeros((3, 64), dtype=np.uint8)
    res = (C.c_int32 * 3)(99, 99, 99)
    rc = fn(h, n, al if algos else None, mb.capi._ptrs(f) if files else None, fl if file_lens else None, pl if part_lens else None,
            sm.ctypes.data if sums else None, res if results else None)
    return rc, list(res)


@pytest.mark.parametrize("name", ["mec_bitrot_verify_parts", "mec_batcher_verify"])
def test_null_handle_first(mb, name):
    fn = getattr(mb.lib(), name)
    for kw in ({}, {"n": 0}, {"n": -1}, {"algos": False, "files": False}, {"sums": False}, {"results": False}):
        rc, res = raw(mb, fn, None, **kw)
        assert rc == INVALID and res == [99, 99, 99]


def test_codec_refusals_leave_results(mb):
    """refused before any device work (none is needed here: a codec is created without touching the GPU)"""
    c = mb.Codec(12, 4, MiB)
    fn = mb.lib().mec_bitrot_verify_parts
    for kw in ({"n": -1}, {"algos": False}, {"files": False}, {"file_lens": False}, {"part_lens": False}, {"sums": False},
               {"sums": False, "algo": BLAKE2B512}):
        rc, res = raw(mb, fn, c.h, **kw)
        assert rc == INVALID and res == [99, 99, 99], kw
    assert raw(mb, fn, c.h, n=0, algos=False, files=False, file_lens=False, part_lens=False, sums=False, results=False)[0] == 0
    c.close()


def test_decisions_without_device(mb):
    """parts decided without hashing: unknown algorithms, negative lengths, NULL files with bytes, wrong streaming lengths and empty
    streaming parts; a call with nothing left to hash returns before any device work"""
    c = mb.Codec(12, 4, MiB)
    S = c.shard_size()
    z = np.zeros(40, dtype=np.uint8)
    files = [z, z, None, z, z, None, z[:0]]
    algos = [0, 7, HIGHWAYHASH256S, HIGHWAYHASH256S, HIGHWAYHASH256S, HIGHWAYHASH256S, HIGHWAYHASH256S]
    plens = [0, 0, 5, 40, -1, 0, 0]
    f = mb.capi._ptrs(files)
    al = (C.c_int32 * 7)(*algos)
    fl = (C.c_int64 * 7)(40, 40, 37, 40, 40, 0, 0)
    pl = (C.c_int64 * 7)(*plens)
    res = (C.c_int32 * 7)()
    assert mb.lib().mec_bitrot_verify_parts(c.h, 7, al, f, fl, pl, None, res) == 0
    assert list(res) == [INVALID, INVALID, INVALID, FILE_CORRUPT, INVALID, 0, 0]
    assert 40 != mb.lib().mec_bitrot_shard_file_size(40, S, HIGHWAYHASH256S)
    fl[1] = -1
    al[1] = SHA256  # a negative length refuses a whole-file part as well; sums may be NULL only without whole-file parts
    assert mb.lib().mec_bitrot_verify_parts(c.h, 7, al, f, fl, pl, None, res) == INVALID
    c.close()


@pytest.fixture
def closed_batcher(mb):
    bat = object.__new__(mb.Batcher)
    bat.h, bat.k, bat.m, bat.n, bat.block_size, bat._dst_sizes = None, 12, 4, 16, MiB, None
    bat._sizes = mb.Codec(12, 4, MiB)
    yield bat
    bat._sizes.close()


def test_wrappers_raise(mb, closed_batcher):
    files = [np.zeros(100, dtype=np.uint8), np.zeros(64, dtype=np.uint8)]
    with pytest.raises(mb.MecError) as ei:
        closed_batcher.verify(files, [SHA256, HIGHWAYHASH256S], [0, 32], [b"\0" * 32, None])
    assert ei.value.code == INVALID
    c = mb.Codec(12, 4, MiB)
    with pytest.raises(mb.MecError) as ei:
        c.bitrot_verify_parts(files, [SHA256, HIGHWAYHASH256S], [0, 32])  # a whole-file part and no sums
    assert ei.value.code == INVALID
    c.close()
