"""CPU-side checks of mec_batcher_decode_mixed / mec_batcher_heal_mixed, the coalesced reads and heals of parts whose drives mix
bitrot formats: the symbols are exported with the header's signatures, a NULL batcher is refused first with MEC_ERR_INVALID_ARGUMENT
(*heal_hint cleared, corrupt[] untouched, as the single-codec calls treat a NULL codec), and the Python wrappers raise MecError with
that code."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MiB = 1 << 20
INVALID = -12
SHA256, HIGHWAYHASH256, HIGHWAYHASH256S, BLAKE2B512 = 1, 2, 3, 4


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


def header_params(name):
    """-> (return type, [parameter types]) of `name`'s prototype in include/minio_ec.h"""
    hdr = open(os.path.join(ROOT, "include", "minio_ec.h")).read()
    m = re.search(r"\n(int64_t|int)\s+" + name + r"\(([^)]*)\);", hdr)
    assert m, name
    params = [" ".join(p.split()[:-1]) + ("*" * p.split()[-1].count("*")) for p in m.group(2).split(",")]
    return m.group(1), [re.sub(r"\s+", " ", p).strip() for p in params]


def ctype_of(t):
    """the ctypes type capi declares for a C parameter type"""
    if "*" in t:
        return "int*" if t.replace(" ", "") == "int*" else "pointer"
    return {"int64_t": "int64", "int": "int"}[t]


def capi_kind(a):
    if a is C.c_int64:
        return "int64"
    if a is C.c_int:
        return "int"
    if a is C.c_void_p:
        return "pointer"
    if a is C.POINTER(C.c_int):
        return "int*"
    raise AssertionError(a)


@pytest.mark.parametrize("name", ["mec_batcher_decode_mixed", "mec_batcher_heal_mixed"])
def test_signature_matches_header(mb, name):
    ret, params = header_params(name)
    fn = getattr(mb.lib(), name)
    assert fn.restype is (C.c_int64 if ret == "int64_t" else C.c_int)
    assert [capi_kind(a) for a in fn.argtypes] == [ctype_of(p) for p in params]


def test_signatures_follow_single_codec_calls(mb):
    """The batcher calls take the arguments of mec_decode_mixed / mec_heal_mixed, the batcher in place of the codec."""
    for single, batched in (("mec_decode_mixed", "mec_batcher_decode_mixed"), ("mec_heal_mixed", "mec_batcher_heal_mixed")):
        r1, p1 = header_params(single)
        r2, p2 = header_params(batched)
        assert r1 == r2 and p1[1:] == p2[1:] and p2[0] == "mec_batcher*"


def decode_raw(mb, b, algos=True, files=True, sums=True, offset=0, length=10, total=12 * 64, dst=True):
    """-> (return code, *heal_hint after the call)"""
    al = (C.c_int32 * 16)(*([SHA256] * 8 + [HIGHWAYHASH256S] * 8))
    f = [np.zeros(64, dtype=np.uint8) for _ in range(16)]
    sm = np.zeros((16, 64), dtype=np.uint8)
    out = np.zeros(max(length, 1), dtype=np.uint8)
    h = C.c_int(99)
    rc = mb.lib().mec_batcher_decode_mixed(b, al if algos else None, mb.capi._ptrs(f) if files else None,
                                           sm.ctypes.data if sums else None, None, offset, length, total,
                                           out.ctypes.data if dst else None, C.byref(h))
    return rc, h.value


def heal_raw(mb, b, algos=True, files=True, sums=True, outs=True, total=12 * 64):
    """-> (return code, corrupt[] pre-filled with 1s)"""
    al = (C.c_int32 * 16)(*([SHA256] * 8 + [HIGHWAYHASH256S] * 8))
    f = [np.zeros(64, dtype=np.uint8) for _ in range(16)]
    o = [np.zeros(64, dtype=np.uint8) if i == 0 else None for i in range(16)]
    sm = np.zeros((16, 64), dtype=np.uint8)
    corrupt = np.ones(16, dtype=np.uint8)
    rc = mb.lib().mec_batcher_heal_mixed(b, al if algos else None, mb.capi._ptrs(f) if files else None,
                                         sm.ctypes.data if sums else None, None, total, mb.capi._ptrs(o) if outs else None,
                                         corrupt.ctypes.data)
    return rc, corrupt


def test_decode_null_batcher_first(mb):
    """A NULL batcher is refused before any other check: a bad range, an empty read, a missing dst or algos do not change that."""
    assert decode_raw(mb, None) == (INVALID, 0)
    assert decode_raw(mb, None, length=0) == (INVALID, 0)
    assert decode_raw(mb, None, offset=-1) == (INVALID, 0)
    assert decode_raw(mb, None, dst=False) == (INVALID, 0)
    assert decode_raw(mb, None, algos=False, files=False, sums=False) == (INVALID, 0)
    assert mb.lib().mec_batcher_decode_mixed(None, None, None, None, None, 0, 10, 100, None, None) == INVALID  # heal_hint may be NULL


def test_heal_null_batcher_first(mb):
    """A NULL batcher is refused first and corrupt[] is left as it was (mec_heal_mixed clears it only for a live codec)."""
    for kw in ({}, {"total": 0}, {"outs": False}, {"algos": False, "files": False, "sums": False}):
        rc, corrupt = heal_raw(mb, None, **kw)
        assert rc == INVALID and corrupt.tolist() == [1] * 16


@pytest.fixture
def closed_batcher(mb):
    """A Batcher object without a handle, as a closed batcher is; its size helper is a real codec (no device needed)"""
    bat = object.__new__(mb.Batcher)
    bat.h, bat.k, bat.m, bat.n, bat.block_size, bat._dst_sizes = None, 12, 4, 16, MiB, None
    bat._sizes = mb.Codec(12, 4, MiB)
    yield bat
    bat._sizes.close()


@pytest.mark.parametrize("walgo", [SHA256, HIGHWAYHASH256, BLAKE2B512])
def test_wrappers_raise(mb, closed_batcher, walgo):
    total = 3 * MiB + 5
    c = closed_batcher._sizes
    files = [np.zeros(c.shard_file_size(total) if i < 6 else c.bitrot_file_size(total), dtype=np.uint8) for i in range(16)]
    algos = [walgo] * 6 + [HIGHWAYHASH256S] * 10
    sums = [b"\0" * 32] * 6 + [None] * 10
    with pytest.raises(mb.MecError) as ei:
        closed_batcher.decode_mixed(files, algos, sums, 0, 100, total)
    assert ei.value.code == INVALID
    stale = [i == 15 for i in range(16)]
    for report in (False, True):
        with pytest.raises(mb.MecError) as ei:
            closed_batcher.heal_mixed(files, algos, sums, stale, total, report=report)
        assert ei.value.code == INVALID
