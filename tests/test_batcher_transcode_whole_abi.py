"""CPU-side checks of mec_batcher_transcode_whole, the coalesced move of a part written with a whole-file bitrot algorithm: the
symbol is exported, refusals that need no batcher return MEC_ERR_INVALID_ARGUMENT with *heal_hint cleared, and the Python wrapper
raises MecError with that code."""
import ctypes as C

import numpy as np
import pytest

INVALID_ARGUMENT = -12
SHA256, HIGHWAYHASH256, HIGHWAYHASH256S, BLAKE2B512 = 1, 2, 3, 4


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


def call(mb, b, algo=SHA256, files=True, sums=True, outs=True, total=10, hint=True):
    """-> (return code, *heal_hint after the call, or None without one)"""
    f = [np.zeros(64, dtype=np.uint8) for _ in range(16)]
    o = [np.zeros(64, dtype=np.uint8) for _ in range(8)]
    sm = np.zeros((16, 64), dtype=np.uint8)
    h = C.c_int(99)
    rc = mb.lib().mec_batcher_transcode_whole(b, algo, mb.capi._ptrs(f) if files else None, sm.ctypes.data if sums else None, None,
                                              total, mb.capi._ptrs(o) if outs else None, 0, C.byref(h) if hint else None)
    return rc, h.value if hint else None


def test_symbol_exported(mb):
    fn = mb.lib().mec_batcher_transcode_whole
    assert fn.restype == C.c_int64 and len(fn.argtypes) == 9


@pytest.mark.parametrize("algo", [SHA256, HIGHWAYHASH256, BLAKE2B512, HIGHWAYHASH256S, 0, 5, -1])
def test_null_batcher(mb, algo):
    """A NULL batcher is refused first, whatever the algorithm (HighwayHash256S and unknown values included), and clears
    *heal_hint."""
    assert call(mb, None, algo) == (INVALID_ARGUMENT, 0)
    assert call(mb, None, algo, hint=False) == (INVALID_ARGUMENT, None)


@pytest.mark.parametrize("missing", ["files", "sums", "outs"])
def test_null_arguments(mb, missing):
    assert call(mb, None, **{missing: False}) == (INVALID_ARGUMENT, 0)


def test_negative_length(mb):
    assert call(mb, None, total=-1) == (INVALID_ARGUMENT, 0)


def test_wrapper_raises(mb):
    """Batcher.transcode_whole turns the refusal into MecError carrying the code: here a batcher object without a handle or a
    destination codec, as a closed batcher is."""
    bat = object.__new__(mb.Batcher)
    bat.h, bat.k, bat.m, bat.n, bat.block_size, bat._dst_sizes = None, 12, 4, 16, 1 << 20, None
    files = [np.zeros(64, dtype=np.uint8) for _ in range(16)]
    with pytest.raises(mb.MecError) as ei:
        bat.transcode_whole(files, [b"\0" * 32] * 16, 12 * 64, mb.SHA256)
    assert ei.value.code == INVALID_ARGUMENT
