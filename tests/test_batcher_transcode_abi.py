"""CPU-side checks of the transcode batcher (mec_batcher_new_transcode, mec_batcher_transcode): every refusal returns its code and
leaves *out NULL, and valid arguments without a GPU fail with MEC_ERR_NO_DEVICE instead of creating a CPU path."""
import ctypes as C

import numpy as np
import pytest

MiB = 1 << 20
INV_SHARD_NUM, MAX_SHARD_NUM, NO_DEVICE, INVALID_ARGUMENT = -1, -2, -101, -12
MIX = 1


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


def new_transcode(mb, k, m, k2, m2, flags=0, bs=MiB, out=True):
    """-> (return code, *out after the call)"""
    h = C.c_void_p(0xDEAD)
    rc = mb.lib().mec_batcher_new_transcode(k, m, k2, m2, bs, 0, 16, 0, flags, C.byref(h) if out else None)
    return rc, h.value


@pytest.mark.parametrize("k,m,k2,m2,want", [
    (0, 4, 6, 2, INV_SHARD_NUM), (12, -1, 6, 2, INV_SHARD_NUM),     # the source geometry
    (12, 4, 0, 2, INV_SHARD_NUM), (12, 4, 6, -1, INV_SHARD_NUM),    # the destination geometry
    (200, 57, 6, 2, MAX_SHARD_NUM), (12, 4, 250, 7, MAX_SHARD_NUM),
])
def test_geometry_errors(mb, k, m, k2, m2, want):
    assert new_transcode(mb, k, m, k2, m2) == (want, None)


def test_flags_and_null_out(mb):
    for flags in (2, MIX | 4, -1):
        assert new_transcode(mb, 12, 4, 6, 2, flags) == (INVALID_ARGUMENT, None)
    assert new_transcode(mb, 12, 4, 6, 2, out=False)[0] == INVALID_ARGUMENT


def test_no_cpu_fallback(mb):
    """Valid arguments without a CUDA device: MEC_ERR_NO_DEVICE, for equal geometries too (rebalance between equal pools)."""
    if mb.device_count() > 0:
        pytest.skip("GPU present")
    for k, m, k2, m2 in ((12, 4, 6, 2), (12, 4, 12, 4)):
        for flags in (0, MIX):
            assert new_transcode(mb, k, m, k2, m2, flags) == (NO_DEVICE, None)
    with pytest.raises(mb.MecError) as ei:
        mb.Batcher(12, 4, dst=(6, 2))
    assert ei.value.code == NO_DEVICE


def test_null_batcher(mb):
    files = [np.zeros(64, dtype=np.uint8) for _ in range(16)]
    outs = [np.zeros(64, dtype=np.uint8) for _ in range(8)]
    hint = C.c_int(99)
    rc = mb.lib().mec_batcher_transcode(None, mb.capi._ptrs(files), None, 10, mb.capi._ptrs(outs), 0, C.byref(hint))
    assert rc == INVALID_ARGUMENT and hint.value == 0
    assert mb.lib().mec_batcher_transcode(None, None, None, 10, None, 0, None) == INVALID_ARGUMENT
