"""CPU-side checks of moves across block sizes: mec_transcode accepts a destination block size that divides the source's and refuses
every other one before any device work; mec_batcher_new_transcode_ex reports its refusals in order (source geometry, destination
geometry, flags, block sizes) and leaves *out NULL; without a GPU a valid call fails with MEC_ERR_NO_DEVICE."""
import ctypes as C

import numpy as np
import pytest

from test_transcode_abi import part, raw_transcode

MiB = 1 << 20
INV_SHARD_NUM, MAX_SHARD_NUM, INVALID_ARGUMENT, WRITE_QUORUM, NO_DEVICE, UNSUPPORTED = -1, -2, -12, -11, -101, -102
MIX = 1


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


def new_ex(mb, k, m, bs, k2, m2, bs2, flags=0, out=True):
    """-> (return code, *out after the call)"""
    h = C.c_void_p(0xDEAD)
    rc = mb.lib().mec_batcher_new_transcode_ex(k, m, bs, k2, m2, bs2, 0, 16, 0, flags, C.byref(h) if out else None)
    return rc, h.value


@pytest.mark.parametrize("k,m,bs,k2,m2,bs2,flags,want", [
    # 1. the source geometry, ahead of every later error
    (0, 4, 10 * MiB, 6, 2, MiB, 0, INV_SHARD_NUM),
    (12, 4, 0, 6, 2, MiB, 0, INVALID_ARGUMENT),
    (200, 57, 10 * MiB, 0, 2, 3 * MiB, 2, MAX_SHARD_NUM),
    # 2. the destination geometry, ahead of flags and block sizes
    (12, 4, 10 * MiB, 0, 2, MiB, 0, INV_SHARD_NUM),
    (12, 4, 10 * MiB, 250, 7, MiB, 0, MAX_SHARD_NUM),
    (12, 4, 10 * MiB, 6, 2, 0, 0, INVALID_ARGUMENT),
    (12, 4, 10 * MiB, 6, -1, 3 * MiB, 2, INV_SHARD_NUM),
    # 3. unknown flags, ahead of block sizes
    (12, 4, 10 * MiB, 6, 2, MiB, 2, INVALID_ARGUMENT),
    (12, 4, 3 * MiB, 6, 2, 2 * MiB, MIX | 4, INVALID_ARGUMENT),
    (12, 4, 10 * MiB, 6, 2, 3 * MiB, -1, INVALID_ARGUMENT),
    # 4. a destination block size that does not divide the source's
    (12, 4, 3 * MiB, 6, 2, 2 * MiB, 0, UNSUPPORTED),
    (12, 4, 10 * MiB, 6, 2, 10 * MiB - 1, 0, UNSUPPORTED),
    (12, 4, MiB, 6, 2, 10 * MiB, MIX, UNSUPPORTED),
])
def test_batcher_refusal_order(mb, k, m, bs, k2, m2, bs2, flags, want):
    assert new_ex(mb, k, m, bs, k2, m2, bs2, flags) == (want, None)


def test_batcher_null_out(mb):
    assert new_ex(mb, 12, 4, 10 * MiB, 6, 2, MiB, out=False)[0] == INVALID_ARGUMENT


def test_batcher_no_cpu_fallback(mb):
    """Valid arguments without a CUDA device, R = 10, R = 4 with odd block sizes and R = 1: MEC_ERR_NO_DEVICE."""
    if mb.device_count() > 0:
        pytest.skip("GPU present")
    for bs, bs2 in ((10 * MiB, MiB), (4 * (MiB - 1), MiB - 1), (MiB, MiB)):
        for flags in (0, MIX):
            assert new_ex(mb, 12, 4, bs, 6, 2, bs2, flags) == (NO_DEVICE, None)
    with pytest.raises(mb.MecError) as ei:
        mb.Batcher(12, 4, 10 * MiB, dst=(6, 2, MiB))
    assert ei.value.code == NO_DEVICE


def test_transcode_refusals_across_block_sizes(mb):
    """mec_transcode: a destination block size larger than the source's, or one that does not divide it, is MEC_ERR_UNSUPPORTED;
    the earlier refusals keep their codes when the block sizes differ."""
    total = 3 * MiB + 5
    src = mb.Codec(12, 4, 10 * MiB)
    files = part(src, total)
    for bs2 in (10 * MiB - 1, 3 * MiB, 20 * MiB, 4 * MiB):
        dst = mb.Codec(6, 2, bs2)
        assert raw_transcode(mb, src, files, total, dst, part(dst, total)) == (UNSUPPORTED, 0)
        dst.close()
    dst = mb.Codec(6, 2, MiB)
    outs = part(dst, total)
    assert raw_transcode(mb, src, None, total, dst, outs) == (INVALID_ARGUMENT, 0)
    assert raw_transcode(mb, src, files, -1, dst, outs) == (INVALID_ARGUMENT, 0)
    for algo in (mb.SHA256, mb.HIGHWAYHASH256, mb.BLAKE2B512):
        whole = mb.Codec(6, 2, MiB, algo)
        assert raw_transcode(mb, src, files, total, whole, outs) == (UNSUPPORTED, 0)
        whole.close()
    other = mb.Codec(6, 2, MiB, device=1)
    assert raw_transcode(mb, src, files, total, other, outs) == (UNSUPPORTED, 0)
    offline = [o if i < 5 else None for i, o in enumerate(outs)]
    assert raw_transcode(mb, src, files, total, dst, offline, write_quorum=6) == (WRITE_QUORUM, 0)
    for c in (src, dst, other):
        c.close()


def test_transcode_no_cpu_fallback(mb):
    """A valid 10 MiB -> 1 MiB move without a CUDA device fails with MEC_ERR_NO_DEVICE: no CPU path."""
    if mb.device_count() > 0:
        pytest.skip("GPU present")
    src, dst = mb.Codec(12, 4, 10 * MiB), mb.Codec(6, 2, MiB)
    total = 2 * 10 * MiB + 4321
    with pytest.raises(mb.MecError) as ei:
        src.transcode(part(src, total), total, dst)
    assert ei.value.code == NO_DEVICE
    src.close()
    dst.close()
