"""CPU-side checks of mec_transcode_whole: every refusal returns its code before any device work, an empty part moves nothing but
still checks the write quorum, and a valid call without a GPU fails with MEC_ERR_NO_DEVICE instead of moving the part on the CPU."""
import ctypes as C

import numpy as np
import pytest

MiB = 1 << 20
INVALID, WRITE_QUORUM, NO_DEVICE, UNSUPPORTED = -12, -11, -101, -102


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


def raw(mb, src, files, sums, total, dst, outs, write_quorum=0, src_h=None, dst_h=None):
    """-> (return code, heal hint); files / sums / outs None pass NULL"""
    L = mb.lib()
    hint = C.c_int(99)
    fp = None if files is None else mb.capi._ptrs(files)
    sp = None if sums is None else sums.ctypes.data
    op = None if outs is None else mb.capi._ptrs(outs)
    rc = L.mec_transcode_whole(src.h if src_h is None else src_h, fp, sp, None, total, dst.h if dst_h is None else dst_h, op,
                               write_quorum, C.byref(hint))
    return rc, hint.value


def shard_files(c, total):
    return [np.zeros(max(c.shard_file_size(total), 1), dtype=np.uint8) for _ in range(c.n)]


def part(c, total):
    return [np.zeros(max(c.bitrot_file_size(total), 1), dtype=np.uint8) for _ in range(c.n)]


@pytest.mark.parametrize("algo", ["SHA256", "HIGHWAYHASH256", "BLAKE2B512"])
def test_refusals_before_device_work(mb, algo):
    src, dst = mb.Codec(12, 4, 10 * MiB, getattr(mb, algo)), mb.Codec(6, 2, MiB)
    total = 3 * MiB + 5
    files, sums, outs = shard_files(src, total), np.zeros((16, 64), dtype=np.uint8), part(dst, total)
    # one handle cannot be both ends
    assert raw(mb, src, files, sums, total, src, part(src, total)) == (INVALID, 0)
    # NULL arrays, NULL handles, negative length
    assert raw(mb, src, None, sums, total, dst, outs) == (INVALID, 0)
    assert raw(mb, src, files, None, total, dst, outs) == (INVALID, 0)
    assert raw(mb, src, files, sums, total, dst, None) == (INVALID, 0)
    assert raw(mb, src, files, sums, total, dst, outs, dst_h=C.c_void_p())[0] == INVALID
    assert raw(mb, src, files, sums, total, dst, outs, src_h=C.c_void_p())[0] == INVALID
    assert raw(mb, src, files, sums, -1, dst, outs) == (INVALID, 0)
    # a streaming source moves through mec_transcode
    streaming = mb.Codec(12, 4, 10 * MiB)
    assert raw(mb, streaming, files, sums, total, dst, outs) == (UNSUPPORTED, 0)
    # whole-file bitrot on the destination side
    for walgo in (mb.SHA256, mb.HIGHWAYHASH256, mb.BLAKE2B512):
        whole = mb.Codec(6, 2, MiB, walgo)
        assert raw(mb, src, files, sums, total, whole, outs) == (UNSUPPORTED, 0)
        whole.close()
    # a destination block size that does not divide the source's: larger, and a non-divisor
    for bd in (20 * MiB, 3 * MiB):
        other = mb.Codec(6, 2, bd)
        assert raw(mb, src, files, sums, total, other, part(other, total)) == (UNSUPPORTED, 0)
        other.close()
    # another device
    far = mb.Codec(6, 2, MiB, device=1)
    assert raw(mb, src, files, sums, total, far, outs) == (UNSUPPORTED, 0)
    # write quorum: 5 writers online, 6 required
    offline = [o if i < 5 else None for i, o in enumerate(outs)]
    assert raw(mb, src, files, sums, total, dst, offline, write_quorum=6) == (WRITE_QUORUM, 0)
    with pytest.raises(mb.MecError) as ei:
        src.transcode_whole(files, [None] * 16, total, dst, online=[True] * 5 + [False] * 3, write_quorum=6)
    assert ei.value.code == WRITE_QUORUM
    for c in (src, dst, streaming, far):
        c.close()


def test_empty_part(mb):
    """total == 0 moves nothing and returns 0; the write quorum is still checked (cmd/erasure-encode.go:59-65)."""
    src, dst = mb.Codec(12, 4, 10 * MiB, mb.SHA256), mb.Codec(6, 2, MiB)
    outs, hint = src.transcode_whole([np.zeros(0, dtype=np.uint8)] * 16, [None] * 16, 0, dst, write_quorum=8)
    assert hint == 0 and len(outs) == 8 and all(o.size == 0 for o in outs)
    assert raw(mb, src, [None] * 16, np.zeros((16, 64), dtype=np.uint8), 0, dst, [None] * 8) == (0, 0)
    with pytest.raises(mb.MecError) as ei:
        src.transcode_whole([None] * 16, [None] * 16, 0, dst, online=[True] * 4 + [False] * 4, write_quorum=5)
    assert ei.value.code == WRITE_QUORUM
    src.close()
    dst.close()


def test_no_cpu_fallback(mb):
    """A valid call without a CUDA device fails with MEC_ERR_NO_DEVICE: the part is never moved through a CPU path."""
    if mb.device_count() > 0:
        pytest.skip("GPU present")
    src, dst = mb.Codec(12, 4, 10 * MiB, mb.BLAKE2B512), mb.Codec(6, 2, MiB)
    total = 2 * MiB + 1
    with pytest.raises(mb.MecError) as ei:
        src.transcode_whole(shard_files(src, total), [bytes(64)] * 16, total, dst)
    assert ei.value.code == NO_DEVICE
    src.close()
    dst.close()
