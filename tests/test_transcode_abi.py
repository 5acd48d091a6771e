"""CPU-side checks of mec_transcode: every refusal returns its code before any device work, and a valid call without a GPU fails
with MEC_ERR_NO_DEVICE instead of moving the part on the CPU."""
import ctypes as C

import numpy as np
import pytest

MiB = 1 << 20


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


def raw_transcode(mb, src, files, total, dst, outs, write_quorum=0, src_h=None, dst_h=None):
    """-> (return code, heal hint); files / outs None pass NULL arrays"""
    L = mb.lib()
    hint = C.c_int(99)
    fp = None if files is None else mb.capi._ptrs(files)
    op = None if outs is None else mb.capi._ptrs(outs)
    rc = L.mec_transcode(src.h if src_h is None else src_h, fp, None, total, dst.h if dst_h is None else dst_h, op, write_quorum,
                         C.byref(hint))
    return rc, hint.value


def part(c, total):
    return [np.zeros(c.bitrot_file_size(total), dtype=np.uint8) for _ in range(c.n)]


def test_refusals_before_device_work(mb):
    src, dst = mb.Codec(12, 4), mb.Codec(6, 2)
    total = 3 * MiB + 5
    files, outs = part(src, total), part(dst, total)
    # one handle cannot be both ends
    assert raw_transcode(mb, src, files, total, src, part(src, total)) == (-12, 0)
    # NULL arrays, NULL handles, negative length
    assert raw_transcode(mb, src, None, total, dst, outs) == (-12, 0)
    assert raw_transcode(mb, src, files, total, dst, None) == (-12, 0)
    assert raw_transcode(mb, src, files, total, dst, outs, dst_h=C.c_void_p())[0] == -12
    assert raw_transcode(mb, src, files, total, dst, outs, src_h=C.c_void_p())[0] == -12
    assert raw_transcode(mb, src, files, -1, dst, outs) == (-12, 0)
    # block sizes differ (a legacy blockSizeV1 source)
    small = mb.Codec(6, 2, 10 * MiB)
    assert raw_transcode(mb, src, files, total, small, part(small, total)) == (-102, 0)
    # whole-file bitrot on either side
    for algo in (mb.SHA256, mb.HIGHWAYHASH256, mb.BLAKE2B512):
        whole = mb.Codec(6, 2, MiB, algo)
        assert raw_transcode(mb, src, files, total, whole, outs) == (-102, 0)
        assert raw_transcode(mb, whole, files[:8], total, dst, outs) == (-102, 0)
        whole.close()
    # another device
    other = mb.Codec(6, 2, MiB, device=1)
    assert raw_transcode(mb, src, files, total, other, outs) == (-102, 0)
    # write quorum: 5 writers online, 6 required
    offline = [o if i < 5 else None for i, o in enumerate(outs)]
    assert raw_transcode(mb, src, files, total, dst, offline, write_quorum=6) == (-11, 0)
    with pytest.raises(mb.MecError) as ei:
        src.transcode(files, total, dst, online=[True] * 5 + [False] * 3, write_quorum=6)
    assert ei.value.code == -11
    for c in (src, dst, small, other):
        c.close()


def test_empty_part(mb):
    """total == 0 moves nothing and returns 0; the write quorum is still checked (cmd/erasure-encode.go:59-65)."""
    src, dst = mb.Codec(12, 4), mb.Codec(6, 2)
    outs, hint = src.transcode([np.zeros(0, dtype=np.uint8)] * 16, 0, dst, write_quorum=8)
    assert hint == 0 and len(outs) == 8 and all(o.size == 0 for o in outs)
    with pytest.raises(mb.MecError) as ei:
        src.transcode([None] * 16, 0, dst, online=[True] * 4 + [False] * 4, write_quorum=5)
    assert ei.value.code == -11
    src.close()
    dst.close()


def test_no_cpu_fallback(mb):
    """A valid call without a CUDA device fails with MEC_ERR_NO_DEVICE: the part is never moved through a CPU path."""
    if mb.device_count() > 0:
        pytest.skip("GPU present")
    src, dst = mb.Codec(12, 4), mb.Codec(6, 2)
    total = 2 * MiB + 1
    with pytest.raises(mb.MecError) as ei:
        src.transcode(part(src, total), total, dst)
    assert ei.value.code == -101
    src.close()
    dst.close()
