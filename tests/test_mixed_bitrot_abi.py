"""CPU-side checks of mec_decode_mixed / mec_heal_mixed: every refusal returns its code before any device work, the empty cases
return as specified, and a valid call without a GPU fails with MEC_ERR_NO_DEVICE instead of reading the part on the CPU."""
import ctypes as C

import numpy as np
import pytest

MiB = 1 << 20
INVALID, NO_DEVICE, UNSUPPORTED = -12, -101, -102


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


def algos_arr(algos):
    return None if algos is None else (C.c_int32 * len(algos))(*algos)


def decode_raw(mb, c, algos, files, sums, offset, length, total, dst=True, prefer=None, h=None):
    """-> (return code, heal hint); algos / files / sums None pass NULL"""
    hint = C.c_int(99)
    out = np.zeros(max(length, 1), dtype=np.uint8) if dst else None
    rc = mb.lib().mec_decode_mixed(c.h if h is None else h, algos_arr(algos), None if files is None else mb.capi._ptrs(files),
                                   None if sums is None else sums.ctypes.data, prefer, offset, length, total,
                                   None if out is None else out.ctypes.data, C.byref(hint))
    return rc, hint.value


def heal_raw(mb, c, algos, files, sums, total, outs, h=None):
    """-> (return code, corrupt[]) with corrupt pre-filled with 1s"""
    corrupt = np.ones(c.n, dtype=np.uint8)
    rc = mb.lib().mec_heal_mixed(c.h if h is None else h, algos_arr(algos), None if files is None else mb.capi._ptrs(files),
                                 None if sums is None else sums.ctypes.data, None, total,
                                 None if outs is None else mb.capi._ptrs(outs), corrupt.ctypes.data)
    return rc, corrupt


def mixed_files(c, total, nwhole):
    """drives [0, nwhole) raw shard files, the rest part.N images"""
    return [np.zeros(max(c.shard_file_size(total) if i < nwhole else c.bitrot_file_size(total), 1), dtype=np.uint8)
            for i in range(c.n)]


@pytest.mark.parametrize("walgo", ["SHA256", "HIGHWAYHASH256", "BLAKE2B512"])
def test_decode_refusals_before_device_work(mb, walgo):
    wa = getattr(mb, walgo)
    c = mb.Codec(12, 4, MiB)
    total = 3 * MiB + 5
    files, sums = mixed_files(c, total, 6), np.zeros((16, 64), dtype=np.uint8)
    algos = [wa] * 6 + [mb.HIGHWAYHASH256S] * 10
    # NULL handle, algos, files
    assert decode_raw(mb, c, algos, files, sums, 0, 10, total, h=C.c_void_p()) == (INVALID, 0)
    assert decode_raw(mb, c, None, files, sums, 0, 10, total) == (INVALID, 0)
    assert decode_raw(mb, c, algos, None, sums, 0, 10, total) == (INVALID, 0)
    # mec_decode_prefer's range checks, in its order: the range before the empty read, the empty read before dst
    assert decode_raw(mb, c, algos, files, sums, -1, 10, total) == (INVALID, 0)
    assert decode_raw(mb, c, algos, files, sums, 0, -1, total) == (INVALID, 0)
    assert decode_raw(mb, c, algos, files, sums, total - 5, 6, total) == (INVALID, 0)
    assert decode_raw(mb, c, algos, files, sums, 5, 0, total, dst=False) == (0, 0)
    assert decode_raw(mb, c, algos, files, None, 5, 0, total) == (0, 0)
    assert decode_raw(mb, c, algos, files, sums, 0, 10, total, dst=False) == (INVALID, 0)
    # an algorithm that is no MEC_* bitrot value on a read drive; the same value on an offline drive is not read
    for bad in (0, 5, -1):
        assert decode_raw(mb, c, [bad] + algos[1:], files, sums, 0, 10, total) == (INVALID, 0)
    offline = [None] + files[1:]
    if mb.device_count() == 0:
        assert decode_raw(mb, c, [0] + algos[1:], offline, sums, 0, 10, total)[0] == NO_DEVICE
    # NULL sums beside a whole-file read drive; with every read drive streaming sums is not needed (reaches the device)
    assert decode_raw(mb, c, algos, files, None, 0, 10, total) == (INVALID, 0)
    # two whole-file algorithms among the read drives
    other = mb.SHA256 if wa != mb.SHA256 else mb.BLAKE2B512
    assert decode_raw(mb, c, [other] + algos[1:], files, sums, 0, 10, total) == (UNSUPPORTED, 0)
    # ... but not when the drive with the other algorithm is offline
    if mb.device_count() == 0:
        assert decode_raw(mb, c, [other] + algos[1:], offline, sums, 0, 10, total)[0] == NO_DEVICE
    # a codec of another algorithm
    for ca in (mb.SHA256, mb.HIGHWAYHASH256, mb.BLAKE2B512):
        w = mb.Codec(12, 4, MiB, ca)
        assert decode_raw(mb, w, algos, files, sums, 0, 10, total) == (UNSUPPORTED, 0)
        w.close()
    c.close()


def test_binding_refusals(mb):
    c = mb.Codec(4, 2, MiB)
    total = MiB
    files = mixed_files(c, total, 2)
    algos = [mb.SHA256] * 2 + [mb.HIGHWAYHASH256S] * 4
    with pytest.raises(mb.MecError) as ei:
        c.decode_mixed(files, algos, None, 0, 10, total)
    assert ei.value.code == INVALID
    with pytest.raises(mb.MecError) as ei:
        c.heal_mixed(files, [mb.SHA256, mb.BLAKE2B512] + algos[2:], [bytes(32)] * 6, [False] * 5 + [True], total)
    assert ei.value.code == UNSUPPORTED
    out, hint = c.decode_mixed(files, algos, None, 7, 0, total)
    assert out.size == 0 and hint == 0
    c.close()


@pytest.mark.parametrize("walgo", ["SHA256", "HIGHWAYHASH256", "BLAKE2B512"])
def test_heal_refusals_before_device_work(mb, walgo):
    wa = getattr(mb, walgo)
    c = mb.Codec(12, 4, MiB)
    total = 3 * MiB + 5
    files, sums = mixed_files(c, total, 6), np.zeros((16, 64), dtype=np.uint8)
    algos = [wa] * 6 + [mb.HIGHWAYHASH256S] * 10
    outs = [None] * 15 + [np.zeros(c.bitrot_file_size(total), dtype=np.uint8)]
    rc, corrupt = heal_raw(mb, c, algos, files, sums, total, outs, h=C.c_void_p())
    assert rc == INVALID
    for args in ((None, files, sums), (algos, None, sums)):
        rc, corrupt = heal_raw(mb, c, *args, total, outs)
        assert rc == INVALID and corrupt.all()  # refused before corrupt[] is touched
    rc, corrupt = heal_raw(mb, c, algos, files, sums, total, None)
    assert rc == INVALID and corrupt.all()
    # corrupt[] is cleared from here on
    rc, corrupt = heal_raw(mb, c, [9] + algos[1:], files, sums, total, outs)
    assert rc == INVALID and not corrupt.any()
    assert heal_raw(mb, c, algos, files, None, total, outs)[0] == INVALID
    other = mb.SHA256 if wa != mb.SHA256 else mb.HIGHWAYHASH256
    assert heal_raw(mb, c, [other] + algos[1:], files, sums, total, outs)[0] == UNSUPPORTED
    # a stale drive is never read: its algos[i] and files[i] are not looked at
    stale0 = [np.zeros(c.bitrot_file_size(total), dtype=np.uint8)] + [None] * 15
    if mb.device_count() == 0:
        assert heal_raw(mb, c, [9] + algos[1:], files, sums, total, stale0)[0] == NO_DEVICE
        assert heal_raw(mb, c, [other] + algos[1:], files, sums, total, stale0)[0] == NO_DEVICE
    # the empty part heals nothing
    for t in (0, -1):
        rc, corrupt = heal_raw(mb, c, algos, files, sums, t, outs)
        assert rc == 0 and not corrupt.any()
    # a codec of another algorithm
    w = mb.Codec(12, 4, MiB, wa)
    assert heal_raw(mb, w, algos, files, sums, total, outs)[0] == UNSUPPORTED
    w.close()
    c.close()


def test_no_cpu_fallback(mb):
    """A valid call without a CUDA device fails with MEC_ERR_NO_DEVICE: the part is never read through a CPU path."""
    if mb.device_count() > 0:
        pytest.skip("GPU present")
    c = mb.Codec(12, 4, 10 * MiB)
    total = 2 * MiB + 1
    files = mixed_files(c, total, 8)
    algos = [mb.BLAKE2B512] * 8 + [mb.HIGHWAYHASH256S] * 8
    with pytest.raises(mb.MecError) as ei:
        c.decode_mixed(files, algos, [bytes(64)] * 16, 0, total, total)
    assert ei.value.code == NO_DEVICE
    with pytest.raises(mb.MecError) as ei:
        c.heal_mixed(files, algos, [bytes(64)] * 16, [True] + [False] * 15, total)
    assert ei.value.code == NO_DEVICE
    c.close()
