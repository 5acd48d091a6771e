"""CPU-side checks of mec_reconstruct_frames: malformed arguments — a last shard length outside [0, S] among them — are refused
before any device work, without touching corrupt[] or the outputs, and a valid call without a GPU fails with MEC_ERR_NO_DEVICE."""
import ctypes as C

import numpy as np
import pytest

MARK = 0xA5


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


def raw_reconstruct(mb, c, frames, nblocks, last, want, outs, corrupt):
    """-> return code; frames / want / outs None pass NULL"""
    return mb.lib().mec_reconstruct_frames(c.h, None if frames is None else mb.capi._ptrs(frames), nblocks, last,
                                           None if want is None else want.ctypes.data, 0,
                                           None if outs is None else mb.capi._ptrs(outs), corrupt.ctypes.data)


def test_refusals_before_device_work(mb):
    c = mb.Codec(12, 4)
    S = c.shard_size()
    files = [np.zeros(2 * (32 + S), dtype=np.uint8) for _ in range(c.n)]
    outs = [np.full(2 * (32 + S), MARK, dtype=np.uint8) for _ in range(c.n)]
    want = np.zeros(c.n, dtype=np.uint8)
    want[1] = 1
    corrupt = np.full(c.n, MARK, dtype=np.uint8)
    for last in (-1, -S, S + 1, 1 << 40):   # a last shard length outside [0, S]
        assert raw_reconstruct(mb, c, files, 2, last, want, outs, corrupt) == -12, last
        assert raw_reconstruct(mb, c, files, 0, last, want, outs, corrupt) == -12, last
    assert raw_reconstruct(mb, c, files, -1, 0, want, outs, corrupt) == -12
    assert raw_reconstruct(mb, c, None, 2, 0, want, outs, corrupt) == -12
    assert raw_reconstruct(mb, c, files, 2, 0, None, outs, corrupt) == -12
    assert raw_reconstruct(mb, c, files, 2, 0, want, None, corrupt) == -12
    assert (corrupt == MARK).all() and all((o == MARK).all() for o in outs)
    with pytest.raises(mb.MecError) as ei:
        c.reconstruct_frames(files, 2, -1, want)
    assert ei.value.code == -12
    c.close()


def test_no_cpu_fallback(mb):
    """Valid arguments without a CUDA device: MEC_ERR_NO_DEVICE, never a CPU rebuild."""
    if mb.device_count() > 0:
        pytest.skip("GPU present")
    c = mb.Codec(12, 4)
    S = c.shard_size()
    files = [np.zeros(2 * (32 + S), dtype=np.uint8) for _ in range(c.n)]
    for last in (0, 1, S):
        with pytest.raises(mb.MecError) as ei:
            c.reconstruct_frames(files, 2, last, [0, 1] + [0] * 14)
        assert ei.value.code == -101
    c.close()
