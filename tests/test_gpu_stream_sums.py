"""mec_sums_device (stream_sums_kernel, obj_hash.cuh) against hashlib: MD5, SHA-1 and SHA-256 of many messages in device memory, one
thread per (message, algorithm).

Where the kernel changes behaviour: a message of fewer than 64 bytes is nothing but its padding block(s) (one below 56 bytes, two from
56 on); from 64 bytes on, the full blocks are read with 16-byte aligned loads realigned by the start's offset within its granule
(0..15, the whole-word part of the shift in two selects, the byte part in funnel shifts), with the next block's loads in flight
(a second block from 128 bytes on).  Lengths 0..257 cover every remainder class with zero to four full blocks; the long messages
cover long runs of prefetched blocks.  Items are sorted by (algorithm, length descending) on the host and run 32 to a CTA."""
import ctypes as C
import hashlib

import numpy as np
import pytest

MiB = 1 << 20
SUM_BYTES = 96
SLOTS = ((8, "md5", 0, 16), (16, "sha1", 32, 20), (32, "sha256", 64, 32))  # bit, hashlib name, offset in the record, length
FILL = 0xA5
LONG_LENS = [4095, 4096, 4097, 65535, 65536, 65537, MiB - 1, MiB + 1, 3 * MiB + 5]


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


@pytest.fixture(scope="module")
def buf():
    import torch
    host = np.random.default_rng(20261017).integers(0, 256, 4 * MiB + 8192, dtype=np.uint8)
    dev = torch.from_numpy(host).to("cuda")
    assert dev.data_ptr() % 256 == 0
    yield host, dev
    del dev
    torch.cuda.empty_cache()


def _messages():
    """(offset, length): every length 0..257 at start offsets cycling 0..15 (and every offset at several lengths), the long lengths
    at an aligned and a misaligned start, and an odd offset past 4 KiB"""
    msgs = [(1024 + 300 * n + n % 16, n) for n in range(258)]
    for off in range(16):
        for n in (1, 55, 56, 63, 64, 65, 127, 128, 129, 1000, 4097):
            msgs.append((100_000 + 5000 * off + off, n))
    for q, n in enumerate(LONG_LENS):
        msgs.append((0 if q % 2 else 7 + q, n))
    msgs += [(4099, 5000), (4099, 64), (4099, 0)]
    return msgs


def _record(host, off, n, which):
    rec = bytearray([FILL]) * SUM_BYTES
    for bit, name, o, ln in SLOTS:
        if which & bit:
            rec[o:o + ln] = hashlib.new(name, host[off:off + n].tobytes()).digest()
    return bytes(rec)


def _run(mb, dev, msgs, which):
    import torch
    c = mb.Codec(12, 4)
    out = torch.full((len(msgs) * SUM_BYTES,), FILL, dtype=torch.uint8, device="cuda")
    c.sums_device(dev.data_ptr(), [o for o, _ in msgs], [n for _, n in msgs], which, out.data_ptr(),
                  torch.cuda.current_stream().cuda_stream)
    got = out.cpu().numpy().tobytes()
    launches = c.launches
    c.close()
    return got, launches


@pytest.mark.gpu
@pytest.mark.parametrize("which", range(8, 64, 8))
def test_sums_device_every_mask(mb, buf, which):
    """one call per non-empty mask over all messages (far more than four warps of mixed lengths): every asked digest equals
    hashlib's, every other byte of every record keeps its guard value"""
    host, dev = buf
    msgs = _messages()
    assert len(msgs) > 4 * 32
    got, launches = _run(mb, dev, msgs, which)
    assert launches == 1
    bad = []
    for i, (off, n) in enumerate(msgs):
        if got[i * SUM_BYTES:(i + 1) * SUM_BYTES] != _record(host, off, n, which):
            bad.append((i, off, n))
    assert not bad, bad[:10]


@pytest.mark.gpu
def test_sums_device_empty_messages_and_null_base(mb):
    """zero-length messages need no base pointer and give the digests of the empty message"""
    import torch
    c = mb.Codec(4, 2)
    out = torch.full((3 * SUM_BYTES,), FILL, dtype=torch.uint8, device="cuda")
    c.sums_device(None, [0, 5, 1 << 40], [0, 0, 0], 56, out.data_ptr())
    got = out.cpu().numpy().tobytes()
    c.close()
    want = _record(np.zeros(0, dtype=np.uint8), 0, 0, 56)
    assert got == want * 3
    assert want[:16].hex() == "d41d8cd98f00b204e9800998ecf8427e"
    assert want[32:52].hex() == "da39a3ee5e6b4b0d3255bfef95601890afd80709"
    assert want[64:96].hex() == "e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855"


@pytest.mark.gpu
def test_sums_device_back_to_back_calls(mb, buf):
    """two calls on one handle without a synchronisation between them: the second refills the work table only after the first
    kernel has read it"""
    import torch
    host, dev = buf
    c = mb.Codec(12, 4)
    a = torch.full((64 * SUM_BYTES,), FILL, dtype=torch.uint8, device="cuda")
    b = torch.full((64 * SUM_BYTES,), FILL, dtype=torch.uint8, device="cuda")
    ma = [(q * 3, 70_000 + 17 * q) for q in range(64)]
    mb_ = [(q * 5 + 1, 1000 + q) for q in range(64)]
    st = torch.cuda.current_stream().cuda_stream
    c.sums_device(dev.data_ptr(), [o for o, _ in ma], [n for _, n in ma], 8, a.data_ptr(), st)
    c.sums_device(dev.data_ptr(), [o for o, _ in mb_], [n for _, n in mb_], 32, b.data_ptr(), st)
    ga, gb = a.cpu().numpy().tobytes(), b.cpu().numpy().tobytes()
    c.close()
    assert ga == b"".join(_record(host, o, n, 8) for o, n in ma)
    assert gb == b"".join(_record(host, o, n, 32) for o, n in mb_)


@pytest.mark.gpu
def test_sums_device_refusals(mb, buf):
    """every refusal returns MEC_ERR_INVALID_ARGUMENT before any device work: the records keep their guard bytes"""
    import torch
    _, dev = buf
    L = mb.lib()
    c = mb.Codec(12, 4)
    out = torch.full((2 * SUM_BYTES,), FILL, dtype=torch.uint8, device="cuda")
    offs = (C.c_int64 * 2)(0, 64)
    lens = (C.c_int64 * 2)(100, 200)
    d, o = dev.data_ptr(), out.data_ptr()
    launches = c.launches
    cases = {
        "null codec": L.mec_sums_device(None, 8, d, offs, lens, 2, o, None),
        "empty mask": L.mec_sums_device(c.h, 0, d, offs, lens, 2, o, None),
        "crc bits": L.mec_sums_device(c.h, 1, d, offs, lens, 2, o, None),
        "crc and sum bits": L.mec_sums_device(c.h, 8 | 4, d, offs, lens, 2, o, None),
        "unknown bit": L.mec_sums_device(c.h, 64, d, offs, lens, 2, o, None),
        "high bit": L.mec_sums_device(c.h, 8 | (1 << 30), d, offs, lens, 2, o, None),
        "negative mask": L.mec_sums_device(c.h, -1, d, offs, lens, 2, o, None),
        "negative count": L.mec_sums_device(c.h, 8, d, offs, lens, -1, o, None),
        "null offsets": L.mec_sums_device(c.h, 8, d, None, lens, 2, o, None),
        "null lens": L.mec_sums_device(c.h, 8, d, offs, None, 2, o, None),
        "null d_sums": L.mec_sums_device(c.h, 8, d, offs, lens, 2, None, None),
        "null base": L.mec_sums_device(c.h, 8, None, offs, lens, 2, o, None),
        "negative offset": L.mec_sums_device(c.h, 8, d, (C.c_int64 * 2)(0, -1), lens, 2, o, None),
        "negative length": L.mec_sums_device(c.h, 8, d, offs, (C.c_int64 * 2)(-5, 1), 2, o, None),
    }
    assert all(rc == -12 for rc in cases.values()), cases
    assert L.mec_sums_device(c.h, 8, None, None, None, 0, None, None) == 0  # nothing to do
    torch.cuda.synchronize()
    assert out.cpu().numpy().tobytes() == bytes([FILL]) * (2 * SUM_BYTES)
    assert c.launches == launches
    c.close()
