"""CPU-side checks of the object-hash entry points (mec_sums_device, mec_batcher_encode_sums): a NULL batcher and bad masks return
MEC_ERR_INVALID_ARGUMENT before anything else, the header's MEC_SUM_* constants are the binding's, and stream_sums_kernel compiles
for sm_90a without spilling."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARGUMENT = -12


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


def _header_defines():
    with open(os.path.join(ROOT, "include", "minio_ec.h")) as f:
        return {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(MEC_\w+)\s+(\d+)", f.read())}


def test_header_constants_match_binding(mb):
    d = _header_defines()
    cap = mb.capi
    assert (d["MEC_SUM_MD5"], d["MEC_SUM_SHA1"], d["MEC_SUM_SHA256"], d["MEC_SUM_BYTES"]) == \
        (cap.SUM_MD5, cap.SUM_SHA1, cap.SUM_SHA256, cap.SUM_BYTES)
    assert (d["MEC_CRC32"], d["MEC_CRC32C"], d["MEC_CRC64NVME"]) == (cap.CRC32, cap.CRC32C, cap.CRC64NVME)
    # the record layout: MD5 at +0, SHA-1 at +32, SHA-256 at +64, each inside the record
    assert cap.SUM_SLOTS == {"md5": (8, 0, 16), "sha1": (16, 32, 20), "sha256": (32, 64, 32)}
    assert all(o + n <= cap.SUM_BYTES for _, o, n in cap.SUM_SLOTS.values())


def test_batcher_encode_sums_refusals(mb):
    L = mb.lib()
    files = (C.c_void_p * 16)()
    crc3 = (C.c_uint64 * 3)()
    rec = (C.c_uint8 * 96)()
    src = (C.c_uint8 * 10)()
    for which in (0, 7, 8, 56, 63):  # a NULL batcher, whatever the mask
        assert L.mec_batcher_encode_sums(None, src, 10, files, None, 0, which, crc3, rec) == INVALID_ARGUMENT
    for which in (64, 128, 63 | 64, 1 << 30, -1):  # unknown bits, refused before the batcher is looked at
        assert L.mec_batcher_encode_sums(None, src, 10, files, None, 0, which, crc3, rec) == INVALID_ARGUMENT
    # a set bit with a NULL destination
    assert L.mec_batcher_encode_sums(None, src, 10, files, None, 0, 8, crc3, None) == INVALID_ARGUMENT
    assert L.mec_batcher_encode_sums(None, src, 10, files, None, 0, 1, None, rec) == INVALID_ARGUMENT
    assert list(crc3) == [0, 0, 0] and bytes(rec) == bytes(96)


def test_sums_device_refusals_without_device_work(mb):
    L = mb.lib()
    c = mb.Codec(12, 4)
    offs = (C.c_int64 * 1)(0)
    lens = (C.c_int64 * 1)(10)
    base, out = C.c_void_p(16), C.c_void_p(4096)  # never dereferenced: every call below is refused first
    assert L.mec_sums_device(None, 8, base, offs, lens, 1, out, None) == INVALID_ARGUMENT
    for which in (0, 1, 2, 4, 7, 64, 8 | 64, -8):
        assert L.mec_sums_device(c.h, which, base, offs, lens, 1, out, None) == INVALID_ARGUMENT, which
    assert L.mec_sums_device(c.h, 8, base, offs, lens, -1, out, None) == INVALID_ARGUMENT
    assert L.mec_sums_device(c.h, 8, base, None, lens, 1, out, None) == INVALID_ARGUMENT
    assert L.mec_sums_device(c.h, 8, base, offs, None, 1, out, None) == INVALID_ARGUMENT
    assert L.mec_sums_device(c.h, 8, base, offs, lens, 1, None, None) == INVALID_ARGUMENT
    assert L.mec_sums_device(c.h, 8, None, offs, lens, 1, out, None) == INVALID_ARGUMENT
    assert L.mec_sums_device(c.h, 56, None, None, None, 0, None, None) == 0
    c.close()


def test_stream_sums_kernel_does_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = tmp_path / "k.cu"
    src.write_text('#include "obj_hash.cuh"\n')
    p = subprocess.run([nvcc, "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-cubin", "-Xptxas", "-v",
                        "-I" + os.path.join(ROOT, "minio_b200", "csrc"), str(src), "-o", str(tmp_path / "k.cubin")],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    lines = p.stderr.splitlines()
    at = [i for i, ln in enumerate(lines) if "Function properties for" in ln and "stream_sums_kernel" in ln]
    assert at, p.stderr[-3000:]
    props = lines[at[0] + 1]
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props, props
