"""CPU-side checks of the Signature V4 streaming entry points (mec_encode_chunked, mec_chunk_signatures_device): the header's codes
are the binding's, the Python reference reproduces AWS's published chunked-upload example, every refusal comes in its order before
any device work (so is an error in the first chunk's header, which no signature precedes), and sigv4_chunk_kernel compiles for
sm_90a without spilling."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import sigv4_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARGUMENT, WRITE_QUORUM = -12, -11
KEY = ref.signing_key("wJalrXUtnFEMI/K7MDENG/bPxRfiCYEXAMPLEKEY")
SEED = b"4f232c4386841ef735655705268965c44a0e4690baa4adea153f7db9fa80a0a9"
SCOPE = ref.scope_of()


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


def test_header_constants_match_binding(mb):
    with open(os.path.join(ROOT, "include", "minio_ec.h")) as f:
        hdr = f.read()
    codes = {m.group(1): int(m.group(2)) for m in re.finditer(r"(MEC_ERR_\w+)\s*=\s*(-?\d+)", hdr)}
    cap = mb.capi
    assert (codes["MEC_ERR_SIGNATURE_MISMATCH"], codes["MEC_ERR_MALFORMED_ENCODING"], codes["MEC_ERR_CHUNK_TOO_BIG"],
            codes["MEC_ERR_INCOMPLETE_BODY"], codes["MEC_ERR_OVERREAD"]) == \
        (cap.SIGNATURE_MISMATCH, cap.MALFORMED_ENCODING, cap.CHUNK_TOO_BIG, cap.INCOMPLETE_BODY, cap.OVERREAD) == \
        (ref.SIGNATURE_MISMATCH, ref.MALFORMED_ENCODING, ref.CHUNK_TOO_BIG, ref.INCOMPLETE_BODY, ref.OVERREAD)
    assert len(set(codes.values())) == len(codes), "every MEC_ERR_* code is distinct"
    defs = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(MEC_SIGV4_\w+)\s+(\d+)", hdr)}
    assert (defs["MEC_SIGV4_PAYLOAD"], defs["MEC_SIGV4_TRAILER"]) == (cap.SIGV4_PAYLOAD, cap.SIGV4_TRAILER)
    assert all(c in cap.ERRORS for c in (-14, -15, -16, -17, -18))


def test_reference_reproduces_aws_example():
    with open(os.path.join(ROOT, "tests", "golden", "sigv4_aws_example.json")) as f:
        ex = json.load(f)
    key = ref.signing_key(ex["secret_key"], ex["date"], ex["region"])
    body = ref.build(b"a" * ex["payload_len"], ex["chunk_sizes"], key, ex["seed_signature"].encode(), ex["date"],
                     ref.scope_of(ex["date"], ex["region"]))
    assert [c["sigval"].decode() for c in body.chunks] == ex["chunk_signatures"]
    code, out, _ = ref.read(body.data, ex["payload_len"], key, ex["seed_signature"].encode(), ex["date"])
    assert code == ref.OK and out == b"a" * ex["payload_len"]


def test_reference_reader_quirks():
    """the serial reader's verdicts the GPU tests rely on, on bodies small enough to reason about by hand"""
    data = bytes(range(200))
    b = ref.build(data, [100, 100], KEY, SEED)
    assert ref.read(b.data, 200, KEY, SEED) == (ref.OK, data, None)
    assert ref.read(b.data, 199, KEY, SEED)[0] == ref.OVERREAD
    assert ref.read(b.data, 201, KEY, SEED)[0] == ref.INCOMPLETE_BODY
    s, _ = b.chunks[0]["crlf2"]
    assert ref.read(b.cut(s), 200, KEY, SEED)[0] == ref.MALFORMED_ENCODING      # the '\r' behind a payload cut off
    assert ref.read(b.cut(s + 1), 200, KEY, SEED)[0] == ref.INCOMPLETE_BODY     # ... its '\n' cut off
    t = ref.build(data, [200], KEY, SEED, trailer=b"x-amz-checksum-crc32:AAAAAA==")
    assert ref.read(t.data, 200, KEY, SEED, trailer=True) == (ref.OK, data, b"x-amz-checksum-crc32:AAAAAA==\n")
    e, _ = t.trailer["end"]
    assert ref.read(t.cut(e + 1), 200, KEY, SEED, trailer=True)[0] == ref.INCOMPLETE_BODY
    assert ref.read(t.cut(e + 2), 200, KEY, SEED, trailer=True)[0] == ref.MALFORMED_ENCODING
    assert ref.go_trim_space(b" \t\xc2\xa0ab\xe3\x80\x80\r\n") == b"ab"


def _call(mb, codec, body, D, key=KEY, seed=SEED, date=ref.DATE, scope=SCOPE, trailer=0, files=None, wq=0, tcap=0, tlen=True):
    L = mb.lib()
    b = np.frombuffer(bytes(body), dtype=np.uint8) if body is not None else None
    fa = (C.c_void_p * 16)(*([1] * 16)) if files is None else files  # never dereferenced: every call below stops first
    n = C.c_int64(-5)
    rc = L.mec_encode_chunked(codec, None if b is None or not b.size else b.ctypes.data, 0 if b is None else b.size, D,
                              None if key is None else key, None if seed is None else seed,
                              None if date is None else date.encode(), None if scope is None else scope.encode(),
                              trailer, fa, wq, None, tcap, C.byref(n) if tlen else None)
    return rc, n.value


def test_encode_chunked_refusals_in_order(mb):
    c = mb.Codec(12, 4)
    good = bytes(ref.build(b"x" * 10, [10], KEY, SEED).data)
    assert _call(mb, None, good, 10)[0] == INVALID_ARGUMENT
    for kw in ({"key": None}, {"seed": None}, {"date": None}, {"scope": None}):
        assert _call(mb, c.h, good, 10, **kw)[0] == INVALID_ARGUMENT, kw
    assert _call(mb, c.h, good, -1)[0] == INVALID_ARGUMENT
    L = mb.lib()
    fa = (C.c_void_p * 16)(*([1] * 16))
    assert L.mec_encode_chunked(c.h, None, 5, 10, KEY, SEED, b"d", b"s", 0, fa, 0, None, 0, None) == INVALID_ARGUMENT
    assert L.mec_encode_chunked(c.h, good, -1, 10, KEY, SEED, b"d", b"s", 0, None, 0, None, 0, None) == INVALID_ARGUMENT
    assert L.mec_encode_chunked(c.h, good, len(good), 10, KEY, SEED, b"d", b"s", 0, None, 0, None, 0, None) == INVALID_ARGUMENT
    # the seed: exactly 64 lowercase hex bytes
    for seed in (SEED.upper(), SEED[:63] + b"g", b"z" * 64, SEED[:63] + b"\0"):
        assert _call(mb, c.h, good, 10, seed=seed)[0] == INVALID_ARGUMENT, seed
    # date "\n" scope "\n" must fit the 256-byte head
    assert _call(mb, c.h, good, 10, scope="s" * 239)[0] == INVALID_ARGUMENT
    # trailer mode needs trailer_len, and a buffer when it has a capacity
    assert _call(mb, c.h, good, 10, trailer=1, tlen=False)[0] == INVALID_ARGUMENT
    assert _call(mb, c.h, good, 10, trailer=1, tcap=8)[0] == INVALID_ARGUMENT
    assert _call(mb, c.h, good, 10, trailer=1, tcap=-1)[0] == INVALID_ARGUMENT
    # an argument error wins over the write quorum, which wins over the body
    off = (C.c_void_p * 16)(*([None] * 8 + [1] * 8))
    assert _call(mb, c.h, good, 10, seed=SEED.upper(), files=off, wq=9)[0] == INVALID_ARGUMENT
    assert _call(mb, c.h, b"zz", 10, files=off, wq=9)[0] == WRITE_QUORUM
    assert _call(mb, c.h, b"zz", 10, files=off, wq=8)[0] == ref.MALFORMED_ENCODING
    assert c.stat("launches") == 0
    c.close()


FIRST_HEADER = [
    (b"", ref.INCOMPLETE_BODY),
    (b"1", ref.INCOMPLETE_BODY),
    (b"1g;", ref.MALFORMED_ENCODING),
    (b" 10;", ref.MALFORMED_ENCODING),
    (b"1000001;", ref.CHUNK_TOO_BIG),                 # 16 MiB + 1
    (b"10000000000", ref.CHUNK_TOO_BIG),              # as soon as it is exceeded, mid-digit and before any ';'
    (b"00000000000001000001;", ref.CHUNK_TOO_BIG),
    (b"10;chunk-signature=" + b"0" * 63, ref.INCOMPLETE_BODY),
    (b"10;chunk-signaturE=" + b"0" * 64 + b"\r\n", ref.MALFORMED_ENCODING),
    (b"10;chunk-signature=" + b"0" * 64, ref.INCOMPLETE_BODY),
    (b"10;chunk-signature=" + b"0" * 64 + b"\r", ref.INCOMPLETE_BODY),
    (b"10;chunk-signature=" + b"0" * 64 + b"\n\n", ref.MALFORMED_ENCODING),
    (b"10;chunk-signature=" + b"0" * 64 + b"\r\r", ref.MALFORMED_ENCODING),
    (b"10;chunk-signature=" + b"0" * 64 + b"\r\n" + b"x" * 15, ref.INCOMPLETE_BODY),
]


@pytest.mark.parametrize("body,code", FIRST_HEADER)
def test_first_header_errors_need_no_device(mb, body, code):
    """no signature precedes an error in the first chunk's header: the call returns it at once, as the serial reader does"""
    assert ref.read(body, 16, KEY, SEED)[0] == code
    c = mb.Codec(12, 4)
    assert _call(mb, c.h, body, 16)[0] == code
    assert c.stat("launches") == 0 and c.stat("sigv4_chunks") == 0
    with pytest.raises(mb.MecError) as ei:
        c.encode_chunked(body, 16, KEY, SEED, ref.DATE, SCOPE)
    assert ei.value.code == code
    c.close()


def test_chunk_signatures_device_refusals(mb):
    L = mb.lib()
    c = mb.Codec(12, 4)
    offs, lens = (C.c_int64 * 1)(0), (C.c_int64 * 1)(10)
    sig = (C.c_uint8 * 64)()
    kinds, out = (C.c_int32 * 1)(0), (C.c_uint8 * 1)(7)
    base = C.c_void_p(16)  # never dereferenced
    args = dict(key=KEY, date=ref.DATE.encode(), scope=SCOPE.encode(), base=base, offs=offs, lens=lens, prev=sig, claim=sig, kinds=kinds,
                count=1, out=out)

    def call(h=c.h, **kw):
        a = dict(args, **kw)
        return L.mec_chunk_signatures_device(h, a["key"], a["date"], a["scope"], a["base"], a["offs"], a["lens"], a["prev"],
                                             a["claim"], a["kinds"], a["count"], a["out"], None)
    assert call(h=None) == INVALID_ARGUMENT
    for name in ("key", "date", "scope", "offs", "lens", "prev", "claim", "kinds", "out"):
        assert call(**{name: None}) == INVALID_ARGUMENT, name
    assert call(base=None) == INVALID_ARGUMENT
    assert call(count=-1) == INVALID_ARGUMENT
    assert call(scope=b"s" * 239) == INVALID_ARGUMENT
    assert call(offs=(C.c_int64 * 1)(-1)) == INVALID_ARGUMENT
    assert call(lens=(C.c_int64 * 1)(-1)) == INVALID_ARGUMENT
    for k in (2, -1):
        assert call(kinds=(C.c_int32 * 1)(k)) == INVALID_ARGUMENT
    assert call(count=0, offs=None, lens=None, prev=None, claim=None, kinds=None, out=None) == 0
    assert out[0] == 7 and c.stat("launches") == 0
    with pytest.raises(mb.MecError):
        c.chunk_signatures_device(KEY, ref.DATE, SCOPE, 16, [0], [-1], [SEED], [SEED], [0])
    c.close()


def test_sigv4_chunk_kernel_does_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = tmp_path / "k.cu"
    src.write_text('#include "sigv4.cuh"\n')
    p = subprocess.run([nvcc, "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-cubin", "-Xptxas", "-v",
                        "-I" + os.path.join(ROOT, "minio_b200", "csrc"), str(src), "-o", str(tmp_path / "k.cubin")],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    log = p.stderr
    i = log.index("sigv4_chunk_kernel")
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log[i:])
    assert m and m.group(1) == "0" and m.group(2) == "0", log
