"""CPU-side checks of the server-side encryption entry points (DARE 2.0, AES-256-GCM; mec_dare_*, mec_encode_sse, mec_decode_sse):
the symbols are declared and exported with the wrappers' signatures, the size helpers follow sio.EncryptedSize / DecryptedSize,
the refusals that need no device, and the host DARE 2.0 reference (tests/dare_ref.py) against MinIO's own bytes: the SSE-C sealed
object key, the DerivePartKey vectors and the single-part rows of TestGetDecryptedRange.  The committed fixture is checked to be
what tests/golden/make_dare_fixtures.py makes."""
import base64
import ctypes as C
import hashlib
import json
import os
import re
import subprocess

import numpy as np
import pytest

import dare_ref as d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "dare_streams.json")
INVALID, NOT_AUTHENTIC = -12, -13
KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30
NAMES = ["mec_dare_encrypted_size", "mec_dare_decrypted_size", "mec_dare_device", "mec_encode_sse", "mec_decode_sse"]


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


@pytest.fixture(scope="module")
def fx():
    with open(FIXTURE) as f:
        return json.load(f)


def proto(name):
    hdr = open(os.path.join(ROOT, "include", "minio_ec.h")).read()
    m = re.search(r"\n(int64_t|int)\s+" + name + r"\(([^)]*)\);", hdr)
    assert m, name
    kinds = []
    for p in m.group(2).split(","):
        p = re.sub(r"/\*.*?\*/", "", p).strip()
        kinds.append("pointer" if ("*" in p or "[" in p) else {"int64_t": "int64", "int": "int"}[" ".join(p.split()[:-1])])
    return m.group(1), kinds


@pytest.mark.parametrize("name", NAMES)
def test_declared_exported_and_wrapped(mb, name):
    ret, kinds = proto(name)
    lib_path = mb.lib_path()
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    assert any(ln.split()[-1] == name for ln in out.splitlines())
    fn = getattr(mb.lib(), name)
    assert fn.restype is (C.c_int64 if ret == "int64_t" else C.c_int)
    got = ["int64" if a is C.c_int64 else "int" if a is C.c_int else "pointer" for a in fn.argtypes]
    assert got == kinds


@pytest.mark.parametrize("n", [0, 1, 15, 16, 17, 65535, 65536, 65537, 131072, 3 * 65536 + 5, MiB + 5, 5 * GiB, (1 << 48)])
def test_size_helpers(mb, n):
    L = mb.lib()
    e = L.mec_dare_encrypted_size(n)
    assert e == d.encrypted_size(n)
    assert L.mec_dare_decrypted_size(e) == n
    assert mb.capi.dare_encrypted_size(n) == e and mb.capi.dare_decrypted_size(e) == n


def test_size_helper_edges(mb):
    L = mb.lib()
    assert L.mec_dare_encrypted_size(0) == 0 and L.mec_dare_encrypted_size(1) == 33
    assert L.mec_dare_encrypted_size(65536) == 65568 and L.mec_dare_encrypted_size(65537) == 65601
    for r in range(1, 33):  # a remainder of 1..32 bytes holds no package
        for q in (0, 1, 7):
            assert L.mec_dare_decrypted_size(q * 65568 + r) == INVALID
            with pytest.raises(ValueError):
                d.decrypted_size(q * 65568 + r)
    assert L.mec_dare_decrypted_size(33) == 1 and L.mec_dare_decrypted_size(65568 + 33) == 65537
    assert L.mec_dare_encrypted_size(-1) == INVALID and L.mec_dare_decrypted_size(-1) == INVALID
    assert L.mec_dare_encrypted_size((1 << 48) + 1) == INVALID  # 2^32 packages at most: sequence numbers are uint32
    with pytest.raises(mb.MecError) as e:
        mb.capi.dare_decrypted_size(65568 + 32)
    assert e.value.code == INVALID


def test_refusals_without_device_work(mb):
    """what mec_dare_device, mec_encode_sse and mec_decode_sse refuse is refused before the device is touched"""
    L = mb.lib()
    c = mb.Codec(12, 4, MiB)
    key, nonce = np.zeros(32, np.uint8), np.zeros(12, np.uint8)
    i64 = lambda *v: (C.c_int64 * len(v))(*v)  # noqa: E731
    seq = (C.c_uint32 * 1)(0)
    st = (C.c_uint8 * 1)(99)
    dev = C.c_void_p(16)
    args = dict(c=c.h, op=1, ns=1, keys=key.ctypes.data, nonces=nonce.ctypes.data, seq=seq, tot=i64(33), din=dev, ino=i64(0),
                lens=i64(10), dout=dev, outo=i64(0), st=st, stream=None)

    def call(**kw):
        a = dict(args, **kw)
        return L.mec_dare_device(a["c"], a["op"], a["ns"], a["keys"], a["nonces"], a["seq"], a["tot"], a["din"], a["ino"], a["lens"],
                                 a["dout"], a["outo"], a["st"], a["stream"])

    assert call(c=None) == INVALID
    assert call(op=3) == INVALID and call(op=0) == INVALID
    assert call(ns=-1) == INVALID
    assert call(ns=0, keys=None) == 0  # nothing to do
    assert call(keys=None) == INVALID and call(seq=None) == INVALID and call(st=None) == INVALID
    assert call(nonces=None) == INVALID                # seal needs the nonces
    assert call(op=2, tot=None) == INVALID             # open needs the stored sizes
    assert call(lens=i64(-1)) == INVALID and call(ino=i64(-5)) == INVALID and call(outo=i64(-5)) == INVALID
    assert call(din=None) == INVALID and call(dout=None) == INVALID
    assert call(seq=(C.c_uint32 * 1)(0xFFFFFFFF), lens=i64(2 * 65536)) == INVALID  # past sequence number 2^32 - 1
    assert st[0] == 99

    files = [np.zeros(64, np.uint8) for _ in range(16)]
    src = np.zeros(10, np.uint8)
    ptrs = (C.c_void_p * 16)(*[f.ctypes.data for f in files])
    assert L.mec_encode_sse(c.h, src.ctypes.data, 10, None, nonce.ctypes.data, ptrs, 0) == INVALID
    assert L.mec_encode_sse(c.h, src.ctypes.data, 10, key.ctypes.data, None, ptrs, 0) == INVALID
    assert L.mec_encode_sse(c.h, src.ctypes.data, -1, key.ctypes.data, nonce.ctypes.data, ptrs, 0) == INVALID
    assert L.mec_encode_sse(c.h, src.ctypes.data, 10, key.ctypes.data, nonce.ctypes.data, ptrs, 17) == -11  # write quorum
    assert L.mec_encode_sse(c.h, None, 0, key.ctypes.data, nonce.ctypes.data, ptrs, 0) == 0

    hint = C.c_int(5)
    dst = np.zeros(16, np.uint8)
    dec = lambda off, ln, tot, k=key.ctypes.data: L.mec_decode_sse(c.h, ptrs, None, off, ln, tot, k, dst.ctypes.data, C.byref(hint))  # noqa: E731
    assert dec(0, 1, 33, k=None) == INVALID and hint.value == 0
    assert dec(0, 1, 20) == NOT_AUTHENTIC         # a stored size that is no DARE size: errObjectTampered
    assert dec(0, 2, 33) == INVALID               # beyond the plaintext
    assert dec(-1, 1, 33) == INVALID
    assert dec(1, 0, 33) == 0
    with pytest.raises(mb.MecError) as e:
        c.decode_sse(files, 0, 1, 65568 + 16, key)
    assert e.value.code == NOT_AUTHENTIC and "NotAuthentic" in str(e.value)
    c.close()


def test_sealed_key_vector(fx):
    """MinIO's SSE-C sealed object key is a one-package DARE 2.0 stream: it opens to the object key under exactly this layout, and
    fails with no additional data or with the whole header as additional data"""
    pytest.importorskip("cryptography")
    from cryptography.exceptions import InvalidTag
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
    s = fx["sealed_key"]
    key = d.ssec_sealing_key(base64.b64decode(s["client_key"]), base64.b64decode(s["iv"]), s["bucket"], s["object"])
    assert key.hex() == s["sealing_key"]
    pkg = base64.b64decode(s["sealed_key"])
    assert len(pkg) == d.encrypted_size(32) and pkg[0] == 0x20 and pkg[1] == 0 and pkg[2:4] == b"\x1f\x00" and pkg[4] & 0x80
    assert d.open_stream(key, pkg).hex() == s["object_key"]
    g = AESGCM(key)
    for aad in (None, pkg[:16]):
        with pytest.raises(InvalidTag):
            g.decrypt(d.aead_nonce(pkg[:16], 0), pkg[16:], aad)
    assert d.seal(key, pkg[4:16], bytes.fromhex(s["object_key"])) == pkg  # the same bytes back from the plaintext


def test_part_keys(fx):
    for v in fx["part_keys"]:
        assert d.derive_part_key(bytes(32), v["part"]).hex() == v["key"]


@pytest.mark.parametrize("size", [0, 1, 64 * KiB - 1, 64 * KiB, 128 * KiB - 1, 5 * MiB, 5 * GiB])
def test_decrypted_range_single_part(size):
    """the single-part rows of TestGetDecryptedRange (cmd/encryption-v1_test.go): whole object, first 10 bytes, 64 KiB after
    32 KiB, 64 KiB after 96 KiB"""
    pkg = 64 * KiB
    esz = d.encrypted_size(size)
    if size > 0:
        assert d.decrypted_range(size, 0, size) == (0, esz, 0, 0)
    if size >= 10:
        assert d.decrypted_range(size, 0, 10) == (0, (pkg + 32) if size >= pkg else size + 32, 0, 0)
    if size >= 96 * KiB:
        rlen = (pkg + 32) * 2 if size >= 2 * pkg else (pkg + 32) + (size - pkg + 32)
        assert d.decrypted_range(size, 32 * KiB, 64 * KiB) == (0, rlen, 32 * KiB, 0)
    if size >= 160 * KiB:
        rlen = (pkg + 32) * 2 if size - pkg >= 2 * pkg else (pkg + 32) + (size - pkg + 64)
        assert d.decrypted_range(size, 96 * KiB, 64 * KiB) == (pkg + 32, rlen, 32 * KiB, 1)


def test_fixture_is_reproducible(fx):
    """every fixture stream is what the host reference seals (and opens back)"""
    pytest.importorskip("cryptography")
    for s in fx["streams"]:
        pt = d.plaintext(s["length"], s["seed"]).tobytes()
        st = d.seal(bytes.fromhex(s["key"]), bytes.fromhex(s["nonce"]), pt, s["seq0"])
        assert hashlib.sha256(st).hexdigest() == s["sha256"]
        assert all(s[f] == v for f, v in d.excerpts(st).items())
        assert d.open_stream(bytes.fromhex(s["key"]), st, s["seq0"]) == pt
