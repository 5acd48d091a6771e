"""CPU-side checks of DARE 2.0 ChaCha20-Poly1305 (cipher 1): the pure-Python reference (tests/chacha_ref.py) against RFC 8439's
AEAD example, the committed fixture streams and, where it is installed, `cryptography`; the device building blocks of chacha.cuh
(block function and Poly1305 field arithmetic) run on the host by tests/cpp/test_chacha against Python integers and the reference;
and option "dare_chacha20" / mec_batcher_set_option refusals, which need no device."""
import ctypes as C
import hashlib
import json
import os
import random
import subprocess

import numpy as np
import pytest

import chacha_ref as cr
import dare_ref as d
from test_batcher_mixed_bitrot_abi import header_params

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
INVALID = -12
P = (1 << 130) - 5
M128 = (1 << 128) - 1


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    return minio_b200


@pytest.fixture(scope="module")
def fx():
    with open(os.path.join(HERE, "golden", "dare_chacha_streams.json")) as f:
        return json.load(f)["streams"]


# ---- the Python reference ------------------------------------------------------------------------------------------------------
def test_rfc8439_aead_vector():
    """RFC 8439 §2.8.2"""
    key = bytes(range(0x80, 0xA0))
    nonce = bytes.fromhex("070000004041424344454647")
    aad = bytes.fromhex("50515253c0c1c2c3c4c5c6c7")
    pt = (b"Ladies and Gentlemen of the class of '99: If I could offer you only one tip for the future, sunscreen would be it.")
    assert len(pt) == 114
    sealed = cr.aead_seal(key, nonce, pt, aad)
    assert sealed[:16].hex() == "d31a8d34648e60db7b86afbc53ef7ec2"
    assert sealed[-16:].hex() == "1ae10b594f09e26a7e902ecbd0600691"
    assert cr.aead_open(key, nonce, sealed, aad) == pt
    assert cr.aead_open(key, nonce, sealed[:-1] + bytes([sealed[-1] ^ 1]), aad) is None


def test_rfc8439_block_vector():
    """RFC 8439 §2.3.2: the serialized block starts 10 f1 e7 e4 and ends 4e"""
    blk = cr.chacha20_blocks(bytes(range(32)), bytes.fromhex("000000090000004a00000000"), 1, 1).tobytes()
    assert blk[:4].hex() == "10f1e7e4" and blk[-4:].hex() == "a2503c4e"


def test_fixture_lengths(fx):
    lengths = {s["length"] for s in fx}
    for n in [1, 15, 16, 17, 63, 64, 65, 65535, 65536, 65537, 3 * 65536 + 5, (1 << 20) + 5]:
        assert n in lengths
    for T in (255, 256, 257, 512, 513):
        assert 16 * (T - 2) in lengths and 16 * (T - 2) - 7 in lengths
    assert any(s["seq0"] for s in fx)


def test_reference_reproduces_fixture(fx):
    for s in fx:
        key, nonce = bytes.fromhex(s["key"]), bytes.fromhex(s["nonce"])
        pt = d.plaintext(s["length"], s["seed"]).tobytes()
        st = cr.seal_chacha(key, nonce, pt, s["seq0"])
        assert hashlib.sha256(st).hexdigest() == s["sha256"], s["length"]
        assert d.excerpts(st) == {f: s[f] for f in ("first_head", "first_tag", "last_head", "last_tag")}
        assert st[1] == 1 and len(st) == d.encrypted_size(s["length"])
        assert cr.open_chacha(key, st, s["seq0"]) == pt
        if s["seq0"]:
            with pytest.raises(ValueError):
                cr.open_chacha(key, st, 0)


def test_reference_against_cryptography():
    ccp = pytest.importorskip("cryptography.hazmat.primitives.ciphers.aead")
    rng = random.Random(7)
    for _ in range(40):
        n = rng.choice([rng.randrange(0, 200), rng.randrange(0, 5000), rng.randrange(60000, 70000)])
        key, nonce, aad = rng.randbytes(32), rng.randbytes(12), rng.randbytes(rng.choice([0, 4, 13]))
        pt = rng.randbytes(n)
        assert cr.aead_seal(key, nonce, pt, aad) == ccp.ChaCha20Poly1305(key).encrypt(nonce, pt, aad), n


# ---- chacha.cuh's building blocks on the host ----------------------------------------------------------------------------------
def value(limbs):
    return sum(int(x) << (26 * i) for i, x in enumerate(limbs))


def words(ws):
    return sum(int(x) << (32 * i) for i, x in enumerate(ws))


@pytest.fixture(scope="module")
def host_run():
    exe = os.path.join(HERE, "cpp", "test_chacha")
    assert os.path.exists(exe), "tests/cpp/test_chacha is built by __graft_entry__.build()"
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = out.stdout.split("\n")
    assert "done" in lines
    cases = {}
    for ln in lines:
        f = ln.split()
        if f and f[0] != "done":
            cases.setdefault(f[0], []).append([int(x) for x in f[1:]])
    return cases


def test_field_mul_and_add(host_run):
    assert len(host_run["mul"]) > 2000 and len(host_run["add"]) > 2000
    for op in ("mul", "add"):
        for v in host_run[op]:
            a, b, r = v[0:5], v[5:10], v[10:15]
            assert max(a + b) < 1 << 28
            want = value(a) * value(b) if op == "mul" else value(a) + value(b)
            assert value(r) % P == want % P, (op, a, b, r)
            assert r[1] < (1 << 26) + (1 << 13) and all(x < 1 << 26 for x in r[:1] + r[2:]), (op, r)


def test_field_finish(host_run):
    crafted = {P - 1, P, P + 1, (1 << 130) - 1}
    seen = set()
    for v in host_run["fin"]:
        a, s, t = v[0:5], v[5:9], v[9:13]
        seen.add(value(a))
        assert words(t) == (value(a) % P + words(s)) & M128, (a, s)
    assert crafted <= seen  # the final subtraction of acc >= p, which random data almost never reaches


def test_clamp(host_run):
    for v in host_run["clamp"]:
        k, r = v[0:4], v[4:9]
        assert value(r) == words(k) & 0x0FFFFFFC0FFFFFFC0FFFFFFC0FFFFFFF and all(x < 1 << 26 for x in r)


def test_block_function(host_run):
    assert len(host_run["blk"]) == 200
    for v in host_run["blk"]:
        key, ctr, nonce, out = v[0:8], v[8], v[9:12], v[12:28]
        kb = np.array(key, dtype="<u4").tobytes()
        nb = np.array(nonce, dtype="<u4").tobytes()
        want = cr.chacha20_blocks(kb, nb, ctr, 1).tobytes()
        assert np.array(out, dtype="<u4").tobytes() == want
    first = np.array(host_run["blk"][0][12:28], dtype="<u4").tobytes()
    assert first[:4].hex() == "10f1e7e4"  # RFC 8439 §2.3.2


# ---- the option and mec_batcher_set_option -------------------------------------------------------------------------------------
def test_codec_option_values(mb):
    c = mb.Codec(12, 4, 1 << 20)
    assert c.stat("dare_chacha20") == 0  # the default
    for v in (1, 2, 0, 2):
        c.set_option("dare_chacha20", v)
        assert c.stat("dare_chacha20") == v
    for bad in (3, -1, 1 << 40):
        with pytest.raises(mb.MecError) as e:
            c.set_option("dare_chacha20", bad)
        assert e.value.code == INVALID and c.stat("dare_chacha20") == 2
    c.close()


def test_batcher_set_option_declared_exported_wrapped(mb):
    ret, params = header_params("mec_batcher_set_option")
    assert ret == "int" and params == ["mec_batcher*", "const char*", "int64_t"]
    out = subprocess.run(["nm", "-D", "--defined-only", mb.lib_path()], capture_output=True, text=True, check=True).stdout
    assert "mec_batcher_set_option" in {ln.split()[-1] for ln in out.splitlines() if ln.strip()}
    fn = mb.lib().mec_batcher_set_option
    assert fn.restype is C.c_int and fn.argtypes == [C.c_void_p, C.c_char_p, C.c_int64]
    assert callable(mb.Batcher.set_option)


def test_batcher_set_option_refusals(mb):
    L = mb.lib()
    for name, v in [(b"dare_chacha20", 1), (b"dare_chacha20", 0), (None, 1), (b"eb", 1), (b"dare_chacha20", 3)]:
        assert L.mec_batcher_set_option(None, name, v) == INVALID
    bat = object.__new__(mb.Batcher)  # a closed batcher: the wrapper reaches the NULL-batcher refusal
    bat.h = None
    with pytest.raises(mb.MecError) as e:
        bat.set_option("dare_chacha20", 1)
    assert e.value.code == INVALID
