"""Server-side encryption through the cross-request coalescer (mec_batcher_encode_sse / mec_batcher_decode_sse), on the GPU.  The oracle
of every output is the single-codec call (mec_encode_sse / mec_decode_sse), whose bytes tests/test_gpu_sse.py checks against the
committed host-made streams; the fixture streams that start at sequence number 0 are also checked here directly.  Only the
pure-Python helpers of tests/dare_ref.py are used (no `cryptography`)."""
import hashlib
import json
import os
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import dare_ref as d

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MiB = 1 << 20
PKG, EPKG = d.PKG, d.EPKG
K, M = 12, 4
INVALID, WRITE_QUORUM, NOT_AUTHENTIC, UNSUPPORTED = -12, -11, -13, -102
# 1 MiB of plaintext is 16 packages, 1049088 bytes of ciphertext: its last package straddles the first erasure block
PUT_LENGTHS = [1, 15, 16, 17, 65535, 65536, 65537, MiB, MiB + 1, 3 * MiB + 12345, 2 * MiB - 5, 5 * MiB + 3]


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    if minio_b200.device_count() == 0:
        pytest.skip("no CUDA device")
    return minio_b200


@pytest.fixture(scope="module")
def fx():
    with open(os.path.join(ROOT, "tests", "golden", "dare_streams.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def codec(mb):
    c = mb.Codec(K, M, MiB)
    yield c
    c.close()


def key_of(i):
    return np.frombuffer(hashlib.sha256(b"key %d" % i).digest(), np.uint8).copy()


def nonce_of(i):
    return np.frombuffer(hashlib.sha256(b"nonce %d" % i).digest()[:12], np.uint8).copy()


def pinned(mb, a):
    p = mb.pinned_array(max(a.size, 1))[:a.size]
    p[:] = a
    return p


def npk(n):
    return -(-n // PKG)


def touched(offset, length):
    return (offset + length - 1) // PKG - offset // PKG + 1


def run_all(fns, workers=64):
    """every callable at once, behind a barrier, so that they queue together"""
    bar = threading.Barrier(len(fns)) if len(fns) <= workers else None

    def go(f):
        if bar is not None:
            bar.wait()
        return f()

    with ThreadPoolExecutor(max_workers=min(workers, len(fns))) as ex:
        return list(ex.map(go, fns))


def sse_part(mb, codec, n, i):
    """plaintext, its part files from mec_encode_sse (page-locked copies) and the stored size"""
    pt = d.plaintext(n, 1000 + i)
    files = codec.encode_sse(pt, key_of(i), nonce_of(i))
    return pt, [pinned(mb, f) for f in files], mb.capi.dare_encrypted_size(n)


def test_refusals_on_the_callers_thread(mb):
    """mec_encode_sse's and mec_decode_sse's refusals with a live batcher; nothing is queued and no counter moves"""
    L = mb.lib()
    b = mb.Batcher(K, M, MiB)
    key, nonce = key_of(0), nonce_of(0)
    files = [np.zeros(64, np.uint8) for _ in range(K + M)]
    ptrs = mb.capi._ptrs(files)
    src = np.zeros(10, np.uint8)
    enc = lambda s, n, k, no, f, q: L.mec_batcher_encode_sse(b.h, s, n, k, no, f, q)  # noqa: E731
    assert enc(src.ctypes.data, 10, None, nonce.ctypes.data, ptrs, 0) == INVALID
    assert enc(src.ctypes.data, 10, key.ctypes.data, None, ptrs, 0) == INVALID
    assert enc(None, 10, key.ctypes.data, nonce.ctypes.data, ptrs, 0) == INVALID
    assert enc(src.ctypes.data, 10, key.ctypes.data, nonce.ctypes.data, None, 0) == INVALID
    assert enc(src.ctypes.data, -1, key.ctypes.data, nonce.ctypes.data, ptrs, 0) == INVALID
    assert enc(src.ctypes.data, (1 << 48) + 1, key.ctypes.data, nonce.ctypes.data, ptrs, 0) == INVALID  # past 2^32 packages
    assert enc(src.ctypes.data, 10, key.ctypes.data, nonce.ctypes.data, ptrs, K + M + 1) == WRITE_QUORUM
    assert enc(None, 0, key.ctypes.data, nonce.ctypes.data, ptrs, 0) == 0
    hint = mb.capi.C.c_int(5)
    dst = np.zeros(16, np.uint8)
    dec = lambda off, ln, tot, k=key.ctypes.data, f=ptrs, o=dst.ctypes.data: L.mec_batcher_decode_sse(  # noqa: E731
        b.h, f, None, off, ln, tot, k, o, mb.capi.C.byref(hint))
    assert dec(0, 1, 33, k=None) == INVALID and hint.value == 0
    assert dec(0, 1, 33, f=None) == INVALID
    assert dec(0, 1, 33, o=None) == INVALID
    assert dec(-1, 1, 33) == INVALID and dec(0, -1, 33) == INVALID and dec(0, 1, -1) == INVALID
    assert dec(0, 1, 20) == NOT_AUTHENTIC  # a stored size that is no DARE size
    assert dec(0, 2, 33) == INVALID        # past the plaintext
    assert dec(1, 0, 33) == 0
    assert b.stat("requests") == 0 and b.stat("sse_serial") == 0 and b.stat("dare_sealed") == 0
    b.close()


def test_concurrent_puts(mb, codec):
    """64 threads, distinct keys and nonces: every part file is mec_encode_sse's, each package is sealed once, and every merged batch
    adds exactly its two cipher launches"""
    b = mb.Batcher(K, M, MiB, max_wait_us=2000)
    # the batcher codec's first encrypted call also builds its AES tables (one more launch): out of the launch counts below
    w = pinned(mb, d.plaintext(100, 1))
    for f in b.encode_sse(w, key_of(0), nonce_of(0), pinned=True):
        mb.lib().mec_free_pinned(f.ctypes.data)
    # one call per batch: two launches (setup, seal) over a plain batch of the same ciphertext layout
    for n in (17, MiB, 3 * MiB + 12345):
        e = mb.capi.dare_encrypted_size(n)
        plain = pinned(mb, np.zeros(e, np.uint8))
        l0, b0 = b.stat("launches"), b.stat("batches")
        b.encode(plain, pinned=True)
        l1, b1 = b.stat("launches"), b.stat("batches")
        b.encode_sse(pinned(mb, d.plaintext(n, 2)), key_of(1), nonce_of(1), pinned=True)
        l2, b2 = b.stat("launches"), b.stat("batches")
        assert b1 - b0 == 1 and b2 - b1 == 1
        assert (l2 - l1) - (l1 - l0) == 2, n
    # one merged batch of eight encrypted PUTs (each under one block of ciphertext, so that the batch is not split): still two
    # launches over the merged plain batch of the same ciphertext lengths
    small = [1, 100, 65535, 65537, 200000, 300001, 500000, 900000]
    slow = mb.Batcher(K, M, MiB, max_wait_us=200000)
    for f in slow.encode_sse(w, key_of(0), nonce_of(0), pinned=True):
        mb.lib().mec_free_pinned(f.ctypes.data)
    plains = [pinned(mb, np.zeros(mb.capi.dare_encrypted_size(n), np.uint8)) for n in small]
    ptxt = [pinned(mb, d.plaintext(n, 3 + i)) for i, n in enumerate(small)]
    l0, b0 = slow.stat("launches"), slow.stat("batches")
    run_all([lambda p=p: slow.encode(p, pinned=True) for p in plains])
    l1, b1 = slow.stat("launches"), slow.stat("batches")
    merged = run_all([lambda i=i: slow.encode_sse(ptxt[i], key_of(i), nonce_of(i), pinned=True) for i in range(len(small))])
    l2, b2 = slow.stat("launches"), slow.stat("batches")
    assert b1 - b0 == 1 and b2 - b1 == 1
    assert (l2 - l1) - (l1 - l0) == 2
    for i, n in enumerate(small):
        assert all(np.array_equal(x, y) for x, y in zip(merged[i], codec.encode_sse(ptxt[i], key_of(i), nonce_of(i)))), n
    slow.close()
    lens = [PUT_LENGTHS[i % len(PUT_LENGTHS)] for i in range(64)]
    srcs = [pinned(mb, d.plaintext(n, 50 + i)) for i, n in enumerate(lens)]
    before = {s: b.stat(s) for s in ("sse_puts", "dare_sealed", "batches", "sse_serial")}
    got = run_all([lambda i=i: b.encode_sse(srcs[i], key_of(i), nonce_of(i), pinned=True) for i in range(64)])
    assert b.stat("sse_puts") - before["sse_puts"] == 64
    assert b.stat("sse_serial") == before["sse_serial"]
    assert b.stat("dare_sealed") - before["dare_sealed"] == sum(npk(n) for n in lens)
    assert b.stat("batches") - before["batches"] < 64  # calls were merged
    for i, n in enumerate(lens):
        want = codec.encode_sse(srcs[i], key_of(i), nonce_of(i))
        for j in range(K + M):
            assert np.array_equal(got[i][j], want[j]), (n, j)
    b.close()


def test_fixture_ciphertext(mb, fx):
    """the fixture streams that start at sequence number 0, sealed by merged batches: mec_decode of the part files is the stream"""
    b = mb.Batcher(K, M, MiB, max_wait_us=2000)
    c = mb.Codec(K, M, MiB)
    ss = [s for s in fx["streams"] if s["seq0"] == 0]
    assert ss
    srcs = [pinned(mb, d.plaintext(s["length"], s["seed"])) for s in ss]
    keys = [np.frombuffer(bytes.fromhex(s["key"]), np.uint8) for s in ss]
    nonces = [np.frombuffer(bytes.fromhex(s["nonce"]), np.uint8) for s in ss]
    parts = run_all([lambda i=i: b.encode_sse(srcs[i], keys[i], nonces[i], pinned=True) for i in range(len(ss))])
    assert b.stat("sse_puts") == len(ss)
    for s, files in zip(ss, parts):
        e = d.encrypted_size(s["length"])
        ct, _ = c.decode(files, 0, e, e)
        got = ct.tobytes()
        assert hashlib.sha256(got).hexdigest() == s["sha256"], s["length"]
        assert d.excerpts(got) == {f: s[f] for f in ("first_head", "first_tag", "last_head", "last_tag")}
    c.close()
    b.close()


def get_cases(D):
    """whole object, single bytes at package edges, a range across packages, the last byte"""
    cases = [(0, D), (0, 1), (D - 1, 1)]
    for e in (PKG - 1, PKG, 2 * PKG - 1):
        if e < D:
            cases.append((e, 1))
    if D > PKG + 10:
        cases.append((PKG - 10, 20))
    if D > 3 * PKG:
        cases.append((PKG // 2, 2 * PKG))
    return cases


@pytest.mark.parametrize("get_out", [0, 1, 2])
@pytest.mark.parametrize("mix", [False, True])
@pytest.mark.parametrize("offline,prefer", [((), False), ((0, 5, 9, 13), False), ((2, 3), True), ((), True)])
def test_concurrent_gets(mb, codec, monkeypatch, mix, offline, prefer, get_out):
    """concurrent encrypted GETs with 0 .. m drives offline, with and without prefer, in every MEC_BATCHER_GET_OUT mode (assembly on
    the device, scatter kernel into the callers' buffers, copy-engine pieces): the plaintext, and results equal to mec_decode_sse's,
    heal_hint included; each touched package is opened once"""
    if get_out:
        monkeypatch.setenv("MEC_BATCHER_GET_OUT", str(get_out))
    else:
        monkeypatch.delenv("MEC_BATCHER_GET_OUT", raising=False)
    b = mb.Batcher(K, M, MiB, max_wait_us=2000, mix_patterns=mix)
    sizes = [1, 65537, MiB, 3 * MiB + 12345]
    objs = [sse_part(mb, codec, n, i) for i, n in enumerate(sizes)]
    pf = None
    if prefer:
        pf = np.zeros(K + M, np.uint8)
        pf[[4, 6, 8, 10, 12, 14]] = 1
    tasks, wants = [], []
    for i, (pt, files, e) in enumerate(objs):
        fl = [None if j in offline else f for j, f in enumerate(files)]
        for off, ln in get_cases(pt.size):
            want, whint = codec.decode_sse(fl, off, ln, e, key_of(i), prefer=pf)
            assert np.array_equal(want, pt[off:off + ln])
            wants.append((pt[off:off + ln], whint, touched(off, ln)))
            tasks.append((fl, off, ln, e, i))
    dsts = [pinned(mb, np.full(max(t[2], 1), 0xAA, np.uint8)) for t in tasks]
    before = {s: b.stat(s) for s in ("sse_gets", "dare_opened", "sse_serial")}
    got = run_all([lambda t=t, o=o: b.decode_sse(t[0], t[1], t[2], t[3], key_of(t[4]), prefer=pf, dst=o) for t, o in zip(tasks, dsts)])
    for (data, hint), (want, whint, _) in zip(got, wants):
        assert np.array_equal(data, want) and hint == whint
    assert b.stat("sse_gets") - before["sse_gets"] == len(tasks)
    assert b.stat("sse_serial") == before["sse_serial"]
    assert b.stat("dare_opened") - before["dare_opened"] == sum(w[2] for w in wants)
    b.close()


def test_first_encrypted_calls_of_a_batcher(mb, codec):
    """no warm-up: the first encrypted calls of a fresh batcher are a large degraded GET beside small GETs and PUTs, which run as
    batches on other slots; the codec's AES tables are complete before any of them reads them"""
    b = mb.Batcher(K, M, MiB)
    big_pt, big_files, big_e = sse_part(mb, codec, 24 * MiB + 5, 40)
    big_fl = [None if j < 4 else f for j, f in enumerate(big_files)]
    smalls = [sse_part(mb, codec, n, 41 + i) for i, n in enumerate([1, 3000, 65537, 70000, 1000, 5, 130000, 64000])]
    srcs = [pinned(mb, d.plaintext(n, 60 + i)) for i, n in enumerate([7, 65536, 100000, 33, 5000, 200000, 1, 65537])]
    big_dst = pinned(mb, np.zeros(big_pt.size, np.uint8))
    fns = [lambda: b.decode_sse(big_fl, 0, big_pt.size, big_e, key_of(40), dst=big_dst)]
    for i, (pt, files, e) in enumerate(smalls):
        o = pinned(mb, np.zeros(pt.size, np.uint8))
        fns.append(lambda files=files, e=e, i=i, o=o, pt=pt: b.decode_sse(files, 0, pt.size, e, key_of(41 + i), dst=o))
    for i, s in enumerate(srcs):
        fns.append(lambda s=s, i=i: b.encode_sse(s, key_of(60 + i), nonce_of(60 + i), pinned=True))
    got = run_all(fns)
    assert np.array_equal(got[0][0], big_pt)
    for (data, hint), (pt, _, _) in zip(got[1:1 + len(smalls)], smalls):
        assert np.array_equal(data, pt) and hint == 0
    for files, s, i in zip(got[1 + len(smalls):], srcs, range(len(srcs))):
        assert all(np.array_equal(x, y) for x, y in zip(files, codec.encode_sse(s, key_of(60 + i), nonce_of(60 + i))))
    assert b.stat("sse_serial") == 0
    b.close()


@pytest.mark.parametrize("dst", [None, (6, 2)])
def test_mixed_traffic(mb, codec, dst):
    """plain and encrypted PUTs and GETs on one batcher (and on a transcode batcher) all give their single-call results"""
    b = mb.Batcher(K, M, MiB, max_wait_us=2000, dst=dst)
    objs = [sse_part(mb, codec, n, i) for i, n in enumerate([70000, 2 * MiB + 5])]
    plain = d.plaintext(3 * MiB + 7, 77)
    pfiles = [pinned(mb, f) for f in codec.encode(plain)]
    srcs = [pinned(mb, d.plaintext(n, 300 + i)) for i, n in enumerate([5, 65536, MiB + 77, 4 * MiB])]
    fns, checks = [], []
    for i, s in enumerate(srcs):
        fns.append(lambda s=s, i=i: b.encode_sse(s, key_of(i), nonce_of(i), pinned=True))
        checks.append(lambda r, s=s, i=i: all(np.array_equal(x, y) for x, y in zip(r, codec.encode_sse(s, key_of(i), nonce_of(i)))))
        fns.append(lambda s=s: b.encode(s, pinned=True))
        checks.append(lambda r, s=s: all(np.array_equal(x, y) for x, y in zip(r, codec.encode(s))))
    for i, (pt, files, e) in enumerate(objs):
        for off, ln in get_cases(pt.size):
            o = pinned(mb, np.zeros(ln, np.uint8))
            fns.append(lambda files=files, off=off, ln=ln, e=e, i=i, o=o: b.decode_sse(files, off, ln, e, key_of(i), dst=o))
            checks.append(lambda r, pt=pt, off=off, ln=ln: np.array_equal(r[0], pt[off:off + ln]) and r[1] == 0)
    for off, ln in get_cases(plain.size):
        o = pinned(mb, np.zeros(ln, np.uint8))
        fns.append(lambda off=off, ln=ln, o=o: b.decode(pfiles, off, ln, plain.size, dst=o))
        checks.append(lambda r, off=off, ln=ln: np.array_equal(r[0], plain[off:off + ln]) and r[1] == 0)
    got = run_all(fns)
    for j, (r, ck) in enumerate(zip(got, checks)):
        assert ck(r), j
    assert b.stat("sse_puts") == len(srcs) and b.stat("sse_gets") == sum(len(get_cases(o[0].size)) for o in objs)
    assert b.stat("sse_serial") == 0
    b.close()


def test_isolation_in_one_batch(mb, codec):
    """tampered ciphertext with valid frames, a wrong key, DARE 1.0, ChaCha20 and a frame failing its digest, among good requests
    queued together: each gets its own result, and every batch-mate succeeds"""
    b = mb.Batcher(K, M, MiB, max_wait_us=20000)
    n = 3 * PKG + 100
    pt, files, e = sse_part(mb, codec, n, 7)
    ct, _ = codec.decode(files, 0, e, e)  # the stored stream

    def restored(mut):
        s = ct.copy()
        mut(s)
        return [pinned(mb, f) for f in codec.encode(s)]

    def flip(s):
        s[EPKG + 500] ^= 1

    def dare10(s):
        s[0] = 0x10

    def chacha(s):
        s[2 * EPKG + 1] = 1

    rot = [f.copy() for f in files]
    rot[0][32 + 7] ^= 0x40  # drive 0's first frame fails its digest
    rot = [pinned(mb, f) for f in rot]
    cases = [  # (files, key index, expected rc)
        (restored(flip), 7, NOT_AUTHENTIC), (files, 8, NOT_AUTHENTIC), (restored(dare10), 7, UNSUPPORTED),
        (restored(chacha), 7, UNSUPPORTED), (rot, 7, n)]
    cases += [(files, 7, n)] * 6
    before = {s: b.stat(s) for s in ("redone", "sse_serial", "batches")}
    dsts = [pinned(mb, np.full(n, 0xAA, np.uint8)) for _ in cases]
    keys = [key_of(ki) for _, ki, _ in cases]  # alive until every call has returned: the worker reads them
    L = mb.lib()

    def call(j):
        return L.mec_batcher_decode_sse(b.h, mb.capi._ptrs(cases[j][0]), None, 0, n, e, keys[j].ctypes.data, dsts[j].ctypes.data, None)

    rcs = run_all([lambda j=j: call(j) for j in range(len(cases))])
    for j, ((_, _, want), rc) in enumerate(zip(cases, rcs)):
        assert rc == want, j
        if want < 0:
            assert not dsts[j].any(), j  # nothing of the range handed out
        else:
            assert np.array_equal(dsts[j], pt), j
    assert b.stat("redone") - before["redone"] == 1
    assert b.stat("sse_serial") - before["sse_serial"] == 1  # the redo
    # the single call agrees on every failure
    for fl, ki, want in cases[:4]:
        with pytest.raises(mb.MecError) as ex:
            codec.decode_sse(fl, 0, n, e, key_of(ki))
        assert ex.value.code == want
    b.close()


def test_private_paths(mb, codec, monkeypatch):
    """pageable buffers, and MEC_BATCHER_MEMCPY, go through mec_encode_sse / mec_decode_sse on the private handle: same bytes"""
    n = 2 * MiB + 33
    src = d.plaintext(n, 9)
    want = codec.encode_sse(src, key_of(3), nonce_of(3))
    e = mb.capi.dare_encrypted_size(n)
    b = mb.Batcher(K, M, MiB)
    got = b.encode_sse(src, key_of(3), nonce_of(3))  # pageable
    assert all(np.array_equal(x, y) for x, y in zip(got, want))
    data, hint = b.decode_sse(want, 100, PKG, e, key_of(3))
    assert np.array_equal(data, src[100:100 + PKG]) and hint == 0
    assert b.stat("sse_serial") == 2 and b.stat("sse_puts") == 0 and b.stat("sse_gets") == 0
    b.close()
    monkeypatch.setenv("MEC_BATCHER_MEMCPY", "1")
    b = mb.Batcher(K, M, MiB)
    got = b.encode_sse(pinned(mb, src), key_of(3), nonce_of(3), pinned=True)
    assert all(np.array_equal(x, y) for x, y in zip(got, want))
    data, _ = b.decode_sse([pinned(mb, f) for f in want], 0, n, e, key_of(3), dst=pinned(mb, np.zeros(n, np.uint8)))
    assert np.array_equal(data, src)
    assert b.stat("sse_serial") == 2 and b.stat("sse_puts") == 0
    b.close()


def test_encrypted_put_beside_pageable_put(mb, codec):
    """an encrypted PUT in a batch with a pageable plain PUT (the batch takes the per-request copy path) is still sealed by the batch"""
    b = mb.Batcher(K, M, MiB, max_wait_us=20000)
    s1, s2 = d.plaintext(MiB + 5, 21), pinned(mb, d.plaintext(2 * MiB + 9, 22))
    r = run_all([lambda: b.encode(s1), lambda: b.encode_sse(s2, key_of(5), nonce_of(5), pinned=True)])
    assert all(np.array_equal(x, y) for x, y in zip(r[0], codec.encode(s1)))
    assert all(np.array_equal(x, y) for x, y in zip(r[1], codec.encode_sse(s2, key_of(5), nonce_of(5))))
    assert b.stat("sse_puts") == 1 and b.stat("sse_serial") == 0
    b.close()
