"""DARE 2.0 ChaCha20-Poly1305 packages (cipher 1) on the GPU under option "dare_chacha20": mec_dare_device, mec_encode_sse /
mec_decode_sse, mec_encode_chunked_sse and the coalescer's encrypted GETs and PUTs.  Streams are checked against the committed
host-made fixture (tests/golden/dare_chacha_streams.json, sealed with `cryptography`) and the pure-Python reference
tests/chacha_ref.py; nothing outside the standard library, numpy, torch and the repository is imported."""
import hashlib
import json
import os
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import chacha_ref as cr
import dare_ref as d
import sigv4_ref as sref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MiB = 1 << 20
PKG, EPKG = d.PKG, d.EPKG
NOT_AUTHENTIC, UNSUPPORTED, INVALID = -13, -102, -12
KEY, NONCE = bytes(range(32)), bytes.fromhex("0123456789abcdeffedcba98")
K, M = 12, 4


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    if minio_b200.device_count() == 0:
        pytest.skip("no CUDA device")
    return minio_b200


@pytest.fixture(scope="module")
def fx():
    with open(os.path.join(ROOT, "tests", "golden", "dare_chacha_streams.json")) as f:
        return json.load(f)["streams"]


def codec_at(mb, v, k=K, m=M, bs=MiB):
    c = mb.Codec(k, m, bs)
    c.set_option("dare_chacha20", v)
    return c


@pytest.fixture(scope="module")
def c1(mb):
    c = codec_at(mb, 1)
    yield c
    c.close()


@pytest.fixture(scope="module")
def c2(mb):
    c = codec_at(mb, 2)
    yield c
    c.close()


def npk(n):
    return -(-n // PKG)


def dev(buf):
    import torch
    return torch.from_numpy(np.frombuffer(bytes(buf), dtype=np.uint8).copy()).to("cuda")


def check_stream(s, got):
    what = f"length {s['length']} seq0 {s['seq0']}"
    assert d.excerpts(got) == {f: s[f] for f in ("first_head", "first_tag", "last_head", "last_tag")}, what
    assert hashlib.sha256(got).hexdigest() == s["sha256"], what


def seal(c, key, nonce, pt, seq0=0):
    """one stream through mec_dare_device SEAL -> sealed bytes"""
    import torch
    pt = bytes(pt)
    src = dev(pt) if pt else torch.zeros(1, dtype=torch.uint8, device="cuda")
    out = torch.zeros(max(d.encrypted_size(len(pt)), 1), dtype=torch.uint8, device="cuda")
    c.dare_device(1, np.frombuffer(key, np.uint8), src.data_ptr(), [0], [len(pt)], out.data_ptr(), [0], seq0=[seq0],
                  nonces=np.frombuffer(nonce, np.uint8))
    return out.cpu().numpy()[:d.encrypted_size(len(pt))].tobytes()


def open_(c, key, stream, enc_total, seq0=0, fill=0xAA, out_len=None):
    """one stream through mec_dare_device OPEN -> (rc, status, plaintext buffer pre-filled with `fill`)"""
    import torch
    st = bytes(stream)
    src = dev(st) if st else torch.zeros(1, dtype=torch.uint8, device="cuda")
    n = out_len if out_len is not None else PKG * (len(st) // EPKG + 1)
    out = torch.full((n,), fill, dtype=torch.uint8, device="cuda")
    rc, status = c.dare_device(2, np.frombuffer(key, np.uint8), src.data_ptr(), [0], [len(st)], out.data_ptr(), [0], seq0=[seq0],
                               enc_totals=[enc_total], check=False)
    return rc, int(status[0]), out.cpu().numpy()


def layout(lens, a=3, b=5, ga=7, gb=9):
    """odd offsets of streams of in-lengths / out-lengths"""
    ins, outs = [], []
    for li, lo in lens:
        ins.append(a); outs.append(b)
        a += li + ga; b += lo + gb
    return ins, outs, a, b


# ---- the option ---------------------------------------------------------------------------------------------------------------
def test_option_values(mb):
    c = mb.Codec(K, M, MiB)
    for v in (0, 1, 2):
        c.set_option("dare_chacha20", v)
        assert c.stat("dare_chacha20") == v
    for bad in (3, -1):
        with pytest.raises(mb.MecError) as e:
            c.set_option("dare_chacha20", bad)
        assert e.value.code == INVALID and c.stat("dare_chacha20") == 2
    c.close()
    b = mb.Batcher(K, M, MiB)
    assert b.stat("dare_chacha20") == 0
    for v in (2, 1, 0, 1):
        b.set_option("dare_chacha20", v)
        assert b.stat("dare_chacha20") == v
    for name, bad in (("dare_chacha20", 3), ("dare_chacha20", -1), ("eb", 1)):
        with pytest.raises(mb.MecError) as e:
            b.set_option(name, bad)
        assert e.value.code == INVALID and b.stat("dare_chacha20") == 1
    b.close()


# ---- mec_dare_device ------------------------------------------------------------------------------------------------------------
def test_open_every_fixture_stream_in_one_call(c1, fx):
    import torch
    sts = [cr.seal_chacha(bytes.fromhex(s["key"]), bytes.fromhex(s["nonce"]), d.plaintext(s["length"], s["seed"]).tobytes(), s["seq0"])
           for s in fx]
    for s, st in zip(fx, sts):
        check_stream(s, st)
    pts = [d.plaintext(s["length"], s["seed"]) for s in fx]
    ins, outs, a, b = layout([(len(st), p.size) for st, p in zip(sts, pts)])
    host = np.zeros(a, np.uint8)
    for o, st in zip(ins, sts):
        host[o:o + len(st)] = np.frombuffer(st, np.uint8)
    src, out = dev(host), torch.full((b,), 0xAA, dtype=torch.uint8, device="cuda")
    keys = np.concatenate([np.frombuffer(bytes.fromhex(s["key"]), np.uint8) for s in fx])
    seal(c1, KEY, NONCE, b"x")  # the codec's AES tables are built
    before, launches = c1.stat("dare_opened"), c1.launches
    rc, status = c1.dare_device(2, keys, src.data_ptr(), ins, [len(st) for st in sts], out.data_ptr(), outs,
                                seq0=[s["seq0"] for s in fx], enc_totals=[s["seq0"] * EPKG + len(st) for s, st in zip(fx, sts)])
    assert rc == 0 and not status.any()
    assert c1.stat("dare_opened") - before == sum(npk(p.size) for p in pts)
    assert c1.launches - launches == 3  # key setup, the AES open, the ChaCha20 open
    o = out.cpu().numpy()
    for off, p in zip(outs, pts):
        assert np.array_equal(o[off:off + p.size], p)


def test_seal_equals_fixture(c2, fx):
    import torch
    pts = [d.plaintext(s["length"], s["seed"]) for s in fx]
    ins, outs, a, b = layout([(p.size, d.encrypted_size(p.size)) for p in pts])
    host = np.zeros(a, np.uint8)
    for o, p in zip(ins, pts):
        host[o:o + p.size] = p
    src, out = dev(host), torch.zeros(b, dtype=torch.uint8, device="cuda")
    keys = np.concatenate([np.frombuffer(bytes.fromhex(s["key"]), np.uint8) for s in fx])
    nonces = np.concatenate([np.frombuffer(bytes.fromhex(s["nonce"]), np.uint8) for s in fx])
    before, launches = c2.stat("dare_sealed"), c2.launches
    c2.dare_device(1, keys, src.data_ptr(), ins, [p.size for p in pts], out.data_ptr(), outs, seq0=[s["seq0"] for s in fx],
                   nonces=nonces)
    assert c2.stat("dare_sealed") - before == sum(npk(p.size) for p in pts)
    assert c2.launches - launches == 1  # no key setup: one ChaCha20 seal launch
    o = out.cpu().numpy()
    for s, off, p in zip(fx, outs, pts):
        check_stream(s, o[off:off + d.encrypted_size(p.size)].tobytes())
    # random lengths against the reference, and a stream sealed one at a time
    rng = np.random.default_rng(5)
    for n in [int(x) for x in rng.integers(1, 300000, 6)] + [4081, 4096, 8161, 8176]:
        pt = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert seal(c2, KEY, NONCE, pt, 3) == cr.seal_chacha(KEY, NONCE, pt, 3), n


def test_aes_and_chacha_streams_in_one_call(mb, c1, c2):
    import torch
    pt = d.plaintext(5 * PKG + 77, 4)
    aes, cha = seal(c1, KEY, NONCE, pt), seal(c2, KEY, NONCE, pt)
    assert aes[1] == 0 and cha[1] == 1
    alt = bytearray(aes)  # packages alternate ciphers: odd packages ChaCha20
    for p in range(1, 6, 2):
        alt[p * EPKG:(p + 1) * EPKG] = cha[p * EPKG:(p + 1) * EPKG]
    sts = [aes, cha, bytes(alt)]
    ins, outs, a, b = layout([(len(s), pt.size) for s in sts])
    host = np.zeros(a, np.uint8)
    for o, s in zip(ins, sts):
        host[o:o + len(s)] = np.frombuffer(s, np.uint8)
    src, out = dev(host), torch.zeros(b, dtype=torch.uint8, device="cuda")
    rc, status = c1.dare_device(2, np.frombuffer(KEY * 3, np.uint8), src.data_ptr(), ins, [len(s) for s in sts], out.data_ptr(), outs,
                                enc_totals=[len(s) for s in sts])
    assert rc == 0 and not status.any()
    o = out.cpu().numpy()
    for off in outs:
        assert np.array_equal(o[off:off + pt.size], pt)
    c0 = codec_at(mb, 0)  # at option 0 only the AES stream opens; the other two are the host's
    rc, status = c0.dare_device(2, np.frombuffer(KEY * 3, np.uint8), src.data_ptr(), ins, [len(s) for s in sts], out.data_ptr(), outs,
                                enc_totals=[len(s) for s in sts], check=False)
    assert rc == UNSUPPORTED and list(status) == [0, 102, 102]
    c0.close()


@pytest.fixture(scope="module")
def four(c2):
    pt = d.plaintext(3 * PKG + 5, 8)
    st = seal(c2, KEY, NONCE, pt)
    assert st == cr.seal_chacha(KEY, NONCE, pt.tobytes())
    return pt, st


def flip(b, i, bit=1):
    b = bytearray(b)
    b[i] ^= bit
    return bytes(b)


# the cases of tests/test_gpu_sse.py's TAMPER on a four-package ChaCha20 stream:
# case -> (stream, stored size, key, packages that still open, packages opened)
TAMPER = {
    "header": lambda st: (flip(st, EPKG + 9), len(st), KEY, {0, 2, 3}, 4),
    "ciphertext": lambda st: (flip(st, 2 * EPKG + 16 + 777, 0x10), len(st), KEY, {0, 1, 3}, 4),
    "tag": lambda st: (flip(st, len(st) - 3, 0x80), len(st), KEY, {0, 1, 2}, 4),
    "aad_length": lambda st: (flip(st, 2, 0x01), len(st), KEY, {1, 2, 3}, 4),          # the length field of package 0
    "swap": lambda st: (st[EPKG:2 * EPKG] + st[:EPKG] + st[2 * EPKG:], len(st), KEY, {2, 3}, 4),
    "drop_final": lambda st: (st[:3 * EPKG], 3 * EPKG, KEY, {0, 1}, 3),
    "move_final": lambda st: (flip(flip(st, 4, 0x80), 3 * EPKG + 4, 0x80), len(st), KEY, {1, 2}, 4),
    "wrong_key": lambda st: (st, len(st), bytes(31) + b"\x01", set(), 4),
    "trailing_40": lambda st: (st + bytes(40), len(st) + 40, KEY, {0, 1, 2}, 4),
    "trailing_10": lambda st: (st + bytes(10), len(st) + 10, KEY, {0, 1, 2}, 4),
    "trailing_beyond_size": lambda st: (st + bytes(50), len(st), KEY, {0, 1, 2, 3}, 4),
    "cut_short": lambda st: (st[:-1], len(st), KEY, {0, 1, 2}, 3),
    "bad_size": lambda st: (st, len(st) - 5, KEY, set(), 0),
}


@pytest.mark.parametrize("case", list(TAMPER))
def test_tamper_not_authentic(c1, four, case):
    pt, st = four
    st, total, key, good, rows = TAMPER[case](st)
    before = c1.stat("dare_opened")
    rc, status, out = open_(c1, key, st, total, out_len=4 * PKG)
    assert rc == NOT_AUTHENTIC and status == 13 and c1.stat("dare_opened") - before == rows
    for p in range(4):
        lo, hi = p * PKG, min(pt.size, (p + 1) * PKG)
        assert np.array_equal(out[lo:hi], pt[lo:hi]) if p in good else (out[lo:hi] == 0xAA).all(), (case, p)


def test_other_cipher_bytes_and_dare10(c1, c2):
    """at option 1, cipher bytes 2..255 are NOT_AUTHENTIC (one call, one stream each) and DARE 1.0 is still UNSUPPORTED"""
    import torch
    pt = d.plaintext(1000, 9)
    st = seal(c2, KEY, NONCE, pt)
    sts = []
    for cb in range(2, 256):
        b = bytearray(st)
        b[1] = cb
        sts.append(bytes(b))
    ins, outs, a, b = layout([(len(s), pt.size) for s in sts])
    host = np.zeros(a, np.uint8)
    for o, s in zip(ins, sts):
        host[o:o + len(s)] = np.frombuffer(s, np.uint8)
    src, out = dev(host), torch.full((b,), 0xAA, dtype=torch.uint8, device="cuda")
    rc, status = c1.dare_device(2, np.frombuffer(KEY * len(sts), np.uint8), src.data_ptr(), ins, [len(s) for s in sts], out.data_ptr(),
                                outs, enc_totals=[len(s) for s in sts], check=False)
    assert rc == NOT_AUTHENTIC and (status == 13).all() and (out.cpu().numpy() == 0xAA).all()
    d10 = bytearray(st)
    d10[0] = 0x10
    rc, status, out = open_(c1, KEY, bytes(d10), len(st))
    assert rc == UNSUPPORTED and status == 102 and (out == 0xAA).all()
    rc, status, out = open_(c1, KEY, st, len(st))
    assert rc == 0 and np.array_equal(out[:pt.size], pt)


def test_option0_leaves_chacha_unsupported(mb, four):
    pt, st = four
    c0 = codec_at(mb, 0)
    seal(c0, KEY, NONCE, b"x")
    launches = c0.launches
    rc, status, out = open_(c0, KEY, st, len(st), out_len=4 * PKG)
    assert rc == UNSUPPORTED and status == 102 and (out == 0xAA).all()
    assert c0.launches - launches == 2  # key setup and the AES open: nothing new at option 0
    c0.close()


# ---- mec_encode_sse / mec_decode_sse / mec_encode_chunked_sse ------------------------------------------------------------------
@pytest.fixture(scope="module")
def part(mb, c2):
    """a 5 MiB + 12345 B object sealed with ChaCha20-Poly1305 and encoded in RS(12,4) with 1 MiB blocks; its part files equal
    mec_encode of the reference stream"""
    pt = d.plaintext(5 * MiB + 12345, 6)
    before, launches = c2.stat("dare_sealed"), c2.launches
    files = c2.encode_sse(pt, KEY, NONCE)
    assert c2.stat("dare_sealed") - before >= npk(pt.size)  # a package across a pipeline chunk boundary is sealed in both
    ref = np.frombuffer(cr.seal_chacha(KEY, NONCE, pt.tobytes()), np.uint8)
    want = c2.encode(ref)
    assert all(np.array_equal(a, b) for a, b in zip(files, want))
    return pt, files, d.encrypted_size(pt.size)


def test_encode_sse_small_chunks(mb, c2):
    """packages across erasure blocks and pipeline chunks, as the AES path seals them"""
    for k, m, bs in [(12, 4, MiB), (4, 2, MiB)]:
        c = codec_at(mb, 2, k, m, bs)
        for cb in (1, 2):
            c.set_option("chunk_blocks", cb)
            for n in (1, 3 * PKG + 5, 3 * bs + 4321):
                pt = d.plaintext(n, 5)
                want = c.encode(np.frombuffer(cr.seal_chacha(KEY, NONCE, pt.tobytes()), np.uint8))
                got = c.encode_sse(pt, KEY, NONCE)
                assert all(np.array_equal(a, b) for a, b in zip(got, want)), (k, m, cb, n)
        c.close()


def test_encode_chunked_sse(mb, c2, part):
    pt, files, E = part
    key = sref.signing_key("wJalrXUtnFEMI/K7MDENG/bPxRfiCYEXAMPLEKEY")
    seed = b"4f232c4386841ef735655705268965c44a0e4690baa4adea153f7db9fa80a0a9"
    for csize in (64 * 1024, 65537):
        sizes = [csize] * (pt.size // csize) + ([pt.size % csize] if pt.size % csize else [])
        body = sref.build(pt.tobytes(), sizes, key, seed).data
        got = c2.encode_chunked_sse(body, pt.size, key, seed, sref.DATE, sref.scope_of(), KEY, NONCE)
        assert all(np.array_equal(a, b) for a, b in zip(got, files)), csize


def ranges(D):
    blk = MiB * PKG // EPKG
    return [(0, D), (100, 70000), (PKG, PKG), (PKG - 1, 2), (15 * PKG + 3, 2 * PKG), (blk - 10, 20), (3 * blk + 5, 2 * MiB),
            (D - 1, 1), (D - 70000, 70000), (0, 1)]


def opened_for(off, ln):
    return (off + ln - 1) // PKG - off // PKG + 1


@pytest.mark.parametrize("cb", [0, 1])
@pytest.mark.parametrize("offline", [(), (0, 1, 2, 3)])
def test_decode_sse_ranges(mb, part, cb, offline):
    pt, files, E = part
    c = codec_at(mb, 1)
    c.set_option("chunk_blocks", cb)
    fs = [None if i in offline else f for i, f in enumerate(files)]
    for off, ln in ranges(pt.size):
        before = c.stat("dare_opened")
        out, hint = c.decode_sse(fs, off, ln, E, KEY)
        assert hint == 0 and np.array_equal(out, pt[off:off + ln]), (off, ln, offline, cb)
        assert c.stat("dare_opened") - before == opened_for(off, ln)
    c.set_option("dare_chacha20", 0)
    with pytest.raises(mb.MecError) as e:
        c.decode_sse(fs, 0, 1000, E, KEY)
    assert e.value.code == UNSUPPORTED
    c.close()


def test_decode_sse_corrupt_frame_and_wrong_key(mb, part):
    pt, files, E = part
    c = codec_at(mb, 2)
    c.set_option("chunk_blocks", 1)
    bad = [f.copy() for f in files]
    bad[2][3 * (32 + c.shard_size()) + 32 + 1000] ^= 0x40
    for off, ln in [(0, pt.size), (3 * MiB - 5000, 10000)]:
        out, hint = c.decode_sse(bad, off, ln, E, KEY)
        assert np.array_equal(out, pt[off:off + ln]) and hint == -7
    with pytest.raises(mb.MecError) as e:
        c.decode_sse(files, 0, 1000, E, bytes(32))
    assert e.value.code == NOT_AUTHENTIC
    c.close()


# ---- the coalescer -------------------------------------------------------------------------------------------------------------
def pinned(mb, a):
    p = mb.pinned_array(max(a.size, 1))[:a.size]
    p[:] = a
    return p


def key_of(i):
    return np.frombuffer(hashlib.sha256(b"key %d" % i).digest(), np.uint8).copy()


def nonce_of(i):
    return np.frombuffer(hashlib.sha256(b"nonce %d" % i).digest()[:12], np.uint8).copy()


def run_all(fns, delays=None):
    """every callable at once (each after its delay in seconds), so that they queue together"""
    def go(j):
        if delays:
            time.sleep(delays[j])
        return fns[j]()

    with ThreadPoolExecutor(max_workers=len(fns)) as ex:
        return list(ex.map(go, range(len(fns))))


def sse_parts(mb, sizes, cipher_of):
    """(plaintext, page-locked part files, stored size) per size, sealed with AES (cipher_of(i) == 0) or ChaCha20 (1)"""
    cs = {0: codec_at(mb, 0), 2: codec_at(mb, 2)}
    out = []
    for i, n in enumerate(sizes):
        pt = d.plaintext(n, 300 + i)
        files = cs[2 * cipher_of(i)].encode_sse(pt, key_of(i), nonce_of(i))
        out.append((pt, [pinned(mb, f) for f in files], d.encrypted_size(n)))
    for c in cs.values():
        c.close()
    return out


SMALL = [1, 100, 65535, 65537, 200000, 300001, 500000, 900000]


def test_batcher_gets_merge_both_ciphers(mb):
    """a GET batch admitted at 1 runs one more launch (the ChaCha20 open) than one admitted at 0, whatever its ciphers; AES and
    ChaCha20 GETs merge into shared batches and each gets its plaintext"""
    parts = sse_parts(mb, SMALL, lambda i: i % 2)
    b = mb.Batcher(K, M, MiB, max_wait_us=200000)

    def gets(idx):
        dsts = [pinned(mb, np.zeros(parts[j][0].size, np.uint8)) for j in idx]
        res = run_all([lambda q=q, j=j: b.decode_sse(parts[j][1], 0, parts[j][0].size, parts[j][2], key_of(j), dst=dsts[q])
                       for q, j in enumerate(idx)])
        for j, (out, hint) in zip(idx, res):
            assert hint == 0 and np.array_equal(out, parts[j][0]), j

    def delta(fn):
        s0 = {s: b.stat(s) for s in ("launches", "batches", "sse_gets", "sse_serial")}
        fn()
        return {s: b.stat(s) - v for s, v in s0.items()}

    gets([0])  # the codec's AES tables: out of the counts below
    one = delta(lambda: gets([2]))  # one AES GET admitted at 0: a batch of its own
    assert one["batches"] == 1
    base = one["launches"]
    b.set_option("dare_chacha20", 1)
    for j in (4, 1):  # an AES and a ChaCha20 GET admitted at 1: setup, AES open, ChaCha20 open
        got = delta(lambda j=j: gets([j]))
        assert got["batches"] == 1 and got["launches"] == base + 1, j
    merged = delta(lambda: gets(list(range(len(SMALL)))))
    assert merged["batches"] < len(SMALL)  # calls were merged, both ciphers in shared batches
    assert merged["launches"] == merged["batches"] * (base + 1)
    assert merged["sse_gets"] == len(SMALL) and b.stat("sse_serial") == 0
    b.close()


def test_batcher_puts_at_option2(mb):
    """PUTs admitted at 2 seal with ONE ChaCha20 launch and no setup; a batch mixing 0 and 2 runs setup, AES and ChaCha20 seals"""
    b = mb.Batcher(K, M, MiB, max_wait_us=200000)
    c0, c2 = codec_at(mb, 0), codec_at(mb, 2)
    w = pinned(mb, d.plaintext(100, 1))
    b.encode_sse(w, key_of(0), nonce_of(0), pinned=True)  # the AES tables
    plains = [pinned(mb, np.zeros(d.encrypted_size(n), np.uint8)) for n in SMALL]
    ptxt = [pinned(mb, d.plaintext(n, 3 + i)) for i, n in enumerate(SMALL)]

    def stats():
        return {s: b.stat(s) for s in ("launches", "batches", "sse_puts", "sse_serial")}

    s0 = stats()
    run_all([lambda p=p: b.encode(p, pinned=True) for p in plains])
    s1 = stats()
    b.set_option("dare_chacha20", 2)
    got = run_all([lambda i=i: b.encode_sse(ptxt[i], key_of(i), nonce_of(i), pinned=True) for i in range(len(SMALL))])
    s2 = stats()
    assert s1["batches"] - s0["batches"] == 1 and s2["batches"] - s1["batches"] == 1
    base = s1["launches"] - s0["launches"]
    assert s2["launches"] - s1["launches"] == base + 1
    assert s2["sse_puts"] - s1["sse_puts"] == len(SMALL) and s2["sse_serial"] == 0
    for i in range(len(SMALL)):
        want = c2.encode_sse(ptxt[i], key_of(i), nonce_of(i))
        assert all(np.array_equal(x, y) for x, y in zip(got[i], want)), SMALL[i]
    # half admitted at 0, then (the batch still open) half at 2
    fns, delays = [], []
    for i in range(len(SMALL)):
        fns.append(lambda i=i: b.encode_sse(ptxt[i], key_of(i), nonce_of(i), pinned=True))
        delays.append(0.0 if i < 4 else 0.05)
    b.set_option("dare_chacha20", 0)
    timer = threading.Timer(0.025, lambda: b.set_option("dare_chacha20", 2))
    timer.start()
    got = run_all(fns, delays)
    timer.join()
    s3 = stats()
    if s3["batches"] - s2["batches"] == 1:  # the late half joined the open batch
        assert s3["launches"] - s2["launches"] == base + 3  # setup, AES seal, ChaCha20 seal
    for i in range(len(SMALL)):
        want = (c0 if i < 4 else c2).encode_sse(ptxt[i], key_of(i), nonce_of(i))
        assert all(np.array_equal(x, y) for x, y in zip(got[i], want)), (i, SMALL[i])
    c0.close(); c2.close()
    b.close()


def test_batcher_isolation(mb):
    """among good ChaCha20 GETs admitted at 1: a tampered one, one admitted at 0 and one redone for bitrot each get their own
    result"""
    n = 3 * PKG + 100
    (pt, files, e), = sse_parts(mb, [n], lambda i: 1)
    c = codec_at(mb, 1)
    ct, _ = c.decode(files, 0, e, e)
    t = ct.copy()
    t[EPKG + 500] ^= 1
    tampered = [pinned(mb, f) for f in c.encode(t)]
    rot = [f.copy() for f in files]
    rot[0][32 + 7] ^= 0x40
    rot = [pinned(mb, f) for f in rot]
    b = mb.Batcher(K, M, MiB, max_wait_us=200000)
    cases = [(files, UNSUPPORTED), (tampered, NOT_AUTHENTIC), (rot, n)] + [(files, n)] * 5  # case 0 is admitted at 0
    dsts = [pinned(mb, np.full(n, 0xAA, np.uint8)) for _ in cases]
    keys = [key_of(0) for _ in cases]
    L = mb.lib()

    def call(j):
        return L.mec_batcher_decode_sse(b.h, mb.capi._ptrs(cases[j][0]), None, 0, n, e, keys[j].ctypes.data, dsts[j].ctypes.data, None)

    before = {s: b.stat(s) for s in ("redone", "sse_serial", "batches")}
    timer = threading.Timer(0.025, lambda: b.set_option("dare_chacha20", 1))
    timer.start()
    rcs = run_all([lambda j=j: call(j) for j in range(len(cases))], [0.0] + [0.05] * (len(cases) - 1))
    timer.join()
    for j, ((_, want), rc) in enumerate(zip(cases, rcs)):
        assert rc == want, j
        assert (not dsts[j].any()) if want < 0 else np.array_equal(dsts[j], pt), j
    assert b.stat("redone") - before["redone"] == 1 and b.stat("sse_serial") - before["sse_serial"] == 1
    c.close()
    b.close()
