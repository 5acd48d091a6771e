"""Server-side encryption on the GPU: DARE 2.0 AES-256-GCM packages sealed by mec_dare_device and mec_encode_sse and opened by
mec_dare_device and mec_decode_sse, checked against the committed host-made streams of tests/golden/dare_streams.json (no
`cryptography` here).  Every case checks the output bytes and the "dare_sealed" / "dare_opened" package counters.

What pins the format: MinIO's SSE-C sealed object key (one final package at sequence 0: header layout, nonce placement, final bit,
additional data, tag) opens on the GPU.  The sequence-number XOR of later packages is not pinned by MinIO's bytes; it follows the
published DARE 2.0 specification, as the fixture streams do."""
import base64
import hashlib
import json
import os

import numpy as np
import pytest

import dare_ref as d

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MiB = 1 << 20
PKG, EPKG = d.PKG, d.EPKG
NOT_AUTHENTIC, UNSUPPORTED = -13, -102
KEY, NONCE = bytes(range(32)), bytes.fromhex("0123456789abcdeffedcba98")


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
    c = mb.Codec(12, 4, MiB)
    yield c
    c.close()


def npk(n):
    return -(-n // PKG)


def dev(buf):
    import torch
    return torch.from_numpy(np.array(buf, dtype=np.uint8)).to("cuda")


def seal(c, key, nonce, pt, seq0=0):
    """one stream through mec_dare_device -> sealed bytes"""
    import torch
    pt = np.frombuffer(bytes(pt), np.uint8) if not isinstance(pt, np.ndarray) else pt
    n = pt.size
    src = dev(pt) if n else torch.zeros(1, dtype=torch.uint8, device="cuda")
    out = torch.zeros(max(d.encrypted_size(n), 1), dtype=torch.uint8, device="cuda")
    before = c.stat("dare_sealed")
    c.dare_device(1, np.frombuffer(key, np.uint8), src.data_ptr(), [0], [n], out.data_ptr(), [0], seq0=[seq0],
                  nonces=np.frombuffer(nonce, np.uint8))
    assert c.stat("dare_sealed") - before == npk(n)
    return out.cpu().numpy()[:d.encrypted_size(n)].tobytes()


def open_(c, key, stream, enc_total, seq0=0, fill=0xAA, out_len=None):
    """one stream through mec_dare_device -> (rc, status, plaintext buffer pre-filled with `fill`)"""
    import torch
    st = np.frombuffer(bytes(stream), np.uint8)
    src = dev(st) if st.size else torch.zeros(1, dtype=torch.uint8, device="cuda")
    n = out_len if out_len is not None else PKG * (len(stream) // EPKG + 1)
    out = torch.full((n,), fill, dtype=torch.uint8, device="cuda")
    rc, status = c.dare_device(2, np.frombuffer(key, np.uint8), src.data_ptr(), [0], [st.size], out.data_ptr(), [0], seq0=[seq0],
                               enc_totals=[enc_total], check=False)
    return rc, int(status[0]), out.cpu().numpy()


def check_stream(s, got):
    what = f"length {s['length']} seq0 {s['seq0']}"
    assert d.excerpts(got) == {f: s[f] for f in ("first_head", "first_tag", "last_head", "last_tag")}, what
    assert hashlib.sha256(got).hexdigest() == s["sha256"], what


# ---- mec_dare_device ------------------------------------------------------------------------------------------------------------
def test_seal_many_streams_one_launch(codec, fx):
    """every fixture stream (three keys, non-zero seq0, lengths 1 B .. 1 MiB + 5) in one call at odd offsets, then one at a time"""
    import torch
    ss = fx["streams"]
    pts = [d.plaintext(s["length"], s["seed"]) for s in ss]
    in_off, out_off, a, b = [], [], 3, 5
    for p in pts:
        in_off.append(a); out_off.append(b)
        a += p.size + 7; b += d.encrypted_size(p.size) + 9
    host = np.zeros(a, np.uint8)
    for o, p in zip(in_off, pts):
        host[o:o + p.size] = p
    seal(codec, KEY, NONCE, b"x")  # the codec's AES tables are built
    src, out = dev(host), torch.zeros(b, dtype=torch.uint8, device="cuda")
    keys = np.concatenate([np.frombuffer(bytes.fromhex(s["key"]), np.uint8) for s in ss])
    nonces = np.concatenate([np.frombuffer(bytes.fromhex(s["nonce"]), np.uint8) for s in ss])
    before, launches = codec.stat("dare_sealed"), codec.launches
    codec.dare_device(1, keys, src.data_ptr(), in_off, [p.size for p in pts], out.data_ptr(), out_off, seq0=[s["seq0"] for s in ss],
                      nonces=nonces)
    assert codec.stat("dare_sealed") - before == sum(npk(p.size) for p in pts)
    assert codec.launches - launches == 2  # the H powers of every stream, then every package
    o = out.cpu().numpy()
    for s, off, p in zip(ss, out_off, pts):
        check_stream(s, o[off:off + d.encrypted_size(p.size)].tobytes())
    # and all of them open again in one call; a stream sealed from sequence number seq0 is the tail of a part of seq0 more packages
    plain = torch.full((a,), 0xAA, dtype=torch.uint8, device="cuda")
    before = codec.stat("dare_opened")
    rc, status = codec.dare_device(2, keys, out.data_ptr(), out_off, [d.encrypted_size(p.size) for p in pts], plain.data_ptr(), in_off,
                                   seq0=[s["seq0"] for s in ss],
                                   enc_totals=[s["seq0"] * EPKG + d.encrypted_size(p.size) for s, p in zip(ss, pts)])
    assert rc == 0 and not status.any()
    assert codec.stat("dare_opened") - before == sum(npk(p.size) for p in pts)
    pl = plain.cpu().numpy()
    for off, p in zip(in_off, pts):
        assert np.array_equal(pl[off:off + p.size], p)
    for s, p in zip(ss, pts):
        check_stream(s, seal(codec, bytes.fromhex(s["key"]), bytes.fromhex(s["nonce"]), p, s["seq0"]))


def test_sealed_key_vector_opens_on_gpu(codec, fx):
    s = fx["sealed_key"]
    rc, st, out = open_(codec, bytes.fromhex(s["sealing_key"]), base64.b64decode(s["sealed_key"]), 64)
    assert rc == 0 and st == 0 and out[:32].tobytes().hex() == s["object_key"]


def test_open_ranged_read(codec, fx):
    """a ranged read starts at the sequence number of its first package: packages 1..2 of a four-package stream"""
    s = next(x for x in fx["streams"] if x["length"] == 3 * PKG + 5 and x["seq0"] == 0)
    pt = d.plaintext(s["length"], s["seed"])
    st = seal(codec, KEY, NONCE, pt)
    before = codec.stat("dare_opened")
    rc, status, out = open_(codec, KEY, st[EPKG:3 * EPKG], len(st), seq0=1, out_len=2 * PKG)
    assert rc == 0 and status == 0 and np.array_equal(out, pt[PKG:3 * PKG])
    assert codec.stat("dare_opened") - before == 2
    rc, status, out = open_(codec, KEY, st[EPKG:3 * EPKG], len(st), seq0=0, out_len=2 * PKG)  # wrong position: nonce differs
    assert rc == NOT_AUTHENTIC and status == 13 and (out == 0xAA).all()


@pytest.fixture(scope="module")
def four(codec):
    pt = d.plaintext(3 * PKG + 5, 8)
    return pt, seal(codec, KEY, NONCE, pt)


def flip(b, i, bit=1):
    b = bytearray(b)
    b[i] ^= bit
    return bytes(b)


# case -> (stream, stored size, key, packages that still open, packages opened) from the four-package stream (3 x 65536 + 5 bytes)
TAMPER = {
    "header": lambda st: (flip(st, EPKG + 9), len(st), KEY, {0, 2, 3}, 4),                  # nonce byte of package 1
    "ciphertext": lambda st: (flip(st, 2 * EPKG + 16 + 777, 0x10), len(st), KEY, {0, 1, 3}, 4),
    "tag": lambda st: (flip(st, len(st) - 3, 0x80), len(st), KEY, {0, 1, 2}, 4),
    "swap": lambda st: (st[EPKG:2 * EPKG] + st[:EPKG] + st[2 * EPKG:], len(st), KEY, {2, 3}, 4),
    "drop_final": lambda st: (st[:3 * EPKG], 3 * EPKG, KEY, {0, 1}, 3),                     # package 2 is the part's last, not final
    "move_final": lambda st: (flip(flip(st, 4, 0x80), 3 * EPKG + 4, 0x80), len(st), KEY, {1, 2}, 4),
    "wrong_key": lambda st: (st, len(st), bytes(31) + b"\x01", set(), 4),
    "trailing_40": lambda st: (st + bytes(40), len(st) + 40, KEY, {0, 1, 2}, 4),              # package 3's length no longer fits
    "trailing_10": lambda st: (st + bytes(10), len(st) + 10, KEY, {0, 1, 2}, 4),
    "trailing_beyond_size": lambda st: (st + bytes(50), len(st), KEY, {0, 1, 2, 3}, 4),      # bytes past the stored size
    "cut_short": lambda st: (st[:-1], len(st), KEY, {0, 1, 2}, 3),
    "bad_size": lambda st: (st, len(st) - 5, KEY, set(), 0),                                  # no DARE size
}


@pytest.mark.parametrize("case", list(TAMPER))
def test_tamper_not_authentic(codec, four, case):
    """each tampered stream is MEC_ERR_NOT_AUTHENTIC, and a package that fails leaves its plaintext untouched"""
    pt, st = four
    st, total, key, good, rows = TAMPER[case](st)
    before = codec.stat("dare_opened")
    rc, status, out = open_(codec, key, st, total, out_len=4 * PKG)
    assert rc == NOT_AUTHENTIC and status == 13 and codec.stat("dare_opened") - before == rows
    for p in range(4):
        lo, hi = p * PKG, min(pt.size, (p + 1) * PKG)
        assert np.array_equal(out[lo:hi], pt[lo:hi]) if p in good else (out[lo:hi] == 0xAA).all(), (case, p)


@pytest.mark.parametrize("field", ["cipher", "version"])
def test_unsupported(codec, four, field):
    """a ChaCha20-Poly1305 package or a DARE 1.0 stream is left to sio: MEC_ERR_UNSUPPORTED"""
    pt, st = four
    b = bytearray(st)
    if field == "cipher":
        b[EPKG + 1] = 1
    else:
        for p in range(4):
            b[p * EPKG] = 0x10
    rc, status, out = open_(codec, KEY, bytes(b), len(b), out_len=4 * PKG)
    assert rc == UNSUPPORTED and status == 102
    if field == "cipher":
        assert (out[PKG:2 * PKG] == 0xAA).all() and np.array_equal(out[:PKG], pt[:PKG])


# ---- mec_encode_sse / mec_decode_sse ---------------------------------------------------------------------------------------------
def reference_stream(c, fx, n, seed):
    """the DARE stream of plaintext(n, seed) under KEY / NONCE: checked against the fixture where it has that stream, otherwise
    sealed by mec_dare_device (which the fixture pins at every length above)"""
    pt = d.plaintext(n, seed)
    st = seal(c, KEY, NONCE, pt)
    for s in fx["streams"]:
        if s["length"] == n and s["seed"] == seed and s["seq0"] == 0 and s["key"] == KEY.hex():
            check_stream(s, st)
    return pt, np.frombuffer(st, np.uint8)


def straddles(E, chunk_bytes):
    return sum(1 for x in range(chunk_bytes, E, chunk_bytes) if x % EPKG)


GEOMS = [(12, 4, MiB), (4, 2, MiB), (16, 4, MiB), (12, 4, 10 * MiB)]


@pytest.mark.parametrize("k,m,bs", GEOMS)
def test_encode_sse_equals_encode_of_stream(mb, fx, k, m, bs):
    c = mb.Codec(k, m, bs)
    fixture_seed = {s["length"]: s["seed"] for s in fx["streams"] if s["key"] == KEY.hex() and s["seq0"] == 0}
    lengths = [0, 1, 2 * PKG, 3 * PKG + 5, MiB + 5, 5 * MiB + 12345, 2 * bs + 777]
    for n in lengths:
        seed = fixture_seed.get(n, 3)
        pt, st = reference_stream(c, fx, n, seed)
        want = c.encode(st)
        before = c.stat("dare_sealed")
        got = c.encode_sse(pt, KEY, NONCE)
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), (k, m, bs, n)
        assert c.stat("dare_sealed") - before >= npk(n)
    # small chunks: packages across erasure blocks and across pipeline chunks are sealed in both chunks
    for cb in (1, 2):
        c.set_option("chunk_blocks", cb)
        n = 3 * bs + 4321
        pt, st = reference_stream(c, fx, n, 5)
        want = c.encode(st)
        before = c.stat("dare_sealed")
        got = c.encode_sse(pt, KEY, NONCE)
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), (k, m, bs, cb)
        assert c.stat("dare_sealed") - before == npk(n) + straddles(len(st), cb * bs)
    c.set_option("chunk_blocks", 0)
    c.close()


def test_encode_sse_checksums_are_of_plaintext(mb, fx):
    c = mb.Codec(12, 4, MiB)
    c.set_option("checksums", 7)
    for cb, n in ((1, 5 * MiB + 12345), (0, 3 * PKG + 5), (3, 7 * MiB)):
        c.set_option("chunk_blocks", cb)
        pt = d.plaintext(n, 4)
        c.encode_sse(pt, KEY, NONCE)
        crcs, ln = c.last_checksums()
        assert ln == n and crcs == c.checksums(pt, 7), (cb, n)
    c.close()


@pytest.fixture(scope="module")
def part(mb, fx):
    """a 5 MiB + 12345 B object sealed and encoded in RS(12,4) with 1 MiB blocks"""
    c = mb.Codec(12, 4, MiB)
    pt = d.plaintext(5 * MiB + 12345, 6)
    files = c.encode_sse(pt, KEY, NONCE)
    c.close()
    return pt, files, d.encrypted_size(pt.size)


def ranges(D):
    blk = MiB * PKG // EPKG  # plaintext offset near the first erasure-block boundary of the ciphertext
    return [(0, D), (100, 70000), (PKG, PKG), (PKG - 1, 2), (15 * PKG + 3, 2 * PKG), (blk - 10, 20), (3 * blk + 5, 2 * MiB),
            (D - 1, 1), (D - 70000, 70000), (0, 1)]


def opened_for(off, ln):
    return (off + ln - 1) // PKG - off // PKG + 1


@pytest.mark.parametrize("cb", [0, 1])
@pytest.mark.parametrize("offline", [(), (0, 5, 13), (0, 1, 2, 3)])
def test_decode_sse_ranges(mb, part, cb, offline):
    pt, files, E = part
    c = mb.Codec(12, 4, MiB)
    c.set_option("chunk_blocks", cb)
    fs = [None if i in offline else f for i, f in enumerate(files)]
    for off, ln in ranges(pt.size):
        before = c.stat("dare_opened")
        out, hint = c.decode_sse(fs, off, ln, E, KEY)
        assert hint == 0 and np.array_equal(out, pt[off:off + ln]), (off, ln, offline, cb)
        assert c.stat("dare_opened") - before == opened_for(off, ln)
    c.close()


def test_decode_sse_prefer_and_corrupt_frame(mb, part):
    pt, files, E = part
    c = mb.Codec(12, 4, MiB)
    c.set_option("chunk_blocks", 1)
    prefer = [0] * 4 + [1] * 12
    for off, ln in ranges(pt.size):
        out, hint = c.decode_sse(files, off, ln, E, KEY, prefer=prefer)
        assert hint == 0 and np.array_equal(out, pt[off:off + ln])
    # a corrupt frame in block 3 of data drive 2: the reader is dropped, the range resumes with drive 12, heal_hint is set
    bad = [f.copy() for f in files]
    S = c.shard_size()
    bad[2][3 * (32 + S) + 32 + 1000] ^= 0x40
    for off, ln in [(0, pt.size), (3 * MiB - 5000, 10000), (2 * MiB, 2 * MiB)]:
        before = c.stat("dare_opened")
        out, hint = c.decode_sse(bad, off, ln, E, KEY)
        assert np.array_equal(out, pt[off:off + ln]) and hint == -7
        assert c.stat("dare_opened") - before == opened_for(off, ln)
    c.close()


def test_decode_sse_wrong_key(mb, part):
    pt, files, E = part
    c = mb.Codec(12, 4, MiB)
    with pytest.raises(mb.MecError) as e:
        c.decode_sse(files, 0, 1000, E, bytes(32))
    assert e.value.code == NOT_AUTHENTIC
    dst = np.full(1000, 0x55, np.uint8)
    import ctypes as C
    ptrs = (C.c_void_p * 16)(*[f.ctypes.data for f in files])
    assert mb.lib().mec_decode_sse(c.h, ptrs, None, 0, 1000, E, bytes(32), dst.ctypes.data, None) == NOT_AUTHENTIC
    assert not dst.any()  # nothing of a range that does not open is handed out
    out, hint = c.decode_sse(files, 0, 1000, E, KEY)  # the failed call left nothing behind that breaks the next
    assert np.array_equal(out, pt[:1000])
    c.close()


def test_multipart_part_keys(mb):
    """three parts sealed with DerivePartKey keys, each read back with its own key, one call per part"""
    c = mb.Codec(4, 2, MiB)
    object_key = hashlib.sha256(b"object key").digest()
    sizes = [5 * MiB, 5 * MiB + 1, 12345]
    parts = []
    for i, n in enumerate(sizes):
        pk = d.derive_part_key(object_key, i + 1)
        pt = d.plaintext(n, 20 + i)
        nonce = hashlib.sha256(b"nonce%d" % i).digest()[:12]
        parts.append((pk, pt, c.encode_sse(pt, pk, nonce)))
    for pk, pt, files in parts:
        E = d.encrypted_size(pt.size)
        out, hint = c.decode_sse(files, 0, pt.size, E, pk)
        assert np.array_equal(out, pt) and hint == 0
        out, _ = c.decode_sse(files, pt.size // 3, pt.size // 2, E, pk)
        assert np.array_equal(out, pt[pt.size // 3:pt.size // 3 + pt.size // 2])
    with pytest.raises(mb.MecError):
        c.decode_sse(parts[1][2], 0, 10, d.encrypted_size(sizes[1]), parts[0][0])  # another part's key
    c.close()


def test_heal_transcode_verify_unchanged(mb, part):
    """an SSE part is an ordinary part whose object bytes are ciphertext: healed, moved and scanned as before, and it still opens"""
    pt, files, E = part
    c = mb.Codec(12, 4, MiB)
    stale = [i in (1, 14) for i in range(16)]
    outs = c.heal([None if s else f for s, f in zip(stale, files)], stale, E)
    for i in (1, 14):
        assert np.array_equal(outs[i], files[i])
    healed = [outs[i] if stale[i] else f for i, f in enumerate(files)]
    out, hint = c.decode_sse([None if i in (0, 2, 3) else f for i, f in enumerate(healed)], 0, pt.size, E, KEY)
    assert np.array_equal(out, pt) and hint == 0
    for f in files:
        assert c.bitrot_verify(f, c.shard_file_size(E)) == 0
    dst = mb.Codec(6, 2, MiB)
    moved, hint = c.transcode(files, E, dst)
    assert hint == 0
    out, hint = dst.decode_sse(moved, 123, pt.size - 246, E, KEY)
    assert np.array_equal(out, pt[123:pt.size - 123]) and hint == 0
    c.close()
    dst.close()
