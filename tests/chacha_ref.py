"""Pure-Python reference of DARE 2.0 ChaCha20-Poly1305 streams (cipher 1; minio/sio, RFC 8439 §2.8): ChaCha20 vectorised with numpy
over every block of a package, Poly1305 with Python integers.  Header, nonce and sizes are dare_ref's; no crypto package needed."""
import struct

import numpy as np

import dare_ref as d

P1305 = (1 << 130) - 5
_SIGMA = np.array([0x61707865, 0x3320646E, 0x79622D32, 0x6B206574], dtype=np.uint32)


def _rotl(x, n):
    return (x << np.uint32(n)) | (x >> np.uint32(32 - n))


def chacha20_blocks(key, nonce, counter0, nblocks):
    """keystream blocks counter0 .. counter0 + nblocks - 1 as an (nblocks, 64) uint8 array (RFC 8439 §2.3)"""
    k = np.frombuffer(bytes(key), dtype="<u4").astype(np.uint32)
    n = np.frombuffer(bytes(nonce), dtype="<u4").astype(np.uint32)
    init = np.zeros((16, nblocks), dtype=np.uint32)
    init[0:4] = _SIGMA[:, None]
    init[4:12] = k[:, None]
    init[12] = (np.arange(nblocks, dtype=np.uint64) + counter0).astype(np.uint32)
    init[13:16] = n[:, None]
    x = init.copy()

    def qr(a, b, c, dd):
        x[a] += x[b]; x[dd] ^= x[a]; x[dd] = _rotl(x[dd], 16)
        x[c] += x[dd]; x[b] ^= x[c]; x[b] = _rotl(x[b], 12)
        x[a] += x[b]; x[dd] ^= x[a]; x[dd] = _rotl(x[dd], 8)
        x[c] += x[dd]; x[b] ^= x[c]; x[b] = _rotl(x[b], 7)

    with np.errstate(over="ignore"):
        for _ in range(10):
            qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
            qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
        x += init
    return np.ascontiguousarray(x.T).astype("<u4").view(np.uint8).reshape(nblocks, 64)


def poly1305(otk, msg):
    """Poly1305 tag of msg under the 32-byte one-time key (RFC 8439 §2.5)"""
    r = int.from_bytes(otk[:16], "little") & 0x0FFFFFFC0FFFFFFC0FFFFFFC0FFFFFFF
    s = int.from_bytes(otk[16:32], "little")
    acc = 0
    for i in range(0, len(msg), 16):
        acc = (acc + int.from_bytes(msg[i:i + 16] + b"\x01", "little")) * r % P1305
    return ((acc + s) & ((1 << 128) - 1)).to_bytes(16, "little")


def _pad16(b):
    return b + bytes(-len(b) % 16)


def aead_mac_data(aad, ct):
    """the Poly1305 message of RFC 8439 §2.8: aad and ciphertext zero padded to 16, then both lengths as uint64 LE"""
    return _pad16(bytes(aad)) + _pad16(bytes(ct)) + struct.pack("<QQ", len(aad), len(ct))


def xor_keystream(key, nonce, data):
    data = np.frombuffer(bytes(data), np.uint8)
    if data.size == 0:
        return b""
    ks = chacha20_blocks(key, nonce, 1, -(-data.size // 64)).reshape(-1)[:data.size]
    return (data ^ ks).tobytes()


def aead_seal(key, nonce, pt, aad):
    """ChaCha20-Poly1305 (RFC 8439 §2.8): ciphertext || tag"""
    otk = chacha20_blocks(key, nonce, 0, 1).tobytes()[:32]
    ct = xor_keystream(key, nonce, pt)
    return ct + poly1305(otk, aead_mac_data(aad, ct))


def aead_open(key, nonce, sealed, aad):
    """plaintext, or None if the tag does not match"""
    sealed = bytes(sealed)
    ct, tag = sealed[:-16], sealed[-16:]
    otk = chacha20_blocks(key, nonce, 0, 1).tobytes()[:32]
    if poly1305(otk, aead_mac_data(aad, ct)) != tag:
        return None
    return xor_keystream(key, nonce, ct)


def seal_chacha(key, nonce, plaintext, seq0=0):
    """the DARE 2.0 ChaCha20-Poly1305 stream of `plaintext`, its first package at sequence number seq0"""
    out = bytearray()
    pt = bytes(plaintext)
    n = len(pt)
    for i, p in enumerate(range(0, n, d.PKG)):
        chunk = pt[p:p + d.PKG]
        h = d.header(len(chunk), nonce, p + d.PKG >= n, cipher=1)
        out += h + aead_seal(key, d.aead_nonce(h, seq0 + i), chunk, h[:4])
    return bytes(out)


def open_chacha(key, stream, seq0=0):
    """plaintext of a DARE 2.0 ChaCha20-Poly1305 stream; raises ValueError on any package that does not authenticate"""
    stream = bytes(stream)
    out = bytearray()
    pos, i = 0, 0
    while pos < len(stream):
        h = stream[pos:pos + 16]
        if h[0] != 0x20 or h[1] != 1:
            raise ValueError("not a DARE 2.0 ChaCha20-Poly1305 package")
        ln = struct.unpack_from("<H", h, 2)[0] + 1
        pt = aead_open(key, d.aead_nonce(h, seq0 + i), stream[pos + 16:pos + 16 + ln + 16], h[:4])
        if pt is None:
            raise ValueError(f"package {i} does not authenticate")
        out += pt
        pos += 16 + ln + 16
        i += 1
    return bytes(out)
