"""Host reference of the DARE 2.0 stream format (minio/sio, AES-256-GCM; layout in include/minio_ec.h).  seal / open_stream need
Python `cryptography` (fixture generation and CPU tests); the GPU tests use only the pure-Python helpers."""
import hashlib
import hmac
import struct

PKG = 65536          # payload bytes of a full package
OVERHEAD = 32        # header + tag
EPKG = PKG + OVERHEAD


def encrypted_size(n):
    """sio.EncryptedSize"""
    if n < 0:
        raise ValueError("negative size")
    return (n // PKG) * EPKG + ((n % PKG) + OVERHEAD if n % PKG else 0)


def decrypted_size(n):
    """sio.DecryptedSize: a remainder of 1..32 bytes is no package"""
    if n < 0:
        raise ValueError("negative size")
    r = n % EPKG
    if 0 < r <= OVERHEAD:
        raise ValueError("invalid encrypted size")
    return (n // EPKG) * PKG + (r - OVERHEAD if r else 0)


def derive_part_key(object_key, part_id):
    """ObjectKey.DerivePartKey: HMAC-SHA256(object key, uint32 LE part id)"""
    return hmac.new(bytes(object_key), struct.pack("<I", part_id), hashlib.sha256).digest()


def ssec_sealing_key(client_key, iv, bucket, obj):
    """the key that seals an SSE-C object key: HMAC-SHA256 over iv | "SSE-C" | "DAREv2-HMAC-SHA256" | bucket/object"""
    return hmac.new(bytes(client_key), bytes(iv) + b"SSE-C" + b"DAREv2-HMAC-SHA256" + f"{bucket}/{obj}".encode(),
                    hashlib.sha256).digest()


def decrypted_range(size, offset, length):
    """GetDecryptedRange of a single-part object of `size` plaintext bytes: (enc_off, enc_len, skip, seq)"""
    start_pkg = offset // PKG
    skip = offset % PKG
    enc_off = start_pkg * EPKG
    end_pkg = (offset + length - 1) // PKG
    end_enc = min((end_pkg + 1) * EPKG, encrypted_size(size))
    return enc_off, end_enc - enc_off, skip, start_pkg


def aead_nonce(header, seq):
    n = bytearray(header[4:16])
    v = struct.unpack_from("<I", n, 8)[0] ^ (seq & 0xFFFFFFFF)
    struct.pack_into("<I", n, 8, v)
    return bytes(n)


def header(length, nonce, final, version=0x20, cipher=0):
    h = bytearray(16)
    h[0], h[1] = version, cipher
    struct.pack_into("<H", h, 2, length - 1)
    h[4:16] = nonce
    h[4] = (h[4] | 0x80) if final else (h[4] & 0x7F)
    return bytes(h)


def seal(key, nonce, plaintext, seq0=0):
    """the DARE 2.0 stream of `plaintext`, its first package at sequence number seq0 (0 for a part)"""
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
    g = AESGCM(bytes(key))
    out = bytearray()
    n = len(plaintext)
    for i, p in enumerate(range(0, n, PKG)):
        chunk = bytes(plaintext[p:p + PKG])
        h = header(len(chunk), nonce, p + PKG >= n)
        out += h + g.encrypt(aead_nonce(h, seq0 + i), chunk, h[:4])
    return bytes(out)


def open_stream(key, stream, seq0=0):
    """plaintext of a DARE 2.0 AES-256-GCM stream; raises on any package that does not authenticate"""
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
    g = AESGCM(bytes(key))
    out = bytearray()
    pos, i = 0, 0
    while pos < len(stream):
        h = bytes(stream[pos:pos + 16])
        ln = struct.unpack_from("<H", h, 2)[0] + 1
        out += g.decrypt(aead_nonce(h, seq0 + i), bytes(stream[pos + 16:pos + 16 + ln + 16]), h[:4])
        pos += 16 + ln + 16
        i += 1
    return bytes(out)


def excerpts(stream):
    """where a stream that differs starts to differ: header + first 32 ciphertext bytes and tag of its first and last packages"""
    stream = bytes(stream)
    first, last = stream[:EPKG], stream[(max(len(stream) - 1, 0) // EPKG) * EPKG:]
    return {"first_head": first[:48].hex(), "first_tag": first[-16:].hex(), "last_head": last[:48].hex(), "last_tag": last[-16:].hex()}


def plaintext(n, seed):
    """the seeded plaintext of the fixture streams: byte j = (j * 131 + seed * 7 + (j >> 16)) mod 256"""
    import numpy as np
    j = np.arange(n, dtype=np.int64)
    return ((j * 131 + seed * 7 + (j >> 16)) & 0xFF).astype(np.uint8)
