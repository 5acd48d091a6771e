#!/usr/bin/env python
"""Generate tests/golden/dare_chacha_streams.json with Python `cryptography`'s ChaCha20Poly1305, so the GPU tests need no crypto
package.  Each stream is dare_ref.plaintext(length, seed) sealed as DARE 2.0 cipher-1 packages from sequence number seq0: SHA-256 of
the stream and dare_ref.excerpts, one line per stream.  The lengths cover the package boundaries and the Poly1305 thread-stride
boundaries of the device kernel (T = ceil(len / 16) + 2 blocks per package at T = 255, 256, 257, 512, 513)."""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import dare_ref as d  # noqa: E402

KEYS = {"a": bytes(range(32)), "b": bytes((0xF0 - 3 * i) & 0xFF for i in range(32)), "c": hashlib.sha256(b"dare c").digest()}
NONCES = {"a": bytes.fromhex("0123456789abcdeffedcba98"), "b": bytes.fromhex("fffefdfcfbfaf9f8f7f6f5f4"), "c": bytes(12)}
LENGTHS = [1, 15, 16, 17, 63, 64, 65, 65535, 65536, 65537, 3 * 65536 + 5, (1 << 20) + 5]
STRIDE = sorted({x for T in (255, 256, 257, 512, 513) for x in (16 * (T - 2), 16 * (T - 2) - 7)})
EXTRA = [(131072 + 100, "b", 5), (70000, "c", 0), (3 * 65536 + 5, "a", 7), (4000, "b", 0xFFFFFFFE)]  # (length, key, seq0)


def seal(key, nonce, plaintext, seq0=0):
    from cryptography.hazmat.primitives.ciphers.aead import ChaCha20Poly1305
    g = ChaCha20Poly1305(bytes(key))
    out = bytearray()
    n = len(plaintext)
    for i, p in enumerate(range(0, n, d.PKG)):
        chunk = bytes(plaintext[p:p + d.PKG])
        h = d.header(len(chunk), nonce, p + d.PKG >= n, cipher=1)
        out += h + g.encrypt(d.aead_nonce(h, seq0 + i), chunk, h[:4])
    return bytes(out)


def main():
    streams = []
    for n, kid, seq0 in [(n, "a", 0) for n in LENGTHS + STRIDE] + EXTRA:
        pt = d.plaintext(n, seed=len(streams)).tobytes()
        st = seal(KEYS[kid], NONCES[kid], pt, seq0)
        assert len(st) == d.encrypted_size(n)
        streams.append({"length": n, "seed": len(streams), "key": KEYS[kid].hex(), "nonce": NONCES[kid].hex(), "seq0": seq0,
                        "sha256": hashlib.sha256(st).hexdigest(), **d.excerpts(st)})
    with open(os.path.join(HERE, "dare_chacha_streams.json"), "w") as f:
        f.write('{"streams": [\n  ' + ",\n  ".join(json.dumps(x) for x in streams) + "]}\n")  # one line per stream


if __name__ == "__main__":
    main()
