#!/usr/bin/env python
"""Generate tests/golden/dare_streams.json with Python `cryptography` (tests/dare_ref.py), so the GPU tests need no crypto package.
  sealed_key  MinIO's SSE-C sealed object key (internal/crypto/sse_test.go) and the object key it opens to: one package at sequence 0
              pinning header layout, nonce and final bit, additional data and tag
  part_keys   DerivePartKey of the all-zero object key (internal/crypto/key_test.go)
  streams     plaintext dare_ref.plaintext(length, seed) sealed from seq0: SHA-256 of the stream and dare_ref.excerpts
Later packages' sequence-number XOR is not pinned by MinIO's bytes; it follows the published DARE 2.0 specification."""
import base64
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import dare_ref as d  # noqa: E402

KEYS = {"a": bytes(range(32)), "b": bytes((0xF0 - 3 * i) & 0xFF for i in range(32)), "c": hashlib.sha256(b"dare c").digest()}
NONCES = {"a": bytes.fromhex("0123456789abcdeffedcba98"), "b": bytes.fromhex("fffefdfcfbfaf9f8f7f6f5f4"), "c": bytes(12)}
LENGTHS = [1, 15, 16, 17, 65535, 65536, 65537, 131072, 3 * 65536 + 5, (1 << 20) + 5]
EXTRA = [(131072 + 100, "b", 5), (70000, "c", 0), (3 * 65536 + 5, "a", 7)]  # (length, key, seq0)


def main():
    sealed = {
        "client_key": "MzJieXRlc2xvbmdzZWNyZXRrZXltdXN0cHJvdmlkZWQ=",
        "iv": "coVfGS3I/CTrqexX5vUN+PQPoP9aUFiPYYrSzqTWfBA=",
        "bucket": "bucket", "object": "object",
        "sealed_key": "IAAfAMBdYor5tf/UlVaQvwYlw5yKbPBeQqfygqsfHqhu1wHD9KDAP4bw38AhL12prFTS23JbbR9Re5Qv26ZnlQ==",
        "object_key": "d4bef6fb18079e63828e8ab5953d9ae6d765d410d70e098d5c3d309731668f4e",
    }
    sk = d.ssec_sealing_key(base64.b64decode(sealed["client_key"]), base64.b64decode(sealed["iv"]), "bucket", "object")
    assert d.open_stream(sk, base64.b64decode(sealed["sealed_key"])).hex() == sealed["object_key"]
    sealed["sealing_key"] = sk.hex()
    part_keys = [{"part": 0, "key": "aa7855e13839dd767cd5da7c1ff5036540c9264b7a803029315e55375287b4af"},
                 {"part": 1, "key": "a3e7181c6eed030fd52f79537c56c4d07da92e56d374ff1dd2043350785b37d8"},
                 {"part": 10000, "key": "f86e65c396ed52d204ee44bd1a0bbd86eb8b01b7354e67a3b3ae0e34dd5bd115"}]
    for pk in part_keys:
        assert d.derive_part_key(bytes(32), pk["part"]).hex() == pk["key"]
    streams = []
    for n, kid, seq0 in [(n, "a", 0) for n in LENGTHS] + EXTRA:
        pt = d.plaintext(n, seed=len(streams)).tobytes()
        st = d.seal(KEYS[kid], NONCES[kid], pt, seq0)
        assert len(st) == d.encrypted_size(n) and d.open_stream(KEYS[kid], st, seq0) == pt
        streams.append({"length": n, "seed": len(streams), "key": KEYS[kid].hex(), "nonce": NONCES[kid].hex(), "seq0": seq0,
                        "sha256": hashlib.sha256(st).hexdigest(), **d.excerpts(st)})
    with open(os.path.join(HERE, "dare_streams.json"), "w") as f:
        f.write('{"sealed_key": ' + json.dumps(sealed) + ',\n "part_keys": ' + json.dumps(part_keys) + ',\n "streams": [\n  ')
        f.write(",\n  ".join(json.dumps(x) for x in streams) + "]}\n")  # one line per stream


if __name__ == "__main__":
    main()
