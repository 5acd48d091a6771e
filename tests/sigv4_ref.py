"""Signature V4 streaming payloads in pure Python (hashlib + hmac only), as MinIO's cmd/streaming-signature-v4.go and
getSigningKey (cmd/signature-v4.go) define them: signing keys, signed aws-chunked bodies whose every structural field can be
found (and tampered with), and a serial reader that returns the verdict s3ChunkedReader + HardLimitReader + Erasure.Encode
reach for a body (the MEC_ERR_* code, the decoded bytes and the signed trailer value)."""
import hashlib
import hmac

EMPTY_SHA256 = hashlib.sha256(b"").hexdigest()
MAX_CHUNK = 16 << 20
OK, SIGNATURE_MISMATCH, MALFORMED_ENCODING, CHUNK_TOO_BIG, INCOMPLETE_BODY, OVERREAD = 0, -14, -15, -16, -17, -18
DATE = "20130524T000000Z"
REGION = "us-east-1"


def _hmac(k, m):
    return hmac.new(k, m, hashlib.sha256).digest()


def signing_key(secret, date=DATE, region=REGION):
    """getSigningKey: HMAC chain over yyyymmdd, region, "s3", "aws4_request" from "AWS4" + secret"""
    k = _hmac(("AWS4" + secret).encode(), date[:8].encode())
    for part in (region, "s3", "aws4_request"):
        k = _hmac(k, part.encode())
    return k


def scope_of(date=DATE, region=REGION):
    return f"{date[:8]}/{region}/s3/aws4_request"


def chunk_signature(key, date, scope, prev, payload):
    """getChunkSignature: 64 lowercase hex bytes"""
    sts = b"AWS4-HMAC-SHA256-PAYLOAD\n" + date.encode() + b"\n" + scope.encode() + b"\n" + prev + b"\n" + EMPTY_SHA256.encode() + \
        b"\n" + hashlib.sha256(payload).hexdigest().encode()
    return hmac.new(key, sts, hashlib.sha256).hexdigest().encode()


def trailer_signature(key, date, scope, prev, value):
    """getTrailerChunkSignature over the trailer value as readTrailers hashes it"""
    sts = b"AWS4-HMAC-SHA256-TRAILER\n" + date.encode() + b"\n" + scope.encode() + b"\n" + prev + b"\n" + \
        hashlib.sha256(value).hexdigest().encode()
    return hmac.new(key, sts, hashlib.sha256).hexdigest().encode()


def signed_trailer_value(value):
    """what readTrailers hashes: the value line with a '\\n' appended when it has none (an empty value stays empty)"""
    return value if not value or value.endswith(b"\n") else value + b"\n"


class Body:
    """A signed aws-chunked body.  chunks[i] holds the byte ranges of chunk i's fields in `data` (the final zero-size chunk
    included): "size" (hex digits), "sig" (the 64 claimed bytes), "crlf1" (behind the signature), "payload", "crlf2" (behind the
    payload; absent for the final chunk) and the chunk's "sigval".  trailer: "value", "sig" (the 64 claimed bytes), "end"
    (the "\\r\\n\\r\\n" behind the signature line)."""

    def __init__(self):
        self.data = bytearray()
        self.chunks = []
        self.trailer = None

    def _put(self, b):
        s = len(self.data)
        self.data += b
        return (s, len(self.data))

    def cut(self, pos):
        return bytes(self.data[:pos])


def build(payload, sizes, key, seed, date=DATE, scope=None, trailer=None, size_text=None):
    """payload split into chunks of `sizes` (their sum is len(payload)), then the final zero-size chunk; signatures chained from
    `seed`.  size_text(i, size) -> the hex digits of chunk i (default lowercase, the final chunk "0").  trailer: the raw trailer
    value line (without its "\\r\\n"), signed after the final chunk."""
    scope = scope or scope_of(date)
    assert sum(sizes) == len(payload)
    b = Body()
    prev, pos = seed, 0
    for i, n in enumerate(list(sizes) + [0]):
        data = bytes(payload[pos:pos + n])
        pos += n
        sig = chunk_signature(key, date, scope, prev, data)
        txt = size_text(i, n) if size_text else f"{n:x}"
        f = {"size": b._put(txt.encode())}
        b._put(b";chunk-signature=")
        f["sig"] = b._put(sig)
        f["crlf1"] = b._put(b"\r\n")
        f["payload"] = b._put(data)
        if n:
            f["crlf2"] = b._put(b"\r\n")
        f["sigval"] = sig
        b.chunks.append(f)
        prev = sig
    if trailer is not None:
        tsig = trailer_signature(key, date, scope, prev, signed_trailer_value(trailer))
        t = {"value": b._put(trailer)}
        b._put(b"\r\nx-amz-trailer-signature:")
        t["sig"] = b._put(tsig)
        t["end"] = b._put(b"\r\n\r\n")
        b.trailer = t
    return b


# bytes.TrimSpace: ASCII white space and Unicode White_Space
_GO_SPACE = "\t\n\v\f\r \x85\xa0\u1680" + "".join(chr(c) for c in range(0x2000, 0x200b)) + "\u2028\u2029\u202f\u205f\u3000"


def go_trim_space(b):
    return b.decode("utf-8", "surrogateescape").strip(_GO_SPACE).encode("utf-8", "surrogateescape")


def read(body, decoded_len, key, seed, date=DATE, scope=None, trailer=False):
    """The serial reader: returns (code, decoded bytes, signed trailer value or None) for `body`, with s3ChunkedReader's checks
    in its order, HardLimitReader's over-read check on each yielded chunk, and IncompleteBody for a short total."""
    scope = scope or scope_of(date)
    body = bytes(body)
    out = bytearray()
    pos, prev, n = 0, seed, len(body)
    while True:
        size = 0
        while True:
            if pos >= n:
                return INCOMPLETE_BODY, bytes(out), None
            c = body[pos]
            pos += 1
            if c == ord(";"):
                break
            ch = chr(c)
            if ch in "0123456789abcdefABCDEF":
                size = size << 4 | int(ch, 16)
            else:
                return MALFORMED_ENCODING, bytes(out), None
            if size > MAX_CHUNK:
                return CHUNK_TOO_BIG, bytes(out), None
        if n - pos < 80:
            return INCOMPLETE_BODY, bytes(out), None
        if body[pos:pos + 16] != b"chunk-signature=":
            return MALFORMED_ENCODING, bytes(out), None
        claim = body[pos + 16:pos + 80]
        pos += 80
        for want in b"\r\n":
            if pos >= n:
                return INCOMPLETE_BODY, bytes(out), None
            if body[pos] != want:
                return MALFORMED_ENCODING, bytes(out), None
            pos += 1
        if n - pos < size:
            return INCOMPLETE_BODY, bytes(out), None
        data = body[pos:pos + size]
        pos += size
        sig = chunk_signature(key, date, scope, prev, data)
        if not hmac.compare_digest(claim, sig):
            return SIGNATURE_MISMATCH, bytes(out), None
        prev = sig
        if size == 0:
            break
        if pos >= n or body[pos] != ord("\r"):
            return MALFORMED_ENCODING, bytes(out), None
        pos += 1
        if pos >= n:
            return INCOMPLETE_BODY, bytes(out), None
        if body[pos] != ord("\n"):
            return MALFORMED_ENCODING, bytes(out), None
        pos += 1
        out += data
        if len(out) > decoded_len:
            return OVERREAD, bytes(out), None
    value = None
    if trailer:
        e = body.find(b"\r", pos)
        if e < 0:
            return INCOMPLETE_BODY, bytes(out), None
        raw = body[pos:e]
        pos = e + 1
        if pos >= n:
            return INCOMPLETE_BODY, bytes(out), None
        if body[pos] != ord("\n"):
            return MALFORMED_ENCODING, bytes(out), None
        pos += 1
        e = body.find(b"\r", pos)
        if e < 0:
            return INCOMPLETE_BODY, bytes(out), None
        line = body[pos:e]
        pos = e + 1
        if pos >= n:
            return INCOMPLETE_BODY, bytes(out), None
        if body[pos:pos + 3] != b"\n\r\n":
            return MALFORMED_ENCODING, bytes(out), None
        if not line.startswith(b"x-amz-trailer-signature:"):
            return MALFORMED_ENCODING, bytes(out), None
        claim = go_trim_space(line[len(b"x-amz-trailer-signature:"):])
        value = signed_trailer_value(raw)
        if not hmac.compare_digest(claim, trailer_signature(key, date, scope, prev, value)):
            return SIGNATURE_MISMATCH, bytes(out), None
    if len(out) < decoded_len:
        return INCOMPLETE_BODY, bytes(out), None
    return OK, bytes(out), value
