"""Signature V4 streaming bodies on the device (mec_chunk_signatures_device, mec_encode_chunked) against the pure-Python reference
of tests/sigv4_ref.py: verdicts of single rows at every length class, part files byte-equal to mec_encode of the decoded bytes, and
the exact error of every kind of damage, in the serial reader's order."""
import numpy as np
import pytest
import torch

import minio_b200 as mb
import sigv4_ref as ref

pytestmark = pytest.mark.gpu

KEY = ref.signing_key("wJalrXUtnFEMI/K7MDENG/bPxRfiCYEXAMPLEKEY")
SEED = b"4f232c4386841ef735655705268965c44a0e4690baa4adea153f7db9fa80a0a9"
SCOPE = ref.scope_of()
TRAILER = b"x-amz-checksum-crc32c:sOO8/Q=="


def rnd(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def test_chunk_signatures_device_one_launch():
    """every payload length class at odd device offsets, mixed with trailer rows, good and bad claims: ONE launch"""
    lens = [0, 1, 55, 56, 63, 64, 65, 8191, 65536, 65537, 1 << 20] * 2
    host = rnd((1 << 21) + 4096, 1)
    buf = torch.from_numpy(host).cuda()
    rng = np.random.default_rng(2)
    offs, kinds, prevs, claims, want = [], [], [], [], []
    pos = 3
    for i, n in enumerate(lens):
        if pos + n > host.size:
            pos = 5
        kind = mb.capi.SIGV4_TRAILER if i % 5 == 4 else mb.capi.SIGV4_PAYLOAD
        msg = bytes(host[pos:pos + n])
        prev = bytes(b"0123456789abcdef"[x] for x in rng.integers(0, 16, 64))
        good = (ref.trailer_signature if kind == mb.capi.SIGV4_TRAILER else ref.chunk_signature)(KEY, ref.DATE, SCOPE, prev, msg)
        if i % 3 == 0:
            claim = good
        elif i % 3 == 1 and good.upper() != good:
            claim = good.upper()  # compareSignatureV4 compares strings
        else:
            claim = good[:63] + (b"0" if good[63:] != b"0" else b"1")
        offs.append(pos); kinds.append(kind); prevs.append(prev); claims.append(claim); want.append(claim == good)
        pos += n + 2 * (i % 7) + 1
    c = mb.Codec(12, 4)
    l0, r0 = c.launches, c.stat("sigv4_chunks")
    got = c.chunk_signatures_device(KEY, ref.DATE, SCOPE, buf.data_ptr(), offs, lens, prevs, claims, kinds)
    assert c.launches - l0 == 1 and c.stat("sigv4_chunks") - r0 == len(offs)
    assert [bool(v) for v in got] == want
    assert any(want) and not all(want)
    assert c.stat("sigv4_key_bytes") == 0
    c.close()


def staged_bytes(sizes, D, step, tlen):
    """the payload bytes chunked_stage copies for pipeline chunks of `step` object bytes (straddling aws-chunks in each)"""
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    total = 0
    for off in range(0, D, step):
        end = min(D, off + step)
        last = end == D
        sel = {j for j, (s, n) in enumerate(zip(starts, sizes)) if (off <= s < end) or (last and s >= end) or (s < end and s + n > off)}
        total += sum(sizes[j] for j in sel) + (tlen if last else 0)
    return total


MIXED = [65536, 1, 8192, 16 << 20, 1000003, 3 * 65536, 777]


@pytest.mark.parametrize("k,m,bs", [(12, 4, 1 << 20), (4, 2, 1 << 20), (16, 4, 1 << 20), (12, 4, 10 << 20)])
def test_encode_chunked_matches_encode(k, m, bs):
    data = rnd(sum(MIXED), 10 + k + m)
    D = data.size
    body = ref.build(data, MIXED, KEY, SEED)
    c = mb.Codec(k, m, bs)
    c.set_option("checksums", 7)
    want = c.encode(data)
    want_ck = c.checksums(data, 7)
    for cb in (0, 1, 2):
        c.set_option("chunk_blocks", cb)
        h0, r0 = c.stat("bytes_h2d"), c.stat("sigv4_chunks")
        got = c.encode_chunked(body.data, D, KEY, SEED, ref.DATE, SCOPE)
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), (k, m, bs, cb)
        assert c.last_checksums() == (want_ck, D)
        assert c.stat("sigv4_chunks") - r0 == len(MIXED) + 1
        if cb:
            assert c.stat("bytes_h2d") - h0 == staged_bytes(MIXED + [0], D, cb * bs, 0)
        assert c.stat("sigv4_key_bytes") == 0
    c.close()


def test_encode_chunked_host_buffers_and_size_quirks():
    """pinned and pageable bodies at misaligned host offsets, upper-case hex sizes with leading zeros, a ';'-only final size"""
    sizes = [65536] * 5 + [12345, 1, 65536 + 7]
    data = rnd(sum(sizes), 20)
    c = mb.Codec(12, 4)
    want = c.encode(data)
    text = lambda i, n: "" if n == 0 else f"{n:08X}"
    body = ref.build(data, sizes, KEY, SEED, size_text=text).data
    assert ref.read(body, data.size, KEY, SEED)[0] == ref.OK
    for pinned in (False, True):
        for lead in (0, 3, 13):
            arr = mb.pinned_array(len(body) + lead) if pinned else np.zeros(len(body) + lead, dtype=np.uint8)
            arr[lead:lead + len(body)] = np.frombuffer(bytes(body), dtype=np.uint8)
            got = c.encode_chunked(arr[lead:lead + len(body)], data.size, KEY, SEED, ref.DATE, SCOPE)
            assert all(np.array_equal(a, b) for a, b in zip(got, want)), (pinned, lead)
    c.close()


def test_encode_chunked_empty_and_trailer():
    c = mb.Codec(12, 4)
    c.set_option("checksums", 7)
    for tr in (None, TRAILER, b"", b"x-amz-checksum-crc32:AAAAAA==\n"):
        body = ref.build(b"", [], KEY, SEED, trailer=tr)
        code, _, val = ref.read(body.data, 0, KEY, SEED, trailer=tr is not None)
        assert code == ref.OK
        if tr is None:
            files = c.encode_chunked(body.data, 0, KEY, SEED, ref.DATE, SCOPE)
        else:
            files, got = c.encode_chunked(body.data, 0, KEY, SEED, ref.DATE, SCOPE, trailer=True)
            assert got == val
        assert all(f.size == 0 for f in files) and c.last_checksums() == ((0, 0, 0), 0)
    # a trailer behind a multi-chunk body at 1-block chunks: the trailer row rides the last pipeline chunk
    data = rnd(3 * (1 << 20) + 5, 30)
    sizes = [1 << 20, 1 << 20, 1 << 20, 5]
    body = ref.build(data, sizes, KEY, SEED, trailer=TRAILER)
    want = c.encode(data)
    c.set_option("chunk_blocks", 1)
    files, got = c.encode_chunked(body.data, data.size, KEY, SEED, ref.DATE, SCOPE, trailer=True)
    assert got == TRAILER + b"\n" and all(np.array_equal(a, b) for a, b in zip(files, want))
    files, got = c.encode_chunked(body.data, data.size, KEY, SEED, ref.DATE, SCOPE, trailer=True, trailer_cap=5)
    assert got == TRAILER[:5]
    assert c.stat("sigv4_key_bytes") == 0
    c.close()


SIZES = [1000, 70000, 5000, 64]


def _base(trailer=None, sizes=SIZES, seed=40):
    data = rnd(sum(sizes), seed)
    return data, ref.build(data, sizes, KEY, SEED, trailer=trailer)


def _flip(b, pos, to=None):
    d = bytearray(b)
    d[pos] = (d[pos] ^ 1) if to is None else to
    return bytes(d)


def _splice(b, s, e, new):
    return bytes(b[:s]) + new + bytes(b[e:])


def tamper_cases():
    data, b = _base()
    D = data.size
    ch = b.chunks
    cases = []
    cases.append(("payload-byte", _flip(b.data, ch[1]["payload"][0] + 4444), D, ref.SIGNATURE_MISMATCH))
    cases.append(("claimed-sig", _flip(b.data, ch[2]["sig"][0] + 10), D, ref.SIGNATURE_MISMATCH))
    s, e = ch[0]["sig"]
    cases.append(("uppercase-sig", _splice(b.data, s, e, bytes(b.data[s:e]).upper()), D, ref.SIGNATURE_MISMATCH))
    s1, e1 = ch[1]["size"][0], ch[2]["size"][0]
    s2, e2 = ch[2]["size"][0], ch[3]["size"][0]
    swapped = bytes(b.data[:s1]) + bytes(b.data[s2:e2]) + bytes(b.data[s1:e1]) + bytes(b.data[e2:])
    cases.append(("swapped-chunks", swapped, D, ref.SIGNATURE_MISMATCH))
    s, e = ch[0]["crlf2"]
    cases.append(("missing-crlf", _splice(b.data, s, e, b""), D, ref.MALFORMED_ENCODING))
    s, e = ch[2]["size"]
    cases.append(("non-hex-size", _splice(b.data, s, e, b"13x8"), D, ref.MALFORMED_ENCODING))
    s, e = ch[1]["size"]
    cases.append(("size-16MiB+1", _splice(b.data, s, e, b"1000001"), D, ref.CHUNK_TOO_BIG))
    cases.append(("above-D", bytes(b.data), D - 1, ref.OVERREAD))
    cases.append(("far-above-D", bytes(b.data), 1000, ref.OVERREAD))
    cases.append(("above-zero-D", bytes(b.data), 0, ref.OVERREAD))
    cases.append(("below-D", bytes(b.data), D + 1, ref.INCOMPLETE_BODY))
    # ordering: a bad signature in chunk 1 beats a malformed header in chunk 3, and the other way round
    s, e = ch[3]["size"]
    bad_sig = _flip(b.data, ch[1]["payload"][0])
    cases.append(("sig1-before-header3", _splice(bad_sig, s, e, b"z"), D, ref.SIGNATURE_MISMATCH))
    bad_sig3 = _flip(b.data, ch[3]["payload"][0])
    s, e = ch[1]["size"]
    cases.append(("header1-before-sig3", _splice(bad_sig3, s, e, b"q"), D, ref.MALFORMED_ENCODING))
    # truncations at every structural position of every chunk
    for i, f in enumerate(ch):
        for name in ("size", "sig", "crlf1", "payload", "crlf2"):
            if name not in f:
                continue
            s, e = f[name]
            for cut in sorted({s, (s + e) // 2, e - 1} - ({e} if e == s else set())):
                if 0 <= cut < len(b.data):
                    cases.append((f"cut-{i}-{name}-{cut - s}", b.cut(cut), D, None))
    return cases


@pytest.fixture(scope="module")
def codec():
    c = mb.Codec(4, 2, 1 << 16)
    yield c
    c.close()


@pytest.mark.parametrize("case", tamper_cases(), ids=lambda x: x[0])
def test_encode_chunked_tampered(codec, case):
    name, body, D, code = case
    want = ref.read(body, D, KEY, SEED)[0]
    if code is not None:
        assert want == code, (name, want)
    assert want != ref.OK
    with pytest.raises(mb.MecError) as ei:
        codec.encode_chunked(body, D, KEY, SEED, ref.DATE, SCOPE)
    assert ei.value.code == want, name
    assert codec.stat("sigv4_key_bytes") == 0


def test_encode_chunked_wrong_credentials(codec):
    data, b = _base()
    for args in ((ref.signing_key("other"), SEED, ref.DATE, SCOPE), (KEY, SEED[:-1] + b"0", ref.DATE, SCOPE),
                 (KEY, SEED, "20130524T000001Z", SCOPE), (KEY, SEED, ref.DATE, ref.scope_of(region="eu-west-1"))):
        assert ref.read(b.data, data.size, args[0], args[1], args[2], args[3])[0] == ref.SIGNATURE_MISMATCH
        with pytest.raises(mb.MecError) as ei:
            codec.encode_chunked(b.data, data.size, *args)
        assert ei.value.code == ref.SIGNATURE_MISMATCH


def test_encode_chunked_stops_at_the_first_failure(codec):
    """a malformed header in chunk 1: only chunk 0's row is verified, chunk 3's bytes are never hashed"""
    data, b = _base()
    s, e = b.chunks[1]["size"]
    r0, l0 = codec.stat("sigv4_chunks"), codec.launches
    with pytest.raises(mb.MecError) as ei:
        codec.encode_chunked(_splice(b.data, s, e, b"q"), data.size, KEY, SEED, ref.DATE, SCOPE)
    assert ei.value.code == ref.MALFORMED_ENCODING and codec.stat("sigv4_chunks") - r0 == 1


def trailer_cases():
    data, b = _base(TRAILER)
    D = data.size
    t = b.trailer
    cases = [("trailer-ok", bytes(b.data), ref.OK)]
    cases.append(("trailer-sig", _flip(b.data, t["sig"][0] + 5), ref.SIGNATURE_MISMATCH))
    cases.append(("trailer-value", _flip(b.data, t["value"][0] + 3), ref.SIGNATURE_MISMATCH))
    s, e = t["sig"]
    cases.append(("trailer-sig-upper", _splice(b.data, s, e, bytes(b.data[s:e]).upper()), ref.SIGNATURE_MISMATCH))
    cases.append(("trailer-sig-spaces", _splice(b.data, s, e, b" \t" + bytes(b.data[s:e]) + b"\xc2\xa0 "), ref.OK))
    cases.append(("trailer-sig-short", _splice(b.data, s, e, bytes(b.data[s:e - 1])), ref.SIGNATURE_MISMATCH))
    ps = b.data.index(b"x-amz-trailer-signature:")
    cases.append(("trailer-prefix", _flip(b.data, ps + 3), ref.MALFORMED_ENCODING))
    s, e = t["end"]
    cases.append(("trailer-end", _splice(b.data, s, e, b"\r\n\r\r"), ref.MALFORMED_ENCODING))
    cases.append(("trailer-end-lf", _splice(b.data, s, e, b"\r\r\r\n"), ref.MALFORMED_ENCODING))
    vs, ve = t["value"]
    cases.append(("trailer-value-cr", _splice(b.data, ve, ve + 2, b"\rx"), ref.MALFORMED_ENCODING))
    for cut in (vs, (vs + ve) // 2, ve, ve + 1, s - 10, s, s + 1, s + 2, s + 3):
        cases.append((f"trailer-cut-{cut - vs}", b.cut(cut), None))
    cases.append(("trailer-bad-chunk-first", _flip(_flip(b.data, t["sig"][0]), b.chunks[2]["payload"][0]), ref.SIGNATURE_MISMATCH))
    return [(n, body, D, code) for n, body, code in cases]


@pytest.mark.parametrize("case", trailer_cases(), ids=lambda x: x[0])
def test_encode_chunked_trailer(codec, case):
    name, body, D, code = case
    want, out, val = ref.read(body, D, KEY, SEED, trailer=True)
    if code is not None:
        assert want == code, (name, want)
    if want == ref.OK:
        files, got = codec.encode_chunked(body, D, KEY, SEED, ref.DATE, SCOPE, trailer=True)
        assert got == val == TRAILER + b"\n"
        ref_files = codec.encode(np.frombuffer(out, dtype=np.uint8))
        assert all(np.array_equal(a, b) for a, b in zip(files, ref_files))
    else:
        with pytest.raises(mb.MecError) as ei:
            codec.encode_chunked(body, D, KEY, SEED, ref.DATE, SCOPE, trailer=True)
        assert ei.value.code == want, name
