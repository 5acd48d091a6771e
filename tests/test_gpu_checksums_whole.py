"""The object-checksum kernels (crc.cuh) and the whole-file hash and gather kernels (whole_hash.cuh) against references that share
no code with the library, at the launch shapes where they loop, fold, fall back to byte loads or spill into a second CTA.

References: zlib for CRC32, the oracle's bit-at-a-time CRC32C / CRC64NVME, hashlib for SHA-256 and (unkeyed) BLAKE2b-512 and the
oracle's HighwayHash-256, which the goldens pin.  The CRCs of many prefixes of one long stream come from the oracle CRCs of the
pieces between consecutive prefix ends, merged by the CRC combine written out below in plain Python (GF(2) polynomial product and
x^(8n) mod P, as zlib does it), which is itself checked against zlib and the oracle.

Where the kernels change behaviour:
  crc_regions_kernel   grid min(regions, 8 x SMs) of 256 KiB regions: a CTA takes a second region only above 8 x SMs x 256 KiB
  crc_fold_kernel      each of 256 threads folds ceil(regions / 256) partials serially: more than one above 64 MiB
  mec_checksums, encode_pipeline   six slots: a slot is retired inside the loop only from the seventh chunk on
  whole_hash_kernel    64 threads per CTA: 32 HighwayHash streams (two threads each) or 64 SHA-256 / BLAKE2b streams per CTA
  gather_shard_files_kernel   at most 4096 x 256 threads: loops only over shard files larger than 1 MiB
"""
import concurrent.futures
import hashlib
import os
import zlib

import numpy as np
import pytest

MiB = 1 << 20
REGION = 256 * 1024                   # kCrcRegion: bytes one CTA pass of crc_regions_kernel covers
LONG = 7 * 64 * MiB + 4321            # seven 64 MiB host chunks and a bit: more regions than 8 x SMs on an H100
CRC_TYPES = ((0xEDB88320, 32), (0x82F63B78, 32), (0x9A6C9329AC4BC9B5, 64))   # reflected polynomials: CRC32, CRC32C, CRC64NVME
SHA256, HIGHWAYHASH256, BLAKE2B512 = 1, 2, 4
ALGOS = {"SHA256": SHA256, "HighwayHash256": HIGHWAYHASH256, "BLAKE2b512": BLAKE2B512}
FILL = 0xA5                           # digest buffers are pre-filled with this byte


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


def rand(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def masked(crcs, which):
    return tuple(v if which & (1 << t) else 0 for t, v in enumerate(crcs))


# ---- CRC combine in plain Python (zlib's multmodp / x2nmodp, for any reflected CRC) --------------------------------------------
def _mulmod(a, b, poly, bits):
    """a(x) * b(x) mod P; reflected: bit bits-1 is x^0."""
    m, p = 1 << (bits - 1), 0
    while m:
        if a & m:
            p ^= b
        m >>= 1
        b = (b >> 1) ^ poly if b & 1 else b >> 1
    return p


def _xpow8n(n, poly, bits):
    """x^(8n) mod P by square-and-multiply."""
    r, sq = 1 << (bits - 1), 1 << (bits - 9)      # x^0, x^8
    while n:
        if n & 1:
            r = _mulmod(r, sq, poly, bits)
        sq = _mulmod(sq, sq, poly, bits)
        n >>= 1
    return r


def crc_combine(t, c1, c2, len2):
    """CRC of type t over A || B from crc(A), crc(B) and |B|."""
    poly, bits = CRC_TYPES[t]
    return _mulmod(_xpow8n(len2, poly, bits), c1, poly, bits) ^ c2 if len2 else c1


def test_python_crc_combine_matches_zlib_and_oracle(oracle):
    rng = np.random.default_rng(17)
    for la, lb in [(0, 0), (0, 5), (5, 0), (1, 1), (3, 1024), (1024, 1023), (4097, 262144), (262145, 17), (100003, 65537)]:
        a = rng.integers(0, 256, la, dtype=np.uint8).tobytes()
        b = rng.integers(0, 256, lb, dtype=np.uint8).tobytes()
        assert crc_combine(0, zlib.crc32(a), zlib.crc32(b), lb) == zlib.crc32(a + b), (la, lb)
        ca, cb, cab = oracle.crcs(a), oracle.crcs(b), oracle.crcs(a + b)
        for t in range(3):
            assert crc_combine(t, ca[t], cb[t], lb) == cab[t], (t, la, lb)


def prefix_crcs(oracle, data, cuts):
    """{p: (CRC32, CRC32C, CRC64NVME) of data[:p]} for every p in cuts: each piece between consecutive cuts is checksummed once,
    in a thread pool (zlib and ctypes release the GIL), and the pieces are merged in order with crc_combine."""
    ends = sorted(set(cuts) | {0})
    pieces = list(zip(ends[:-1], ends[1:]))
    L, base, mv = oracle.lib(), data.ctypes.data, memoryview(data)
    one = (lambda a, b: zlib.crc32(mv[a:b]), lambda a, b: L.orc_crc32c(base + a, b - a), lambda a, b: L.orc_crc64nvme(base + a, b - a))
    with concurrent.futures.ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as pool:
        jobs = sorted(((a, b, t) for a, b in pieces for t in range(3)), key=lambda j: j[0] - j[1])   # longest first
        futs = {(a, t): pool.submit(one[t], a, b) for a, b, t in jobs}
        seg = {(a, t): f.result() for (a, t), f in futs.items()}
    acc, out = [0, 0, 0], {0: (0, 0, 0)}
    for a, b in pieces:
        acc = [crc_combine(t, acc[t], seg[(a, t)], b - a) for t in range(3)]
        out[b] = tuple(acc)
    return out


# prefix lengths of the long stream, by name (the last ones depend on the SM count)
PREFIXES = {"0": lambda g: 0, "1": lambda g: 1, "15": lambda g: 15, "16": lambda g: 16, "17": lambda g: 17,
            "1023": lambda g: 1023, "1024": lambda g: 1024, "1025": lambda g: 1025,
            "256K-1": lambda g: REGION - 1, "256K": lambda g: REGION, "256K+1": lambda g: REGION + 1,
            "64M-1": lambda g: 64 * MiB - 1, "64M": lambda g: 64 * MiB, "64M+1": lambda g: 64 * MiB + 1,
            # 515 regions: folds in runs of 3, the short last region shares its run with two full ones
            "514x256K+1": lambda g: 514 * REGION + 1,
            # g = 8 x SMs x 256 KiB: above it a CTA of the region kernel takes a second region
            "grid-1": lambda g: g - 1, "grid": lambda g: g, "grid+1": lambda g: g + 1}


@pytest.fixture(scope="module")
def long_stream(mb, oracle):
    """LONG random bytes on the host and on the device (offset 0 of a 16-byte aligned buffer), with the reference CRCs of every
    prefix in PREFIXES and of the whole stream."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid_bytes = 8 * sms * REGION
    assert LONG > grid_bytes, f"{sms} SMs: the long stream no longer reaches a second pass of the CRC region kernel"
    data = rand(LONG, 2024)
    ref = prefix_crcs(oracle, data, [f(grid_bytes) for f in PREFIXES.values()] + [LONG])
    dev = torch.from_numpy(data).to("cuda")
    assert dev.data_ptr() % 16 == 0
    shifted = torch.empty(LONG + 64, dtype=torch.uint8, device="cuda")
    assert shifted.data_ptr() % 16 == 0
    ls = dict(data=data, dev=dev, shifted=shifted, ref=ref, grid_bytes=grid_bytes)
    yield ls
    ls.clear()
    del dev, shifted
    torch.cuda.empty_cache()


def at_offset(ls, off, n):
    """Device address of the first n bytes of the long stream copied to a buffer at byte offset `off` from 16-byte alignment."""
    if off == 0:
        return ls["dev"].data_ptr()
    ls["shifted"][off:off + n].copy_(ls["dev"][:n])
    return ls["shifted"].data_ptr() + off


@pytest.mark.gpu
@pytest.mark.parametrize("off", range(16))
def test_checksums_device_whole_long_stream(mb, long_stream, off):
    """All LONG bytes, from every alignment: the grid-stride loop of the region kernel, runs of 8 in the fold, and (off != 0)
    every thread's chunk read byte by byte."""
    c = mb.Codec(12, 4)
    assert c.checksums_device(at_offset(long_stream, off, LONG), LONG, 7) == long_stream["ref"][LONG]
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("off", [0, 1, 8, 15])
@pytest.mark.parametrize("prefix", list(PREFIXES))
def test_checksums_device_prefixes(mb, long_stream, prefix, off):
    n = PREFIXES[prefix](long_stream["grid_bytes"])
    c = mb.Codec(12, 4)
    assert c.checksums_device(at_offset(long_stream, off, n), n, 7) == long_stream["ref"][n], (prefix, n, off)
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which", range(8))
def test_checksums_device_masks(mb, long_stream, which):
    """Every subset of the three types over the whole stream and over the 515-region prefix; unrequested types are 0."""
    c = mb.Codec(12, 4)
    for n in (LONG, 514 * REGION + 1):
        assert c.checksums_device(long_stream["dev"].data_ptr(), n, which) == masked(long_stream["ref"][n], which), (n, which)
    c.close()


@pytest.mark.gpu
def test_checksums_device_follows_the_callers_stream(mb, long_stream):
    """The bytes are written by a torch copy on a side stream and checksummed on that stream with no synchronisation between."""
    import torch
    c = mb.Codec(12, 4)
    buf = long_stream["shifted"]
    buf.zero_()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        buf[:LONG].copy_(long_stream["dev"])
        got = c.checksums_device(buf.data_ptr(), LONG, 7, side.cuda_stream)
    assert got == long_stream["ref"][LONG]
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which", range(8))
def test_checksums_host_long_stream(mb, long_stream, which):
    """mec_checksums stages 64 MiB chunks through six slots: the seventh and eighth chunks reuse a slot retired inside the loop."""
    c = mb.Codec(12, 4)
    assert c.checksums(long_stream["data"], which) == masked(long_stream["ref"][LONG], which)
    c.close()


@pytest.mark.gpu
def test_checksums_host_misaligned_source(mb, long_stream):
    c = mb.Codec(12, 4)
    buf = np.empty(LONG + 1, dtype=np.uint8)
    buf[1:] = long_stream["data"]
    src = buf[1:]
    assert src.ctypes.data % 16 != 0
    assert c.checksums(src, 7) == long_stream["ref"][LONG]
    c.close()


# ---- checksums carried by the host-buffer encode ---------------------------------------------------------------------------------
ENC_GEOMS = {
    "rs12_4-1M-cb2": (12, 4, MiB, 2, 15 * MiB + 4321),     # 8 chunks of 2 blocks, the last block short
    "rs4_2-4K-cb1": (4, 2, 4096, 1, 50 * 4096 + 1234),     # 51 chunks of 1 block
}
_ENC_CACHE = {}


def enc_reference(oracle, geom):
    """(data, CRCs, oracle part files, per-block digests [nb][n][32], per-block shard lengths) of one geometry."""
    if geom not in _ENC_CACHE:
        k, m, bs, _, size = ENC_GEOMS[geom]
        data = rand(size, 77 + k)
        files, _ = oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, data)
        S, nb = -(-bs // k), -(-size // bs)
        tail = size % bs
        lens = [S] * nb
        if tail:
            lens[-1] = -(-tail // k)
        dig = np.stack([np.stack([f[b * (32 + S):b * (32 + S) + 32] for f in files]) for b in range(nb)])
        _ENC_CACHE[geom] = (data, oracle.crcs(data), files, dig, lens)
    return _ENC_CACHE[geom]


def enc_codec(mb, geom, which):
    k, m, bs, cb, _ = ENC_GEOMS[geom]
    c = mb.Codec(k, m, bs)
    c.set_option("chunk_blocks", cb)
    c.set_option("checksums", which)
    return c


def run_encode(c, entry, data, k, m, want_files, want_dig, lens):
    """Encode through one host entry point and compare what it returns with the oracle's part files."""
    S = c.shard_size()
    if entry == "encode":
        files = c.encode(data)
        for i in range(k + m):
            assert np.array_equal(files[i], want_files[i]), (entry, i)
    elif entry == "encode_sg":
        files, dd = c.encode_sg(data)
        assert np.array_equal(dd, want_dig[:, :k]), entry
        for i in range(k, k + m):
            assert np.array_equal(files[i], want_files[i]), (entry, i)
    else:
        parity, dig = c.encode_blocks(data)
        assert np.array_equal(dig, want_dig), entry
        for b, sb in enumerate(lens):
            for j in range(m):
                f = want_files[k + j]
                assert np.array_equal(parity[b, j, :sb], f[b * (32 + S) + 32:b * (32 + S) + 32 + sb]), (entry, b, j)


@pytest.mark.gpu
@pytest.mark.parametrize("which", [1, 2, 4, 5, 6, 7])
@pytest.mark.parametrize("entry", ["encode", "encode_sg", "encode_blocks"])
@pytest.mark.parametrize("geom", list(ENC_GEOMS))
def test_encode_carries_checksums(mb, oracle, geom, entry, which):
    """Option "checksums": the CRCs of more than six chunks, merged on the host across reused slots, for every entry point and
    every mask; the encode itself still matches the oracle."""
    k, m, _, _, size = ENC_GEOMS[geom]
    data, crcs, files, dig, lens = enc_reference(oracle, geom)
    c = enc_codec(mb, geom, which)
    run_encode(c, entry, data, k, m, files, dig, lens)
    assert c.last_checksums() == (masked(crcs, which), size)
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["encode", "encode_sg", "encode_blocks"])
def test_empty_object_resets_carried_checksums(mb, oracle, entry):
    """An empty object after another one reports the checksums of the empty stream, not those of the previous object."""
    geom = "rs4_2-4K-cb1"
    k, m, _, _, size = ENC_GEOMS[geom]
    data, crcs, files, dig, lens = enc_reference(oracle, geom)
    c = enc_codec(mb, geom, 7)
    run_encode(c, entry, data, k, m, files, dig, lens)
    assert c.last_checksums() == (crcs, size)
    getattr(c, entry)(np.zeros(0, dtype=np.uint8))
    assert c.last_checksums() == ((0, 0, 0), 0)
    c.close()


# ---- whole-file hashes -----------------------------------------------------------------------------------------------------------
def ref_digest(oracle, algo, msg):
    if algo == SHA256:
        return hashlib.sha256(msg.tobytes()).digest()
    if algo == BLAKE2B512:
        return hashlib.blake2b(msg.tobytes(), digest_size=64).digest()
    return oracle.bitrot_hash(HIGHWAYHASH256, msg)


def digest_size(algo):
    return 64 if algo == BLAKE2B512 else 32


def round_up(x, a):
    return (x + a - 1) // a * a


# lengths at the padding edges: SHA-256 (55/56, 64-byte blocks), BLAKE2b (128-byte blocks), HighwayHash (32-byte packets, 16-byte
# halves of the remainder)
LENGTHS = [0, 1, 31, 32, 55, 56, 63, 64, 65, 111, 112, 119, 120, 127, 128, 129, 4097]
FEW_LENGTHS = [0, 56, 119, 129, 4097]
COUNTS = [1, 31, 32, 33, 63, 64, 65, 1000]


def whole_hash_device_case(oracle, c, algo, count, n, pitch, seed):
    """count messages of n bytes at `pitch` in a buffer of random bytes (so a read past n changes a digest), hashed on a side
    stream into a 0xA5-filled digest array with a 64-byte guard on each side."""
    import torch
    host = rand(count * pitch + 256, seed)                  # 128 readable bytes behind the last message, and then some
    d_msgs = torch.from_numpy(host).to("cuda")
    dig = torch.full((64 + count * 64 + 64,), FILL, dtype=torch.uint8, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    c.whole_hash_device(algo, d_msgs.data_ptr(), pitch, n, count, dig.data_ptr() + 64, side.cuda_stream)
    side.synchronize()
    out = dig.cpu().numpy()
    ds = digest_size(algo)
    assert (out[:64] == FILL).all() and (out[-64:] == FILL).all(), ("guard", algo, count, n, pitch)
    slots = out[64:-64].reshape(count, 64)
    assert (slots[:, ds:] == FILL).all(), ("digest slot tail", algo, count, n, pitch)
    for i in range(count):
        assert slots[i, :ds].tobytes() == ref_digest(oracle, algo, host[i * pitch:i * pitch + n]), (algo, count, n, pitch, i)


@pytest.mark.gpu
@pytest.mark.parametrize("count", COUNTS)
@pytest.mark.parametrize("algo", list(ALGOS))
def test_whole_hash_device(mb, oracle, algo, count):
    """mec_whole_hash_device at CTA-edge counts (32 HighwayHash or 64 SHA-256 / BLAKE2b streams per CTA), padding-edge lengths
    (all of them at 65 streams) and the pitches round_up(len, 16), that + 16, and 4144."""
    a = ALGOS[algo]
    c = mb.Codec(2, 2)
    for n in (LENGTHS if count == 65 else FEW_LENGTHS):
        for pitch in (round_up(n, 16), round_up(n, 16) + 16, 4144):
            whole_hash_device_case(oracle, c, a, count, n, pitch, seed=count * 7919 + n * 31 + pitch)
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("algo", list(ALGOS))
def test_whole_hash_device_many_streams(mb, oracle, algo):
    """BASELINE config 5 scale: 20 000 streams of 256 bytes at pitch == msg_len."""
    c = mb.Codec(8, 8)
    whole_hash_device_case(oracle, c, ALGOS[algo], 20000, 256, 256, seed=5)
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("count", [65, 1000])
@pytest.mark.parametrize("algo", list(ALGOS))
def test_whole_hash_host_many_streams(mb, oracle, algo, count):
    a = ALGOS[algo]
    c = mb.Codec(2, 2)
    for n in FEW_LENGTHS:
        msgs = rand(count * n, count + n)
        got = c.whole_hash(a, msgs, n, count)
        for i in range(count):
            assert got[i].tobytes() == ref_digest(oracle, a, msgs[i * n:(i + 1) * n]), (algo, count, n, i)
    c.close()


def test_whole_hash_device_rejects_unusable_pointers():
    """A message base that is not 16-byte aligned, a NULL message base with bytes to read, and a NULL or not 8-byte aligned
    digest array are refused before any device work (the addresses are never dereferenced)."""
    import minio_b200 as mb
    L = mb.lib()
    for algo in ALGOS.values():
        c = mb.Codec(12, 4, algo=algo)
        for d_msgs, d_digests in ((0x1001, 0x2000), (0x1008, 0x2000), (0x100F, 0x2000), (None, 0x2000), (0x1000, None),
                                  (0x1000, 0x2001), (0x1000, 0x2004)):
            rc = L.mec_whole_hash_device(c.h, algo, d_msgs, 87392, 87382, 16, d_digests, None)
            assert rc == -12, (algo, hex(d_msgs or 0), hex(d_digests or 0), rc)
        c.close()


# ---- encode_whole / gather / decode_whole / heal_whole ---------------------------------------------------------------------------
WHOLE_GEOMS = {
    "rs4_2-1M": (4, 2, MiB, 9 * MiB + 4321),          # shard files of 2.3 MB
    "rs12_4-1M": (12, 4, MiB, 40 * MiB + 777),        # 3.6 MB
    "rs3_0-64K": (3, 0, 64 * 1024, 4 * MiB + 5),      # 1.4 MB, no parity
    "rs20_12-1M": (20, 12, MiB, 3 * MiB + 777),       # 32 shard files
    "rs32_16-1M": (32, 16, MiB, 3 * MiB + 777),       # 48 shard files: two CTAs of HighwayHash streams
}


@pytest.mark.gpu
@pytest.mark.parametrize("algo", list(ALGOS))
@pytest.mark.parametrize("geom", list(WHOLE_GEOMS))
def test_encode_whole_decode_heal(mb, oracle, geom, algo):
    """Shard files over 1 MiB make the gather kernel loop; 32 and 48 shard files make multi-CTA hash launches on a production path.
    Files and sums against the oracle (and hashlib), a read across the 1 MiB mark of the shard files with m shards offline, and
    a heal of m stale shards."""
    k, m, bs, size = WHOLE_GEOMS[geom]
    a, n = ALGOS[algo], k + m
    data = rand(size, size % 1000)
    want_files, want_sums = oracle.erasure_encode(k, m, bs, a, data)
    c = mb.Codec(k, m, bs, algo=a)
    files, sums = c.encode_whole(data)
    for i in range(n):
        assert np.array_equal(files[i], want_files[i]), (geom, algo, "file", i)
        assert sums[i] == want_sums[i], (geom, algo, "sum", i)
        if a != HIGHWAYHASH256:
            assert sums[i] == ref_digest(oracle, a, files[i]), (geom, algo, "hashlib", i)
    S = c.shard_size()
    b1 = MiB // S                                    # the block holding byte 1 MiB of every shard file
    lo, hi = (max(0, b1 * bs - 777), min(size, (b1 + 2) * bs + 123)) if files[0].size > MiB else (1000, size - 2000)
    srcs = [None if i < m else files[i] for i in range(n)]
    out, hint = c.decode_whole(srcs, sums, lo, hi - lo, size)
    assert hint == 0 and np.array_equal(out, data[lo:hi]), (geom, algo, lo, hi)
    if m:
        stale = [i in range(0, n, max(1, n // m))[:m] for i in range(n)]
        outs, osums, rc, corrupt = c.heal_whole([None if stale[i] else files[i] for i in range(n)], sums, stale, size)
        assert rc == 0 and not corrupt.any()
        for i in range(n):
            if stale[i]:
                assert np.array_equal(outs[i], files[i]) and osums[i] == sums[i], (geom, algo, "heal", i)
    c.close()
