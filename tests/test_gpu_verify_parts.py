"""mec_bitrot_verify_parts (VerifyFile in one call: every part of an object on one drive, each with its own bitrot algorithm and sum)
against the CPU oracle's bitrotVerify, part by part.

Streaming parts are HighwayHash256S frames of the codec's shard size S built with the oracle's HighwayHash; whole-file parts are
random files with the oracle's SHA256 / HighwayHash256 / BLAKE2b512 digest as their sum.  Covered: RS(4,2) and RS(12,4) at 1 MiB
and RS(12,4) at 10 MiB; part lengths 0, 1, S-1, S, S+1 and several blocks with a short tail; streaming damage (a digest byte, the
first / middle / last byte of a full frame, the last byte of a short last frame, file lengths +-1 and +-32); whole-file damage (first
and last byte, a wrong sum, an empty file, a NULL file of length 0); unknown algorithms per part; the inline frames of
tests/golden/inline_frames.json; one call that mixes all four algorithms at every hash-block edge in ONE whole_hash_kernel launch,
equal to per-part mec_bitrot_verify_batch / mec_bitrot_verify_whole; and whole files of more than 256 MiB in total, which take more than
one staging group."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
MiB = 1 << 20
SHA256, HIGHWAYHASH256, HIGHWAYHASH256S, BLAKE2B512 = 1, 2, 3, 4
WHOLE = (SHA256, HIGHWAYHASH256, BLAKE2B512)
FILE_CORRUPT, INVALID = -7, -12
GEOMS = {"rs4_2_1m": (4, 2, MiB), "rs12_4_1m": (12, 4, MiB), "rs12_4_10m": (12, 4, 10 * MiB)}
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


def stream_file(oracle, data, S):
    """the HighwayHash256S part.N image of `data`: [32-byte digest][up to S bytes] per frame"""
    out = bytearray()
    for o in range(0, len(data), S):
        chunk = bytes(data[o:o + S])
        out += oracle.hh256(chunk) + chunk
    return np.frombuffer(bytes(out), dtype=np.uint8).copy()


def flip(a, i):
    b = a.copy()
    b[i] ^= 0x40
    return b


class Case:
    """one part of a verify call: (algo, file or None, part_len, sum or None)"""

    def __init__(self, algo, file, part_len, want=None):
        self.algo, self.file, self.part_len, self.want = algo, file, part_len, want

    def oracle(self, oracle, S):
        if self.algo not in (SHA256, HIGHWAYHASH256, HIGHWAYHASH256S, BLAKE2B512):
            return INVALID
        f = np.zeros(0, dtype=np.uint8) if self.file is None else self.file
        return oracle.bitrot_verify(self.algo, f, self.part_len, S, self.want)


def streaming_cases(oracle, rng, S, plen):
    data = rng.integers(0, 256, plen, dtype=np.uint8)
    f = stream_file(oracle, data, S)
    cases = [Case(HIGHWAYHASH256S, f, plen)]
    if plen == 0:
        return cases + [Case(HIGHWAYHASH256S, None, 0), Case(HIGHWAYHASH256S, np.zeros(32, dtype=np.uint8), 0)]
    nb = -(-plen // S)
    last = plen - (nb - 1) * S
    cases.append(Case(HIGHWAYHASH256S, flip(f, 5), plen))  # a digest byte
    if nb > 1 or last == S:  # a full frame: its first, middle and last byte
        for x in (32, 32 + S // 2, 32 + S - 1):
            cases.append(Case(HIGHWAYHASH256S, flip(f, x), plen))
    if last < S:  # the last byte of the short last frame
        cases.append(Case(HIGHWAYHASH256S, flip(f, f.size - 1), plen))
    for d in (-32, -1, 1, 32):  # wrong file lengths
        g = f[:f.size + d].copy() if d < 0 else np.concatenate([f, np.zeros(d, dtype=np.uint8)])
        if g.size >= 0:
            cases.append(Case(HIGHWAYHASH256S, g, plen))
    return cases


def whole_cases(oracle, rng, algo, flen):
    f = rng.integers(0, 256, flen, dtype=np.uint8)
    want = oracle.bitrot_hash(algo, f)
    cases = [Case(algo, f, 12345, want), Case(algo, f, 0, bytes(64))]  # part_len is not read; a wrong sum
    if flen:
        cases += [Case(algo, flip(f, 0), 0, want), Case(algo, flip(f, flen - 1), 0, want)]
    else:
        cases += [Case(algo, None, 0, want), Case(algo, None, 7, bytes(64))]  # a NULL file of length 0
    cases.append(Case(algo, np.zeros(0, dtype=np.uint8), 0, want))  # an empty file against a non-empty file's sum
    return cases


def run(c, cases):
    return c.bitrot_verify_parts([x.file for x in cases], [x.algo for x in cases], [x.part_len for x in cases],
                                 [x.want for x in cases])


@pytest.mark.parametrize("geom", GEOMS, ids=list(GEOMS))
def test_every_algorithm_length_and_damage(mb, oracle, geom):
    k, m, bs = GEOMS[geom]
    S = -(-bs // k)
    rng = np.random.default_rng(k * 1000 + bs // MiB)
    lens = (0, 1, S - 1, S, S + 1, 3 * S + 17)
    cases = []
    for plen in lens:
        cases += streaming_cases(oracle, rng, S, plen)
        for a in WHOLE:
            cases += whole_cases(oracle, rng, a, plen)
    cases += [Case(a, np.zeros(10, dtype=np.uint8), 10, bytes(64)) for a in (0, 5, -1, 99)]  # unknown algorithms
    rng.shuffle(cases)
    c = mb.Codec(k, m, bs)
    w0 = c.stat("whole_hash_launches")
    got = run(c, cases)
    want = [x.oracle(oracle, S) for x in cases]
    assert got == want
    assert c.stat("whole_hash_launches") - w0 == 1  # every whole-file part in one group: one launch
    assert FILE_CORRUPT in got and 0 in got and INVALID in got
    c.close()


def test_inline_frames(mb, oracle):
    """xl.meta inline data is verified as a streaming part of one frame (cmd/erasure-healing-common.go:398-406)"""
    frames = json.load(open(os.path.join(GOLD, "inline_frames.json")))
    c = mb.Codec(4, 2, MiB)
    S = c.shard_size()
    cases = []
    for f in frames:
        shard = bytes.fromhex(f["shard"])
        assert len(shard) == f["len"] <= S
        img = np.frombuffer(bytes.fromhex(f["digest"]) + shard, dtype=np.uint8).copy()
        cases.append(Case(HIGHWAYHASH256S, img, len(shard)))
        if img.size > 32:
            cases.append(Case(HIGHWAYHASH256S, flip(img, img.size - 1), len(shard)))
    got = run(c, cases)
    assert got == [x.oracle(oracle, S) for x in cases]
    assert got[0] == 0 and FILE_CORRUPT in got
    c.close()


EDGES = {SHA256: (0, 1, 55, 56, 63, 64, 65, 119, 120, 128), BLAKE2B512: (0, 1, 127, 128, 129, 255, 256, 257),
         HIGHWAYHASH256: (0, 1, 31, 32, 33, 63, 64, 65), HIGHWAYHASH256S: (0, 1, 31, 32, 33, 1000)}


@pytest.mark.parametrize("count", [1, 31, 32, 33, 65])
def test_four_algorithms_one_launch(mb, oracle, count):
    """count parts of each algorithm, lengths at every hash-block edge, interleaved, in ONE call: one whole_hash_kernel launch, and
    every result equal to the per-part single-algorithm calls"""
    rng = np.random.default_rng(count)
    c = mb.Codec(12, 4, MiB)
    S = c.shard_size()
    per = {a: [] for a in EDGES}
    for a, edges in EDGES.items():
        for q in range(count):
            n = edges[q % len(edges)]
            data = rng.integers(0, 256, n, dtype=np.uint8)
            if a == HIGHWAYHASH256S:
                f = stream_file(oracle, data, S)
                x = Case(a, f if q % 5 != 3 or n == 0 else flip(f, f.size - 1), n)
            else:
                want = oracle.bitrot_hash(a, data)
                x = Case(a, data if q % 5 != 3 or n == 0 else flip(data, n // 2), 0, want)
            per[a].append(x)
    cases = [per[a][q] for q in range(count) for a in (SHA256, HIGHWAYHASH256S, BLAKE2B512, HIGHWAYHASH256)]
    w0 = c.stat("whole_hash_launches")
    got = run(c, cases)
    assert c.stat("whole_hash_launches") - w0 == 1
    single = []
    for x in cases:
        if x.algo == HIGHWAYHASH256S:
            single.append(c.bitrot_verify_batch([x.file], [x.part_len])[0])  # mec_bitrot_verify refuses the NULL file of an empty part
        else:
            single.append(c.bitrot_verify_whole(x.algo, x.file, np.frombuffer(x.want, dtype=np.uint8)))
    assert got == single
    assert got == [x.oracle(oracle, S) for x in cases]
    c.close()


def test_more_than_256mib_takes_several_groups(mb, oracle):
    """three 90 MiB HighwayHash256 files: the first two share a staging group, the third is staged and hashed in a second one"""
    rng = np.random.default_rng(7)
    c = mb.Codec(12, 4, MiB)
    files = [rng.integers(0, 256, 90 * MiB, dtype=np.uint8) for _ in range(3)]
    sums = [oracle.bitrot_hash(HIGHWAYHASH256, f) for f in files]
    files[2][-1] ^= 1
    w0 = c.stat("whole_hash_launches")
    got = c.bitrot_verify_parts(files, [HIGHWAYHASH256] * 3, [0] * 3, sums)
    assert got == [0, 0, FILE_CORRUPT]
    assert c.stat("whole_hash_launches") - w0 == 2
    c.close()


def test_verify_batch_is_verify_parts(mb, oracle):
    """mec_bitrot_verify_batch equals mec_bitrot_verify_parts with every part HighwayHash256S"""
    rng = np.random.default_rng(3)
    c = mb.Codec(12, 4, MiB)
    S = c.shard_size()
    cases = []
    for plen in (0, 1, S, S + 1, 5 * S + 3):
        cases += streaming_cases(oracle, rng, S, plen)
    cases = [x for x in cases if x.file is not None]
    files, plens = [x.file for x in cases], [x.part_len for x in cases]
    assert c.bitrot_verify_batch(files, plens) == c.bitrot_verify_parts(files, [HIGHWAYHASH256S] * len(files), plens)
    c.close()
