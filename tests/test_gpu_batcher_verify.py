"""mec_batcher_verify (VerifyFile through the cross-request coalescer) against the CPU oracle's bitrotVerify, part by part.

Files live in page-locked arenas so that calls ride in merged verify batches.  Covered: 64 threads of VerifyFile-shaped calls that
mix streaming and whole-file parts with some corrupted ones ("verifies" = calls, at most one whole_hash_kernel launch per batch);
every private path ("verifies_serial": a pageable file, MEC_BATCHER_MEMCPY, an oversize part); MEC_SMALL_BLOCKS=0, where the shared
frame check takes its multi-launch branch; PUT, GET, heal and verify threads together on one batcher, every output bit-exact; and a
transcode batcher serving verifies."""
import numpy as np
import pytest

from test_gpu_batcher_transcode_blocksize import concurrently
from test_gpu_verify_parts import Case, flip, stream_file

pytestmark = pytest.mark.gpu
KiB, MiB = 1 << 10, 1 << 20
SHA256, HIGHWAYHASH256, HIGHWAYHASH256S, BLAKE2B512 = 1, 2, 3, 4
FILE_CORRUPT = -7
ENV = ("MEC_BATCHER_DEPTH", "MEC_BATCHER_MEMCPY", "MEC_SMALL_BLOCKS", "MEC_BATCHER_GET_OUT")


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


@pytest.fixture(autouse=True)
def clean_env(monkeypatch):
    for name in ENV:
        monkeypatch.delenv(name, raising=False)


class Arena:
    """page-locked bump allocator (freed at the end of the test)"""

    def __init__(self, mb, nbytes):
        self.mb, self.buf, self.at = mb, mb.pinned_array(nbytes), 0

    def put(self, a):
        if a is None:
            return None
        n = a.size
        out = self.buf[self.at:self.at + n]
        out[:] = a
        self.at += (n + 63) // 64 * 64 + 64
        assert self.at <= self.buf.size
        return out

    def free(self):
        self.mb.lib().mec_free_pinned(self.buf.ctypes.data)


def object_parts(oracle, rng, S, nparts, legacy, corrupt):
    """one VerifyFile: nparts parts of one object on one drive; legacy parts use a whole-file algorithm, the others HighwayHash256S"""
    cases = []
    for p in range(nparts):
        n = int(rng.choice([0, 1, 100, 4 * KiB, 128 * KiB, S - 1, S, S + 1, 3 * S + 5]))
        data = rng.integers(0, 256, n, dtype=np.uint8)
        algo = [SHA256, HIGHWAYHASH256, BLAKE2B512][p % 3] if legacy else HIGHWAYHASH256S
        if algo == HIGHWAYHASH256S:
            f = stream_file(oracle, data, S)
            x = Case(algo, flip(f, f.size - 1) if corrupt and p == 0 and f.size else f, n)
        else:
            x = Case(algo, flip(data, n - 1) if corrupt and p == 0 and n else data, 0, oracle.bitrot_hash(algo, data))
        cases.append(x)
    return cases


def hashed(oracle, S, cases):
    """does the call leave a part to hash once the decisions that need no device are made (else it returns at once)?"""
    return any(x.algo != HIGHWAYHASH256S or (x.part_len > 0 and x.file is not None and
                                             x.file.size == oracle.bitrot_shard_file_size(x.part_len, S, HIGHWAYHASH256S))
               for x in cases)


def verify(b, cases):
    return b.verify([x.file for x in cases], [x.algo for x in cases], [x.part_len for x in cases], [x.want for x in cases])


def pinned(arena, cases):
    return [Case(x.algo, arena.put(x.file), x.part_len, x.want) for x in cases]


def test_64_threads_mixed_formats(mb, oracle):
    b = mb.Batcher(12, 4, MiB)
    S = -(-MiB // 12)
    rng = np.random.default_rng(1)
    calls = [object_parts(oracle, rng, S, 1 + q % 4, legacy=q % 3 == 1 or (q % 3 == 2 and q % 2 == 0), corrupt=q % 5 == 0)
             for q in range(64)]
    # a call that mixes both formats: a legacy part beside healed (streaming) parts
    calls[2] = object_parts(oracle, rng, S, 2, True, False) + object_parts(oracle, rng, S, 2, False, True)
    arena = Arena(mb, sum(sum((0 if x.file is None else x.file.size) + 128 for x in c) for c in calls) + MiB)
    calls = [pinned(arena, c) for c in calls]
    stat = {k: b.stat(k) for k in ("verifies", "verifies_serial", "batches", "whole_hash_launches", "blocks_read")}
    got = concurrently([lambda c=c: verify(b, c) for c in calls])
    for c, g in zip(calls, got):
        assert g == [x.oracle(oracle, S) for x in c]
    assert FILE_CORRUPT in sum(got, []) and 0 in sum(got, [])
    assert b.stat("verifies") - stat["verifies"] == sum(hashed(oracle, S, c) for c in calls) and b.stat("verifies_serial") == stat["verifies_serial"]
    batches = b.stat("batches") - stat["batches"]
    assert 1 <= batches <= 64
    assert 1 <= b.stat("whole_hash_launches") - stat["whole_hash_launches"] <= batches
    frames = sum(-(-x.part_len // S) for c in calls for x in c
                 if x.algo == HIGHWAYHASH256S and x.file.size == oracle.bitrot_shard_file_size(x.part_len, S, HIGHWAYHASH256S))
    assert b.stat("blocks_read") - stat["blocks_read"] == frames
    b.close()
    arena.free()


def test_private_paths(mb, oracle, monkeypatch):
    rng = np.random.default_rng(2)
    b = mb.Batcher(12, 4, MiB, max_batch_blocks=4)  # slots of 8 blocks: at most 8 MiB - 1 KiB staged per batch
    S = -(-MiB // 12)
    arena = Arena(mb, 32 * MiB)
    small = object_parts(oracle, rng, S, 3, True, True)
    # a pageable file
    v0 = b.stat("verifies_serial")
    assert verify(b, small) == [x.oracle(oracle, S) for x in small]
    assert b.stat("verifies_serial") == v0 + 1
    # an oversize part: a whole file larger than a slot's staging buffer
    big = rng.integers(0, 256, 9 * MiB, dtype=np.uint8)
    over = pinned(arena, [Case(SHA256, big, 0, oracle.bitrot_hash(SHA256, big)), Case(SHA256, flip(big, 3), 0, oracle.bitrot_hash(SHA256, big))])
    assert verify(b, over) == [0, FILE_CORRUPT]
    assert b.stat("verifies_serial") == v0 + 2
    # a call that fits rides a merged batch
    ok = pinned(arena, small)
    v1 = b.stat("verifies")
    assert verify(b, ok) == [x.oracle(oracle, S) for x in ok]
    assert b.stat("verifies") == v1 + 1 and b.stat("verifies_serial") == v0 + 2
    b.close()
    # MEC_BATCHER_MEMCPY: every call takes the private path
    monkeypatch.setenv("MEC_BATCHER_MEMCPY", "1")
    b = mb.Batcher(12, 4, MiB)
    monkeypatch.delenv("MEC_BATCHER_MEMCPY")
    assert verify(b, ok) == [x.oracle(oracle, S) for x in ok]
    assert b.stat("verifies_serial") == 1 and b.stat("verifies") == 0
    b.close()
    arena.free()


def test_small_blocks_zero(mb, oracle, monkeypatch):
    """options that rule out the latency kernel: the shared frame check runs one launch per run of full frames and per short frame"""
    monkeypatch.setenv("MEC_SMALL_BLOCKS", "0")
    b = mb.Batcher(4, 2, MiB)
    monkeypatch.delenv("MEC_SMALL_BLOCKS")
    S = -(-MiB // 4)
    rng = np.random.default_rng(3)
    calls = [object_parts(oracle, rng, S, 3, q % 4 == 3, q % 3 == 0) for q in range(16)]
    arena = Arena(mb, sum(sum((0 if x.file is None else x.file.size) + 128 for x in c) for c in calls) + MiB)
    calls = [pinned(arena, c) for c in calls]
    got = concurrently([lambda c=c: verify(b, c) for c in calls])
    for c, g in zip(calls, got):
        assert g == [x.oracle(oracle, S) for x in c]
    assert b.stat("verifies") == sum(hashed(oracle, S, c) for c in calls) and b.stat("small_launches") == 0
    b.close()
    arena.free()


def test_mixed_traffic_one_batcher(mb, oracle):
    """PUT, GET, heal and verify threads together on one batcher: every output bit-exact"""
    k, m, bs = 12, 4, MiB
    S = -(-bs // k)
    b = mb.Batcher(k, m, bs)
    rng = np.random.default_rng(4)
    objs = [rng.integers(0, 256, n, dtype=np.uint8) for n in (100, 300 * KiB, 2 * MiB + 7)]
    enc = [oracle.erasure_encode(k, m, bs, HIGHWAYHASH256S, d)[0] for d in objs]
    arena = Arena(mb, 256 * MiB)
    pfiles = [[arena.put(f) for f in files] for files in enc]
    vcalls = [pinned(arena, object_parts(oracle, rng, S, 2, q % 2 == 1, q % 3 == 0)) for q in range(12)]
    srcs = [arena.put(d) for d in objs]
    calls, checks = [], []
    for q in range(24):
        o = q % 3
        kind = q % 4
        if kind == 0:
            calls.append(lambda o=o: b.encode(srcs[o], pinned=True))
            checks.append(lambda r, o=o: all(np.array_equal(r[i], enc[o][i]) for i in range(k + m)))
        elif kind == 1:
            files = [None] * 2 + pfiles[o][2:]
            dst = arena.put(np.zeros(objs[o].size, dtype=np.uint8))  # allocated here: the arena is not shared between threads
            calls.append(lambda files=files, o=o, dst=dst: b.decode(files, 0, objs[o].size, objs[o].size, dst=dst)[0])
            checks.append(lambda r, o=o: np.array_equal(r, objs[o]))
        elif kind == 2:
            stale = [i in (0, 13) for i in range(k + m)]
            files = [None if stale[i] else f for i, f in enumerate(pfiles[o])]
            calls.append(lambda files=files, stale=stale, o=o: b.heal(files, stale, objs[o].size, pinned=True))
            checks.append(lambda r, o=o: r[1] == 0 and np.array_equal(r[0][0], enc[o][0]) and np.array_equal(r[0][13], enc[o][13]))
        else:
            c = vcalls[q % len(vcalls)]
            calls.append(lambda c=c: verify(b, c))
            checks.append(lambda r, c=c: r == [x.oracle(oracle, S) for x in c])
    got = concurrently(calls)
    for q, (chk, r) in enumerate(zip(checks, got)):
        assert r is not None and chk(r), q
    assert b.stat("verifies") == sum(hashed(oracle, S, vcalls[q % len(vcalls)]) for q in range(3, 24, 4))
    b.close()
    arena.free()


def test_transcode_batcher_serves_verifies(mb, oracle):
    b = mb.Batcher(12, 4, MiB, dst=(8, 4))
    S = -(-MiB // 12)
    rng = np.random.default_rng(5)
    calls = [object_parts(oracle, rng, S, 2, q % 2 == 0, q % 4 == 1) for q in range(8)]
    arena = Arena(mb, sum(sum((0 if x.file is None else x.file.size) + 128 for x in c) for c in calls) + MiB)
    calls = [pinned(arena, c) for c in calls]
    got = concurrently([lambda c=c: verify(b, c) for c in calls])
    for c, g in zip(calls, got):
        assert g == [x.oracle(oracle, S) for x in c]
    assert b.stat("verifies") == sum(hashed(oracle, S, c) for c in calls)
    b.close()
    arena.free()
