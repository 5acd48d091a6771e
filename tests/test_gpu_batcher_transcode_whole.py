"""Whole-file-bitrot parts moved between pools through the cross-request coalescer (mec_batcher_transcode_whole): concurrent moves
of parts written with SHA256, HighwayHash256 and BLAKE2b512 (raw shard files, one digest per file) share merged batches, one
hash launch per batch, and every out file must be byte for byte what the oracle's streaming Erasure.Encode of the destination
geometry and block size writes, inside guard bytes.  Covered: merged batches per algorithm and block-size pair, shard files at
every hash block edge in one launch, offline drives with and without MEC_BATCHER_MIX_PATTERNS, bitrot redone on the private pair,
the private paths, traffic of every kind on one batcher, and the refusals.  Batchers at 10 MiB source blocks keep
max_batch_blocks <= 8."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_batcher_transcode_blocksize import concurrently
from test_gpu_transcode import assert_oracle_exact, rand

pytestmark = pytest.mark.gpu
MiB = 1 << 20
V1 = 10 * MiB
GUARD = 61
SHA256, HIGHWAYHASH256, HIGHWAYHASH256S, BLAKE2B512 = 1, 2, 3, 4
ALGOS = {"sha256": SHA256, "hh256": HIGHWAYHASH256, "blake2b": BLAKE2B512}
FILE_CORRUPT, READ_QUORUM, WRITE_QUORUM, INVALID_ARGUMENT, UNSUPPORTED = -7, -10, -11, -12, -102
PAIRS = [(12, 4, V1, 6, 2, MiB), (12, 4, MiB, 6, 2, MiB), (12, 4, MiB, 12, 4, MiB)]
PAIR_IDS = ["rs12_4@10M-rs6_2@1M", "rs12_4@1M-rs6_2@1M", "rs12_4@1M-rs12_4@1M"]


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


def lengths(bs, bd):
    """1 byte, half a destination block, a destination block, a source block - 1, a source block + 1, two source blocks + tail"""
    return [1, bd // 2 + 13, bd, bs - 1, bs + 1, 2 * bs + 4321]


def guarded(n):
    return (np.arange(n, dtype=np.int64) * 131 + 7).astype(np.uint8)


class Part:
    """a part written by the oracle with a whole-file algorithm in the source geometry (raw shard files in page-locked buffers,
    the expected digests n x 64) and the oracle's streaming files of the destination geometry"""

    def __init__(self, mb, oracle, pair, algo, total, seed):
        k1, m1, bs, k2, m2, bd = pair
        self.mb, self.total, self.algo, self.n = mb, total, algo, k1 + m1
        self.data = rand(total, seed)
        files, sums = oracle.erasure_encode(k1, m1, bs, algo, self.data)
        self.want, _ = oracle.erasure_encode(k2, m2, bd, oracle.HIGHWAYHASH256S, self.data)
        self.files = [mb.pinned_array(max(f.size, 1))[:f.size] for f in files]
        for a, f in zip(self.files, files):
            a[:] = f
        self.sums = np.zeros((self.n, 64), dtype=np.uint8)
        for i, d in enumerate(sums):
            self.sums[i, :len(d)] = np.frombuffer(d, dtype=np.uint8)

    def free(self):
        for a in self.files:
            self.mb.lib().mec_free_pinned(a.ctypes.data)


def move(mb, bat, part, n2, offline=(), prefer=None, pinned=True, online=None, write_quorum=0, algo=None, files=None):
    """mec_batcher_transcode_whole into guarded out files (page-locked unless pinned=False; online: the destination writers) ->
    (rc, heal_hint, outs); asserts that nothing outside an out file was written"""
    fsz = part.want[0].size
    fill = guarded(fsz + 2 * GUARD)
    online = [True] * n2 if online is None else online
    bufs = []
    for i in range(n2):
        b = None
        if online[i]:
            b = mb.pinned_array(fsz + 2 * GUARD) if pinned else np.empty(fsz + 2 * GUARD, dtype=np.uint8)
            b[:] = fill
        bufs.append(b)
    src = part.files if files is None else files
    fp = (C.c_void_p * part.n)(*[None if i in offline or src[i] is None else src[i].ctypes.data for i in range(part.n)])
    op = (C.c_void_p * n2)(*[b.ctypes.data + GUARD if b is not None else None for b in bufs])
    pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
    hint = C.c_int(-1)
    rc = mb.lib().mec_batcher_transcode_whole(bat.h, part.algo if algo is None else algo, fp, part.sums.ctypes.data,
                                              None if pf is None else pf.ctypes.data, part.total, op, write_quorum, C.byref(hint))
    outs = []
    for b in bufs:
        if b is None:
            outs.append(None)
            continue
        outs.append(b[GUARD:GUARD + fsz].copy())
        assert np.array_equal(b[:GUARD], fill[:GUARD]) and np.array_equal(b[GUARD + fsz:], fill[GUARD + fsz:]), "guard bytes written"
        if pinned:
            mb.lib().mec_free_pinned(b.ctypes.data)
    return rc, hint.value, outs


def exact(part, outs):
    return all(o is None or np.array_equal(o, w) for o, w in zip(outs, part.want))


NAMES = ("batches", "requests", "transcodes", "transcodes_whole", "transcodes_whole_serial", "transcodes_serial", "redone",
         "whole_hash_launches", "mixed_batches", "blocks_read", "bytes_h2d", "dst_blocks_encoded")


def counters(bat):
    return {s: bat.stat(s) for s in NAMES}


def delta(bat, before):
    return {s: v - before[s] for s, v in counters(bat).items()}


@pytest.fixture(scope="module", params=PAIRS, ids=PAIR_IDS)
def pair_batcher(request, mb):
    k1, m1, bs, k2, m2, bd = request.param
    bat = mb.Batcher(k1, m1, bs, max_batch_blocks=8, max_wait_us=200_000, dst=(k2, m2, bd))
    yield request.param, bat
    bat.close()


@pytest.mark.parametrize("algo", list(ALGOS))
def test_merged_vs_oracle(mb, oracle, pair_batcher, algo):
    """Every length twice at once through merged batches: every out file equals the oracle's, every move completes merged, the
    batches are fewer than the moves and each added exactly one hash launch; the source side stages k shard files per move."""
    pair, bat = pair_batcher
    k1, m1, bs, k2, m2, bd = pair
    parts = [Part(mb, oracle, pair, ALGOS[algo], t, 1000 + q) for q, t in enumerate(lengths(bs, bd) * 2)]
    try:
        before = counters(bat)
        res = concurrently([lambda p=p: move(mb, bat, p, k2 + m2) for p in parts])
        d = delta(bat, before)
        for p, (rc, hint, outs) in zip(parts, res):
            assert rc == p.total and hint == 0, (p.total, rc, hint)
            assert_oracle_exact(oracle, outs, k2, m2, bd, p.data)
        assert d["transcodes_whole"] == len(parts) and d["transcodes_whole_serial"] == 0 and d["redone"] == 0, d
        assert d["requests"] == len(parts) and d["transcodes"] == 0 and 0 < d["batches"] < len(parts), d
        assert d["whole_hash_launches"] == d["batches"], d
        assert d["blocks_read"] == sum(-(-p.total // bs) for p in parts), d
        sizes = mb.Codec(k1, m1, bs, ALGOS[algo])
        assert d["bytes_h2d"] == sum(k1 * sizes.shard_file_size(p.total) for p in parts), d
        sizes.close()
        assert d["dst_blocks_encoded"] == sum(-(-p.total // bd) for p in parts), d
    finally:
        for p in parts:
            p.free()


@pytest.mark.parametrize("algo", list(ALGOS))
def test_hash_block_edges_one_launch(mb, oracle, monkeypatch, algo):
    """One merged batch of moves whose shard files are exactly 1 .. 4097 bytes, across every algorithm's block edges (32 for
    HighwayHash, 64 and the 56-byte padding edge for SHA256, 128 for BLAKE2b): one hash launch over files of different lengths,
    no redo, exact outputs."""
    monkeypatch.setenv("MEC_BATCHER_DEPTH", "0")  # one batch of everything queued: cut at max_batch_blocks only
    lens = [1, 31, 32, 33, 55, 56, 63, 64, 65, 127, 128, 129, 4097]
    pair = PAIRS[1]
    k1, m1, bs, k2, m2, bd = pair
    bat = mb.Batcher(k1, m1, bs, max_batch_blocks=len(lens), max_wait_us=2_000_000, dst=(k2, m2, bd))
    parts = [Part(mb, oracle, pair, ALGOS[algo], k1 * n, 2000 + n) for n in lens]
    try:
        assert all(p.files[0].size == n for p, n in zip(parts, lens))
        before = counters(bat)
        res = concurrently([lambda p=p: move(mb, bat, p, k2 + m2) for p in parts])
        d = delta(bat, before)
        for p, (rc, hint, outs) in zip(parts, res):
            assert rc == p.total and hint == 0, (p.total, rc, hint)
            assert_oracle_exact(oracle, outs, k2, m2, bd, p.data)
        assert d["batches"] == 1 and d["whole_hash_launches"] == 1, d
        assert d["transcodes_whole"] == len(lens) and d["redone"] == 0, d
    finally:
        for p in parts:
            p.free()
        bat.close()


@pytest.mark.parametrize("use_prefer", [False, True])
def test_offline_same_pattern(mb, oracle, pair_batcher, use_prefer):
    """Data and parity drives offline, the same for every move of the batch, with and without `prefer`: the missing data shards
    are rebuilt from the raw rows of every move in one merged reconstruct."""
    pair, bat = pair_batcher
    k1, m1, bs, k2, m2, bd = pair
    parts = [Part(mb, oracle, pair, SHA256 if q % 2 else HIGHWAYHASH256, t, 3000 + q)
             for q, t in enumerate([bd // 2 + 5, bs + 1, 2 * bs + 4321])]
    prefer = [1 if i in (3, 14, 15) else 0 for i in range(k1 + m1)] if use_prefer else None
    try:
        before = counters(bat)
        res = concurrently([lambda p=p: move(mb, bat, p, k2 + m2, offline=(1, 7, 12, 13), prefer=prefer) for p in parts])
        d = delta(bat, before)
        for p, (rc, hint, outs) in zip(parts, res):
            assert rc == p.total and hint == 0 and exact(p, outs), (p.total, rc, hint)
        assert d["transcodes_whole"] == len(parts) and d["redone"] == 0, d
    finally:
        for p in parts:
            p.free()


@pytest.mark.parametrize("mix", [False, True])
def test_offline_rotated(mb, oracle, mix):
    """One source drive offline, rotating with the move: with MEC_BATCHER_MIX_PATTERNS the patterns share batches
    ("mixed_batches" > 0), without it they never do; every out file is exact either way."""
    pair = PAIRS[1]
    k1, m1, bs, k2, m2, bd = pair
    bat = mb.Batcher(k1, m1, bs, max_batch_blocks=64, max_wait_us=200_000, mix_patterns=mix, dst=(k2, m2, bd))
    parts = [Part(mb, oracle, pair, BLAKE2B512, t, 4000 + q) for q, t in enumerate([bd // 3, bs - 1, bs + 1, 2 * bs + 99] * 2)]
    try:
        before = counters(bat)
        res = concurrently([lambda q=q, p=p: move(mb, bat, p, k2 + m2, offline=((q * 3) % (k1 + m1),)) for q, p in enumerate(parts)])
        d = delta(bat, before)
        for p, (rc, hint, outs) in zip(parts, res):
            assert rc == p.total and hint == 0 and exact(p, outs), (p.total, rc, hint)
        assert d["transcodes_whole"] == len(parts) and d["redone"] == 0, d
        assert (d["mixed_batches"] > 0) == mix, d
        assert d["whole_hash_launches"] == d["batches"], d
    finally:
        for p in parts:
            p.free()
        bat.close()


def test_bitrot_redone(mb, oracle, pair_batcher):
    """A flipped byte in a chosen reader's shard file: that move is redone alone on the private pair (heal_hint = -7, exact, counted
    in redone and transcodes_whole_serial) while its batch-mates complete merged.  A move with more corrupt and offline readers
    than parity drives returns MEC_ERR_READ_QUORUM."""
    pair, bat = pair_batcher
    k1, m1, bs, k2, m2, bd = pair
    parts = [Part(mb, oracle, pair, algo, t, 5000 + q)
             for q, (algo, t) in enumerate([(SHA256, bd), (HIGHWAYHASH256, bs + 1), (SHA256, 2 * bs + 4321), (SHA256, bs - 1)])]
    bad = parts[2]
    f = bad.files[5]
    f[f.size // 2] ^= 0x20
    try:
        before = counters(bat)
        res = concurrently([lambda p=p: move(mb, bat, p, k2 + m2) for p in parts])
        d = delta(bat, before)
        for p, (rc, hint, outs) in zip(parts, res):
            assert rc == p.total and hint == (FILE_CORRUPT if p is bad else 0) and exact(p, outs), (p.total, rc, hint)
        assert d["redone"] == 1 and d["transcodes_whole_serial"] == 1 and d["transcodes_whole"] == len(parts) - 1, d
        # five readers gone: drive 9 offline, drives 0, 4, 11 and 14 fail their digests
        q = parts[3]
        files = [a.copy() for a in q.files]
        for i in (0, 4, 11, 14):
            files[i][i * 7 % files[i].size] ^= 0x01
        pinned = [mb.pinned_array(a.size) for a in files]
        for a, b in zip(pinned, files):
            a[:] = b
        try:
            rc, hint, _ = move(mb, bat, q, k2 + m2, offline=(9,), files=pinned)
        finally:
            for a in pinned:
                mb.lib().mec_free_pinned(a.ctypes.data)
        assert rc == READ_QUORUM
    finally:
        f[f.size // 2] ^= 0x20
        for p in parts:
            p.free()


def test_private_paths(mb, oracle):
    """Pageable out files, and a part of more source blocks than max_batch_blocks, move on the private pair (the source handle of
    the part's algorithm) with exact outputs."""
    pair = PAIRS[1]
    k1, m1, bs, k2, m2, bd = pair
    bat = mb.Batcher(k1, m1, bs, max_batch_blocks=2, max_wait_us=0, dst=(k2, m2, bd))
    small = Part(mb, oracle, pair, HIGHWAYHASH256, bd // 2 + 1, 6001)
    big = Part(mb, oracle, pair, BLAKE2B512, 3 * bs + 17, 6002)
    try:
        for p, pinned in ((small, False), (big, True), (big, False)):
            before = counters(bat)
            rc, hint, outs = move(mb, bat, p, k2 + m2, pinned=pinned)
            d = delta(bat, before)
            assert rc == p.total and hint == 0 and exact(p, outs)
            assert d["requests"] == 0 and d["transcodes_whole_serial"] == 1 and d["transcodes_whole"] == 0, d
    finally:
        small.free()
        big.free()
        bat.close()


def test_mixed_traffic(mb, oracle):
    """Whole-file moves of two algorithms, streaming moves, PUTs and GETs at once on one batcher: every result is exact, streaming
    moves are counted as such, and every whole-file batch launched its own hash (at least one batch per algorithm)."""
    pair = PAIRS[1]
    k1, m1, bs, k2, m2, bd = pair
    bat = mb.Batcher(k1, m1, bs, max_batch_blocks=64, max_wait_us=100_000, dst=(k2, m2, bd))
    wparts = [Part(mb, oracle, pair, SHA256 if q % 2 else HIGHWAYHASH256, t, 7000 + q)
              for q, t in enumerate([bd // 2, bs + 3, 2 * bs + 5, bs - 7, 77, bs])]
    sdata = [rand(t, 7100 + q) for q, t in enumerate([bs // 3, 2 * bs + 1, 5000])]
    sfiles = []
    for data in sdata:
        files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
        pf = [mb.pinned_array(f.size) for f in files]
        for a, f in zip(pf, files):
            a[:] = f
        sfiles.append(pf)
    put_data = [mb.pinned_array(t) for t in (bs // 2, bs + 11)]
    for q, a in enumerate(put_data):
        a[:] = rand(a.size, 7200 + q)
    keep = []
    try:
        def stream_move(q):
            outs, hint = bat.transcode(sfiles[q], sdata[q].size, pinned=True)
            keep.append(outs)
            return outs, hint

        def put(q):
            files = bat.encode(put_data[q], pinned=True)
            keep.append(files)
            return files

        def get(q):
            dst = mb.pinned_array(sdata[q].size)
            keep.append([dst])
            return bat.decode([None, None] + sfiles[q][2:], 0, sdata[q].size, sdata[q].size, dst=dst)

        calls = [lambda p=p: move(mb, bat, p, k2 + m2) for p in wparts]
        calls += [lambda q=q: stream_move(q) for q in range(len(sdata))]
        calls += [lambda q=q: put(q) for q in range(len(put_data))]
        calls += [lambda q=q: get(q) for q in range(len(sdata))]
        before = counters(bat)
        res = concurrently(calls)
        d = delta(bat, before)
        nw = len(wparts)
        for p, (rc, hint, outs) in zip(wparts, res[:nw]):
            assert rc == p.total and hint == 0 and exact(p, outs), (p.algo, p.total, rc, hint)
        for q, (outs, hint) in enumerate(res[nw:nw + len(sdata)]):
            assert hint == 0
            assert_oracle_exact(oracle, outs, k2, m2, bd, sdata[q])
        for q, files in enumerate(res[nw + len(sdata):nw + len(sdata) + len(put_data)]):
            want, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, np.asarray(put_data[q]))
            assert all(np.array_equal(f, w) for f, w in zip(files, want))
        for q, (got, hint) in enumerate(res[nw + len(sdata) + len(put_data):]):
            assert hint == 0 and np.array_equal(got, sdata[q])
        assert d["transcodes_whole"] == nw and d["transcodes_whole_serial"] == 0 and d["redone"] == 0, d
        assert d["transcodes"] == len(sdata) and d["transcodes_serial"] == 0, d
        assert d["whole_hash_launches"] >= 2, d  # SHA256 and HighwayHash256 moves never share a batch
    finally:
        for p in wparts:
            p.free()
        for pf in sfiles:
            for a in pf:
                mb.lib().mec_free_pinned(a.ctypes.data)
        for a in put_data:
            mb.lib().mec_free_pinned(a.ctypes.data)
        for files in keep:
            for f in files:
                if f is not None and f.size:
                    mb.lib().mec_free_pinned(f.ctypes.data)
        bat.close()


def test_refusals(mb, oracle):
    """With a real batcher, in the documented order: HighwayHash256S is MEC_ERR_UNSUPPORTED and an unknown algorithm
    MEC_ERR_INVALID_ARGUMENT; a plain batcher MEC_ERR_INVALID_ARGUMENT; too few writers MEC_ERR_WRITE_QUORUM; an empty part returns
    0 with every out file and guard untouched; fewer than k source files MEC_ERR_READ_QUORUM.  Offline destination writers are
    skipped and count against the write quorum."""
    pair = PAIRS[1]
    k1, m1, bs, k2, m2, bd = pair
    bat = mb.Batcher(k1, m1, bs, max_batch_blocks=8, max_wait_us=1000, dst=(k2, m2, bd))
    plain = mb.Batcher(k1, m1, bs, max_batch_blocks=8, max_wait_us=1000)
    p = Part(mb, oracle, pair, SHA256, bs + 5, 8001)
    try:
        n2 = k2 + m2
        assert move(mb, bat, p, n2, algo=HIGHWAYHASH256S)[:2] == (UNSUPPORTED, 0)
        assert move(mb, bat, p, n2, algo=5)[:2] == (INVALID_ARGUMENT, 0)
        assert move(mb, bat, p, n2, algo=0)[:2] == (INVALID_ARGUMENT, 0)
        assert move(mb, plain, p, n2)[:2] == (INVALID_ARGUMENT, 0)
        assert move(mb, plain, p, n2, algo=HIGHWAYHASH256S)[:2] == (INVALID_ARGUMENT, 0)  # the batcher is checked first
        online = [i not in (0, 3, 7) for i in range(n2)]
        assert move(mb, bat, p, n2, online=online, write_quorum=6)[0] == WRITE_QUORUM
        # the empty part: nothing is written, guards and out files keep their fill
        empty = Part(mb, oracle, pair, SHA256, 0, 8002)
        fill = guarded(empty.want[0].size + 2 * GUARD)[GUARD:GUARD + empty.want[0].size]
        rc, hint, outs = move(mb, bat, empty, n2)
        assert rc == 0 and hint == 0 and all(np.array_equal(o, fill) for o in outs)
        empty.free()
        rc, hint, _ = move(mb, bat, p, n2, offline=(0, 1, 2, 3, 4))
        assert rc == READ_QUORUM
        # offline writers are skipped
        online = [i not in (1, 6) for i in range(n2)]
        rc, hint, outs = move(mb, bat, p, n2, online=online, write_quorum=6)
        assert rc == p.total and hint == 0 and outs[1] is None and outs[6] is None and exact(p, outs)
        # the Python binding
        outs, hint = bat.transcode_whole(p.files, [p.sums[i].tobytes() for i in range(p.n)], p.total, SHA256, pinned=True)
        assert hint == 0 and exact(p, outs)
        for o in outs:
            mb.lib().mec_free_pinned(o.ctypes.data)
        with pytest.raises(mb.MecError) as ei:
            bat.transcode_whole(p.files, [p.sums[i].tobytes() for i in range(p.n)], p.total, HIGHWAYHASH256S)
        assert ei.value.code == UNSUPPORTED
    finally:
        p.free()
        bat.close()
        plain.close()
