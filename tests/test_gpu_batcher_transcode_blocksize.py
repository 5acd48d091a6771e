"""Moves across block sizes through the cross-request coalescer (mec_batcher_new_transcode_ex, mec_batcher_transcode): legacy parts
written with 10 MiB erasure blocks moved concurrently into a pool that writes 1 MiB blocks, in merged batches and on the private
path, every out file byte for byte against the CPU oracle's Erasure.Encode of the destination geometry and block size, with guard
bytes around each file.  Batchers stay at max_batch_blocks <= 8: at 10 MiB source blocks their slots already take about 3 GiB."""
import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
MiB = 1 << 20
V1 = 10 * MiB
GUARD = 64
PAIRS = [(12, 4, V1, 6, 2, MiB), (10, 1, 4 * (MiB - 1), 5, 3, MiB - 1)]
FILE_CORRUPT = -7


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


def rand(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def lengths(bs, bd):
    """one byte, half a destination block, 3.5 destination blocks, one source block, one more byte, two source blocks and a tail"""
    return [1, bd // 2 + 13, 3 * bd + bd // 2, bs, bs + 1, 2 * bs + 4321]


class Part:
    """a part written by the oracle in the source geometry, its page-locked copy, and the oracle's destination files"""

    def __init__(self, mb, oracle, pair, total, seed):
        k1, m1, bs, k2, m2, bd = pair
        self.mb, self.total = mb, total
        self.data = rand(total, seed)
        files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, self.data)
        self.want, _ = oracle.erasure_encode(k2, m2, bd, oracle.HIGHWAYHASH256S, self.data)
        self.files = [mb.pinned_array(f.size) for f in files]
        for a, f in zip(self.files, files):
            a[:] = f

    def free(self):
        for a in self.files:
            self.mb.lib().mec_free_pinned(a.ctypes.data)


def move(mb, bat, part, n2, offline=(), pinned=True):
    """mec_batcher_transcode into guarded out files (page-locked unless pinned=False) -> (rc, heal_hint, outs); asserts that
    nothing outside an out file was written"""
    fsz = part.want[0].size
    fill = (np.arange(fsz + 2 * GUARD) * 37 + 11).astype(np.uint8)
    bufs = []
    for _ in range(n2):
        b = mb.pinned_array(fsz + 2 * GUARD) if pinned else np.empty(fsz + 2 * GUARD, dtype=np.uint8)
        b[:] = fill
        bufs.append(b)
    fp = (C.c_void_p * len(part.files))(*[None if i in offline else f.ctypes.data for i, f in enumerate(part.files)])
    op = (C.c_void_p * n2)(*[b.ctypes.data + GUARD for b in bufs])
    hint = C.c_int(-1)
    rc = mb.lib().mec_batcher_transcode(bat.h, fp, None, part.total, op, 0, C.byref(hint))
    outs = [b[GUARD:GUARD + fsz].copy() for b in bufs]
    for b in bufs:
        assert np.array_equal(b[:GUARD], fill[:GUARD]) and np.array_equal(b[GUARD + fsz:], fill[GUARD + fsz:]), "guard bytes written"
        if pinned:
            mb.lib().mec_free_pinned(b.ctypes.data)
    return rc, hint.value, outs


def concurrently(calls):
    """all callers released together -> their results"""
    bar = threading.Barrier(len(calls))
    res = [None] * len(calls)

    def run(q):
        bar.wait()
        res[q] = calls[q]()
    th = [threading.Thread(target=run, args=(q,)) for q in range(len(calls))]
    [t.start() for t in th]
    [t.join() for t in th]
    return res


@pytest.fixture(scope="module", params=PAIRS, ids=lambda p: f"rs{p[0]}_{p[1]}@{p[2]}-rs{p[3]}_{p[4]}@{p[5]}")
def setup(request, mb, oracle):
    pair = request.param
    parts = [Part(mb, oracle, pair, total, 900 + q) for q, total in enumerate(lengths(pair[2], pair[5]))]
    yield pair, parts
    for p in parts:
        p.free()


def counters(bat):
    return {s: bat.stat(s) for s in ("requests", "transcodes", "transcodes_serial", "redone", "dst_blocks_encoded")}


@pytest.mark.parametrize("mix", [False, True])
def test_concurrent_moves(mb, setup, mix):
    """Every length twice at once, the second copy with one source drive offline (rotating with the request, so with MIX the
    patterns differ and still share batches); every out file equals the oracle's, dst_blocks_encoded counts destination blocks."""
    (k1, m1, bs, k2, m2, bd), parts = setup
    bat = mb.Batcher(k1, m1, bs, max_batch_blocks=8, max_wait_us=200_000, mix_patterns=mix, dst=(k2, m2, bd))
    plan = [(p, ()) for p in parts] + [(p, ((q * 3) % (k1 + m1),)) for q, p in enumerate(parts)]
    before = counters(bat)
    res = concurrently([lambda p=p, off=off: move(mb, bat, p, k2 + m2, off) for p, off in plan])
    d = {s: v - before[s] for s, v in counters(bat).items()}
    for (p, off), (rc, hint, outs) in zip(plan, res):
        assert rc == p.total and hint == 0, (p.total, off, rc, hint)
        for i, o in enumerate(outs):
            assert np.array_equal(o, p.want[i]), f"part of {p.total} bytes, offline {off}: destination file {i} differs from the oracle"
    assert d["requests"] == len(plan) and d["transcodes"] == len(plan) and d["transcodes_serial"] == 0 and d["redone"] == 0, d
    assert d["dst_blocks_encoded"] == sum(-(-p.total // bd) for p, _ in plan), d
    bat.close()


def test_corrupt_reader_redone(mb, setup):
    """A move whose chosen reader fails its digest in its last source block is redone alone on the private pair (heal_hint = -7,
    counted in redone and transcodes_serial); it and the moves merged with it are still exact."""
    (k1, m1, bs, k2, m2, bd), parts = setup
    p = parts[-1]  # three source blocks
    S = -(-bs // k1)
    orig = p.files[1][2 * (32 + S) + 40]
    p.files[1][2 * (32 + S) + 40] ^= 0x5A
    try:
        bat = mb.Batcher(k1, m1, bs, max_batch_blocks=8, max_wait_us=200_000, dst=(k2, m2, bd))
        before = counters(bat)
        res = concurrently([lambda q=q: move(mb, bat, parts[q], k2 + m2) for q in (0, 2, len(parts) - 1)])
        d = {s: v - before[s] for s, v in counters(bat).items()}
    finally:
        p.files[1][2 * (32 + S) + 40] = orig
    for q, (rc, hint, outs) in zip((0, 2, len(parts) - 1), res):
        assert rc == parts[q].total and hint == (FILE_CORRUPT if q == len(parts) - 1 else 0)
        assert all(np.array_equal(o, w) for o, w in zip(outs, parts[q].want))
    assert d["redone"] == 1 and d["transcodes_serial"] == 1 and d["transcodes"] == 2, d
    bat.close()


def test_private_paths(mb, setup):
    """A part of more source blocks than max_batch_blocks, and pageable out files: both move on the private pair, whose codecs
    carry both block sizes, with the same bytes."""
    (k1, m1, bs, k2, m2, bd), parts = setup
    big = parts[-1]  # three source blocks
    bat = mb.Batcher(k1, m1, bs, max_batch_blocks=2, max_wait_us=0, dst=(k2, m2, bd))
    for pinned in (True, False):
        before = counters(bat)
        rc, hint, outs = move(mb, bat, big, k2 + m2, pinned=pinned)
        d = {s: v - before[s] for s, v in counters(bat).items()}
        assert rc == big.total and hint == 0
        assert all(np.array_equal(o, w) for o, w in zip(outs, big.want))
        assert d["requests"] == 0 and d["transcodes_serial"] == 1, d
    # pageable out files on a part that would fit a batch
    small = parts[1]
    before = counters(bat)
    rc, hint, outs = move(mb, bat, small, k2 + m2, pinned=False)
    d = {s: v - before[s] for s, v in counters(bat).items()}
    assert rc == small.total and hint == 0 and all(np.array_equal(o, w) for o, w in zip(outs, small.want))
    assert d["requests"] == 0 and d["transcodes_serial"] == 1, d
    bat.close()


def test_equal_block_sizes_match_plain_constructor(mb, oracle):
    """An _ex batcher with R = 1 writes exactly what a mec_batcher_new_transcode batcher writes."""
    k1, m1, k2, m2, bs = 12, 4, 6, 2, MiB
    pair = (k1, m1, bs, k2, m2, bs)
    parts = [Part(mb, oracle, pair, total, 950 + q) for q, total in enumerate((1, bs // 2 + 13, bs, 3 * bs + 12345))]
    got = []
    for dst in ((k2, m2), (k2, m2, bs)):
        bat = mb.Batcher(k1, m1, bs, max_batch_blocks=8, max_wait_us=200_000, dst=dst)
        before = counters(bat)
        res = concurrently([lambda p=p: move(mb, bat, p, k2 + m2) for p in parts])
        d = {s: v - before[s] for s, v in counters(bat).items()}
        assert d["transcodes"] == len(parts) and d["dst_blocks_encoded"] == sum(-(-p.total // bs) for p in parts), d
        got.append(res)
        bat.close()
    for p, a, b in zip(parts, *got):
        assert a[0] == b[0] == p.total and a[1] == b[1] == 0
        assert all(np.array_equal(x, y) and np.array_equal(x, w) for x, y, w in zip(a[2], b[2], p.want))
    for p in parts:
        p.free()
