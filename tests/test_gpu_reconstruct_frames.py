"""mec_reconstruct_frames against the oracle's part files: pass-through of wanted readers, reader fail-over inside one call, short
last frames, the MEC_ERR_READ_QUORUM + corrupt[] contract and the launches of the frame sink.

This is the entry point the C++ binding (include/minio_erasure.hpp, readAndReconstruct) builds Erasure::Decode and Erasure::Heal on.
Its inputs are the part files the oracle writes for the same bytes, and those files are also the expected output of every wanted
shard: a shard passed through, rebuilt, or passed through up to a bad frame and rebuilt from there must equal the original part
file byte for byte, digests included.  Every shard gets an output buffer one frame longer than its file, pre-filled with a marker
byte, so a write past the last frame and any write to a shard that is not wanted (or to parity under data_only that was not read)
shows up.  corrupt[] is pre-filled with a non-zero byte, so a stale verdict shows up too.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
MiB = 1 << 20
MARK = 0xA5
READ_QUORUM = -10
FULL = 13                            # full blocks of data behind every geometry's part files
GEOMS = {
    "12+4": (12, 4, MiB),            # compiled kernels, S = 87382
    "16+4": (16, 4, MiB),            # more than 16 streams
    "5+3": (5, 3, MiB - 1),          # no compiled kernel; S = 209715 is odd, so frames sit at odd host offsets
    "32+16": (32, 16, 256 * 1024),   # the widest geometry of the GPU path
}
LAST_LENS = ("0", "1", "7", "8", "31", "33", "S-1", "S")


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


def last_len(name, S):
    return {"S": S, "S-1": S - 1}.get(name) or int(name)


class Part:
    """The oracle's part files of one geometry, cut to any number of blocks and any last shard length.  A frame depends on its own
    block's bytes only, so the files of (nblocks, L) are the first nblocks - 1 frames of an encode of FULL full blocks followed by
    the frame of a last block whose shards are L bytes long."""

    def __init__(self, oracle, k, m, bs):
        self.k, self.m, self.n, self.bs = k, m, k + m, bs
        self.S = oracle.shard_size(bs, k)
        self.fs = 32 + self.S
        self.oracle = oracle
        rng = np.random.default_rng(k * 1000 + m)
        self.data = rng.integers(0, 256, FULL * bs, dtype=np.uint8)
        self.full, _ = oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, self.data)
        self.tails = {}

    def tail_bytes(self, L):
        # ceil(tail / k) == L: the last data shards are shorter than L, so Split's zero padding is part of the frame
        return self.bs if L == self.S else self.k * L - (self.k - 1) // 2

    def tail(self, L):
        if L not in self.tails:
            data = np.random.default_rng(L).integers(0, 256, self.tail_bytes(L), dtype=np.uint8)
            self.tails[L] = (data, self.oracle.erasure_encode(self.k, self.m, self.bs, self.oracle.HIGHWAYHASH256S, data)[0])
        return self.tails[L][1]

    def files(self, nblocks, L):
        if L == self.S:
            return [f[:nblocks * self.fs].copy() for f in self.full]
        return [np.concatenate([f[:(nblocks - 1) * self.fs], t]) for f, t in zip(self.full, self.tail(L))]


@pytest.fixture(scope="module")
def parts(oracle):
    cache = {}

    def get(name):
        if name not in cache:
            p = Part(oracle, *GEOMS[name])
            # the cut-and-join files are what the oracle writes for the same object
            want, _ = oracle.erasure_encode(p.k, p.m, p.bs, oracle.HIGHWAYHASH256S, p.data[:p.bs])
            assert all(np.array_equal(a, b) for a, b in zip(p.files(1, p.S), want)), "oracle self-check: one full block"
            joined = p.files(2, 33)
            want, _ = oracle.erasure_encode(p.k, p.m, p.bs, oracle.HIGHWAYHASH256S, np.concatenate([p.data[:p.bs], p.tails[33][0]]))
            assert all(np.array_equal(a, b) for a, b in zip(joined, want)), "oracle self-check: a full and a short block"
            cache[name] = p
        return cache[name]
    return get


def codec(mb, p, **opts):
    c = mb.Codec(p.k, p.m, p.bs)
    assert c.shard_size() == p.S
    for name, v in opts.items():
        c.set_option(name, v)
    return c


def ptrs(arrs):
    return (C.c_void_p * len(arrs))(*[None if a is None else a.ctypes.data for a in arrs])


def reconstruct(mb, c, frames, nblocks, last, want, data_only=False, flen=0):
    """mec_reconstruct_frames with an output for EVERY shard, each one frame longer than `flen` and filled with MARK."""
    S = c.shard_size()
    outs = [np.full(flen + 32 + S, MARK, dtype=np.uint8) for _ in range(c.n)]
    corrupt = np.full(c.n, 0xEE, dtype=np.uint8)
    w = np.zeros(c.n, dtype=np.uint8)
    w[list(want)] = 1
    rc = mb.capi.lib().mec_reconstruct_frames(c.h, ptrs(frames), nblocks, last, w.ctypes.data, 1 if data_only else 0, ptrs(outs),
                                               corrupt.ctypes.data)
    return rc, outs, corrupt


def assert_outputs(outs, expect, written, fs):
    """outs[i] == expect[i] followed by untouched guard bytes for i in `written`; every other output untouched."""
    for i, o in enumerate(outs):
        if i not in written:
            assert (o == MARK).all(), f"shard {i} was written although it is not a wanted output"
            continue
        e = expect[i]
        got = o[:e.size]
        if not np.array_equal(got, e):
            off = int(np.nonzero(got != e)[0][0])
            b, pos = divmod(off, fs)
            where = f"digest byte {pos}" if pos < 32 else f"shard byte {pos - 32}"
            raise AssertionError(f"shard {i}: {int((got != e).sum())} bytes differ; first in block {b}, {where} "
                                 f"(got {got[off]:#04x}, want {e[off]:#04x})")
        assert (o[e.size:] == MARK).all(), f"shard {i}: written past its last frame"


def corrupt_set(corrupt):
    return {i for i, v in enumerate(corrupt) if v}


def plan(k, m, r):
    """(offline, wanted) with r rebuilt shards: data shards offline and, from r = 2 on, the last parity shard (online but not one
    of the first k readers) wanted too.  Two readers are always wanted as well, data shard 2 and parity shard k (data shard 3 when
    nothing is offline and parity is not read), so every call passes shards through."""
    offline = set([1, k - 1, k // 2][:r - 1] if r >= 2 else [1][:r])
    wanted = offline | {2, k if offline else 3}
    if r >= 2:
        wanted.add(k + m - 1)
    return offline, wanted


def readers(n, k, offline):
    return [i for i in range(n) if i not in offline][:k]


@pytest.mark.parametrize("chunking", ["auto", "whole"])
@pytest.mark.parametrize("nblocks", [1, 2, 5, 8, 9, 13])
@pytest.mark.parametrize("geom", list(GEOMS))
def test_targets_and_ranges(mb, parts, geom, nblocks, chunking):
    """r = 0..4 rebuilt shards beside two passed-through readers, for full and short last frames.  "whole" runs the range as one
    chunk: 8 blocks are staged with one batched copy call, 9 with 2-D copies.  With auto chunks a short last frame of 5, 9 or 13
    blocks is alone in its chunk."""
    p = parts(geom)
    c = codec(mb, p, chunk_blocks=nblocks if chunking == "whole" else 0)
    try:
        for L in (p.S, 33):
            files = p.files(nblocks, L)
            for r in range(min(4, p.m) + 1):
                offline, wanted = plan(p.k, p.m, r)
                frames = [None if i in offline else f for i, f in enumerate(files)]
                rc, outs, corrupt = reconstruct(mb, c, frames, nblocks, 0 if L == p.S else L, wanted, flen=files[0].size)
                assert rc == 0, (L, r, rc)
                assert corrupt_set(corrupt) == set(), (L, r)
                assert len(wanted - set(readers(p.n, p.k, offline))) == r
                assert_outputs(outs, files, wanted, p.fs)
    finally:
        c.close()


@pytest.mark.parametrize("last", LAST_LENS)
@pytest.mark.parametrize("geom", list(GEOMS))
def test_short_last_frame(mb, parts, geom, last):
    """Every short-frame length, as the only block of a chunk (5 blocks: chunks of 4 and 1) and next to a full block in one launch
    (2 blocks).  Odd lengths end the last frame at an odd offset and leave a hash remainder."""
    p = parts(geom)
    L = last_len(last, p.S) or p.S
    c = codec(mb, p, chunk_blocks=4)
    try:
        for nblocks in (2, 5):
            files = p.files(nblocks, L)
            for r in (1, 3):
                offline, wanted = plan(p.k, p.m, r)
                frames = [None if i in offline else f for i, f in enumerate(files)]
                rc, outs, corrupt = reconstruct(mb, c, frames, nblocks, last_len(last, p.S), wanted, flen=files[0].size)
                assert rc == 0 and corrupt_set(corrupt) == set(), (nblocks, r, rc)
                assert_outputs(outs, files, wanted, p.fs)
    finally:
        c.close()


@pytest.mark.parametrize("geom", list(GEOMS))
def test_sub_range(mb, parts, geom):
    """frames[i] point at a later frame of the part: a range in the middle (its last frame is a full one, last_shard_len = 0) and
    a range that runs to the part's short last frame."""
    p = parts(geom)
    L = 7
    part = p.files(FULL, L)
    c = codec(mb, p)
    try:
        for start, nblocks, last in ((3, 5, 0), (6, FULL - 6, L)):
            files = [f[start * p.fs:(start + nblocks) * p.fs] for f in part]
            offline, wanted = plan(p.k, p.m, 2)
            frames = [None if i in offline else f[start * p.fs:] for i, f in enumerate(part)]
            rc, outs, corrupt = reconstruct(mb, c, frames, nblocks, last, wanted, flen=files[0].size)
            assert rc == 0 and corrupt_set(corrupt) == set(), (start, rc)
            assert_outputs(outs, files, wanted, p.fs)
    finally:
        c.close()


@pytest.mark.parametrize("case", ["all-data-lost", "parity-unread"])
def test_data_only(mb, parts, oracle, case):
    """ReconstructData semantics: parity is never rebuilt.  RS(8,8) with every data shard lost rebuilds eight shards and passes the
    eight parity readers through; RS(12,4) with two data shards lost reads parity 12 and 13 (passed through) and leaves the
    outputs of the unread, wanted parity 14 and 15 untouched."""
    if case == "all-data-lost":
        p = Part(oracle, 8, 8, 256 * 1024)
        offline, nblocks, L = set(range(8)), 9, 31
    else:
        p = parts("12+4")
        offline, nblocks, L = {3, 7}, 5, 8
    files = p.files(nblocks, L)
    frames = [None if i in offline else f for i, f in enumerate(files)]
    c = codec(mb, p, chunk_blocks=4)
    try:
        rc, outs, corrupt = reconstruct(mb, c, frames, nblocks, L, range(p.n), data_only=True, flen=files[0].size)
        assert rc == 0 and corrupt_set(corrupt) == set()
        assert_outputs(outs, files, set(range(p.k)) | set(readers(p.n, p.k, offline)), p.fs)
        # a parity shard only wanted and not read: nothing at all to do
        rc, outs, corrupt = reconstruct(mb, c, files, nblocks, L, {p.n - 1}, data_only=True, flen=files[0].size)
        assert rc == 0 and corrupt_set(corrupt) == set()
        assert_outputs(outs, files, set(), p.fs)
    finally:
        c.close()


def frame_offset(p, files, block, where):
    if where == "data":
        return block * p.fs + 32 + 1000
    if where == "digest":
        return block * p.fs + 5
    return files[0].size - 1     # "tail": the last byte of the short last frame


@pytest.mark.parametrize("case", ["data", "digest", "tail", "two-readers"])
@pytest.mark.parametrize("geom", ["12+4", "5+3"])
def test_failover(mb, parts, geom, case):
    """A wanted reader (data shard 2) fails its digest in the second chunk: its frames before the bad one are passed through, the
    rest are rebuilt with recomputed digests, and the output equals the original file — also when the corrupted byte was the
    stored digest itself, or the last byte of the short frame.  "two-readers": data shard 2 and data shard 0 (not wanted) fail in
    the same block and both are dropped."""
    p = parts(geom)
    nblocks, L = FULL, 31
    files = p.files(nblocks, L)
    offline, wanted = plan(p.k, p.m, 2)          # shard 1 offline; 1 and the last parity rebuilt; 2 and k passed through
    bad = {"data": {2: ("data", 5)}, "digest": {2: ("digest", 5)}, "tail": {2: ("tail", nblocks - 1)},
           "two-readers": {2: ("data", 6), 0: ("digest", 6)}}[case]
    inputs = [f.copy() for f in files]
    for i, (where, block) in bad.items():
        inputs[i][frame_offset(p, files, block, where)] ^= 0x40
    frames = [None if i in offline else f for i, f in enumerate(inputs)]
    c = codec(mb, p, chunk_blocks=4)
    try:
        rc, outs, corrupt = reconstruct(mb, c, frames, nblocks, L, wanted, flen=files[0].size)
        assert rc == 0
        assert corrupt_set(corrupt) == set(bad)
        assert c.stat("corrupt_shards") == len(bad)
        assert_outputs(outs, files, wanted, p.fs)
    finally:
        c.close()


def test_binding_retry_loop(mb, parts):
    """What readAndReconstruct (include/minio_erasure.hpp) does: hand over only the first k readable files; on MEC_ERR_READ_QUORUM
    drop every reader corrupt[] names and call again with the next ones.  The first call must name exactly the bad reader."""
    p = parts("12+4")
    nblocks, L = 9, 33
    files = p.files(nblocks, L)
    inputs = [f.copy() for f in files]
    inputs[4][frame_offset(p, files, 6, "data")] ^= 1
    wanted = {1, 4, 15}
    alive = [i != 1 for i in range(p.n)]
    c = codec(mb, p, chunk_blocks=4)
    try:
        rcs = []
        for _ in range(p.m + 1):
            use = [i for i in range(p.n) if alive[i]][:p.k]
            frames = [inputs[i] if i in use else None for i in range(p.n)]
            rc, outs, corrupt = reconstruct(mb, c, frames, nblocks, L, wanted, flen=files[0].size)
            rcs.append((rc, corrupt_set(corrupt)))
            if rc != READ_QUORUM:
                break
            assert corrupt_set(corrupt), "MEC_ERR_READ_QUORUM without a dropped reader: the caller cannot make progress"
            for i in corrupt_set(corrupt):
                alive[i] = False
        assert rcs == [(READ_QUORUM, {4}), (0, set())]
        assert_outputs(outs, files, wanted, p.fs)
    finally:
        c.close()


@pytest.mark.parametrize("case", ["same-block", "second-round"])
def test_read_quorum(mb, parts, case):
    """m + 1 bad readers: MEC_ERR_READ_QUORUM with exactly those readers in corrupt[].  "second-round": four data readers fail at
    block 4, the call resumes there with parity 12..15, and parity 12 fails at block 6 — a reader that was only read after the
    first drop must be named as well.  Outputs never grow past their files and shards that are not wanted stay untouched."""
    p = parts("12+4")
    nblocks, L = 9, 8
    files = p.files(nblocks, L)
    if case == "same-block":
        bad = {0: 4, 3: 4, 5: 4, 8: 4, 11: 4}
    else:
        bad = {0: 4, 1: 4, 2: 4, 3: 4, 12: 6}
    inputs = [f.copy() for f in files]
    for i, block in bad.items():
        inputs[i][frame_offset(p, files, block, "data")] ^= 0x80
    wanted = {1, 14}
    c = codec(mb, p, chunk_blocks=4)
    try:
        rc, outs, corrupt = reconstruct(mb, c, inputs, nblocks, L, wanted, flen=files[0].size)
        assert rc == READ_QUORUM
        assert corrupt_set(corrupt) == set(bad)
        for i, o in enumerate(outs):
            assert (o[files[0].size:] == MARK).all(), f"shard {i}: written past its last frame"
            if i not in wanted:
                assert (o == MARK).all(), f"shard {i} was written although it is not a wanted output"
        # nothing to do: corrupt[] is still cleared, nothing is written
        rc, outs, corrupt = reconstruct(mb, c, inputs, 0, 0, wanted, flen=0)
        assert rc == 0 and corrupt_set(corrupt) == set()
        assert_outputs(outs, files, set(), p.fs)
    finally:
        c.close()


def test_unread_readers_are_not_checked(mb, parts):
    """Only the first k readable files are read: a corrupt frame in parity 13 is neither flagged nor copied — wanted, that shard is
    rebuilt from the k readers and equals the original file."""
    p = parts("12+4")
    nblocks, L = 5, 7
    files = p.files(nblocks, L)
    inputs = [f.copy() for f in files]
    inputs[13][frame_offset(p, files, 1, "data")] ^= 0xFF
    inputs[13][frame_offset(p, files, 2, "digest")] ^= 0xFF
    c = codec(mb, p)
    try:
        rc, outs, corrupt = reconstruct(mb, c, inputs, nblocks, L, {3, 13}, flen=files[0].size)
        assert rc == 0 and corrupt_set(corrupt) == set()
        assert c.stat("corrupt_shards") == 0
        assert_outputs(outs, files, {3, 13}, p.fs)
    finally:
        c.close()


@pytest.mark.parametrize("form", ["latency", "throughput"])
@pytest.mark.parametrize("nblocks,chunk", [(2, 4), (5, 4), (8, 4), (9, 3), (13, 4)])
@pytest.mark.parametrize("last", ["S", "33"])
def test_launches(mb, parts, form, nblocks, chunk, last):
    """One launch per chunk through the latency kernel (a chunk ending in the short frame carries it as its tail block); with
    small_blocks = 0 the throughput kernel takes the short frame in a launch of its own, one more for that chunk unless the
    short frame is alone in it."""
    p = parts("12+4")
    L = last_len(last, p.S)
    files = p.files(nblocks, L)
    opts = dict(chunk_blocks=chunk)
    if form == "throughput":
        opts.update(small_blocks=0, jit=0)      # jit = 0: no kernel specialisation compiled in the background
    c = codec(mb, p, **opts)
    try:
        offline, wanted = plan(p.k, p.m, 2)
        frames = [None if i in offline else f for i, f in enumerate(files)]
        launches, small = c.launches, c.stat("form_small")
        rc, outs, corrupt = reconstruct(mb, c, frames, nblocks, L, wanted, flen=files[0].size)
        assert rc == 0 and corrupt_set(corrupt) == set()
        assert_outputs(outs, files, wanted, p.fs)
        nchunks = -(-nblocks // chunk)
        last_chunk = nblocks - (nchunks - 1) * chunk
        split = form == "throughput" and L != p.S and last_chunk > 1
        assert c.launches - launches == nchunks + split
        assert c.stat("form_small") - small == (nchunks if form == "latency" else 0)
    finally:
        c.close()
