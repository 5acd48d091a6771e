"""Whole-file decode and heal (mec_decode_whole / mec_heal_whole) on both kernels, against the CPU oracle.

Parts written with the whole-file bitrot algorithms (SHA256, BLAKE2b512, HighwayHash256) carry no frames and no per-block digests:
their rebuild (launch_whole_rebuild, ec_api.cu) hands Engine::launch_fused the raw shard files as staged on the device, blocks S
bytes apart from the start of each file.  A range that begins at block b > 0 is read at b * S bytes into the file, so every
loader sees shard offsets far larger than any frame-based caller makes (those all read 32 bytes in).  The rebuild runs in up to
two launches: the full blocks, then the short last block with its own shard length.

Truth is the oracle: files and sums come from oracle.erasure_encode, the expected decode output is the slice of the object and
the expected heal output the oracle's files and sums.  Each case asserts from the dispatch counters which rebuild form ran:

  shards not 16-byte multiples (S % 16 != 0), or k > 16       dyn_bytewise, loader 0 (byte-wise)
  S % 16 == 0, range from block 0, more than one block          dyn_aligned (jit = 0) / jit (jit = 1); TMA with one 3-D map per
                                                                run of survivors at a uniform arena stride (loader 3) when a CTA
                                                                takes a multiple of 4 blocks and there are at most kMaxRuns = 6
                                                                runs, else one map per survivor (loader 2)
  a launch that starts at a block > 0                           dyn_bytewise: the shard does not lie in the row its map covers
  at most 5 blocks per SM and default options                   small (latency kernel)

The output buffer and every out file are longer than asked for and pre-filled with MARK; the guard bytes must survive, and so
must every out-sum slot that was not asked for.  Source files must come back unchanged.  Every test sets jit to 0 or 1 and
points MEC_JIT_CACHE_DIR at its own directory; the NVRTC specialisations it compiles are two decode matrices (one RS(4,2), one
RS(8,8)), shared in-process by every test that needs them.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_kernel_forms import (TMA_BYTEWISE, TMA_PER_INPUT, TMA_RUNS, ceil_div, form_counts, form_delta, jit_cache, last_launch,
                                   mb, num_sms, round_up)

pytestmark = pytest.mark.gpu
KiB, MiB = 1 << 10, 1 << 20
MARK = 0x5A          # out buffers, out files and out sums are pre-filled with this byte
GUARD = 64           # bytes past the end of every out buffer and out file
SHA256, HIGHWAYHASH256, BLAKE2B512 = 1, 2, 4
ALGOS = {"sha256": SHA256, "hh256": HIGHWAYHASH256, "blake2b": BLAKE2B512}
FILE_CORRUPT, READ_QUORUM = -7, -10
DISPATCH_ENV = ("MEC_SMALL_BLOCKS", "MEC_EB", "MEC_FORCE_BYTEWISE", "MEC_FORCE_DYNAMIC", "MEC_JIT", "MEC_GRID_MULT",
                "MEC_BALANCE_GRID", "MEC_NO_ROWS3D", "MEC_USE_AUTO", "MEC_STATIC_GROUPS", "MEC_CHUNK_BLOCKS")
THROUGHPUT = dict(jit=0, small_blocks=0)                # the throughput kernel for every launch
ONE_BLOCK = dict(jit=1, eb=1, small_blocks=0)           # ... and one erasure block per CTA, NVRTC kernels where TMA runs
LATENCY = dict(jit=0)                                   # default dispatch: small launches take the latency kernel


@pytest.fixture(autouse=True)
def clean_dispatch(monkeypatch, jit_cache):
    """Codec reads these when it is created: only the options a test sets may steer a launch."""
    for name in DISPATCH_ENV:
        monkeypatch.delenv(name, raising=False)


_PARTS = {}


def part(oracle, k, m, bs, algo, size):
    """(object, shard files, whole-file sums) of a part from the oracle, cached across tests."""
    key = (k, m, bs, algo, size)
    if key not in _PARTS:
        data = np.random.default_rng(size % 100003 + 7 * k + m + algo).integers(0, 256, size, dtype=np.uint8)
        files, sums = oracle.erasure_encode(k, m, bs, algo, data)
        _PARTS[key] = (data, files, sums)
    return _PARTS[key]


def codec(mb, k, m, bs, algo, opts):
    c = mb.Codec(k, m, bs, algo=algo)
    for name, v in opts.items():
        c.set_option(name, v)
    return c


def lib():
    import minio_b200
    return minio_b200.lib()


def _ptrs(arrs):
    return (C.c_void_p * len(arrs))(*[None if a is None else a.ctypes.data for a in arrs])


def _sums(n, sums):
    sm = np.zeros((n, 64), dtype=np.uint8)
    for i, d in enumerate(sums):
        sm[i, :len(d)] = np.frombuffer(d, dtype=np.uint8)
    return sm


def _call(c, fn, srcs):
    before = form_counts(c)
    copies = [None if f is None else f.copy() for f in srcs]
    rc = fn()
    for i, (f, g) in enumerate(zip(srcs, copies)):
        assert f is None or np.array_equal(f, g), f"source file {i} was written"
    return rc, dict(delta=form_delta(before, form_counts(c)), last=last_launch(c))


def decode(c, srcs, sums, offset, length, total):
    """mec_decode_whole into a MARK-filled buffer GUARD bytes longer than `length`.  -> (rc, bytes, heal hint, dispatch)"""
    dst = np.full(length + GUARD, MARK, dtype=np.uint8)
    hint = C.c_int(MARK)
    sm = _sums(c.n, sums)
    rc, run = _call(c, lambda: lib().mec_decode_whole(c.h, _ptrs(srcs), sm.ctypes.data, offset, length, total,
                                                               dst.ctypes.data, C.byref(hint)), srcs)
    assert (dst[length:] == MARK).all(), "decode wrote past the end of the range"
    return rc, dst[:length], hint.value, run


def heal(c, srcs, sums, stale, total):
    """mec_heal_whole into MARK-filled out files GUARD bytes longer than a shard file.  -> (rc, out files, out sums [n, 64],
    corrupt[n], dispatch)"""
    flen = c.shard_file_size(total)
    outs = [np.full(flen + GUARD, MARK, dtype=np.uint8) if i in stale else None for i in range(c.n)]
    osum = np.full((c.n, 64), MARK, dtype=np.uint8)
    corrupt = np.full(c.n, MARK, dtype=np.uint8)
    sm = _sums(c.n, sums)
    rc, run = _call(c, lambda: lib().mec_heal_whole(c.h, _ptrs(srcs), sm.ctypes.data, total, _ptrs(outs), osum.ctypes.data,
                                                             corrupt.ctypes.data), srcs)
    for i in stale:
        assert (outs[i][flen:] == MARK).all(), f"heal wrote past the end of out file {i}"
    for i in range(c.n):
        if i not in stale:
            assert (osum[i] == MARK).all(), f"heal wrote the out sum of shard {i}, which was not asked for"
    return rc, [None if o is None else o[:flen] for o in outs], osum, corrupt, run


def check_decode(res, data, offset, length, hint=0):
    rc, out, got_hint, _ = res
    assert rc == length, rc
    if not np.array_equal(out, data[offset:offset + length]):
        bad = np.nonzero(out != data[offset:offset + length])[0]
        raise AssertionError(f"decode [{offset}, {offset + length}): {bad.size} bytes differ, first at object byte {offset + bad[0]}")
    assert got_hint == hint, got_hint


def check_heal(res, files, sums, stale, ds, rc=0, dropped=()):
    got_rc, outs, osum, corrupt, _ = res
    assert got_rc == rc, got_rc
    assert list(np.nonzero(corrupt)[0]) == sorted(dropped), corrupt
    for i in stale:
        if not np.array_equal(outs[i], files[i]):
            bad = np.nonzero(outs[i] != files[i])[0]
            raise AssertionError(f"healed shard file {i}: {bad.size} bytes differ, first at byte {bad[0]}")
        assert osum[i, :ds].tobytes() == sums[i], f"sum of healed shard {i}"


def digest_size(algo):
    return 64 if algo == BLAKE2B512 else 32


# ---------------------------------------------------------------- what launch_fused runs for a whole-file rebuild
def small_ok(opts, nblocks, num_sms):
    limit = opts["small_blocks"] if opts.get("small_blocks", -1) >= 0 else 5 * num_sms
    return nblocks <= limit and opts.get("eb", 0) <= 0 and opts.get("jit", -1) != 1


def rebuild_passes(S, first, nb, last_len):
    """launch_whole_rebuild's launches: (shard offset in the file, blocks, shard bytes)."""
    nfull = nb - 1 if last_len != S else nb
    out = [(first * S, nfull, S)] if nfull else []
    return out + ([((first + nfull) * S, 1, last_len)] if nfull < nb else [])


def rebuild_form(k, S, off, nblocks, S_pass, opts, num_sms):
    if small_ok(opts, nblocks, num_sms):
        return "small"
    row_bytes = S if nblocks > 1 else round_up(S_pass, 16) + 64
    if k > 16 or S % 16 or off + S_pass > row_bytes:
        return "dyn_bytewise"
    return "jit" if opts.get("jit") == 1 else "dyn_aligned"


def expected_forms(k, bs, S, sfs, offset, length, opts, num_sms):
    """Form counter deltas of the rebuild of a decode of [offset, offset + length) (length None: a heal of the whole part)."""
    if length is None:
        first, nb = 0, ceil_div(sfs, S)
    else:
        first, nb = offset // bs, (offset + length - 1) // bs - offset // bs + 1
    last_len = min(S, sfs - (first + nb - 1) * S)
    forms = {}
    for off, cnt, sp in rebuild_passes(S, first, nb, last_len):
        f = rebuild_form(k, S, off, cnt, sp, opts, num_sms)
        forms[f] = forms.get(f, 0) + 1
    return forms


def test_rebuild_passes_model():
    """The model above, on the shapes the tests rely on (pure host arithmetic)."""
    assert rebuild_passes(4096, 0, 10, 4096) == [(0, 10, 4096)]
    assert rebuild_passes(4096, 3, 2, 100) == [(3 * 4096, 1, 4096), (4 * 4096, 1, 100)]
    assert rebuild_passes(4096, 4, 1, 100) == [(4 * 4096, 1, 100)]
    one = dict(ONE_BLOCK)
    assert rebuild_form(4, 4096, 0, 10, 4096, one, 132) == "jit"
    assert rebuild_form(4, 4096, 0, 1, 4096, one, 132) == "jit"            # block 0 alone fits its one-block map
    assert rebuild_form(4, 4096, 4096, 1, 4096, one, 132) == "dyn_bytewise"
    assert rebuild_form(4, 4096, 4096, 2, 4096, one, 132) == "dyn_bytewise"
    assert rebuild_form(12, 1026, 0, 10, 1026, THROUGHPUT, 132) == "dyn_bytewise"
    assert rebuild_form(20, 4096, 0, 10, 4096, THROUGHPUT, 132) == "dyn_bytewise"
    assert rebuild_form(4, 4096, 0, 660, 4096, LATENCY, 132) == "small"
    assert rebuild_form(4, 4096, 0, 661, 4096, LATENCY, 132) == "dyn_aligned"


# ---------------------------------------------------------------- 1. default options: the throughput kernel without any switch
# (id, k, m, block size, algorithm, shards offline for the decodes and stale for the heal)
DEFAULT_GEOMS = {"rs4_2-aligned": (4, 2, 16 * KiB, SHA256, (1, 3)),                 # S = 4096
                 "rs12_4-bytewise": (12, 4, 12 * KiB + 17, BLAKE2B512, (0, 5, 6, 11))}  # S = 1026
# (id, blocks as a function of the SM count, options beyond jit, erasure blocks per CTA, CTAs as a function of the SM count)
DEFAULT_SHAPES = {"eb2": (lambda s: 5 * s + 37, {}, 2, None),         # 661-1055 blocks: the CTA shrinks to two blocks
                  "multipass": (lambda s: 8 * s + 5, dict(eb=4, grid_mult=1), 4, lambda s: s)}
DEFAULT_CASES = [pytest.param(g, s, 0, id=f"{g}-{s}-jit0") for g in DEFAULT_GEOMS for s in DEFAULT_SHAPES] + \
                [pytest.param("rs4_2-aligned", "eb2", 1, id="rs4_2-aligned-eb2-jit1")]


@pytest.mark.parametrize("geom,shape,jit", DEFAULT_CASES)
def test_default_options_throughput(mb, oracle, num_sms, geom, shape, jit):
    """A part too large for the latency kernel: the decode of its full blocks from block 0 with m shards offline, a range of
    them from block 3, the whole part (with its short last block), and a heal of m stale shards."""
    k, m, bs, algo, lost = DEFAULT_GEOMS[geom]
    blocks, extra, eb, grid = DEFAULT_SHAPES[shape]
    nfull = blocks(num_sms)
    size = nfull * bs + bs // 3 + 5
    data, files, sums = part(oracle, k, m, bs, algo, size)
    opts = dict(extra, jit=jit)
    c = codec(mb, k, m, bs, algo, opts)
    try:
        S, sfs = c.shard_size(), c.shard_file_size(size)
        srcs = [None if i in lost else files[i] for i in range(k + m)]
        for offset, length in ((0, nfull * bs), (3 * bs + 5, (nfull - 3) * bs - 12), (0, size)):
            res = decode(c, srcs, sums, offset, length, size)
            check_decode(res, data, offset, length)
            run = res[3]
            assert run["delta"] == expected_forms(k, bs, S, sfs, offset, length, opts, num_sms), (offset, length, run)
            if offset == 0 and length == nfull * bs:      # one launch: the record is the throughput pass
                last = run["last"]
                # the survivors sit at one arena stride, but a 3-D box needs eb x 288-byte rows to fill 128-byte granules
                mode = TMA_BYTEWISE if S % 16 else (TMA_RUNS if eb % 4 == 0 else TMA_PER_INPUT)
                assert last["last_eb"] == eb and last["last_tma_mode"] == mode, last
                if grid:
                    assert last["last_grid"] == grid(num_sms) and ceil_div(nfull, eb) > last["last_grid"], last
        res = heal(c, srcs, sums, set(lost), size)
        check_heal(res, files, sums, lost, digest_size(algo))
        assert res[4]["delta"] == expected_forms(k, bs, S, sfs, 0, None, opts, num_sms), res[4]
    finally:
        c.close()


# ---------------------------------------------------------------- 2. one-block launches at a shard offset > 0
# (id, k, m, block size, shards offline / stale): S % 16 == 0 in all three
ONE_BLOCK_GEOMS = {"rs4_2-1M": (4, 2, MiB, (1, 3)), "rs8_8-1M": (8, 8, MiB, (0, 3, 5, 6)), "rs8_8-10M": (8, 8, 10 * MiB, (0, 3, 5, 6))}
NFULL_ONE = 4


def one_block_ranges(bs, size):
    return {"inside_block3": (3 * bs + 7, bs - 16),
            "inside_short": (NFULL_ONE * bs + 5, size - NFULL_ONE * bs - 8),
            "full_into_short": (3 * bs + bs // 2 + 3, size - 3 * bs - bs // 2 - 4)}


@pytest.mark.parametrize("kernel", ["throughput", "latency"])
@pytest.mark.parametrize("op", ["heal", "inside_block3", "inside_short", "full_into_short"])
@pytest.mark.parametrize("geom", list(ONE_BLOCK_GEOMS))
def test_one_block_rebuild(mb, oracle, num_sms, geom, op, kernel):
    """Four full blocks and a short one.  With jit = 1, eb = 1 and small_blocks = 0 every rebuild runs on the throughput kernel,
    and the short last block of a heal, a range inside block 3, a range inside the short block and a range from block 3 into it
    are each launched as one block at a shard offset of 3 or 4 blocks into the file; the latency kernel is the control."""
    k, m, bs, lost = ONE_BLOCK_GEOMS[geom]
    size = NFULL_ONE * bs + bs // 2 + 12345
    algo = HIGHWAYHASH256
    data, files, sums = part(oracle, k, m, bs, algo, size)
    opts = ONE_BLOCK if kernel == "throughput" else LATENCY
    c = codec(mb, k, m, bs, algo, opts)
    try:
        S, sfs = c.shard_size(), c.shard_file_size(size)
        assert S % 16 == 0 and ceil_div(size - NFULL_ONE * bs, k) * (k - 1) < size - NFULL_ONE * bs
        srcs = [None if i in lost else files[i] for i in range(k + m)]
        if op == "heal":
            res = heal(c, srcs, sums, set(lost), size)
            check_heal(res, files, sums, lost, digest_size(algo))
            run, want = res[4], expected_forms(k, bs, S, sfs, 0, None, opts, num_sms)
        else:
            offset, length = one_block_ranges(bs, size)[op]
            res = decode(c, srcs, sums, offset, length, size)
            check_decode(res, data, offset, length)
            run, want = res[3], expected_forms(k, bs, S, sfs, offset, length, opts, num_sms)
        assert run["delta"] == want, run
        if kernel == "throughput":
            assert "small" not in want and want.get("dyn_bytewise", 0) >= 1, want
            assert run["last"]["last_eb"] == 1 and run["last"]["last_tma_mode"] == TMA_BYTEWISE, run
        else:
            assert set(want) == {"small"}, want
    finally:
        c.close()


# ---------------------------------------------------------------- 3. 10 MiB blocks on the latency kernel
# (k, m, shards offline for the decodes, stale sets for the heals)
TEN_MIB = {"rs12_4": (12, 4, (0, 5, 6, 11), {"data": (0, 5, 6, 11), "parity": (12, 13, 14, 15), "mixed": (2, 9, 13, 14)}),
           "rs8_8": (8, 8, (0, 2, 3, 5, 6, 7), {"data": tuple(range(8)), "parity": tuple(range(8, 16)),
                                                "mixed": (1, 3, 6, 8, 11, 12, 14, 15)})}


def ten_mib_size(nfull):
    return nfull * 10 * MiB + 3 * MiB + 4321


@pytest.mark.parametrize("algo", list(ALGOS))
@pytest.mark.parametrize("nfull", [3, 1], ids=["3_blocks", "1_block"])
@pytest.mark.parametrize("geom", list(TEN_MIB))
def test_ten_mib_blocks(mb, oracle, num_sms, geom, nfull, algo):
    """blockSizeV1 parts of three blocks and a tail and of one block and a tail: decodes from byte 0, from mid-block, from a
    block boundary and inside the tail with the most data shards the code allows offline; heals of data, parity and mixed sets.
    Every call hashes k or more shard files on one GPU thread each, which takes most of a second for SHA-256 and BLAKE2b-512 at
    three blocks; the hash does not change the rebuild, so those two run only the mid-block decode and the mixed heal there."""
    k, m, lost, stale_sets = TEN_MIB[geom]
    bs, a = 10 * MiB, ALGOS[algo]
    size = ten_mib_size(nfull)
    data, files, sums = part(oracle, k, m, bs, a, size)
    c = codec(mb, k, m, bs, a, LATENCY)
    try:
        S, sfs = c.shard_size(), c.shard_file_size(size)
        srcs = [None if i in lost else files[i] for i in range(k + m)]
        boundary = (nfull - 1) * bs if nfull > 1 else bs
        ranges = [(0, bs + 777), (bs // 2 + 3, nfull * bs - bs // 2), (boundary, size - boundary - 1),
                  (nfull * bs + 1000, size - nfull * bs - 2000)]
        if nfull == 3 and a != HIGHWAYHASH256:
            ranges, stale_sets = ranges[1:2], {"mixed": stale_sets["mixed"]}
        for offset, length in ranges:
            res = decode(c, srcs, sums, offset, length, size)
            check_decode(res, data, offset, length)
            assert res[3]["delta"] == expected_forms(k, bs, S, sfs, offset, length, LATENCY, num_sms), res[3]
        for name, stale in stale_sets.items():
            res = heal(c, [None if i in stale else files[i] for i in range(k + m)], sums, set(stale), size)
            check_heal(res, files, sums, stale, digest_size(a))
            assert res[4]["delta"] == {"small": 2}, (name, res[4])
    finally:
        c.close()


@pytest.mark.parametrize("bs", [64 * KiB, MiB, 10 * MiB], ids=["64K", "1M", "10M"])
def test_misaligned_shards_take_bytewise(mb, oracle, num_sms, bs):
    """RS(12,4) shards are not 16-byte multiples at any of these block sizes: the throughput kernel's byte-wise loader."""
    k, m, lost = 12, 4, (1, 4, 8, 11)
    nfull = 1 if bs == 10 * MiB else 3
    size = ten_mib_size(1) if bs == 10 * MiB else nfull * bs + bs // 2 + 99
    data, files, sums = part(oracle, k, m, bs, HIGHWAYHASH256, size)
    c = codec(mb, k, m, bs, HIGHWAYHASH256, THROUGHPUT)
    try:
        assert c.shard_size() % 16
        res = decode(c, [None if i in lost else files[i] for i in range(k + m)], sums, 0, size, size)
        check_decode(res, data, 0, size)
        assert res[3]["delta"] == {"dyn_bytewise": 2}, res[3]
        assert res[3]["last"]["last_tma_mode"] == TMA_BYTEWISE, res[3]
    finally:
        c.close()


# ---------------------------------------------------------------- 4. fail-over that reorders the staging arena
# The first k readers are staged at arena positions 0..k-1; a reader whose file or sum is wrong is dropped and the next alive
# reader takes its position, so the survivors, in index order, no longer sit at ascending positions.  (id, k, m, block size,
# readers with a flipped file byte, readers with a flipped sum byte, readers that must be dropped, survivor maps on TMA)
FAILOVER = [
    # 4 steps into position 0: two runs.  Reader 5's sum is wrong too, but reader 5 is never read: not reported
    ("rs4_2-two_runs", 4, 2, 16 * KiB, (0,), (5,), (0,), TMA_RUNS),
    # 4 steps into position 0 and is dropped in turn; 5 steps in
    ("rs4_2-newcomer_dropped", 4, 2, 16 * KiB, (0,), (4,), (0, 4), TMA_RUNS),
    ("rs12_4-five_runs", 12, 4, 12 * KiB, (4, 10), (1, 7), (1, 4, 7, 10), TMA_RUNS),
    # survivor positions 0,2 3,5 6,8 9,10 12..15 1,4,7 11: more than kMaxRuns = 6 runs, one map per input
    ("rs16_4-per_input", 16, 4, 16 * KiB, (1, 7), (4, 11), (1, 4, 7, 11), TMA_PER_INPUT),
]
FAILOVER_BLOCKS = 24


def corrupted(files, sums, bad_files, bad_sums):
    files = [f.copy() if i in bad_files else f for i, f in enumerate(files)]
    for i in bad_files:
        files[i][(i * 7919) % files[i].size] ^= 0x10
    sums = [bytes([s[0] ^ 0x01]) + s[1:] if i in bad_sums else s for i, s in enumerate(sums)]
    return files, sums


@pytest.mark.parametrize("kernel", ["throughput", "latency"])
@pytest.mark.parametrize("name,k,m,bs,bad_files,bad_sums,dropped,tma", [pytest.param(*f, id=f[0]) for f in FAILOVER])
def test_failover_reorders_arena(mb, oracle, num_sms, name, k, m, bs, bad_files, bad_sums, dropped, tma, kernel):
    """Decode of the full blocks and of the whole part, and a heal of the dropped readers from all n files: the dropped readers
    are rebuilt from survivors at shuffled arena positions, the heal hint / return code is errFileCorrupt and corrupt[] names
    exactly the dropped readers."""
    size = FAILOVER_BLOCKS * bs + bs // 2 + 3
    data, files, sums = part(oracle, k, m, bs, SHA256, size)
    srcs, bsums = corrupted(files, sums, bad_files, bad_sums)
    opts = dict(THROUGHPUT, eb=4) if kernel == "throughput" else LATENCY     # eb = 4: 3-D maps are possible (see above)
    c = codec(mb, k, m, bs, SHA256, opts)
    try:
        S, sfs = c.shard_size(), c.shard_file_size(size)
        assert S % 16 == 0
        for length in (FAILOVER_BLOCKS * bs, size):
            res = decode(c, srcs, bsums, 0, length, size)
            check_decode(res, data, 0, length, hint=FILE_CORRUPT)
            want = expected_forms(k, bs, S, sfs, 0, length, opts, num_sms)
            assert res[3]["delta"] == want, res[3]
            if kernel == "throughput" and length == FAILOVER_BLOCKS * bs:
                assert want == {"dyn_aligned": 1} and res[3]["last"]["last_tma_mode"] == tma, res[3]
        res = heal(c, srcs, bsums, set(dropped), size)
        check_heal(res, files, sums, dropped, digest_size(SHA256), rc=FILE_CORRUPT, dropped=dropped)
        assert res[4]["delta"] == expected_forms(k, bs, S, sfs, 0, None, opts, num_sms), res[4]
    finally:
        c.close()


@pytest.mark.parametrize("kernel", ["throughput", "latency"])
def test_failover_read_quorum(mb, oracle, kernel):
    """One offline reader and four corrupt ones of RS(12,4): decode and heal fail with errErasureReadQuorum, launch no rebuild
    and write nothing."""
    k, m, bs = 12, 4, 12 * KiB
    size = FAILOVER_BLOCKS * bs + 5
    _, files, sums = part(oracle, k, m, bs, SHA256, size)
    srcs, bsums = corrupted(files, sums, (3, 13), (5, 8))
    srcs[0] = None
    c = codec(mb, k, m, bs, SHA256, THROUGHPUT if kernel == "throughput" else LATENCY)
    try:
        rc, out, hint, run = decode(c, srcs, bsums, 0, size, size)
        assert rc == READ_QUORUM and (out == MARK).all() and run["delta"] == {}, (rc, run)
        rc, outs, osum, _, run = heal(c, srcs, bsums, {0, 1}, size)
        assert rc == READ_QUORUM and run["delta"] == {}, (rc, run)
        assert all((outs[i] == MARK).all() and (osum[i] == MARK).all() for i in (0, 1)), "a failed heal wrote its outputs"
    finally:
        c.close()


# ---------------------------------------------------------------- 5. wide stripes: k > 16 inputs, no tensor maps
@pytest.mark.parametrize("eb", [4, 1])
@pytest.mark.parametrize("k,m", [(20, 12), (32, 16)], ids=["rs20_12", "rs32_16"])
def test_wide_stripes(mb, oracle, k, m, eb):
    """Heal of m stale shards: the runtime-matrix kernel with four output rows per pass runs m / 4 passes over the matrix."""
    n = k + m
    bs = k * 1001 - 3                  # S = 1001
    size = 40 * bs                     # one launch: the record is of the 40-block pass
    stale = tuple(range(1, n, 2))[:m // 2] + tuple(range(k, n, 2))[:m - m // 2]
    assert len(set(stale)) == m
    data, files, sums = part(oracle, k, m, bs, BLAKE2B512, size)
    c = codec(mb, k, m, bs, BLAKE2B512, dict(THROUGHPUT, eb=eb))
    try:
        res = heal(c, [None if i in stale else files[i] for i in range(n)], sums, set(stale), size)
        check_heal(res, files, sums, stale, digest_size(BLAKE2B512))
        run = res[4]
        assert run["delta"] == {"dyn_bytewise": 1}, run
        want_eb = eb
        while want_eb > 1 and 2 * n * want_eb > 256:
            want_eb -= 1
        assert (run["last"]["last_eb"], run["last"]["last_tma_mode"], run["last"]["last_row_chunk"]) == (want_eb, TMA_BYTEWISE, 2), run
        lost = tuple(i for i in stale if i < k)
        res = decode(c, [None if i in lost else files[i] for i in range(n)], sums, 0, size, size)
        check_decode(res, data, 0, size)
    finally:
        c.close()


# ---------------------------------------------------------------- 6. no parity
def test_no_parity_read_quorum(mb, oracle):
    """RS(3,0): every reader is needed and nothing can be rebuilt; a corrupt file is errErasureReadQuorum."""
    k, bs = 3, 64 * KiB
    size = 5 * bs + 7
    data, files, sums = part(oracle, k, 0, bs, HIGHWAYHASH256, size)
    c = codec(mb, k, 0, bs, HIGHWAYHASH256, THROUGHPUT)
    try:
        res = decode(c, list(files), sums, 100, size - 200, size)
        check_decode(res, data, 100, size - 200)
        assert res[3]["delta"] == {}, res[3]
        srcs, _ = corrupted(files, sums, (1,), ())
        rc, out, hint, run = decode(c, srcs, sums, 0, size, size)
        assert rc == READ_QUORUM and (out == MARK).all() and run["delta"] == {}, (rc, run)
    finally:
        c.close()
