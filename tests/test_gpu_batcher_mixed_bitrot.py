"""Reads and heals of parts whose drives mix bitrot formats through the cross-request coalescer (mec_batcher_decode_mixed /
mec_batcher_heal_mixed), against the CPU oracle only.

A legacy part (SHA256, BLAKE2b512 or HighwayHash256: raw shard files with whole-file sums) of which some drives were healed holds
HighwayHash256S frames on those drives.  Sources are the oracle's Erasure.Encode of one object twice: with HighwayHash256S for the
streaming ("healed") drives and with the whole-file algorithm for the rest.  GET output must be the object slice, heal output the
oracle's HighwayHash256S part.N images of the stale drives.  Out buffers are page-locked, MARK-filled and GUARD bytes longer than
asked for on both sides; the guards must survive and every source must come back unchanged.

Calls with a whole-file reader among their k chosen share batches of one algorithm: the whole-file readers' shard files are staged
whole and hashed by ONE whole_hash_kernel launch per batch.  Covered: three geometries (RS(12,4) at 10 MiB with max_batch_blocks
<= 8), all three whole-file algorithms, three drive layouts, part lengths across block edges, GET ranges and heals of one and two
stale drives at once, shard files at every hash block edge in one launch, both kernel forms, offline drives with and without
`prefer`, rotated patterns with and without MEC_BATCHER_MIX_PATTERNS, bitrot redone on the private handle, the read quorum, every
refusal on a live batcher, the private paths, mixed traffic of every kind on one batcher, and all-streaming parts, which must ride
ordinary batches exactly as mec_batcher_decode_prefer / mec_batcher_heal requests do."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_batcher_transcode_blocksize import concurrently

pytestmark = pytest.mark.gpu
KiB, MiB = 1 << 10, 1 << 20
MARK = 0x5A
GUARD = 64
SHA256, HIGHWAYHASH256, HIGHWAYHASH256S, BLAKE2B512 = 1, 2, 3, 4
ALGOS = {"sha256": SHA256, "hh256": HIGHWAYHASH256, "blake2b": BLAKE2B512}
FILE_CORRUPT, READ_QUORUM, INVALID, UNSUPPORTED = -7, -10, -12, -102
GEOMS = {"rs4_2_1m": (4, 2, MiB, 64), "rs12_4_1m": (12, 4, MiB, 64), "rs12_4_10m": (12, 4, 10 * MiB, 8)}
FORMS = ("small", "fast3d", "fast3d_auto", "fast3d_semi", "fast", "fast_auto", "aligned", "aligned_auto", "runtime", "bytewise",
         "dyn_aligned", "dyn_runtime", "dyn_bytewise", "jit")
ENV = ("MEC_BATCHER_DEPTH", "MEC_BATCHER_MEMCPY", "MEC_BATCHER_GET_OUT", "MEC_BATCHER_DMA_BLOCKS", "MEC_SMALL_BLOCKS", "MEC_JIT")


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


@pytest.fixture(autouse=True)
def clean_env(monkeypatch, tmp_path):
    for name in ENV:
        monkeypatch.delenv(name, raising=False)
    monkeypatch.setenv("MEC_JIT_CACHE_DIR", str(tmp_path))


def layouts(n):
    """drive kinds: 'w' whole-file, 's' streaming (healed)"""
    return {"all_whole": "w" * n, "half_healed": "sw" * (n // 2), "one_healed": "s" + "w" * (n - 1)}


_ORACLE = {}


class Part:
    """one object encoded by the oracle in both formats, both kept in page-locked buffers"""

    def __init__(self, mb, oracle, k, m, bs, walgo, total, seed):
        key = (k, m, bs, walgo, total, seed)
        if key not in _ORACLE:
            data = np.random.default_rng(seed).integers(0, 256, total, dtype=np.uint8)
            sfiles, _ = oracle.erasure_encode(k, m, bs, HIGHWAYHASH256S, data)
            wfiles, sums = oracle.erasure_encode(k, m, bs, walgo, data)
            _ORACLE[key] = (data, sfiles, wfiles, sums)
        self.data, self.want, wfiles, sums = _ORACLE[key]
        self.mb, self.k, self.m, self.n, self.bs, self.walgo, self.total = mb, k, m, k + m, bs, walgo, total
        self.S = -(-bs // k)
        self.sfs = wfiles[0].size
        self.stream = [self._pin(f) for f in self.want]
        self.whole = [self._pin(f) for f in wfiles]
        self.sums = np.zeros((self.n, 64), dtype=np.uint8)
        for i, d in enumerate(sums):
            self.sums[i, :len(d)] = np.frombuffer(d, dtype=np.uint8)
        self._copies = [f.copy() for f in self.stream + self.whole]

    def _pin(self, f):
        a = self.mb.pinned_array(max(f.size, 1))[:f.size]
        a[:] = f
        return a

    def files(self, kinds, offline=()):
        """kinds[i]: 's' / 'w' -> (files, algos); offline drives are None"""
        files = [None if i in offline else self.stream[i] if t == "s" else self.whole[i] for i, t in enumerate(kinds)]
        algos = [HIGHWAYHASH256S if t == "s" else self.walgo for t in kinds]
        return files, algos

    def unchanged(self):
        return all(np.array_equal(a, b) for a, b in zip(self.stream + self.whole, self._copies))

    def free(self):
        for a in self.stream + self.whole:
            self.mb.lib().mec_free_pinned(a.ctypes.data)


def _ptrs(arrs):
    return (C.c_void_p * len(arrs))(*[None if a is None else a.ctypes.data for a in arrs])


def _buf(mb, n, pinned):
    b = mb.pinned_array(n) if pinned else np.empty(n, dtype=np.uint8)
    b[:] = MARK
    return b


def _free(mb, b, pinned):
    if pinned:
        mb.lib().mec_free_pinned(b.ctypes.data)


def get(mb, bat, p, kinds, offset, length, offline=(), prefer=None, pinned=True, files=None):
    """mec_batcher_decode_mixed into a guarded buffer -> (rc, bytes, heal_hint)"""
    f, algos = p.files(kinds, offline)
    if files is not None:
        f = [None if a is None else files[i] for i, a in enumerate(f)]
    dst = _buf(mb, length + 2 * GUARD, pinned)
    hint = C.c_int(MARK)
    pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
    rc = mb.lib().mec_batcher_decode_mixed(bat.h, (C.c_int32 * p.n)(*algos), _ptrs(f), p.sums.ctypes.data,
                                           None if pf is None else pf.ctypes.data, offset, length, p.total,
                                           dst.ctypes.data + GUARD, C.byref(hint))
    assert (dst[:GUARD] == MARK).all() and (dst[GUARD + length:] == MARK).all(), "GET wrote outside its range"
    out = dst[GUARD:GUARD + length].copy()
    _free(mb, dst, pinned)
    return rc, out, hint.value


def heal(mb, bat, p, kinds, stale, offline=(), prefer=None, pinned=True, files=None):
    """mec_batcher_heal_mixed into guarded out files -> (rc, outs, corrupt)"""
    f, algos = p.files(kinds, offline)
    if files is not None:
        f = [None if a is None else files[i] for i, a in enumerate(f)]
    flen = p.want[0].size
    bufs = [_buf(mb, flen + 2 * GUARD, pinned) if i in stale else None for i in range(p.n)]
    corrupt = np.full(p.n, MARK, dtype=np.uint8)
    pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
    op = (C.c_void_p * p.n)(*[None if b is None else b.ctypes.data + GUARD for b in bufs])
    rc = mb.lib().mec_batcher_heal_mixed(bat.h, (C.c_int32 * p.n)(*algos), _ptrs(f), p.sums.ctypes.data,
                                         None if pf is None else pf.ctypes.data, p.total, op, corrupt.ctypes.data)
    outs = [None] * p.n
    for i, b in enumerate(bufs):
        if b is None:
            continue
        assert (b[:GUARD] == MARK).all() and (b[GUARD + flen:] == MARK).all(), f"heal wrote outside out file {i}"
        outs[i] = b[GUARD:GUARD + flen].copy()
        _free(mb, b, pinned)
    return rc, outs, corrupt


def check_get(res, p, offset, length, hint=0):
    rc, out, h = res
    assert rc == length and h == hint, (p.total, offset, length, rc, h)
    if not np.array_equal(out, p.data[offset:offset + length]):
        bad = np.nonzero(out != p.data[offset:offset + length])[0]
        raise AssertionError(f"GET [{offset}, {offset + length}) of {p.total}: {bad.size} bytes differ, first at {bad[0]}")


def check_heal(res, p, stale, rc=0, corrupt=()):
    got_rc, outs, cr = res
    assert got_rc == rc, (p.total, stale, got_rc)
    assert cr.tolist() == [1 if i in corrupt else 0 for i in range(p.n)], cr
    for i in stale:
        assert np.array_equal(outs[i], p.want[i]), f"healed drive {i} of a {p.total}-byte part differs from the oracle"


NAMES = ("batches", "requests", "redone", "reads_whole", "reads_whole_serial", "whole_hash_launches", "mixed_batches", "launches",
         "bytes_h2d") + tuple("form_" + f for f in FORMS)


def counters(bat):
    return {s: bat.stat(s) for s in NAMES}


def delta(bat, before):
    return {s: v - before[s] for s, v in counters(bat).items()}


def lengths(bs):
    return [1, bs - 1, bs + 1, 2 * bs + 4321]


def ranges(total, bs):
    """inside a block, across a block edge, over the tail, the whole part"""
    out = [(min(5, total - 1), min(1000, total - min(5, total - 1)))]
    if total > bs:
        out.append((bs - 100, min(200, total - bs + 100)))
    t = min(total, 777)
    out.append((total - t, t))
    out.append((0, total))
    return out


def read_range(p, offset, length):
    """Erasure.Decode's blocks of [offset, offset + length): -> (nblocks, last shard length)"""
    b0 = offset // p.bs
    b1 = (offset + length) // p.bs - (1 if (offset + length) % p.bs == 0 else 0)
    b1 = min(b1, -(-p.sfs // p.S) - 1)
    return b1 - b0 + 1, min(p.S, p.sfs - b1 * p.S)


def h2d(p, kinds, readers, offset, length):
    """mec_decode_mixed's bytes_h2d for readers `readers`: one shard file per whole-file reader, frames of the range per streaming"""
    nb, last = read_range(p, offset, length)
    frames = (nb - 1) * (32 + p.S) + 32 + last
    return sum(p.sfs if kinds[i] == "w" else frames for i in readers)


def first_k(p, usable):
    return [i for i in range(p.n) if usable(i)][:p.k]


@pytest.fixture(scope="module", params=list(GEOMS))
def geom_batcher(request, mb):
    k, m, bs, mbb = GEOMS[request.param]
    bat = mb.Batcher(k, m, bs, max_batch_blocks=mbb, max_wait_us=200_000)
    yield (k, m, bs), bat
    bat.close()


@pytest.mark.parametrize("layout", ["all_whole", "half_healed", "one_healed"])
@pytest.mark.parametrize("algo", list(ALGOS))
def test_merged_vs_oracle(mb, oracle, geom_batcher, algo, layout):
    """GET ranges and heals of one and two stale drives (data and parity) of every part length at once: exact bytes and part.N
    images, every call completed merged, fewer batches than calls, one hash launch per batch, and mec_decode_mixed's bytes_h2d."""
    (k, m, bs), bat = geom_batcher
    n = k + m
    kinds = layouts(n)[layout]
    parts = [Part(mb, oracle, k, m, bs, ALGOS[algo], t, 100 + q) for q, t in enumerate(lengths(bs))]
    stales = [(k - 1,), (1, n - 1)]
    try:
        calls, checks, want_h2d = [], [], 0
        for p in parts:
            for off, ln in ranges(p.total, bs):
                calls.append(lambda p=p, off=off, ln=ln: get(mb, bat, p, kinds, off, ln))
                checks.append(lambda res, p=p, off=off, ln=ln: check_get(res, p, off, ln))
                want_h2d += h2d(p, kinds, first_k(p, lambda i: True), off, ln)
            for st in stales:
                calls.append(lambda p=p, st=st: heal(mb, bat, p, kinds, st))
                checks.append(lambda res, p=p, st=st: check_heal(res, p, st))
                want_h2d += h2d(p, kinds, first_k(p, lambda i, st=st: i not in st), 0, p.total)
        before = counters(bat)
        res = concurrently(calls)
        d = delta(bat, before)
        for chk, r in zip(checks, res):
            chk(r)
        assert all(p.unchanged() for p in parts), "a source was written"
        assert d["reads_whole"] == len(calls) and d["requests"] == len(calls) and 0 < d["batches"] < len(calls), d
        assert d["whole_hash_launches"] == d["batches"] and d["redone"] == 0 and d["reads_whole_serial"] == 0, d
        assert d["bytes_h2d"] == want_h2d, (d["bytes_h2d"], want_h2d)
    finally:
        for p in parts:
            p.free()


@pytest.mark.parametrize("algo", list(ALGOS))
def test_hash_block_edges_one_launch(mb, oracle, monkeypatch, algo):
    """One merged batch of GETs whose shard files are exactly 1 .. 4097 bytes, across every algorithm's block edges: one hash launch
    over files of different lengths, no redo, exact bytes."""
    monkeypatch.setenv("MEC_BATCHER_DEPTH", "0")
    lens = [1, 31, 32, 33, 55, 56, 63, 64, 65, 127, 128, 129, 4097]
    k, m = 12, 4
    bat = mb.Batcher(k, m, MiB, max_batch_blocks=len(lens), max_wait_us=2_000_000)
    kinds = layouts(k + m)["half_healed"]
    parts = [Part(mb, oracle, k, m, MiB, ALGOS[algo], k * ln, 200 + ln) for ln in lens]
    try:
        assert [p.sfs for p in parts] == lens
        before = counters(bat)
        res = concurrently([lambda p=p: get(mb, bat, p, kinds, 0, p.total) for p in parts])
        d = delta(bat, before)
        for p, r in zip(parts, res):
            check_get(r, p, 0, p.total)
        assert d["batches"] == 1 and d["whole_hash_launches"] == 1 and d["reads_whole"] == len(lens) and d["redone"] == 0, d
    finally:
        for p in parts:
            p.free()
        bat.close()


@pytest.mark.parametrize("form", ["throughput", "latency"])
def test_kernel_forms(mb, oracle, monkeypatch, form):
    """Merged batches with whole-file readers on the throughput kernel (MEC_SMALL_BLOCKS=0) and on the latency kernel."""
    monkeypatch.setenv("MEC_JIT", "0")
    if form == "throughput":
        monkeypatch.setenv("MEC_SMALL_BLOCKS", "0")
    k, m = 12, 4
    bat = mb.Batcher(k, m, MiB, max_batch_blocks=64, max_wait_us=200_000)
    kinds = layouts(k + m)["half_healed"]
    parts = [Part(mb, oracle, k, m, MiB, SHA256, t, 300 + t % 97) for t in (MiB - 1, 2 * MiB + 4321, 3 * MiB)]
    try:
        before = counters(bat)
        calls = [lambda p=p: get(mb, bat, p, kinds, 0, p.total, offline=(2,)) for p in parts]
        calls += [lambda p=p: heal(mb, bat, p, kinds, (3, 14)) for p in parts]
        res = concurrently(calls)
        d = delta(bat, before)
        for p, r in zip(parts, res[:3]):
            check_get(r, p, 0, p.total)
        for p, r in zip(parts, res[3:]):
            check_heal(r, p, (3, 14))
        forms = {f: d["form_" + f] for f in FORMS if d["form_" + f]}
        if form == "latency":
            assert forms.get("small", 0) > 0, forms
        else:
            assert forms and "small" not in forms, forms
        assert d["reads_whole"] == len(calls) and d["redone"] == 0, d
    finally:
        for p in parts:
            p.free()
        bat.close()


@pytest.mark.parametrize("use_prefer", [False, True])
def test_offline_drives(mb, oracle, use_prefer):
    """Data and parity drives offline, the same for every call, with and without `prefer`: exact, all merged."""
    k, m = 12, 4
    bat = mb.Batcher(k, m, MiB, max_batch_blocks=64, max_wait_us=200_000)
    kinds = layouts(k + m)["half_healed"]
    prefer = [1 if i in (3, 8, 14, 15) else 0 for i in range(k + m)] if use_prefer else None
    off = (1, 7, 12)
    parts = [Part(mb, oracle, k, m, MiB, BLAKE2B512, t, 400 + q) for q, t in enumerate([5000, MiB + 1, 2 * MiB + 4321])]
    try:
        before = counters(bat)
        calls = [lambda p=p: get(mb, bat, p, kinds, 3, p.total - 3, offline=off, prefer=prefer) for p in parts]
        calls += [lambda p=p: heal(mb, bat, p, kinds, (0,), offline=off, prefer=prefer) for p in parts]
        res = concurrently(calls)
        d = delta(bat, before)
        for p, r in zip(parts, res[:3]):
            check_get(r, p, 3, p.total - 3)
        for p, r in zip(parts, res[3:]):
            check_heal(r, p, (0,))
        assert d["reads_whole"] == len(calls) and d["redone"] == 0 and d["reads_whole_serial"] == 0, d
    finally:
        for p in parts:
            p.free()
        bat.close()


@pytest.mark.parametrize("mix", [False, True])
def test_rotated_patterns(mb, oracle, mix):
    """One drive offline, rotating with the call: with MEC_BATCHER_MIX_PATTERNS the reader sets share batches ("mixed_batches" > 0),
    without it they never do; exact either way."""
    k, m = 12, 4
    bat = mb.Batcher(k, m, MiB, max_batch_blocks=64, max_wait_us=200_000, mix_patterns=mix)
    kinds = layouts(k + m)["half_healed"]
    parts = [Part(mb, oracle, k, m, MiB, SHA256, t, 500 + q) for q, t in enumerate([MiB // 3, MiB - 1, MiB + 1, 2 * MiB + 99] * 2)]
    try:
        before = counters(bat)
        calls = [lambda q=q, p=p: get(mb, bat, p, kinds, 0, p.total, offline=((q * 3) % 16,)) for q, p in enumerate(parts)]
        res = concurrently(calls)
        d = delta(bat, before)
        for p, r in zip(parts, res):
            check_get(r, p, 0, p.total)
        assert d["reads_whole"] == len(calls) and d["redone"] == 0, d
        assert (d["mixed_batches"] > 0) == mix and d["whole_hash_launches"] == d["batches"], d
    finally:
        for p in parts:
            p.free()
        bat.close()


@pytest.mark.parametrize("where", ["whole_file", "healed_frame"])
def test_bitrot_redone(mb, oracle, where):
    """A flipped byte in a chosen whole-file reader, or in a frame of a chosen healed drive: that GET and that heal are redone alone
    through mec_decode_mixed / mec_heal_mixed (heal_hint / rc -7, corrupt[i], exact output) while their neighbours complete merged."""
    k, m = 12, 4
    bat = mb.Batcher(k, m, MiB, max_batch_blocks=64, max_wait_us=200_000)
    kinds = layouts(k + m)["half_healed"]   # drive 4 streams, drive 5 is whole-file
    parts = [Part(mb, oracle, k, m, MiB, SHA256, t, 600 + q) for q, t in enumerate([MiB - 1, MiB + 1, 2 * MiB + 4321, 3000])]
    bad = parts[2]
    drive = 5 if where == "whole_file" else 4
    f = bad.whole[drive] if where == "whole_file" else bad.stream[drive]
    pos = f.size // 2 if where == "whole_file" else 32 + 1000   # inside the first frame's shard
    f[pos] ^= 0x20
    try:
        before = counters(bat)
        calls = [lambda p=p: get(mb, bat, p, kinds, 0, p.total) for p in parts]
        calls += [lambda p=p: heal(mb, bat, p, kinds, (15,)) for p in parts]
        res = concurrently(calls)
        d = delta(bat, before)
        for p, r in zip(parts, res[:4]):
            check_get(r, p, 0, p.total, hint=FILE_CORRUPT if p is bad else 0)
        for p, r in zip(parts, res[4:]):
            check_heal(r, p, (15,), rc=FILE_CORRUPT if p is bad else 0, corrupt=(drive,) if p is bad else ())
        assert d["redone"] == 2 and d["reads_whole_serial"] == 2 and d["reads_whole"] == len(calls) - 2, d
    finally:
        f[pos] ^= 0x20
        for p in parts:
            p.free()
        bat.close()


def test_read_quorum(mb, oracle):
    """Fewer than k readable drives is MEC_ERR_READ_QUORUM before anything is queued; exactly k readable with one of them failing
    its digest is MEC_ERR_READ_QUORUM from the redo."""
    k, m = 4, 2
    bat = mb.Batcher(k, m, MiB, max_batch_blocks=64, max_wait_us=1000)
    kinds = layouts(k + m)["half_healed"]
    p = Part(mb, oracle, k, m, MiB, SHA256, MiB + 77, 700)
    try:
        before = counters(bat)
        assert get(mb, bat, p, kinds, 0, p.total, offline=(0, 1, 2))[0] == READ_QUORUM
        assert heal(mb, bat, p, kinds, (0, 1), offline=(2,))[0] == READ_QUORUM
        assert delta(bat, before)["requests"] == 0
        p.whole[1][10] ^= 1
        assert get(mb, bat, p, kinds, 0, p.total, offline=(4, 5))[0] == READ_QUORUM
        rc, _, corrupt = heal(mb, bat, p, kinds, (5,), offline=(4,))
        assert rc == READ_QUORUM
        p.whole[1][10] ^= 1
        assert delta(bat, before)["redone"] == 2
    finally:
        p.free()
        bat.close()


def test_refusals_live_batcher(mb, oracle):
    """Every refusal, in the single-codec calls' order, before anything is queued: "requests" does not grow."""
    k, m = 12, 4
    bat = mb.Batcher(k, m, MiB, max_batch_blocks=64, max_wait_us=1000)
    p = Part(mb, oracle, k, m, MiB, SHA256, 2 * MiB + 5, 800)
    kinds = layouts(k + m)["half_healed"]
    L = mb.lib()
    files, algos = p.files(kinds)
    fp = _ptrs(files)
    al = (C.c_int32 * 16)(*algos)
    bad_al = (C.c_int32 * 16)(*([9] + algos[1:]))
    two_al = (C.c_int32 * 16)(*[SHA256 if i % 4 == 1 else BLAKE2B512 if i % 2 else HIGHWAYHASH256S for i in range(16)])
    dst = mb.pinned_array(4096)
    sm = p.sums.ctypes.data

    def dec(al_, fp_, sums, off, ln, total, d, hint=True):
        h = C.c_int(MARK)
        rc = L.mec_batcher_decode_mixed(bat.h, al_, fp_, sums, None, off, ln, total, d, C.byref(h) if hint else None)
        return rc, h.value if hint else 0

    outs = [None] * 16
    outs[15] = mb.pinned_array(p.want[0].size)
    op = _ptrs(outs)

    def hl(al_, fp_, sums, total, op_):
        corrupt = np.full(16, MARK, dtype=np.uint8)
        rc = L.mec_batcher_heal_mixed(bat.h, al_, fp_, sums, None, total, op_, corrupt.ctypes.data)
        return rc, corrupt
    try:
        before = counters(bat)
        D = dst.ctypes.data
        assert dec(None, fp, sm, 0, 10, p.total, D) == (INVALID, 0)
        assert dec(al, None, sm, 0, 10, p.total, D) == (INVALID, 0)
        assert dec(bad_al, fp, sm, -1, 10, p.total, D) == (INVALID, 0)          # the range before the formats
        assert dec(bad_al, fp, sm, 0, -1, p.total, D) == (INVALID, 0)
        assert dec(bad_al, fp, sm, p.total - 5, 10, p.total, D) == (INVALID, 0)
        assert dec(bad_al, fp, sm, 0, 0, p.total, D) == (0, 0)                  # the empty read before dst and the formats
        assert dec(bad_al, fp, sm, 0, 10, p.total, None) == (INVALID, 0)       # dst before the formats
        assert dec(bad_al, fp, sm, 0, 10, p.total, D) == (INVALID, 0)
        assert dec(al, fp, None, 0, 10, p.total, D) == (INVALID, 0)             # NULL sums beside a whole-file reader
        assert dec(two_al, fp, sm, 0, 10, p.total, D) == (UNSUPPORTED, 0)
        off = _ptrs([None if i < 5 else f for i, f in enumerate(files)])
        assert dec(al, off, sm, 0, 10, p.total, D) == (READ_QUORUM, 0)
        assert dec(two_al, off, sm, 0, 10, p.total, D) == (UNSUPPORTED, 0)     # the formats before the quorum
        assert hl(None, fp, sm, p.total, op)[0] == INVALID
        assert hl(al, fp, sm, p.total, None)[0] == INVALID
        rc, corrupt = hl(bad_al, fp, sm, p.total, op)
        assert rc == INVALID and corrupt.tolist() == [0] * 16                   # corrupt[] cleared before the formats
        assert hl(two_al, fp, sm, 0, op)[0] == UNSUPPORTED                      # the formats before the empty heal
        assert hl(al, fp, sm, 0, op)[0] == 0
        assert hl(al, off, sm, p.total, op)[0] == READ_QUORUM
        # a stale drive is never read: its format does not matter
        st_al = (C.c_int32 * 16)(*(algos[:15] + [BLAKE2B512]))
        assert hl(st_al, fp, sm, 0, op)[0] == 0
        assert delta(bat, before)["requests"] == 0
    finally:
        L.mec_free_pinned(dst.ctypes.data)
        L.mec_free_pinned(outs[15].ctypes.data)
        p.free()
        bat.close()


@pytest.mark.parametrize("path", ["pageable", "oversize", "memcpy"])
def test_private_paths(mb, oracle, monkeypatch, path):
    """Pageable buffers, a part of more blocks than max_batch_blocks and MEC_BATCHER_MEMCPY run on the private handle
    ("reads_whole_serial"), with exact outputs."""
    if path == "memcpy":
        monkeypatch.setenv("MEC_BATCHER_MEMCPY", "1")
    k, m = 12, 4
    bat = mb.Batcher(k, m, MiB, max_batch_blocks=2, max_wait_us=1000)
    kinds = layouts(k + m)["one_healed"]
    total = 3 * MiB + 9 if path == "oversize" else MiB + 9
    p = Part(mb, oracle, k, m, MiB, HIGHWAYHASH256, total, 900)
    try:
        before = counters(bat)
        pinned = path != "pageable"
        check_get(get(mb, bat, p, kinds, 7, total - 7, pinned=pinned), p, 7, total - 7)
        check_heal(heal(mb, bat, p, kinds, (2, 13), pinned=pinned), p, (2, 13))
        d = delta(bat, before)
        assert d["reads_whole_serial"] == 2 and d["reads_whole"] == 0 and d["requests"] == 0, d
        assert p.unchanged()
    finally:
        p.free()
        bat.close()


def test_mixed_traffic(mb, oracle):
    """PUTs, plain GETs and heals, and SHA256 and BLAKE2b512 mixed calls on one batcher at once: every output exact and no redo
    (a batch hashing two algorithms would fail the other algorithm's sums and redo its calls)."""
    k, m = 12, 4
    bat = mb.Batcher(k, m, MiB, max_batch_blocks=64, max_wait_us=200_000)
    kinds = layouts(k + m)["half_healed"]
    sha = [Part(mb, oracle, k, m, MiB, SHA256, t, 1000 + q) for q, t in enumerate([5000, MiB + 1, 2 * MiB + 7])]
    blk = [Part(mb, oracle, k, m, MiB, BLAKE2B512, t, 1100 + q) for q, t in enumerate([777, MiB - 1, 2 * MiB + 7])]
    objs = [np.random.default_rng(1200 + q).integers(0, 256, t, dtype=np.uint8) for q, t in enumerate([3000, MiB + 5, 2 * MiB])]
    srcs = [mb.pinned_array(max(o.size, 1))[:o.size] for o in objs]
    for a, o in zip(srcs, objs):
        a[:] = o
    plain = sha  # their streaming images, read through the old calls
    try:
        before = counters(bat)
        calls = [lambda p=p: get(mb, bat, p, kinds, 1, p.total - 1) for p in sha + blk]
        calls += [lambda p=p: heal(mb, bat, p, kinds, (0, 15)) for p in sha + blk]
        calls += [lambda a=a: bat.encode(a, pinned=True) for a in srcs]
        calls += [lambda p=p: bat.decode(p.stream, 0, p.total, p.total, dst=mb.pinned_array(p.total)) for p in plain]
        calls += [lambda p=p: bat.heal([None if i == 3 else f for i, f in enumerate(p.stream)], [i == 3 for i in range(16)], p.total,
                                       pinned=True) for p in plain]
        res = concurrently(calls)
        d = delta(bat, before)
        for p, r in zip(sha + blk, res[:6]):
            check_get(r, p, 1, p.total - 1)
        for p, r in zip(sha + blk, res[6:12]):
            check_heal(r, p, (0, 15))
        for o, files in zip(objs, res[12:15]):
            want, _ = oracle.erasure_encode(k, m, MiB, HIGHWAYHASH256S, o)
            assert all(np.array_equal(f, w) for f, w in zip(files, want))
            for f in files:
                mb.lib().mec_free_pinned(f.ctypes.data)
        for p, (out, hint) in zip(plain, res[15:18]):
            assert hint == 0 and np.array_equal(out, p.data)
        for p, (outs, rc, _) in zip(plain, res[18:21]):
            assert rc == 0 and np.array_equal(outs[3], p.want[3])
        assert d["reads_whole"] == 12 and d["redone"] == 0 and d["reads_whole_serial"] == 0, d
    finally:
        for a in srcs:
            mb.lib().mec_free_pinned(a.ctypes.data)
        for p in sha + blk:
            p.free()
        bat.close()


def test_all_streaming_rides_ordinary_batches(mb, oracle, monkeypatch):
    """All-streaming parts through the new calls give the bytes of mec_batcher_decode_prefer / mec_batcher_heal and ride ordinary
    batches: no hash launch, no "reads_whole", and the same launches as the same workload through the old calls (one GET batch and
    one heal batch each: MEC_BATCHER_DEPTH=0 and max_batch_blocks equal to the workload's blocks)."""
    monkeypatch.setenv("MEC_BATCHER_DEPTH", "0")
    k, m = 12, 4
    parts = [Part(mb, oracle, k, m, MiB, SHA256, t, 1300 + q) for q, t in enumerate([4000, MiB + 1, 2 * MiB + 4321])]
    kinds = "s" * 16
    get_blocks = sum((p.total - 2) // MiB + 2 for p in parts)
    heal_blocks = sum(-(-p.total // MiB) for p in parts)
    stale = (2, 13)
    try:
        runs = {}
        for how in ("old", "new"):
            deltas = []
            for what, blocks in (("get", get_blocks), ("heal", heal_blocks)):
                bat = mb.Batcher(k, m, MiB, max_batch_blocks=blocks, max_wait_us=2_000_000)
                before = counters(bat)
                if what == "get":
                    if how == "new":
                        calls = [lambda p=p: get(mb, bat, p, kinds, 2, p.total - 2) for p in parts]
                    else:
                        calls = [lambda p=p: bat.decode(p.stream, 2, p.total - 2, p.total, dst=mb.pinned_array(p.total)) for p in parts]
                else:
                    if how == "new":
                        calls = [lambda p=p: heal(mb, bat, p, kinds, stale) for p in parts]
                    else:
                        calls = [lambda p=p: bat.heal([None if i in stale else f for i, f in enumerate(p.stream)],
                                                      [i in stale for i in range(16)], p.total, pinned=True) for p in parts]
                res = concurrently(calls)
                d = delta(bat, before)
                bat.close()
                for p, r in zip(parts, res):
                    if what == "get":
                        out, hint = (r[1], r[2]) if how == "new" else r
                        if how == "new":
                            assert r[0] == p.total - 2
                        assert hint == 0 and np.array_equal(out[:p.total - 2], p.data[2:])
                    else:
                        outs, rc = (r[1], r[0]) if how == "new" else (r[0], r[1])
                        assert rc == 0 and all(np.array_equal(outs[i][:p.want[i].size], p.want[i]) for i in stale)
                assert d["batches"] == 1 and d["whole_hash_launches"] == 0 and d["reads_whole"] == 0 and d["redone"] == 0, d
                deltas.append(d["launches"])
            runs[how] = deltas
        assert runs["new"] == runs["old"], runs
    finally:
        for p in parts:
            p.free()
