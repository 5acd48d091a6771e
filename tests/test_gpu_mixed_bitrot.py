"""Decode and heal of parts whose drives mix bitrot formats (mec_decode_mixed / mec_heal_mixed), against the CPU oracle.

A legacy part (SHA256, BLAKE2b512 or HighwayHash256: raw shard files with whole-file sums) of which some drives were healed holds
HighwayHash256S frames on those drives: healObject heals into the streaming format.  Sources are the oracle's Erasure.Encode of one
object twice: with HighwayHash256S for the streaming ("healed") drives and with the whole-file algorithm for the rest.  Decode
output must be the object slice; heal output the oracle's HighwayHash256S part.N images of the stale drives.

Fail-over is parallelReader's over both reader kinds: a whole-file reader is hashed when first chosen (one whole_hash_kernel launch
per round of newcomers), a streaming reader is checked frame by frame, and a whole-file reader that is never chosen is never
hashed.  Output buffers and out files are MARK-filled and GUARD bytes longer than asked for; the guard must survive, and every
source must come back unchanged.  Both kernel forms run: the throughput form (small_blocks = 0, jit = 0) and the latency form.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_kernel_forms import form_counts, form_delta, jit_cache, mb  # noqa: F401

pytestmark = pytest.mark.gpu
KiB, MiB = 1 << 10, 1 << 20
MARK = 0x5A
GUARD = 64
SHA256, HIGHWAYHASH256, HIGHWAYHASH256S, BLAKE2B512 = 1, 2, 3, 4
ALGOS = {"sha256": SHA256, "hh256": HIGHWAYHASH256, "blake2b": BLAKE2B512}
FILE_CORRUPT, READ_QUORUM = -7, -10
DISPATCH_ENV = ("MEC_SMALL_BLOCKS", "MEC_EB", "MEC_FORCE_BYTEWISE", "MEC_FORCE_DYNAMIC", "MEC_JIT", "MEC_GRID_MULT",
                "MEC_BALANCE_GRID", "MEC_NO_ROWS3D", "MEC_USE_AUTO", "MEC_STATIC_GROUPS", "MEC_CHUNK_BLOCKS")
THROUGHPUT = dict(jit=0, small_blocks=0)
LATENCY = dict(jit=0)
FORMS = {"throughput": THROUGHPUT, "latency": LATENCY}
GEOMS = {"rs4_2_1m": (4, 2, MiB), "rs12_4_1m": (12, 4, MiB), "rs12_4_10m": (12, 4, 10 * MiB)}


@pytest.fixture(autouse=True)
def clean_dispatch(monkeypatch, jit_cache):  # noqa: F811
    for name in DISPATCH_ENV:
        monkeypatch.delenv(name, raising=False)


_PARTS = {}


def part(oracle, k, m, bs, walgo, total):
    """(object, HighwayHash256S part.N images, raw shard files, whole-file sums) of one object, cached across tests"""
    key = (k, m, bs, walgo, total)
    if key not in _PARTS:
        data = np.random.default_rng(total % 100003 + 7 * k + m + walgo).integers(0, 256, total, dtype=np.uint8)
        sfiles, _ = oracle.erasure_encode(k, m, bs, HIGHWAYHASH256S, data)
        wfiles, sums = oracle.erasure_encode(k, m, bs, walgo, data)
        _PARTS[key] = (data, sfiles, wfiles, sums)
    return _PARTS[key]


def drives(p, kinds, walgo):
    """kinds[i]: 's' streaming, 'w' whole-file, '-' offline -> (files, algos)"""
    _, sfiles, wfiles, _ = p
    files = [sfiles[i] if t == "s" else wfiles[i] if t == "w" else None for i, t in enumerate(kinds)]
    algos = [HIGHWAYHASH256S if t == "s" else walgo for t in kinds]
    return files, algos


def codec(mb, k, m, bs, opts):  # noqa: F811
    c = mb.Codec(k, m, bs)
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
    for i, d in enumerate(sums or []):
        if d is not None:
            sm[i, :len(d)] = np.frombuffer(d, dtype=np.uint8)
    return sm


def _pf(prefer):
    return None if prefer is None else np.asarray(prefer, dtype=np.uint8)


STATS = ("whole_hash_launches", "corrupt_shards", "bytes_h2d", "bytes_d2h", "blocks_read", "shards_rebuilt")


def _call(c, fn, srcs):
    before = {s: c.stat(s) for s in STATS}
    forms = form_counts(c)
    copies = [None if f is None else f.copy() for f in srcs]
    rc = fn()
    for i, (f, g) in enumerate(zip(srcs, copies)):
        assert f is None or np.array_equal(f, g), f"source file {i} was written"
    run = {s: c.stat(s) - before[s] for s in STATS}
    run["forms"] = form_delta(forms, form_counts(c))
    return rc, run


def decode(c, files, algos, sums, offset, length, total, prefer=None):
    """mec_decode_mixed into a MARK-filled buffer GUARD bytes longer than `length`.  -> (rc, bytes, hint, run)"""
    dst = np.full(length + GUARD, MARK, dtype=np.uint8)
    hint = C.c_int(MARK)
    sm, pf, al = _sums(c.n, sums), _pf(prefer), (C.c_int32 * c.n)(*algos)
    rc, run = _call(c, lambda: lib().mec_decode_mixed(c.h, al, _ptrs(files), sm.ctypes.data, None if pf is None else pf.ctypes.data,
                                                      offset, length, total, dst.ctypes.data, C.byref(hint)), files)
    assert (dst[length:] == MARK).all(), "decode wrote past the end of the range"
    return rc, dst[:length], hint.value, run


def heal(c, files, algos, sums, stale, total, prefer=None):
    """mec_heal_mixed into MARK-filled out files GUARD bytes longer than a part.N image.  -> (rc, outs, corrupt, run)"""
    flen = c.bitrot_file_size(total)
    outs = [np.full(flen + GUARD, MARK, dtype=np.uint8) if i in stale else None for i in range(c.n)]
    corrupt = np.full(c.n, MARK, dtype=np.uint8)
    sm, pf, al = _sums(c.n, sums), _pf(prefer), (C.c_int32 * c.n)(*algos)
    rc, run = _call(c, lambda: lib().mec_heal_mixed(c.h, al, _ptrs(files), sm.ctypes.data, None if pf is None else pf.ctypes.data,
                                                    total, _ptrs(outs), corrupt.ctypes.data), files)
    for i in stale:
        assert (outs[i][flen:] == MARK).all(), f"heal wrote past the end of out file {i}"
    return rc, [None if o is None else o[:flen] for o in outs], corrupt, run


def check_bytes(out, want, what):
    if not np.array_equal(out, want):
        bad = np.nonzero(out != want)[0]
        raise AssertionError(f"{what}: {bad.size} bytes differ, first at {bad[0]}")


def check_decode(res, data, offset, length, hint=0):
    rc, out, got_hint, _ = res
    assert rc == length, rc
    check_bytes(out, data[offset:offset + length], f"decode [{offset}, {offset + length})")
    assert got_hint == hint, got_hint


def check_heal(res, sfiles, stale, rc=0, dropped=()):
    got_rc, outs, corrupt, _ = res
    assert got_rc == rc, got_rc
    assert list(np.nonzero(corrupt)[0]) == sorted(dropped), corrupt
    for i in stale:
        check_bytes(outs[i], sfiles[i], f"healed part file {i}")


def check_form(run, form):
    forms = run["forms"]
    assert sum(forms.values()) > 0, forms
    if form == "throughput":
        assert "small" not in forms, forms
    else:
        assert set(forms) == {"small"}, forms


def sizes(bs):
    """under one block, a whole number of blocks, a short last block"""
    return {"sub_block": bs // 3 + 7, "whole_blocks": 3 * bs, "short_last": 2 * bs + bs // 2 + 13}


def ranges(bs, total):
    """from block 0 (the whole part), from a block > 0, the last bytes"""
    out = [(0, total)]
    if total > bs:
        out.append((bs + 100, total - bs - 150))
    out.append((max(0, total - 777), min(777, total)))
    return out


def mixes(n, k):
    """all whole-file; part-healed (every other drive streams); part-healed with two drives offline"""
    healed = "".join("s" if i % 2 == 0 else "w" for i in range(n))
    return {"all_whole": "w" * n, "part_healed": healed, "offline": "--" + healed[2:]}


# ---------------------------------------------------------------- decode and heal against the oracle
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("size", ["sub_block", "whole_blocks", "short_last"])
@pytest.mark.parametrize("walgo", list(ALGOS))
@pytest.mark.parametrize("geom", list(GEOMS))
def test_decode_vs_oracle(mb, oracle, geom, walgo, size, form):  # noqa: F811
    k, m, bs = GEOMS[geom]
    total = sizes(bs)[size]
    p = part(oracle, k, m, bs, ALGOS[walgo], total)
    c = codec(mb, k, m, bs, FORMS[form])
    for name, kinds in mixes(k + m, k).items():
        files, algos = drives(p, kinds, ALGOS[walgo])
        for offset, length in ranges(bs, total):
            res = decode(c, files, algos, p[3], offset, length, total)
            check_decode(res, p[0], offset, length)
            check_form(res[3], form)
            assert res[3]["corrupt_shards"] == 0
    c.close()


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("size", ["sub_block", "whole_blocks", "short_last"])
@pytest.mark.parametrize("walgo", list(ALGOS))
@pytest.mark.parametrize("geom", list(GEOMS))
def test_heal_vs_oracle(mb, oracle, geom, walgo, size, form):  # noqa: F811
    k, m, bs = GEOMS[geom]
    n = k + m
    total = sizes(bs)[size]
    p = part(oracle, k, m, bs, ALGOS[walgo], total)
    c = codec(mb, k, m, bs, FORMS[form])
    healed = mixes(n, k)["part_healed"]
    cases = [
        ("w" * n, [1]),                                   # the first heal of a legacy part: one data drive
        (healed, [1]),                                    # a part already half healed
        (healed, list(range(n - m, n))),                  # m stale drives, the parity drives
        (healed, [0] + list(range(3, 3 + m - 1))),        # m stale drives among the data drives
    ]
    for kinds, stale in cases:
        files, algos = drives(p, kinds, ALGOS[walgo])
        res = heal(c, files, algos, p[3], stale, total)
        check_heal(res, p[1], stale)
        check_form(res[3], form)
    # a stale drive whose files[i] is also given (a garbage file in a format that does not match algos[i]) is never read
    files, algos = drives(p, healed, ALGOS[walgo])
    junk = np.full(max(files[1].size, 1), 0xEE, dtype=np.uint8)
    files[1] = junk
    res = heal(c, files, algos, p[3], [1], total)
    check_heal(res, p[1], [1])
    c.close()


@pytest.mark.parametrize("chunk_blocks", [1, 2])
@pytest.mark.parametrize("walgo", list(ALGOS))
def test_multi_chunk(mb, oracle, walgo, chunk_blocks):  # noqa: F811
    """Parts of many chunks: the verified files stay on the device while the chunks cycle through the slots; each chunk's whole-file
    rows come from the right file rows."""
    k, m, bs = 4, 2, MiB
    total = 9 * bs + 12345
    p = part(oracle, k, m, bs, ALGOS[walgo], total)
    c = codec(mb, k, m, bs, dict(THROUGHPUT, chunk_blocks=chunk_blocks))
    for kinds in ("wswsws", "swswsw", "-wswsw", "wwwwww"):
        files, algos = drives(p, kinds, ALGOS[walgo])
        for offset, length in [(0, total), (3 * bs + 5, 5 * bs), (total - 3 * bs - 1, 3 * bs + 1)]:
            res = decode(c, files, algos, p[3], offset, length, total)
            check_decode(res, p[0], offset, length)
            assert res[3]["whole_hash_launches"] == 1
        res = heal(c, files, algos, p[3], [5], total)
        check_heal(res, p[1], [5])
    c.close()


# ---------------------------------------------------------------- fail-over
def flip_sum(sums, i):
    s = list(sums)
    s[i] = bytes([s[i][0] ^ 1]) + s[i][1:]
    return s


def flip_frame(f, block, S):
    g = f.copy()
    g[block * (32 + S) + 32 + 5] ^= 0x40
    return g


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("walgo", list(ALGOS))
def test_chosen_whole_reader_wrong_sum(mb, oracle, walgo, form):  # noqa: F811
    """A chosen whole-file reader fails its sum: dropped, corrupt[i] set, the next reader hashed in a second round."""
    k, m, bs = 12, 4, MiB
    n, total = k + m, 2 * bs + 4321
    p = part(oracle, k, m, bs, ALGOS[walgo], total)
    c = codec(mb, k, m, bs, FORMS[form])
    sfs = c.shard_file_size(total)
    sums = flip_sum(p[3], 2)
    files, algos = drives(p, "w" * n, ALGOS[walgo])
    res = decode(c, files, algos, sums, 0, total, total)
    check_decode(res, p[0], 0, total, hint=FILE_CORRUPT)
    run = res[3]
    assert run["whole_hash_launches"] == 2 and run["corrupt_shards"] == 1
    assert run["bytes_h2d"] == (k + 1) * sfs, run
    res = heal(c, files, algos, sums, [15], total)
    check_heal(res, p[1], [15], rc=FILE_CORRUPT, dropped=[2])
    assert res[3]["whole_hash_launches"] == 2
    c.close()


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("walgo", list(ALGOS))
def test_streaming_failure_hands_over_to_whole(mb, oracle, walgo, form):  # noqa: F811
    """A streaming reader fails a frame in a chunk after the first; the next reader is whole-file: it is hashed at that point (not
    before: the clean chunks ran without it) and the bytes are still exact."""
    k, m, bs = 4, 2, MiB
    total = 7 * bs + 999
    p = part(oracle, k, m, bs, ALGOS[walgo], total)
    c = codec(mb, k, m, bs, dict(FORMS[form], chunk_blocks=2))
    S, sfs = c.shard_size(), c.shard_file_size(total)
    files, algos = drives(p, "ssssws", ALGOS[walgo])
    files[1] = flip_frame(files[1], 5, S)
    res = decode(c, files, algos, p[3], 0, total, total)
    check_decode(res, p[0], 0, total, hint=FILE_CORRUPT)
    run = res[3]
    assert run["whole_hash_launches"] == 1 and run["corrupt_shards"] == 1
    # frames: 4 readers for blocks [0, 4) (chunks 0 and 1), and chunk 2 is submitted again after the drop with 3 streaming readers
    fb = 32 + S
    assert run["bytes_h2d"] >= 4 * 4 * fb + 3 * 2 * fb + sfs
    res = heal(c, files, algos, p[3], [5], total)
    check_heal(res, p[1], [5], rc=FILE_CORRUPT, dropped=[1])
    assert res[3]["whole_hash_launches"] == 1
    # the same failure with a streaming successor: the whole-file reader of the first set is the only one hashed
    files, algos = drives(p, "wsssss", ALGOS[walgo])
    files[2] = flip_frame(files[2], 6, S)
    res = decode(c, files, algos, p[3], 0, total, total)
    check_decode(res, p[0], 0, total, hint=FILE_CORRUPT)
    assert res[3]["whole_hash_launches"] == 1
    c.close()


@pytest.mark.parametrize("walgo", list(ALGOS))
def test_unchosen_whole_reader_wrong_sum(mb, oracle, walgo):  # noqa: F811
    """A whole-file reader that is never chosen is never hashed or reported, whatever its sum."""
    k, m, bs = 12, 4, 10 * MiB
    n, total = k + m, bs + 77
    p = part(oracle, k, m, bs, ALGOS[walgo], total)
    c = codec(mb, k, m, bs, THROUGHPUT)
    sfs = c.shard_file_size(total)
    sums = flip_sum(p[3], n - 1)
    files, algos = drives(p, "w" * n, ALGOS[walgo])
    res = decode(c, files, algos, sums, 0, total, total)
    check_decode(res, p[0], 0, total)
    assert res[3]["whole_hash_launches"] == 1 and res[3]["corrupt_shards"] == 0 and res[3]["bytes_h2d"] == k * sfs
    res = heal(c, files, algos, sums, [3], total)
    check_heal(res, p[1], [3])
    assert res[3]["whole_hash_launches"] == 1
    c.close()


@pytest.mark.parametrize("walgo", list(ALGOS))
def test_readers_exhausted(mb, oracle, walgo):  # noqa: F811
    k, m, bs = 4, 2, MiB
    total = 3 * bs + 1
    p = part(oracle, k, m, bs, ALGOS[walgo], total)
    c = codec(mb, k, m, bs, THROUGHPUT)
    S = c.shard_size()
    files, algos = drives(p, "swswsw", ALGOS[walgo])
    sums = flip_sum(flip_sum(p[3], 1), 3)  # two whole-file readers fail their sums
    files[0] = flip_frame(files[0], 2, S)  # and a streaming reader fails a frame: five readers left of six, three good
    rc = decode(c, files, algos, sums, 0, total, total)[0]
    assert rc == READ_QUORUM
    rc = heal(c, files, algos, sums, [4], total)[0]
    assert rc == READ_QUORUM
    c.close()


@pytest.mark.parametrize("walgo", list(ALGOS))
def test_prefer_chooses_what_is_hashed(mb, oracle, walgo):  # noqa: F811
    """prefer puts a reader with a wrong sum into the first set: now it is hashed, dropped and reported, and its successor in
    preferReaders' order (4, 5, 2, 3, 0, 1: each preferred reader swapped to the front) is hashed in a second round."""
    k, m, bs = 4, 2, MiB
    n, total = k + m, 2 * bs + 3
    p = part(oracle, k, m, bs, ALGOS[walgo], total)
    c = codec(mb, k, m, bs, THROUGHPUT)
    sums = flip_sum(p[3], 5)
    files, algos = drives(p, "wssssw", ALGOS[walgo])
    res = decode(c, files, algos, sums, 0, total, total)
    check_decode(res, p[0], 0, total)
    assert res[3]["whole_hash_launches"] == 1 and res[3]["corrupt_shards"] == 0
    prefer = [0, 0, 0, 0, 1, 1]
    res = decode(c, files, algos, sums, 0, total, total, prefer=prefer)
    check_decode(res, p[0], 0, total, hint=FILE_CORRUPT)
    assert res[3]["whole_hash_launches"] == 2 and res[3]["corrupt_shards"] == 1
    res = heal(c, files, algos, sums, [2], total, prefer=prefer)
    check_heal(res, p[1], [2], rc=FILE_CORRUPT, dropped=[5])
    # preferring the four streaming readers: no whole-file reader is chosen, none is hashed
    res = decode(c, files, algos, p[3], 0, total, total, prefer=[0, 1, 1, 1, 1, 0])
    check_decode(res, p[0], 0, total)
    assert res[3]["whole_hash_launches"] == 0
    c.close()


# ---------------------------------------------------------------- equivalences
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("geom", list(GEOMS))
def test_all_streaming_equals_prefer(mb, oracle, geom, form):  # noqa: F811
    """Every drive HighwayHash256S: mec_decode_mixed is mec_decode_prefer and mec_heal_mixed is mec_heal_prefer, failures included."""
    k, m, bs = GEOMS[geom]
    n, total = k + m, 2 * bs + bs // 2 + 13
    p = part(oracle, k, m, bs, SHA256, total)
    c = codec(mb, k, m, bs, FORMS[form])
    S = c.shard_size()
    algos = [HIGHWAYHASH256S] * n
    base = list(p[1])
    bad = list(base)
    bad[1] = flip_frame(bad[1], 1, S)
    bad[0] = None
    for files in (base, bad):
        for prefer in (None, [0] * (n - 2) + [1, 1]):
            for offset, length in ranges(bs, total):
                got = decode(c, files, algos, None, offset, length, total, prefer)
                dst = np.zeros(max(length, 1), dtype=np.uint8)
                hint = C.c_int(MARK)
                pf = _pf(prefer)
                rc = lib().mec_decode_prefer(c.h, _ptrs(files), None if pf is None else pf.ctypes.data, offset, length, total,
                                             dst.ctypes.data, C.byref(hint))
                assert (got[0], got[2]) == (rc, hint.value)
                check_bytes(got[1], dst[:length], "decode_mixed vs decode_prefer")
            stale = [n - 1] if prefer is None else [2]
            got = heal(c, files, algos, None, stale, total, prefer)
            flen = c.bitrot_file_size(total)
            outs = [np.full(flen, MARK, dtype=np.uint8) if i in stale else None for i in range(n)]
            corrupt = np.full(n, MARK, dtype=np.uint8)
            pf = _pf(prefer)
            rc = lib().mec_heal_prefer(c.h, _ptrs([f if i not in stale else None for i, f in enumerate(files)]),
                                       None if pf is None else pf.ctypes.data, total, _ptrs(outs), corrupt.ctypes.data)
            assert got[0] == rc and np.array_equal(got[2], corrupt), (got[0], rc)
            for i in stale:
                check_bytes(got[1][i], outs[i], "heal_mixed vs heal_prefer")
    c.close()


@pytest.mark.parametrize("walgo", list(ALGOS))
@pytest.mark.parametrize("geom", list(GEOMS))
def test_all_whole_equals_decode_whole(mb, oracle, geom, walgo):  # noqa: F811
    """Every drive whole-file and prefer NULL: mec_decode_mixed is mec_decode_whole, a dropped reader included."""
    k, m, bs = GEOMS[geom]
    n, total = k + m, 2 * bs + bs // 2 + 13
    p = part(oracle, k, m, bs, ALGOS[walgo], total)
    c = codec(mb, k, m, bs, THROUGHPUT)
    w = mb.Codec(k, m, bs, algo=ALGOS[walgo])
    w.set_option("jit", 0)
    w.set_option("small_blocks", 0)
    files, algos = drives(p, "w" * n, ALGOS[walgo])
    files[3] = None
    for sums in (p[3], flip_sum(p[3], 0)):
        for offset, length in ranges(bs, total):
            got = decode(c, files, algos, sums, offset, length, total)
            want = w.decode_whole(files, sums, offset, length, total)
            assert got[0] == length and got[2] == want[1]
            check_bytes(got[1], want[0], "decode_mixed vs decode_whole")
    w.close()
    c.close()


def test_binding(mb, oracle):  # noqa: F811
    """Codec.decode_mixed / Codec.heal_mixed."""
    k, m, bs = 4, 2, MiB
    total = 2 * bs + 5
    p = part(oracle, k, m, bs, SHA256, total)
    c = mb.Codec(k, m, bs)
    files, algos = drives(p, "wsws-w", SHA256)
    out, hint = c.decode_mixed(files, algos, p[3], 10, total - 20, total)
    assert hint == 0 and np.array_equal(out, p[0][10:total - 10])
    outs = c.heal_mixed(files, algos, p[3], [False, False, False, False, True, False], total)
    assert outs[4] is not None and np.array_equal(outs[4], p[1][4])
    outs, rc, corrupt = c.heal_mixed(files, algos, flip_sum(p[3], 2), [False] * 4 + [True, False], total, report=True)
    assert rc == FILE_CORRUPT and list(corrupt) == [0, 0, 1, 0, 0, 0] and np.array_equal(outs[4], p[1][4])
    c.close()
