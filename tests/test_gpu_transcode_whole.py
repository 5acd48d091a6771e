"""mec_transcode_whole on the GPU: a part written with a whole-file bitrot algorithm (SHA256, HighwayHash256, BLAKE2b512 — raw
shard files, one digest per file kept in xl.meta) moved to a streaming-bitrot pool must be byte for byte what Erasure.Encode of the
destination geometry and block size writes for the object (the CPU oracle), through offline drives and readers that fail their
whole-file digest, and the same as mec_decode_whole followed by mec_encode.  Sources come from the oracle's Erasure.Encode with the
whole-file algorithm; every out file sits inside a pattern-filled buffer whose guard bytes must survive."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_transcode import GUARD, assert_oracle_exact, pattern, rand
from test_gpu_transcode_blocksize import PAIRS as BLOCKSIZE_PAIRS

pytestmark = pytest.mark.gpu
MiB = 1 << 20
V1 = 10 * MiB
SHA256, HIGHWAYHASH256, BLAKE2B512 = 1, 2, 4
ALGOS = {"sha256": SHA256, "hh256": HIGHWAYHASH256, "blake2b": BLAKE2B512}
FILE_CORRUPT, READ_QUORUM, WRITE_QUORUM = -7, -10, -11
PAIRS = BLOCKSIZE_PAIRS + [(12, 4, MiB, 12, 4, MiB)]  # the legacy block-size moves, and one between equal block sizes
LENGTHS = ["1", "half dst block", "dst block", "src block - 1", "src block + 1", "2 src blocks + tail", "7 src blocks, 7 chunks"]


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


def length_of(name, bs, bd):
    return {"1": 1, "half dst block": bd // 2 + 13, "dst block": bd, "src block - 1": bs - 1, "src block + 1": bs + 1,
            "2 src blocks + tail": 2 * bs + 4321, "7 src blocks, 7 chunks": 6 * bs + 777}[name]


_PARTS = {}


def whole_part(oracle, k, m, bs, algo, total, seed):
    """(object, raw shard files, whole-file sums) from the oracle's Erasure.Encode, cached across tests"""
    key = (k, m, bs, algo, total, seed)
    if key not in _PARTS:
        data = rand(total, seed)
        files, sums = oracle.erasure_encode(k, m, bs, algo, data)
        _PARTS[key] = (data, files, sums)
    return _PARTS[key]


def transcode_whole(mb, src, files, sums, total, dst, online=None, prefer=None, write_quorum=0):
    """mec_transcode_whole into guarded out files -> (rc, outs, heal_hint); asserts that nothing outside an out file was written"""
    fsz = dst.bitrot_file_size(total)
    online = [True] * dst.n if online is None else online
    bufs = [pattern(fsz + 2 * GUARD) if online[i] else None for i in range(dst.n)]
    ptrs = (C.c_void_p * dst.n)(*[b.ctypes.data + GUARD if b is not None else None for b in bufs])
    files = [None if f is None else np.ascontiguousarray(f) for f in files]
    sm = np.zeros((src.n, 64), dtype=np.uint8)
    for i, d in enumerate(sums):
        sm[i, :len(d)] = np.frombuffer(d, dtype=np.uint8)
    pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
    hint = C.c_int(0)
    rc = mb.lib().mec_transcode_whole(src.h, mb.capi._ptrs(files), sm.ctypes.data, None if pf is None else pf.ctypes.data, total,
                                      dst.h, ptrs, write_quorum, C.byref(hint))
    ref = pattern(fsz + 2 * GUARD)
    for b in bufs:
        if b is not None:
            assert np.array_equal(b[:GUARD], ref[:GUARD]) and np.array_equal(b[GUARD + fsz:], ref[GUARD + fsz:]), "guard bytes written"
    return rc, [b[GUARD:GUARD + fsz] if b is not None else None for b in bufs], hint.value


def via_host(mb, src, files, sums, total, k2, m2, bd):
    """the Decode -> Encode pipe mec_transcode_whole replaces: mec_decode_whole into a host buffer, mec_encode of it"""
    got, hint = src.decode_whole(files, sums, 0, total, total)
    d = mb.Codec(k2, m2, bd)
    outs = d.encode(got)
    d.close()
    return outs, hint


def nblocks(total, bs):
    return -(-total // bs)


def untouched(outs, fsz):
    ref = pattern(fsz + 2 * GUARD)[GUARD:GUARD + fsz]
    return all(np.array_equal(o, ref) for o in outs if o is not None)


# every pair meets every algorithm and every length meets every algorithm (the algorithm rotates with the case)
CASES = [(algo, pair, length) for p, pair in enumerate(PAIRS) for l, length in enumerate(LENGTHS)
         for algo in [list(ALGOS)[(p + l) % 3]]]


@pytest.mark.parametrize("algo,pair,length", CASES,
                         ids=[f"{a}-RS{p[0]},{p[1]}@{p[2]}->RS{p[3]},{p[4]}@{p[5]}-{l}" for a, p, l in CASES])
def test_vs_oracle(mb, oracle, algo, pair, length):
    k1, m1, bs, k2, m2, bd = pair
    total = length_of(length, bs, bd)
    data, files, sums = whole_part(oracle, k1, m1, bs, ALGOS[algo], total, k1 * 100 + k2 + total % 97)
    src, dst = mb.Codec(k1, m1, bs, ALGOS[algo]), mb.Codec(k2, m2, bd)
    if length.endswith("7 chunks"):
        src.set_option("chunk_blocks", 1)  # seven chunks of one source block: the ring of six slots wraps
    rc, outs, hint = transcode_whole(mb, src, files, sums, total, dst)
    assert rc == total and hint == 0
    assert_oracle_exact(oracle, outs, k2, m2, bd, data)
    assert src.stat("blocks_read") == nblocks(total, bs) and dst.stat("blocks_encoded") == nblocks(total, bd)
    assert src.stat("whole_hash_launches") == 1 and src.stat("corrupt_shards") == 0
    src.close()
    dst.close()


@pytest.mark.parametrize("use_prefer", [False, True])
@pytest.mark.parametrize("algo", list(ALGOS))
def test_offline_source_drives(mb, oracle, algo, use_prefer):
    """m source drives offline, data and parity: the missing data shards are rebuilt from the raw shard rows chunk by chunk,
    `prefer` reorders the readers, and the result equals mec_decode_whole + mec_encode."""
    k1, m1, bs, k2, m2, bd = PAIRS[0]
    total = 3 * bs + 5 * bd + 999
    data, files, sums = whole_part(oracle, k1, m1, bs, ALGOS[algo], total, 21)
    files = [None if i in (1, 7, 12, 13) else f for i, f in enumerate(files)]
    prefer = [1 if i in (3, 14, 15) else 0 for i in range(16)] if use_prefer else None
    src, dst = mb.Codec(k1, m1, bs, ALGOS[algo]), mb.Codec(k2, m2, bd)
    rc, outs, hint = transcode_whole(mb, src, files, sums, total, dst, prefer=prefer)
    assert rc == total and hint == 0
    assert_oracle_exact(oracle, outs, k2, m2, bd, data)
    assert src.stat("shards_rebuilt") == 2 * nblocks(total, bs)  # data shards 1 and 7 of every source block
    want, whint = via_host(mb, src, files, sums, total, k2, m2, bd)
    assert whint == hint and all(np.array_equal(a, b) for a, b in zip(outs, want))
    src.close()
    dst.close()


@pytest.mark.parametrize("use_prefer", [False, True])
@pytest.mark.parametrize("kind", ["flipped byte", "wrong sum"])
def test_corrupt_reader(mb, oracle, kind, use_prefer):
    """A chosen reader fails its whole-file digest (a flipped byte in its file, or a wrong expected sum): it is dropped, the next
    reader in parallelReader's order takes its place, every destination byte is still the oracle's, heal_hint = -7, corrupt_shards
    grows by one, and the result equals mec_decode_whole + mec_encode.  Two rounds of readers: two hash launches."""
    k1, m1, bs, k2, m2, bd = PAIRS[0]
    total = 2 * bs + 3 * bd + 17
    data, files, sums = whole_part(oracle, k1, m1, bs, SHA256, total, 33)
    files, sums = list(files), list(sums)
    bad = 13 if use_prefer else 2
    if kind == "flipped byte":
        files[bad] = files[bad].copy()
        files[bad][files[bad].size // 2] ^= 0x10
    else:
        sums[bad] = bytes(b ^ 0xFF for b in sums[bad])
    prefer = [1 if i >= 12 else 0 for i in range(16)] if use_prefer else None  # parity first: reader 13 is chosen
    src, dst = mb.Codec(k1, m1, bs, SHA256), mb.Codec(k2, m2, bd)
    rc, outs, hint = transcode_whole(mb, src, files, sums, total, dst, prefer=prefer)
    assert rc == total and hint == FILE_CORRUPT
    assert_oracle_exact(oracle, outs, k2, m2, bd, data)
    assert src.stat("corrupt_shards") == 1 and src.stat("whole_hash_launches") == 2
    assert src.stat("blocks_read") == nblocks(total, bs) and dst.stat("blocks_encoded") == nblocks(total, bd)
    ref = mb.Codec(k1, m1, bs, SHA256)
    want, whint = via_host(mb, ref, files, sums, total, k2, m2, bd)
    assert all(np.array_equal(a, b) for a, b in zip(outs, want))
    assert whint == (0 if use_prefer else hint)  # mec_decode_whole has no `prefer`: it reads drives 0..11 and never meets reader 13
    for c in (src, dst, ref):
        c.close()


@pytest.mark.parametrize("algo", list(ALGOS))
def test_read_quorum(mb, oracle, algo):
    """More readers fail their digest than there are parity drives (with one drive offline on top): MEC_ERR_READ_QUORUM, and since
    verification comes before anything is written, every out file is untouched."""
    k1, m1, bs, k2, m2, bd = PAIRS[0]
    total = bs + 2 * bd + 5
    data, files, sums = whole_part(oracle, k1, m1, bs, ALGOS[algo], total, 44)
    files = [None if i == 9 else f.copy() for i, f in enumerate(files)]
    for i in (0, 4, 11, 14):
        files[i][i * 1000 + 7] ^= 0x01
    src, dst = mb.Codec(k1, m1, bs, ALGOS[algo]), mb.Codec(k2, m2, bd)
    rc, outs, hint = transcode_whole(mb, src, files, sums, total, dst)
    assert rc == READ_QUORUM
    assert untouched(outs, dst.bitrot_file_size(total))
    assert src.stat("corrupt_shards") == 4 and dst.stat("blocks_encoded") == 0 and dst.stat("bytes_d2h") == 0
    src.close()
    dst.close()


def test_destination_writers(mb, oracle):
    """Offline destination writers are skipped while the others stay exact; below the write quorum nothing is written."""
    k1, m1, bs, k2, m2, bd = PAIRS[0]
    total = bs + 6 * bd + 77
    data, files, sums = whole_part(oracle, k1, m1, bs, HIGHWAYHASH256, total, 55)
    src, dst = mb.Codec(k1, m1, bs, HIGHWAYHASH256), mb.Codec(k2, m2, bd)
    online = [i not in (1, 6) for i in range(8)]
    rc, outs, hint = transcode_whole(mb, src, files, sums, total, dst, online=online, write_quorum=6)
    assert rc == total and hint == 0 and outs[1] is None and outs[6] is None
    assert_oracle_exact(oracle, outs, k2, m2, bd, data)
    online = [i not in (0, 3, 7) for i in range(8)]
    rc, outs, _ = transcode_whole(mb, src, files, sums, total, dst, online=online, write_quorum=6)
    assert rc == WRITE_QUORUM
    assert untouched(outs, dst.bitrot_file_size(total))
    src.close()
    dst.close()


@pytest.mark.parametrize("algo", list(ALGOS))
def test_same_as_decode_then_encode(mb, oracle, algo):
    """Through the Python binding: the same part files as mec_decode_whole into a host buffer followed by mec_encode."""
    k1, m1, bs, k2, m2, bd = PAIRS[0]
    total = 4 * bs + 3 * bd + 1234
    data, files, sums = whole_part(oracle, k1, m1, bs, ALGOS[algo], total, 66)
    src, dst = mb.Codec(k1, m1, bs, ALGOS[algo]), mb.Codec(k2, m2, bd)
    outs, hint = src.transcode_whole(files, sums, total, dst)
    want, whint = via_host(mb, src, files, sums, total, k2, m2, bd)
    assert hint == whint == 0 and all(np.array_equal(a, b) for a, b in zip(outs, want))
    src.close()
    dst.close()


def test_object_stays_on_the_device(mb, oracle):
    """On a clean move the source never copies object bytes back, the destination never stages them, the source stages its k
    readers' shard files exactly once and hashes them in exactly one launch."""
    k1, m1, bs, k2, m2, bd = PAIRS[0]
    total = 2 * bs + 3 * bd + 5
    data, files, sums = whole_part(oracle, k1, m1, bs, BLAKE2B512, total, 77)
    src, dst = mb.Codec(k1, m1, bs, BLAKE2B512), mb.Codec(k2, m2, bd)
    src.transcode_whole(files, sums, total, dst)  # warm both codecs
    names = ("bytes_h2d", "bytes_d2h", "whole_hash_launches")
    before = {(c, s): c.stat(s) for c in (src, dst) for s in names}
    rc, outs, hint = transcode_whole(mb, src, files, sums, total, dst)
    assert rc == total and hint == 0
    assert_oracle_exact(oracle, outs, k2, m2, bd, data)
    delta = {(c, s): c.stat(s) - before[(c, s)] for c in (src, dst) for s in names}
    assert delta[(src, "bytes_d2h")] == 0 and delta[(dst, "bytes_h2d")] == 0
    assert delta[(src, "bytes_h2d")] == k1 * src.shard_file_size(total)
    assert delta[(src, "whole_hash_launches")] == 1 and delta[(dst, "whole_hash_launches")] == 0
    assert delta[(dst, "bytes_d2h")] > 0
    src.close()
    dst.close()
