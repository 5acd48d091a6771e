"""mec_transcode on the GPU: a part moved from one erasure geometry to another must be byte for byte what Erasure.Encode of the
destination geometry writes for the object (the CPU oracle), through every source fault parallelReader survives, and the same as
mec_decode_prefer followed by mec_encode on the same inputs."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
MiB = 1 << 20
GUARD = 61  # every out file starts at an odd offset inside a pattern-filled buffer, with this many guard bytes on each side


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


def rand(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def pattern(n):
    return (np.arange(n, dtype=np.int64) * 131 + 7).astype(np.uint8)


def transcode(mb, src, files, total, dst, online=None, prefer=None, write_quorum=0):
    """mec_transcode into guarded out files -> (rc, outs, heal_hint); asserts that nothing outside an out file was written"""
    fsz = dst.bitrot_file_size(total)
    online = [True] * dst.n if online is None else online
    bufs = [pattern(fsz + 2 * GUARD) if online[i] else None for i in range(dst.n)]
    ptrs = (C.c_void_p * dst.n)(*[b.ctypes.data + GUARD if b is not None else None for b in bufs])
    files = [None if f is None else np.ascontiguousarray(f) for f in files]
    pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
    hint = C.c_int(0)
    rc = mb.lib().mec_transcode(src.h, mb.capi._ptrs(files), None if pf is None else pf.ctypes.data, total, dst.h, ptrs,
                                write_quorum, C.byref(hint))
    ref = pattern(fsz + 2 * GUARD)
    for b in bufs:
        if b is not None:
            assert np.array_equal(b[:GUARD], ref[:GUARD]) and np.array_equal(b[GUARD + fsz:], ref[GUARD + fsz:]), "guard bytes written"
    return rc, [b[GUARD:GUARD + fsz] if b is not None else None for b in bufs], hint.value


def assert_oracle_exact(oracle, outs, k2, m2, bs, data):
    want, _ = oracle.erasure_encode(k2, m2, bs, oracle.HIGHWAYHASH256S, data)
    for i, o in enumerate(outs):
        if o is not None:
            assert np.array_equal(o, want[i]), f"destination part file {i} differs from the oracle"


PAIRS = [
    (12, 4, 6, 2, MiB),       # a 16-drive pool drained into an 8-drive pool
    (6, 2, 12, 4, MiB),       # and back
    (12, 4, 12, 4, MiB),      # rebalance between equal pools
    (16, 4, 7, 5, MiB),       # odd destination shard size 149797: frames at every alignment mod 4
    (10, 1, 5, 3, MiB - 1),   # block size not a multiple of 16
]
LENGTHS = ["1", "sub-block", "3 blocks", "4 blocks + tail", "7 chunks"]


def length_of(name, bs):
    return {"1": 1, "sub-block": bs // 2 + 13, "3 blocks": 3 * bs, "4 blocks + tail": 4 * bs + 12345,
            "7 chunks": 20 * bs + 4321}[name]


@pytest.mark.parametrize("length", LENGTHS)
@pytest.mark.parametrize("k1,m1,k2,m2,bs", PAIRS)
def test_transcode_vs_oracle(mb, oracle, k1, m1, k2, m2, bs, length):
    total = length_of(length, bs)
    data = rand(total, k1 * 100 + k2 + total % 97)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bs)
    if length == "7 chunks":
        src.set_option("chunk_blocks", 3)  # 21 blocks in seven chunks: every slot of the ring carries one
    nblocks = -(-total // bs)
    rc, outs, hint = transcode(mb, src, files, total, dst)
    assert rc == total and hint == 0
    assert_oracle_exact(oracle, outs, k2, m2, bs, data)
    assert dst.stat("blocks_encoded") == nblocks and src.stat("blocks_read") == nblocks
    src.close()
    dst.close()


@pytest.mark.parametrize("use_prefer", [False, True])
def test_offline_source_drives(mb, oracle, use_prefer):
    """Data and parity drives of the source offline: the missing data shards are rebuilt on the device; `prefer` reorders the
    readers exactly as mec_decode_prefer does, and the result equals mec_decode_prefer + mec_encode."""
    k1, m1, k2, m2, bs = 12, 4, 6, 2, MiB
    total = 5 * MiB + 999
    data = rand(total, 21)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    files = [None if i in (1, 7, 13) else f for i, f in enumerate(files)]
    prefer = [1 if i in (3, 12, 14, 15) else 0 for i in range(16)] if use_prefer else None
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bs)
    rc, outs, hint = transcode(mb, src, files, total, dst, prefer=prefer)
    assert rc == total and hint == 0
    assert_oracle_exact(oracle, outs, k2, m2, bs, data)
    got, ghint = src.decode(files, 0, total, total, prefer=prefer)
    via_host = dst.encode(got)
    assert ghint == hint and all(np.array_equal(a, b) for a, b in zip(outs, via_host))
    assert src.stat("shards_rebuilt") > 0
    src.close()
    dst.close()


def test_corrupt_frame_mid_pipeline(mb, oracle):
    """A corrupt frame of a chosen reader in the middle of the third chunk, with the chunks behind it in flight: the reader is
    dropped, the part resumes at that block with the next reader, every destination byte is still the oracle's, heal_hint = -7,
    and all of it equals mec_decode_prefer + mec_encode."""
    k1, m1, k2, m2, bs = 12, 4, 6, 2, MiB
    total = 20 * MiB + 4321
    data = rand(total, 33)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    S = oracle.shard_size(bs, k1)
    bad = [f.copy() for f in files]
    bad[2][7 * (32 + S) + 32 + 500] ^= 0x10   # reader 2, block 7: the middle block of chunk 2 (blocks 6..8)
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bs)
    src.set_option("chunk_blocks", 3)
    rc, outs, hint = transcode(mb, src, bad, total, dst)
    assert rc == total and hint == -7
    assert_oracle_exact(oracle, outs, k2, m2, bs, data)
    assert dst.stat("blocks_encoded") == 21 and src.stat("corrupt_shards") == 1
    ref = mb.Codec(k1, m1, bs)
    ref.set_option("chunk_blocks", 3)
    got, ghint = ref.decode(bad, 0, total, total)
    via_host = mb.Codec(k2, m2, bs).encode(got)
    assert ghint == hint and all(np.array_equal(a, b) for a, b in zip(outs, via_host))
    # more corrupt readers than parity drives: the part cannot be read
    for i in (0, 5, 9, 14):
        bad[i][3 * (32 + S) + 40] ^= 0xFF
    rc, _, _ = transcode(mb, src, bad, total, dst)
    assert rc == -10
    for c in (src, dst, ref):
        c.close()


def test_destination_writers(mb, oracle):
    """Offline destination writers are skipped while the others stay exact; below the write quorum nothing is written."""
    k1, m1, k2, m2, bs = 12, 4, 6, 2, MiB
    total = 6 * MiB + 77
    data = rand(total, 44)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bs)
    online = [i not in (1, 6) for i in range(8)]
    rc, outs, hint = transcode(mb, src, files, total, dst, online=online, write_quorum=6)
    assert rc == total and hint == 0 and outs[1] is None and outs[6] is None
    assert_oracle_exact(oracle, outs, k2, m2, bs, data)
    online = [i not in (0, 3, 7) for i in range(8)]
    rc, outs, _ = transcode(mb, src, files, total, dst, online=online, write_quorum=6)
    assert rc == -11
    fsz = dst.bitrot_file_size(total)
    ref = pattern(fsz + 2 * GUARD)[GUARD:GUARD + fsz]
    assert all(np.array_equal(o, ref) for o in outs if o is not None)
    src.close()
    dst.close()


def test_object_stays_on_the_device(mb, oracle):
    """The point of the call: the source never copies object bytes back and the destination never stages them."""
    k1, m1, k2, m2, bs = 12, 4, 6, 2, MiB
    total = 9 * MiB + 5
    data = rand(total, 55)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    files[4] = None
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bs)
    src.transcode(files, total, dst)  # warm both codecs
    before = {(c, s): c.stat(s) for c in (src, dst) for s in ("bytes_h2d", "bytes_d2h")}
    outs, hint = src.transcode(files, total, dst)
    assert hint == 0
    assert_oracle_exact(oracle, outs, k2, m2, bs, data)
    assert src.stat("bytes_d2h") == before[(src, "bytes_d2h")]
    assert dst.stat("bytes_h2d") == before[(dst, "bytes_h2d")]
    assert src.stat("bytes_h2d") - before[(src, "bytes_h2d")] == 12 * src.bitrot_file_size(total)  # k whole part files, once
    assert dst.stat("bytes_d2h") > before[(dst, "bytes_d2h")]
    src.close()
    dst.close()


FORMS = ["small", "fast3d", "fast3d_auto", "fast3d_semi", "fast", "fast_auto", "aligned", "aligned_auto", "runtime", "bytewise",
         "dyn_aligned", "dyn_runtime", "dyn_bytewise", "jit"]


def forms(c):
    return {f: c.stat("form_" + f) for f in FORMS}


@pytest.mark.parametrize("shape", ["small part", "long part"])
def test_dispatch(mb, oracle, shape):
    """Which forms of the fused kernel ran.  A part of at most five blocks per SM takes the latency kernel on both ends; the long
    part runs with the latency kernel switched off (small_blocks = 0): the pipeline's chunks never exceed 128 blocks, so by default
    every chunk would take it, and this keeps the throughput forms of reconstruct and encode covered on the transcode path."""
    k1, m1, k2, m2, bs = 12, 4, 6, 2, MiB
    total = 4 * MiB + 3 if shape == "small part" else 40 * MiB + 3
    data = rand(total, 66)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    files[0] = None
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bs)
    if shape == "long part":
        for c in (src, dst):
            c.set_option("small_blocks", 0)
    s0, d0 = forms(src), forms(dst)
    outs, hint = src.transcode(files, total, dst)
    assert hint == 0
    assert_oracle_exact(oracle, outs, k2, m2, bs, data)
    ds = {f: forms(src)[f] - s0[f] for f in FORMS}
    dd = {f: forms(dst)[f] - d0[f] for f in FORMS}
    if shape == "small part":
        assert ds["small"] > 0 and dd["small"] > 0
        assert sum(ds.values()) == ds["small"] and sum(dd.values()) == dd["small"]
    else:
        assert ds["small"] == 0 and dd["small"] == 0 and sum(ds.values()) > 0 and sum(dd.values()) > 0
    assert dst.stat("blocks_encoded") == -(-total // bs)
    src.close()
    dst.close()
