"""mec_transcode across block sizes on the GPU: a legacy part written with 10 MiB erasure blocks (blockSizeV1) moved into a pool
that writes 1 MiB blocks (blockSizeV2) must be byte for byte what Erasure.Encode of the destination geometry and block size writes
(the CPU oracle), through every source fault parallelReader survives, and the same as mec_decode_prefer followed by mec_encode.
Also: the 10 MiB-block codec's other read paths (a decode across a block boundary, heal, bitrot verification) against the oracle."""
import numpy as np
import pytest

from test_gpu_transcode import FORMS, assert_oracle_exact, forms, pattern, rand, transcode, GUARD

pytestmark = pytest.mark.gpu
MiB = 1 << 20
V1 = 10 * MiB  # blockSizeV1, cmd/object-api-common.go:34


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


PAIRS = [
    (12, 4, V1, 6, 2, MiB),                 # a legacy 16-drive pool drained into an 8-drive pool
    (12, 4, V1, 12, 4, MiB),                # the same geometry, only the block size changes
    (16, 4, V1, 7, 5, MiB),                 # odd destination shard size 149797: frames at every alignment mod 4
    (10, 1, 4 * (MiB - 1), 5, 3, MiB - 1),  # R = 4 with block sizes that are not multiples of 16
]
LENGTHS = ["1", "half dst block", "dst block", "3.5 dst blocks", "src block", "src block + 1", "2 src blocks + tail",
           "7 src blocks, 7 chunks"]


def length_of(name, bs, bd):
    return {"1": 1, "half dst block": bd // 2 + 13, "dst block": bd, "3.5 dst blocks": 3 * bd + bd // 2, "src block": bs,
            "src block + 1": bs + 1, "2 src blocks + tail": 2 * bs + 4321, "7 src blocks, 7 chunks": 6 * bs + 777}[name]


def nblocks(total, bs):
    return -(-total // bs)


@pytest.mark.parametrize("length", LENGTHS)
@pytest.mark.parametrize("k1,m1,bs,k2,m2,bd", PAIRS)
def test_transcode_vs_oracle(mb, oracle, k1, m1, bs, k2, m2, bd, length):
    total = length_of(length, bs, bd)
    data = rand(total, k1 * 100 + k2 + total % 97)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bd)
    if length.endswith("7 chunks"):
        src.set_option("chunk_blocks", 1)  # seven chunks of one source block: every slot of the ring carries one
    rc, outs, hint = transcode(mb, src, files, total, dst)
    assert rc == total and hint == 0
    assert_oracle_exact(oracle, outs, k2, m2, bd, data)
    assert src.stat("blocks_read") == nblocks(total, bs) and dst.stat("blocks_encoded") == nblocks(total, bd)
    src.close()
    dst.close()


def via_host(mb, src_codec, files, total, k2, m2, bd, prefer=None):
    got, hint = src_codec.decode(files, 0, total, total, prefer=prefer)
    d = mb.Codec(k2, m2, bd)
    outs = d.encode(got)
    d.close()
    return outs, hint


@pytest.mark.parametrize("use_prefer", [False, True])
def test_offline_source_drives(mb, oracle, use_prefer):
    """Data and parity drives of the source offline: the missing data shards are rebuilt on the device, `prefer` reorders the
    readers as mec_decode_prefer does, and the result equals mec_decode_prefer + mec_encode."""
    k1, m1, bs, k2, m2, bd = PAIRS[0]
    total = 3 * bs + 5 * bd + 999
    data = rand(total, 21)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    files = [None if i in (1, 7, 13) else f for i, f in enumerate(files)]
    prefer = [1 if i in (3, 12, 14, 15) else 0 for i in range(16)] if use_prefer else None
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bd)
    rc, outs, hint = transcode(mb, src, files, total, dst, prefer=prefer)
    assert rc == total and hint == 0
    assert_oracle_exact(oracle, outs, k2, m2, bd, data)
    want, whint = via_host(mb, src, files, total, k2, m2, bd, prefer)
    assert whint == hint and all(np.array_equal(a, b) for a, b in zip(outs, want))
    assert src.stat("shards_rebuilt") > 0
    src.close()
    dst.close()


def test_corrupt_frame_mid_pipeline(mb, oracle):
    """A corrupt frame of a chosen reader in source block 4, with the chunks behind it in flight: the reader is dropped, the part
    resumes at that source block (a destination block boundary) with the next reader, every destination byte is still the
    oracle's, heal_hint = -7, and all of it equals mec_decode_prefer + mec_encode.  Then more corrupt readers than parity drives."""
    k1, m1, bs, k2, m2, bd = PAIRS[0]
    total = 6 * bs + 4321
    data = rand(total, 33)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    S = oracle.shard_size(bs, k1)
    bad = [f.copy() for f in files]
    bad[2][4 * (32 + S) + 32 + 500] ^= 0x10   # reader 2, source block 4: the first block of chunk 2 (blocks 4..5), chunk 3 behind it
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bd)
    src.set_option("chunk_blocks", 2)
    rc, outs, hint = transcode(mb, src, bad, total, dst)
    assert rc == total and hint == -7
    assert_oracle_exact(oracle, outs, k2, m2, bd, data)
    assert src.stat("corrupt_shards") == 1
    assert src.stat("blocks_read") == nblocks(total, bs) and dst.stat("blocks_encoded") == nblocks(total, bd)
    ref = mb.Codec(k1, m1, bs)
    ref.set_option("chunk_blocks", 2)
    want, whint = via_host(mb, ref, bad, total, k2, m2, bd)
    assert whint == hint and all(np.array_equal(a, b) for a, b in zip(outs, want))
    for i in (0, 5, 9, 14):
        bad[i][3 * (32 + S) + 40] ^= 0xFF
    rc, _, _ = transcode(mb, src, bad, total, dst)
    assert rc == -10
    for c in (src, dst, ref):
        c.close()


def test_destination_writers(mb, oracle):
    """Offline destination writers are skipped while the others stay exact; below the write quorum nothing is written."""
    k1, m1, bs, k2, m2, bd = PAIRS[0]
    total = bs + 6 * bd + 77
    data = rand(total, 44)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bd)
    online = [i not in (1, 6) for i in range(8)]
    rc, outs, hint = transcode(mb, src, files, total, dst, online=online, write_quorum=6)
    assert rc == total and hint == 0 and outs[1] is None and outs[6] is None
    assert_oracle_exact(oracle, outs, k2, m2, bd, data)
    online = [i not in (0, 3, 7) for i in range(8)]
    rc, outs, _ = transcode(mb, src, files, total, dst, online=online, write_quorum=6)
    assert rc == -11
    fsz = dst.bitrot_file_size(total)
    ref = pattern(fsz + 2 * GUARD)[GUARD:GUARD + fsz]
    assert all(np.array_equal(o, ref) for o in outs if o is not None)
    src.close()
    dst.close()


def test_object_stays_on_the_device(mb, oracle):
    """The source never copies object bytes back, the destination never stages them, and the source stages its k readers' part
    files exactly once."""
    k1, m1, bs, k2, m2, bd = PAIRS[0]
    total = 2 * bs + 3 * bd + 5
    data = rand(total, 55)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    files[4] = None
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bd)
    src.transcode(files, total, dst)  # warm both codecs
    before = {(c, s): c.stat(s) for c in (src, dst) for s in ("bytes_h2d", "bytes_d2h")}
    outs, hint = src.transcode(files, total, dst)
    assert hint == 0
    assert_oracle_exact(oracle, outs, k2, m2, bd, data)
    assert src.stat("bytes_d2h") == before[(src, "bytes_d2h")]
    assert dst.stat("bytes_h2d") == before[(dst, "bytes_h2d")]
    assert src.stat("bytes_h2d") - before[(src, "bytes_h2d")] == k1 * src.bitrot_file_size(total)
    assert dst.stat("bytes_d2h") > before[(dst, "bytes_d2h")]
    src.close()
    dst.close()


@pytest.mark.parametrize("shape", ["small part", "long part"])
def test_dispatch(mb, oracle, shape):
    """Which forms of the fused kernel ran: a short part takes the latency kernel on both ends; a long part with the latency
    kernel switched off (small_blocks = 0) runs only throughput forms on both ends."""
    k1, m1, bs, k2, m2, bd = PAIRS[0]
    total = bs + 3 * bd + 3 if shape == "small part" else 6 * bs + 3
    data = rand(total, 66)
    files, _ = oracle.erasure_encode(k1, m1, bs, oracle.HIGHWAYHASH256S, data)
    files[0] = None
    src, dst = mb.Codec(k1, m1, bs), mb.Codec(k2, m2, bd)
    if shape == "long part":
        for c in (src, dst):
            c.set_option("small_blocks", 0)
    s0, d0 = forms(src), forms(dst)
    outs, hint = src.transcode(files, total, dst)
    assert hint == 0
    assert_oracle_exact(oracle, outs, k2, m2, bd, data)
    ds = {f: forms(src)[f] - s0[f] for f in FORMS}
    dd = {f: forms(dst)[f] - d0[f] for f in FORMS}
    if shape == "small part":
        assert ds["small"] > 0 and dd["small"] > 0
        assert sum(ds.values()) == ds["small"] and sum(dd.values()) == dd["small"]
    else:
        assert ds["small"] == 0 and dd["small"] == 0 and sum(ds.values()) > 0 and sum(dd.values()) > 0
    assert dst.stat("blocks_encoded") == nblocks(total, bd)
    src.close()
    dst.close()


# ---- the 10 MiB-block codec's other read paths ----------------------------------------------------------------------------------

@pytest.mark.parametrize("call", ["decode across a block boundary", "heal", "bitrot verify batch"])
def test_legacy_block_size_vs_oracle(mb, oracle, call):
    """RS(12,4) at blockSizeV1 = 10 MiB against the oracle: mec_decode of a range that crosses a source block boundary, with a data
    drive offline; mec_heal_prefer of two stale drives; mec_bitrot_verify_batch of every shard file, clean and with a flipped byte."""
    k, m, bs = 12, 4, V1
    total = 2 * bs + 12345
    data = rand(total, 77)
    files, _ = oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, data)
    c = mb.Codec(k, m, bs)
    if call == "decode across a block boundary":
        offset, length = bs - 1000, bs + 5000
        got, hint = c.decode([None if i == 3 else f for i, f in enumerate(files)], offset, length, total)
        rc, want, _ = oracle.erasure_decode(k, m, bs, oracle.HIGHWAYHASH256S, files, [i != 3 for i in range(k + m)], offset, length,
                                            total)
        assert hint == 0 and rc == length and np.array_equal(got, want) and np.array_equal(got, data[offset:offset + length])
    elif call == "heal":
        stale = [i in (2, 13) for i in range(k + m)]
        outs = c.heal([None if stale[i] else f for i, f in enumerate(files)], stale, total, prefer=[i >= 8 for i in range(k + m)])
        for i in range(k + m):
            if stale[i]:
                assert np.array_equal(outs[i], files[i]), f"healed shard file {i} differs from the oracle"
    else:
        part_len = oracle.shard_file_size(bs, k, total)
        assert c.bitrot_verify_batch(files, [part_len] * (k + m)) == [0] * (k + m)
        S = oracle.shard_size(bs, k)
        bad = [f.copy() for f in files]
        bad[5][(32 + S) + 32 + S // 2] ^= 1   # shard 5, block 1
        bad[15][-1] ^= 0x80                    # parity shard 15, the last byte of the short last frame
        want = [-7 if i in (5, 15) else 0 for i in range(k + m)]
        assert c.bitrot_verify_batch(bad, [part_len] * (k + m)) == want
        assert [oracle.bitrot_verify(oracle.HIGHWAYHASH256S, f, part_len, S) for f in bad] == want
    c.close()
