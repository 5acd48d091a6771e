"""GPU tests of the round-2 host paths: pipelined Decode / Heal with DMA sinks, scatter-gather Encode, Heal's bitrot side-band,
NUMA-local pinned buffers, the parity-only tail block, dynamic group claiming — each bit-exact against the CPU oracle."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
MiB = 1 << 20


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


def rand(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


@pytest.mark.parametrize("k,m,bs,length", [(12, 4, MiB, 5 * MiB + 4321), (12, 4, MiB, 70 * MiB + 17), (4, 2, MiB, 4 * MiB),
                                           (6, 2, 512 * 1024, MiB + 3), (16, 4, MiB, 3 * MiB), (8, 8, 256 * 1024, 9 * MiB + 1),
                                           (2, 2, MiB, 5), (12, 4, MiB, MiB - 1)])
def test_encode_sg_vs_oracle(mb, oracle, k, m, bs, length):
    """mec_encode_sg: parity frames by DMA, data digests separately; data frames = digest + the caller's own slice."""
    data = rand(length, length % 1009)
    want, _ = oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, data)
    c = mb.Codec(k, m, bs)
    files, dd = c.encode_sg(data)
    S = c.shard_size()
    for j in range(m):
        assert np.array_equal(files[k + j], want[k + j]), j
    # rebuild the data drives' part files the way a writer would: digest, then the slice of the source (zero padded)
    nb = -(-length // bs)
    for i in range(k):
        out, pos = np.zeros(want[i].size, dtype=np.uint8), 0
        for b in range(nb):
            blen = min(bs, length - b * bs)
            per = -(-blen // k)
            out[pos:pos + 32] = dd[b, i]
            lo = min(i * per, blen); hi = min((i + 1) * per, blen)
            out[pos + 32:pos + 32 + (hi - lo)] = data[b * bs + lo:b * bs + hi]
            pos += 32 + per
        assert pos == want[i].size and np.array_equal(out, want[i]), i
    c.close()


def test_encode_frames_into_pinned_numa_buffers(mb, oracle):
    """mec_encode writing every frame by DMA into mec_alloc_pinned_on buffers; decode straight back out of them."""
    k, m, bs, length = 12, 4, MiB, 37 * MiB + 12345
    L = mb.lib()
    node = L.mec_device_numa_node(0)
    assert node >= -1
    data = mb.capi.pinned_array(length, device=0)
    data[:] = rand(length, 5)
    assert L.mec_is_pinned(data.ctypes.data) == 1
    want, _ = oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, data)
    c = mb.Codec(k, m, bs)
    fsz = c.bitrot_file_size(length)
    files = [mb.capi.pinned_array(fsz, device=0) for _ in range(k + m)]
    for f in files:
        f[:] = 0xA5
    ptrs = (C.c_void_p * (k + m))(*[f.ctypes.data for f in files])
    rc = L.mec_encode(c.h, data.ctypes.data, length, ptrs, k + 1)
    assert rc == length
    for i in range(k + m):
        assert np.array_equal(files[i], want[i]), i
    dst = mb.capi.pinned_array(length, device=0)
    fptrs = (C.c_void_p * (k + m))(*[None if i in (1, 4, 9, 13) else files[i].ctypes.data for i in range(k + m)])
    hint = C.c_int(0)
    rc = L.mec_decode(c.h, fptrs, 0, length, length, dst.ctypes.data, C.byref(hint))
    assert rc == length and hint.value == 0 and np.array_equal(dst, data)
    c.close()
    for a in files + [data, dst]:
        L.mec_free_pinned(a.ctypes.data)


def test_bind_thread_to_device_is_harmless(mb):
    L = mb.lib()
    import os
    before = os.sched_getaffinity(0)
    node = L.mec_bind_thread_to_device(0)
    after = os.sched_getaffinity(0)
    assert after <= before and len(after) > 0
    assert node == -1 or node == L.mec_device_numa_node(0)
    os.sched_setaffinity(0, before)


@pytest.mark.parametrize("offset,length", [(0, 70 * MiB + 17), (MiB - 1, 2), (3 * MiB + 5, 40 * MiB), (69 * MiB, MiB + 17),
                                           (70 * MiB, 17), (12345, 66 * MiB), (35 * MiB, 0), (0, 1)])
def test_pipelined_decode_ranges(mb, oracle, offset, length):
    """Multi-chunk Decode (3 slots x 32-block chunks) over every kind of range edge, with four shards offline."""
    k, m, bs, size = 12, 4, MiB, 70 * MiB + 17
    data = rand(size, 77)
    c = mb.Codec(k, m, bs)
    files = c.encode(data)
    srcs = [None if i in (0, 3, 11, 14) else files[i] for i in range(k + m)]
    out, hint = c.decode(srcs, offset, length, size)
    assert hint == 0 and np.array_equal(out, data[offset:offset + length])
    c.close()


def test_pipelined_decode_failover_mid_stream(mb, oracle):
    """Bitrot in the middle of a long part: chunks submitted behind the bad block are discarded, the range resumes at
    the bad block with the next reader, and the bytes match the oracle's block-sequential parallelReader."""
    k, m, bs, size = 12, 4, MiB, 100 * MiB + 1000
    data = rand(size, 78)
    c = mb.Codec(k, m, bs)
    files = c.encode(data)
    S = c.shard_size()
    bad = [f.copy() for f in files]
    bad[2][50 * (32 + S) + 32 + 999] ^= 0x10     # data shard 2, block 50
    bad[7][51 * (32 + S) + 3] ^= 0x01            # digest of shard 7, block 51
    bad[12][97 * (32 + S) + 40] ^= 0xFF          # parity shard 12 (first stand-in), block 97
    out, hint = c.decode(bad, 0, size, size)
    assert hint == -7 and np.array_equal(out, data)
    rc, ref, corrupt = oracle.erasure_decode(k, m, bs, oracle.HIGHWAYHASH256S, bad, [1] * 16, 0, size, size)
    assert rc == size and np.array_equal(ref, data)
    assert c.stat("corrupt_shards") == int(sum(corrupt))
    c.close()


def test_heal_reports_bitrot_in_a_source(mb, oracle):
    """Erasure.Heal returns errFileCorrupt AFTER writing the healed shards when a source reader failed its digest
    (cmd/erasure-decode.go:338-341,366); the drop-in must not swallow it (ADVICE r1)."""
    k, m, bs, size = 12, 4, MiB, 40 * MiB + 333
    data = rand(size, 79)
    c = mb.Codec(k, m, bs)
    files = c.encode(data)
    S = c.shard_size()
    stale = [i in (0, 15) for i in range(16)]
    srcs = [None if stale[i] else files[i].copy() for i in range(16)]
    srcs[4][20 * (32 + S) + 32 + 5] ^= 0x02
    outs, rc, corrupt = c.heal(srcs, stale, size, report=True)
    assert rc == -7 and list(np.nonzero(corrupt)[0]) == [4]
    for i in (0, 15):
        assert np.array_equal(outs[i], files[i])
    with pytest.raises(mb.MecError) as ei:
        c.heal(srcs, stale, size)
    assert ei.value.code == -7
    # clean sources: MEC_OK, and the prefer hint does not change the bytes
    srcs[4] = files[4]
    outs, rc, corrupt = c.heal(srcs, stale, size, prefer=[i % 2 for i in range(16)], report=True)
    assert rc == 0 and not corrupt.any()
    for i in (0, 15):
        assert np.array_equal(outs[i], files[i])
    c.close()


def test_parity_only_tail_block(mb, oracle):
    """mec_encode_blocks_device with d_digests == NULL and a length that is not a block multiple: the tail launch must not
    hash either (ADVICE r1, high)."""
    import torch
    k, m, bs = 12, 4, MiB
    length = 2 * bs + 4321
    data = rand(length, 80)
    dev = torch.device("cuda:0")
    src = torch.zeros(length + 4096, dtype=torch.uint8, device=dev)
    src[:length] = torch.from_numpy(data).to(dev)
    c = mb.Codec(k, m, bs)
    S = c.shard_size()
    pitch = (S + 15) // 16 * 16
    par = torch.zeros((3 * m, pitch), dtype=torch.uint8, device=dev)
    guard = torch.zeros(1 << 20, dtype=torch.uint8, device=dev)
    c.encode_blocks_device(src.data_ptr(), length, par.data_ptr(), pitch, 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert int(guard.sum().item()) == 0
    hp = par.cpu().numpy()
    for b in range(3):
        blk = data[b * bs:(b + 1) * bs]
        sh = oracle.encode_data(k, m, blk, fast=True)
        per = sh[0].size
        for j in range(m):
            assert np.array_equal(hp[b * m + j, :per], sh[k + j]), (b, j)
    # d_corrupt without d_digests is refused instead of silently skipping the bitrot check
    fp = (32 + S + 15) // 16 * 16
    rc = mb.lib().mec_reconstruct_device(c.h, (C.c_void_p * 16)(*[par.data_ptr()] * 16), fp, 1,
                                         np.ones(16, dtype=np.uint8).ctypes.data, 0, par.data_ptr(), pitch, None, par.data_ptr(), None)
    assert rc == -12
    c.close()


@pytest.mark.parametrize("static_groups", [0, 1])
def test_group_claiming_modes_agree(mb, oracle, static_groups):
    """Dynamic group claiming (several passes per CTA) and the static deal produce the same bytes."""
    import torch
    k, m, bs, nblocks = 12, 4, MiB, 9000   # > 7 CTAs x 132 SMs x 4 blocks: every CTA claims at least one more group
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev); g.manual_seed(1234)
    src = torch.randint(0, 256, (nblocks * bs,), dtype=torch.uint8, device=dev, generator=g)
    S = 87382
    pitch = (S + 15) // 16 * 16
    par = torch.zeros((nblocks * m, pitch), dtype=torch.uint8, device=dev)
    dig = torch.zeros((nblocks, k + m, 32), dtype=torch.uint8, device=dev)
    c = mb.Codec(k, m, bs)
    c.set_option("static_groups", static_groups)
    c.encode_blocks_device(src.data_ptr(), src.numel(), par.data_ptr(), pitch, dig.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for b in (0, 4143, 4144, 4147, 8287, 8288, 8999):
        blk = src[b * bs:(b + 1) * bs].cpu().numpy()
        sh = oracle.encode_data(k, m, blk, fast=True)
        hp = par[b * m:(b + 1) * m, :S].cpu().numpy()
        hd = dig[b].cpu().numpy()
        for j in range(m):
            assert np.array_equal(hp[j], sh[k + j]), (b, j)
        for i in range(k + m):
            assert hd[i].tobytes() == oracle.hh256(sh[i], fast=True), (b, i)
    # every block was written exactly once: no digest row is left zero
    assert bool((dig.view(torch.int64).reshape(nblocks, -1) != 0).any(dim=1).all().item())
    c.close()


# cmd/erasure-decode_test.go:44-83, all 38 rows: (dataBlocks, onDisks, offDisks, blocksize, data, offset, length, algorithm,
# shouldFail, shouldFailQuorum).  DefaultBitrotAlgorithm = HighwayHash256S (streaming frames); BLAKE2b512 / SHA256 = whole-file
# readers.  First pass: every drive online.  Second pass (only when the first may pass): the first offDisks drives fail
# (badDisk) and reader 0 is nil — here both are "offline".
H, B2, SH = "HighwayHash256S", "BLAKE2b512", "SHA256"
DECODE_TABLE_FULL = [
    (2, 4, 0, MiB, MiB, 0, MiB, B2, False, False), (3, 6, 0, MiB, MiB, 0, MiB, SH, False, False), (4, 8, 0, MiB, MiB, 0, MiB, H, False, False),
    (5, 10, 0, MiB, MiB, 1, MiB - 1, B2, False, False), (6, 12, 0, MiB, MiB, MiB, 0, B2, False, False), (7, 14, 0, MiB, MiB, 3, 1024, H, False, False),
    (8, 16, 0, MiB, MiB, 4, 8 * 1024, H, False, False), (7, 14, 7, MiB, MiB, MiB, 1, H, True, False), (6, 12, 6, MiB, MiB, 0, MiB, H, False, False),
    (5, 10, 5, MiB, MiB, 0, MiB, B2, False, False), (4, 8, 4, MiB, MiB, 0, MiB, SH, False, False), (3, 6, 3, MiB, MiB, 0, MiB, H, False, False),
    (2, 4, 2, MiB, MiB, 0, MiB, H, False, False), (2, 4, 1, MiB, MiB, 0, MiB, H, False, False), (3, 6, 2, MiB, MiB, 0, MiB, H, False, False),
    (4, 8, 3, 2 * MiB, MiB, 0, MiB, H, False, False), (5, 10, 6, MiB, MiB, 0, MiB, H, False, True), (5, 10, 2, MiB, 2 * MiB, MiB, MiB, H, False, False),
    (5, 10, 1, MiB, MiB, 0, MiB, B2, False, False), (6, 12, 3, MiB, MiB, 0, MiB, SH, False, False), (6, 12, 7, MiB, MiB, 0, MiB, H, False, True),
    (8, 16, 8, MiB, MiB, 0, MiB, H, False, False), (8, 16, 9, MiB, MiB, 0, MiB, H, False, True), (8, 16, 7, MiB, MiB, 0, MiB, H, False, False),
    (2, 4, 1, MiB, MiB, 0, MiB, H, False, False), (2, 4, 0, MiB, MiB, 0, MiB, H, False, False), (2, 4, 0, MiB, MiB + 1, 0, MiB + 1, B2, False, False),
    (2, 4, 0, MiB, 2 * MiB, 12, MiB + 17, B2, False, False), (3, 6, 0, MiB, 2 * MiB, 1023, MiB + 1024, H, False, False),
    (4, 8, 0, MiB, 2 * MiB, 11, MiB + 2 * 1024, H, False, False), (6, 12, 0, MiB, 2 * MiB, 512, MiB + 8 * 1024, H, False, False),
    (8, 16, 0, MiB, 2 * MiB, MiB, MiB - 1, H, False, False), (2, 4, 0, MiB, MiB, -1, 3, H, True, False), (2, 4, 0, MiB, MiB, 1024, -1, H, True, False),
    (4, 6, 0, MiB, MiB, 0, MiB, B2, False, False), (4, 6, 1, MiB, 2 * MiB, 12, MiB + 17, B2, False, False),
    (4, 6, 3, MiB, 2 * MiB, 1023, MiB + 1024, H, False, True), (8, 12, 4, MiB, 2 * MiB, 11, MiB + 2 * 1024, H, False, False),
]


@pytest.mark.parametrize("row", range(len(DECODE_TABLE_FULL)))
def test_erasure_decode_full_table(mb, oracle, row):
    k, n, off, bs, size, offset, length, algo, should_fail, should_fail_quorum = DECODE_TABLE_FULL[row]
    m = n - k
    data = rand(size, 1000 + row)
    whole = algo != H
    if whole:
        code = {B2: mb.BLAKE2B512, SH: mb.SHA256}[algo]
        c = mb.Codec(k, m, bs, algo=code)
        files, sums = c.encode_whole(data)
        ofiles, osums = oracle.erasure_encode(k, m, bs, {B2: oracle.BLAKE2B512, SH: oracle.SHA256}[algo], data)
        for i in range(n):
            assert np.array_equal(files[i], ofiles[i]) and sums[i] == osums[i]
        run = lambda fl: c.decode_whole(fl, sums, offset, length, size)
    else:
        c = mb.Codec(k, m, bs)
        files = c.encode(data)
        run = lambda fl: c.decode(fl, offset, length, size)
    try:
        out, hint = run(files)
        assert not should_fail, "should fail but it passed"
        assert hint == 0 and np.array_equal(out, data[offset:offset + length])
    except mb.MecError as e:
        assert should_fail, f"should pass but failed with {e}"
        c.close()
        return
    fl = [None if (j < off or (off > 0 and j == 0)) else files[j] for j in range(n)]
    try:
        out, hint = run(fl)
        assert not should_fail_quorum, "should fail with a quorum error but it passed"
        assert np.array_equal(out, data[offset:offset + length])
    except mb.MecError as e:
        assert should_fail_quorum and e.code == -10, f"should pass but failed with {e}"
    c.close()


@pytest.mark.parametrize("algo", ["SHA256", "BLAKE2b512", "HighwayHash256"])
def test_whole_file_decode_and_heal_with_bitrot(mb, oracle, algo):
    """wholeBitrotReader: a shard file whose whole-file digest is wrong is errFileCorrupt — dropped, replaced by the next drive,
    reported; Heal rebuilds stale shard files and their sums and still returns the side-band error."""
    code = {"SHA256": mb.SHA256, "BLAKE2b512": mb.BLAKE2B512, "HighwayHash256": mb.HIGHWAYHASH256}[algo]
    k, m, bs, size = 6, 4, MiB, 5 * MiB + 777
    n = k + m
    data = rand(size, 4242)
    c = mb.Codec(k, m, bs, algo=code)
    files, sums = c.encode_whole(data)
    bad = [f.copy() for f in files]
    bad[1][12345] ^= 0x20
    bad[7][0] ^= 0x01
    srcs = [None if i in (0, 3) else bad[i] for i in range(n)]        # readers 1,2,4,5,6,7 first; 1 and 7 are corrupt -> 8, 9 step in
    out, hint = c.decode_whole(srcs, sums, 3, size - 10, size)
    assert hint == -7 and np.array_equal(out, data[3:size - 7])
    out, hint = c.decode_whole([None if i in (0, 3) else files[i] for i in range(n)], sums, 0, size, size)
    assert hint == 0 and np.array_equal(out, data)
    stale = [i in (0, 9) for i in range(n)]
    srcs = [None if stale[i] else bad[i] for i in range(n)]
    outs, osums, rc, corrupt = c.heal_whole(srcs, sums, stale, size)
    assert rc == -7 and list(np.nonzero(corrupt)[0]) == [1, 7]         # readers 1..6 first: 1 drops, 7 steps in and drops, 8 steps in
    for i in (0, 9):
        assert np.array_equal(outs[i], files[i]) and osums[i] == sums[i]
    stale = [i in (0, 3, 9) for i in range(n)]
    outs, osums, rc, corrupt = c.heal_whole([None if stale[i] else files[i] for i in range(n)], sums, stale, size)
    assert rc == 0 and not corrupt.any()
    for i in (0, 3, 9):
        assert np.array_equal(outs[i], files[i]) and osums[i] == sums[i]
    # too many corrupt files: read quorum
    for i in (2, 4, 5, 6):
        bad[i][99] ^= 0xFF
    with pytest.raises(mb.MecError) as ei:
        c.decode_whole([None if i in (0, 3) else bad[i] for i in range(n)], sums, 0, size, size)
    assert ei.value.code == -10
    c.close()


@pytest.mark.parametrize("pinned", [False, True])
def test_batcher_merges_concurrent_puts(mb, oracle, pinned):
    """Many threads PUT objects of different sizes through one mec_batcher: every caller gets exactly the frames a private
    mec_encode would have produced, and the calls were merged into far fewer launches than there were requests.
    pinned: page-locked buffers -> the gather / scatter kernels move the batch; pageable -> per-request copies."""
    import threading
    k, m, bs = 12, 4, MiB
    sizes = [MiB, 2 * MiB, MiB + 4321, 3 * MiB + 7, 100, MiB - 1, 5 * MiB, MiB, 33, 2 * MiB + 1]
    nthreads, rounds = 32, 6
    bat = mb.Batcher(k, m, bs, max_batch_blocks=128, max_wait_us=2000)
    datas = [rand(sizes[t % len(sizes)], 900 + t) for t in range(nthreads)]
    if pinned:
        pd = []
        for d in datas:
            a = mb.pinned_array(d.size)[:d.size]
            a[:] = d
            pd.append(a)
        datas = pd
    want = [oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, d)[0] for d in datas]
    errs = []

    def worker(t):
        try:
            for _ in range(rounds):
                files = bat.encode(datas[t], pinned=pinned)
                for i in range(k + m):
                    if not np.array_equal(files[i], want[t][i]):
                        errs.append((t, i))
                if pinned:
                    for f in files:
                        mb.lib().mec_free_pinned(f.ctypes.data)
        except Exception as e:  # noqa: BLE001
            errs.append((t, repr(e)))
    th = [threading.Thread(target=worker, args=(t,)) for t in range(nthreads)]
    [x.start() for x in th]
    [x.join() for x in th]
    assert not errs, errs[:5]
    assert bat.stat("requests") == nthreads * rounds
    assert bat.stat("batches") < bat.stat("requests")        # callers were coalesced
    assert (bat.stat("kernel_batches") > 0) == pinned
    # quorum and empty objects behave like mec_encode
    with pytest.raises(mb.MecError) as ei:
        bat.encode(rand(1000, 1), online=[True] * 12 + [False] * 4, write_quorum=13)
    assert ei.value.code == -11
    assert all(f.size == 0 for f in bat.encode(b""))
    bat.close()


def test_jit_disk_cache_across_processes(tmp_path):
    """A specialised kernel compiled by one process is loaded from MEC_JIT_CACHE_DIR by the next one (no NVRTC compile)."""
    import os
    import subprocess
    import sys
    script = r'''
import sys, json
sys.path.insert(0, %r); sys.path.insert(0, %r)
import numpy as np, minio_b200 as mb
k, m, bs, size = 10, 4, 1 << 20, 6 * (1 << 20) + 99
d = np.random.default_rng(3).integers(0, 256, size, dtype=np.uint8)
c = mb.Codec(k, m, bs); c.set_option("jit", 1)
files = c.encode(d)                                   # RS(10,4) has no compiled kernel: NVRTC-specialised encode
stale = [i in (1, 12) for i in range(k + m)]
outs = c.heal([None if stale[i] else files[i] for i in range(k + m)], stale, size)   # and a specialised decode matrix
ok = all(np.array_equal(outs[i], files[i]) for i in (1, 12))
print(json.dumps({"ok": bool(ok), "disk_hits": c.stat("jit_disk_hits"), "jit_ms": c.stat("jit_ms"), "jit_launches": c.stat("jit_launches")}))
''' % (os.path.dirname(os.path.dirname(os.path.abspath(__file__))), os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, MEC_JIT_CACHE_DIR=str(tmp_path))
    import json
    r1 = json.loads(subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, check=True).stdout.strip().split("\n")[-1])
    assert r1["ok"] and r1["disk_hits"] == 0 and r1["jit_launches"] > 0
    assert len([f for f in os.listdir(tmp_path) if f.endswith(".cubin")]) >= 1
    r2 = json.loads(subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, check=True).stdout.strip().split("\n")[-1])
    assert r2["ok"] and r2["disk_hits"] >= 1 and r2["jit_launches"] > 0
    assert r2["jit_ms"] < r1["jit_ms"]


def test_jit_prewarm_serves_first_degraded_get(mb, oracle, tmp_path, monkeypatch):
    """mec_jit_prewarm: after the background compiles finish, the FIRST degraded GET of a single-drive failure already runs a
    specialised kernel (default jit = -1 would otherwise serve it with the runtime-matrix kernel until 32 MiB have been seen)."""
    import time
    k, m, bs, size = 4, 2, MiB, 3 * MiB + 5
    c = mb.Codec(k, m, bs)
    c.set_option("small_blocks", 0)  # a 3-block GET would otherwise take the latency kernel, which never uses specialised matrices
    queued = mb.lib().mec_jit_prewarm(c.h)
    assert queued == k * 4
    c0 = c.stat("jit_compiles")
    deadline = time.time() + 120
    while c.stat("jit_compiles") + c.stat("jit_disk_hits") - c0 < 1 and time.time() < deadline:
        time.sleep(0.2)
    # wait for the queue to drain: compiles are sequential on one background thread
    last, stable = -1, 0
    while stable < 5 and time.time() < deadline:
        cur = c.stat("jit_compiles")
        stable = stable + 1 if cur == last else 0
        last = cur
        time.sleep(0.5)
    data = rand(size, 31)
    files = c.encode(data)
    j0 = c.stat("jit_launches")
    out, hint = c.decode([files[0], None] + files[2:], 0, size, size)     # data drive 1 is gone: its first GET
    assert hint == 0 and np.array_equal(out, data)
    assert c.stat("jit_launches") > j0
    c.close()


@pytest.mark.parametrize("pinned", [True, False])
def test_batcher_merges_concurrent_gets(mb, oracle, pinned):
    """Concurrent GETs through one mec_batcher: requests that see the same drives online share a launch; different ranges, sizes with
    short last blocks, two different failure patterns, and one object with bitrot (redone alone with exact fail-over)."""
    import threading
    k, m, bs = 12, 4, MiB
    sizes = [MiB, 3 * MiB + 4321, 2 * MiB, 100, 5 * MiB + 1, MiB - 1]
    nthreads, rounds = 24, 4
    enc = mb.Codec(k, m, bs)
    bat = mb.Batcher(k, m, bs, max_batch_blocks=128, max_wait_us=2000)
    mk = (lambda a: (lambda p: (p.__setitem__(slice(None), a), p)[1])(mb.pinned_array(a.size)[:a.size])) if pinned else (lambda a: a)
    objs = []
    for t in range(nthreads):
        d = rand(sizes[t % len(sizes)], 700 + t)
        files = [mk(f) for f in enc.encode(d)]
        objs.append((d, files))
    S = enc.shard_size()
    # thread 5's object has a corrupt frame on a reader that WILL be used
    objs[5][1][4][1 * 0 + 40] ^= 0x08
    errs = []

    def worker(t):
        d, files = objs[t]
        n = d.size
        offline = (0, 3, 13) if t % 4 else (1, 2)          # two failure patterns -> two reader sets
        fl = [None if i in offline else files[i] for i in range(k + m)]
        rng = np.random.default_rng(t)
        try:
            for it in range(rounds):
                off = 0 if it == 0 else int(rng.integers(0, n))
                ln = n - off if it == 0 else int(rng.integers(0, n - off + 1))
                dst = mb.pinned_array(max(ln, 1))[:max(ln, 1)] if pinned else None
                out, hint = bat.decode(fl, off, ln, n, dst=dst)
                if not np.array_equal(out, d[off:off + ln]):
                    errs.append((t, it, "bytes"))
                want_hint = -7 if (t == 5 and 4 not in offline and ln > 0 and off < MiB) else 0
                if t != 5 and hint != 0:
                    errs.append((t, it, "hint", hint))
                if t == 5 and it == 0 and hint != want_hint:
                    errs.append((t, it, "hint5", hint))
                if pinned and dst is not None:
                    mb.lib().mec_free_pinned(dst.ctypes.data)
        except Exception as e:  # noqa: BLE001
            errs.append((t, repr(e)))
    th = [threading.Thread(target=worker, args=(t,)) for t in range(nthreads)]
    [x.start() for x in th]
    [x.join() for x in th]
    assert not errs, errs[:6]
    if pinned:
        assert bat.stat("kernel_batches") > 0 and bat.stat("batches") < nthreads * rounds
    with pytest.raises(mb.MecError) as ei:
        bat.decode([None] * 5 + list(objs[0][1][5:]), 0, 10, objs[0][0].size)
    assert ei.value.code == -10
    bat.close(); enc.close()


def test_full_size_properties_config2_and_3(mb, oracle):
    """BASELINE.json's full sizes (config 2: 10 GiB stream = 10240 blocks; config 3: 4 shards erased) through size-independent
    properties: encode -> erase -> reconstruct round trip over EVERY block (rebuilt shards and their digests equal the originals,
    no frame flagged), linearity of the parity (parity(a ^ b) == parity(a) ^ parity(b)), oracle spot checks at both ends."""
    import torch
    k, m, bs, nblocks = 12, 4, MiB, 10240
    dev = torch.device("cuda:0")
    S = 87382
    pitch = (S + 15) // 16 * 16
    fp = (32 + S + 15) // 16 * 16
    g = torch.Generator(device=dev); g.manual_seed(0x4D494E494F00 + 2)
    src = torch.empty(nblocks * bs, dtype=torch.uint8, device=dev)
    for o0 in range(0, nblocks * bs, 1 << 30):
        n = min(1 << 30, nblocks * bs - o0)
        src[o0:o0 + n] = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev, generator=g)
    par = torch.zeros((nblocks * m, pitch), dtype=torch.uint8, device=dev)
    dig = torch.zeros((nblocks, k + m, 32), dtype=torch.uint8, device=dev)
    c = mb.Codec(k, m, bs)
    c.set_option("jit", 1)
    st = torch.cuda.current_stream().cuda_stream
    c.encode_blocks_device(src.data_ptr(), src.numel(), par.data_ptr(), pitch, dig.data_ptr(), st)
    torch.cuda.synchronize()
    for b in (0, nblocks - 1):   # oracle at both ends of the stream
        sh = oracle.encode_data(k, m, src[b * bs:(b + 1) * bs].cpu().numpy(), fast=True)
        for j in range(m):
            assert np.array_equal(par[b * m + j, :S].cpu().numpy(), sh[k + j])
        for i in range(k + m):
            assert dig[b, i].cpu().numpy().tobytes() == oracle.hh256(sh[i], fast=True)
    # linearity on a slice of 256 blocks: GF(2^8) encode is linear over XOR
    nb2 = 256
    a, bsl = src[:nb2 * bs], src[4096 * bs:(4096 + nb2) * bs]
    x = a ^ bsl
    px = torch.zeros((nb2 * m, pitch), dtype=torch.uint8, device=dev)
    dx = torch.zeros((nb2, k + m, 32), dtype=torch.uint8, device=dev)
    c.encode_blocks_device(x.data_ptr(), x.numel(), px.data_ptr(), pitch, dx.data_ptr(), st)
    torch.cuda.synchronize()
    assert torch.equal(px[:, :S], par[:nb2 * m, :S] ^ par[4096 * m:(4096 + nb2) * m, :S])
    del x, px, dx
    # frames of all 16 drives in one arena, erase {0, 5, 12, 15}, rebuild all four, compare with what was erased
    arena = torch.zeros((k + m, nblocks, fp), dtype=torch.uint8, device=dev)
    src2, par3 = src.view(nblocks, bs), par.view(nblocks, m, pitch)
    for i in range(k + m):
        arena[i, :, :32] = dig[:, i]
        if i < k:
            lo, hi = i * S, min((i + 1) * S, bs)
            arena[i, :, 32:32 + hi - lo] = src2[:, lo:hi]
        else:
            arena[i, :, 32:32 + S] = par3[:, i - k, :S]
    erased = [0, 5, 12, 15]
    ptrs = [0 if i in erased else arena[i].data_ptr() for i in range(k + m)]
    want = [1 if i in erased else 0 for i in range(k + m)]
    out = torch.zeros((nblocks * 4, pitch), dtype=torch.uint8, device=dev)
    odig = torch.zeros((nblocks, k + 4, 32), dtype=torch.uint8, device=dev)
    cor = torch.zeros((nblocks, k), dtype=torch.uint8, device=dev)
    c.reconstruct_device(ptrs, fp, nblocks, want, 0, out.data_ptr(), pitch, odig.data_ptr(), cor.data_ptr(), st)
    torch.cuda.synchronize()
    assert int(cor.sum().item()) == 0
    o3 = out.view(nblocks, 4, pitch)
    for q, i in enumerate(erased):
        assert torch.equal(o3[:, q, :S], arena[i, :, 32:32 + S]), i
        assert torch.equal(odig[:, k + q], arena[i, :, :32]), i
    # a single flipped bit anywhere in a survivor is flagged for exactly that frame
    arena[7, 9999, 32 + 12345] ^= 4
    c.reconstruct_device(ptrs, fp, nblocks, want, 0, out.data_ptr(), pitch, odig.data_ptr(), cor.data_ptr(), st)
    torch.cuda.synchronize()
    assert int(cor.sum().item()) == 1 and int(cor[9999, 5].item()) == 1   # shard 7 is reader position 5 (0 and 5 are offline)
    c.close()


def test_bitrot_verify_batch_deep_scan(mb, oracle):
    """Deep scan of every part file of several objects in one call (pipelined chunks, launches shared across files): good files,
    a flipped data byte, a flipped digest byte, a truncated file, an empty part; against the oracle's bitrotVerify."""
    k, m, bs = 12, 4, MiB
    c = mb.Codec(k, m, bs)
    S = c.shard_size()
    files, plens, want = [], [], []
    for size, seed in ((40 * MiB + 777, 1), (MiB, 2), (3 * MiB + 5, 3), (100, 4)):
        d = rand(size, 600 + seed)
        fs = c.encode(d)
        for i in range(k + m):
            files.append(fs[i]); plens.append(c.shard_file_size(size)); want.append(0)
    bad = [f.copy() for f in files]
    bad[3][17 * (32 + S) + 32 + 99] ^= 1; want[3] = -7           # data byte of frame 17
    bad[20][5] ^= 0x10; want[20] = -7                             # digest byte of the only frame of a 1 MiB object's shard
    bad[40] = bad[40][:-1].copy(); want[40] = -7                  # wrong length (cmd/bitrot.go:183)
    bad[50][bad[50].size - 1] ^= 0x80; want[50] = -7              # last byte of a short last frame
    got = c.bitrot_verify_batch(bad, plens)
    assert got == want
    for i in (0, 3, 20, 50):
        assert oracle.bitrot_verify(oracle.HIGHWAYHASH256S, bad[i], plens[i], S) == want[i]
        assert c.bitrot_verify(bad[i], plens[i]) == want[i]
    assert c.bitrot_verify_batch([np.zeros(0, dtype=np.uint8)], [0]) == [0]
    c.close()


def test_handles_of_different_width_share_the_runtime_matrix_kernels(mb, oracle):
    """The runtime-matrix kernels (heal / degraded GET of small objects) are one function for every (k, r); their dynamic
    shared-memory limit is a per-function attribute.  A narrow handle used between two calls of a wide one must not lower it."""
    rng = np.random.default_rng(77)
    wide, narrow = mb.Codec(12, 4, MiB), mb.Codec(4, 2, MiB)
    dw, dn = rng.integers(0, 256, 3 * MiB + 11, dtype=np.uint8), rng.integers(0, 256, 2 * MiB + 5, dtype=np.uint8)
    fw, fn = wide.encode(dw), narrow.encode(dn)
    for _ in range(2):
        for c, d, f, k in ((wide, dw, fw, 12), (narrow, dn, fn, 4), (wide, dw, fw, 12)):
            n = len(f)
            off = [None if i in (0, k) else f[i] for i in range(n)]
            out, hint = c.decode(off, 0, d.size, d.size)
            assert np.array_equal(out, d)
            healed = c.heal(off, [i in (0, k) for i in range(n)], d.size)
            assert np.array_equal(healed[0], f[0]) and np.array_equal(healed[k], f[k])
    wide.close()
    narrow.close()


def test_deep_scan_over_many_small_part_files_is_one_launch_per_chunk(mb, oracle):
    """A scan over hundreds of part files of one short frame each (small objects of odd sizes): every frame of a chunk is staged by one
    batched copy call and hashed by ONE launch with a per-frame length table (latency kernel, FusedParams::block_len); verdicts equal the
    oracle's, with and without that path."""
    k, m, bs = 12, 4, MiB
    c = mb.Codec(k, m, bs)
    S = c.shard_size()
    rng = np.random.default_rng(12)
    files, plens = [], []
    for o in range(24):
        size = int(rng.integers(1, 2 * MiB + 500_000))   # 1 to 3 frames per part file, the last one short
        fs = c.encode(rng.integers(0, 256, size, dtype=np.uint8))
        files += fs
        plens += [c.shard_file_size(size)] * len(fs)
    want = [0] * len(files)
    for i, pos in ((5, 3), (77, 40), (200, -1), (333, 31)):
        files[i] = files[i].copy()
        files[i][pos] ^= 0x20
        want[i] = -7
    for i in (5, 77, 200, 333):
        assert oracle.bitrot_verify(oracle.HIGHWAYHASH256S, files[i], plens[i], S) == -7
    l0 = c.launches
    assert c.bitrot_verify_batch(files, plens) == want
    one = c.launches - l0
    c.set_option("small_blocks", 0)
    l0 = c.launches
    assert c.bitrot_verify_batch(files, plens) == want
    assert one <= 3 and c.launches - l0 > 100, (one, c.launches - l0)
    c.close()


def test_split_padding_is_zero_over_stale_staging(mb, oracle):
    """The latency kernel fetches with cp.async whose source size is trimmed at the last valid byte of every row (hardware zero fill
    for the rest: Split's padding, cmd/erasure-coding.go:81).  The staging buffer of a handle is reused: after a large object of
    0xFF bytes, small objects whose last shards are partly or wholly padding must still match the oracle bit for bit."""
    k, m, bs = 12, 4, MiB
    c = mb.Codec(k, m, bs)
    c.encode(np.full(5 * MiB + 77, 0xFF, dtype=np.uint8))          # every staging byte a later call could over-read is now 0xFF
    for size in (1, 11, 12, 13, 33, 100, 4097, 65536 + 5, 87382 * 11 + 3, MiB - 1, MiB + 1, 2 * MiB + 87382 * 5 + 9):
        d = rand(size, 4000 + size % 97)
        files = c.encode(d)
        want, _ = oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, d)
        for i in range(k + m):
            assert np.array_equal(files[i], want[i]), (size, i)
        out, hint = c.decode([None, files[1], None] + files[3:], 0, size, size)
        assert hint == 0 and np.array_equal(out, d), size
        c.encode(np.full(3 * MiB, 0xFF, dtype=np.uint8))            # dirty the staging again
    c.close()


@pytest.mark.parametrize("k,m", [(10, 4), (7, 5), (6, 3), (8, 2)])
def test_nvrtc_specialised_encode_fetches_tiles_with_one_request(mb, oracle, k, m):
    """Geometries without a compiled kernel: with jit = 1 the encode runs the NVRTC-specialised kernel, which since round 2 uses the
    one-3-D-TMA-request-per-tile fetch of the compiled ones (S mod 16 = 10, 5, 11, 0 here).  Frames equal the oracle's for whole and
    ragged objects; the option no_rows3d selects the row-by-row fetch of the same specialisation."""
    bs = MiB
    for rows3d_off in (0, 1):
        c = mb.Codec(k, m, bs)
        c.set_option("jit", 1)
        c.set_option("eb", 4)   # the CTA shape of the specialised kernels, also for launches this small (the default would shrink it)
        c.set_option("no_rows3d", rows3d_off)
        for size in (8 * MiB, 12 * MiB + 777, 4 * MiB - 5):   # host pipeline chunks of four blocks: 2 + 3 specialised launches, the rest generic
            d = rand(size, 600 + k + size % 13)
            files = c.encode(d)
            want, _ = oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, d)
            for i in range(k + m):
                assert np.array_equal(files[i], want[i]), (k, m, size, i, rows3d_off)
        assert c.stat("jit_launches") >= 3
        c.close()
