#!/bin/bash
cd "${GRAFT_REPO_ROOT:-/root/repo}"
mkdir -p gpurun_out
cat > /tmp/san_case.py <<'PY'
import sys, numpy as np
sys.path.insert(0, '.'); sys.path.insert(0, 'tests')
import minio_b200 as mb, oracle_lib as o
rng = np.random.default_rng(3)
for (k, m, bs, n) in [(12, 4, 1 << 20, (1 << 20) + 4321), (8, 4, 1 << 20, 2 * (1 << 20) + 999), (4, 2, 65536, 3 * 65536 + 17), (7, 5, 1 << 20, 600000)]:
    data = rng.integers(0, 256, n, dtype=np.uint8)
    c = mb.Codec(k, m, bs)
    files = c.encode(data)
    want, _ = o.erasure_encode(k, m, bs, 3, data)
    assert all(np.array_equal(a, b) for a, b in zip(files, want))
    off = [None if i in (0, k) else files[i] for i in range(k + m)]
    out, hint = c.decode(off, 0, n, n)
    assert np.array_equal(out, data)
    for jit in (0, 1):
        c.set_option("jit", jit)
        healed = c.heal(off, [i in (0, k) for i in range(k + m)], n)
        assert np.array_equal(healed[0], files[0]) and np.array_equal(healed[k], files[k])
    assert c.bitrot_verify(files[1], c.shard_file_size(n)) == 0
    c.close()
c = mb.Codec(8, 8, 65536, algo=1)
d = rng.integers(0, 256, 200000, dtype=np.uint8)
f, s = c.encode_whole(d)
out, hint = c.decode_whole([None, None] + f[2:], s, 5, 150000, 200000)       # whole-file readers: verify + rebuild from raw shards
assert hint == 0 and np.array_equal(out, d[5:150005])
c.close()
# round 2: multi-chunk pipelined decode with fail-over (run-wise 3-D fetch from the arena), scatter-gather encode, CRCs, the batcher
k, m, bs, n = 12, 4, 1 << 20, 40 * (1 << 20) + 77
c = mb.Codec(k, m, bs); c.set_option("checksums", 7); c.set_option("chunk_blocks", 8)
data = rng.integers(0, 256, n, dtype=np.uint8)
files, dd = c.encode_sg(data)
crc, ln = c.last_checksums()
import zlib
assert ln == n and crc[0] == zlib.crc32(data.tobytes())
full = c.encode(data)
bad = [x.copy() for x in full]; bad[3][20 * (32 + c.shard_size()) + 40] ^= 1
out, hint = c.decode([None if i in (0, 9) else bad[i] for i in range(16)], 12345, n - 20000, n)
assert hint == -7 and np.array_equal(out, data[12345:n - 7655])
c.close()
import threading
bat = mb.Batcher(k, m, bs, max_batch_blocks=32, max_wait_us=500)
pin = [mb.pinned_array(sz)[:sz] for sz in ((1 << 20), (1 << 20) + 333, 2 * (1 << 20), 4097)]
for a in pin: a[:] = rng.integers(0, 256, a.size, dtype=np.uint8)
want = [o.erasure_encode(k, m, bs, 3, a)[0] for a in pin]
errs = []
def work(t):
    for _ in range(2):
        fs = bat.encode(pin[t % 4], pinned=(t < 4))
        if not all(np.array_equal(x, y) for x, y in zip(fs, want[t % 4])): errs.append(t)
th = [threading.Thread(target=work, args=(t,)) for t in range(8)]
[x.start() for x in th]; [x.join() for x in th]
assert not errs, errs
bat.close()
# one merged heal round: four heals of stale drive 1 in one batch (staging, fused reconstruct with digests, heal scatter kernel)
bat = mb.Batcher(k, m, bs, max_batch_blocks=sum(-(-a.size // bs) for a in pin), max_wait_us=500000)
rd = [[None if i == 1 else mb.pinned_array(w[i].size) for i in range(k + m)] for w in want]
for r, w in zip(rd, want):
    for i, f in enumerate(r):
        if f is not None: f[:] = w[i]
res = [None] * 4
def heal(t): res[t] = bat.heal(rd[t], [i == 1 for i in range(k + m)], pin[t].size, pinned=True)
th = [threading.Thread(target=heal, args=(t,)) for t in range(4)]
[x.start() for x in th]; [x.join() for x in th]
assert all(r[1] == 0 and np.array_equal(r[0][1], want[t][1]) for t, r in enumerate(res)), [r[1] for r in res]
assert bat.stat("kernel_batches") == 1 and bat.stat("requests") == 4
bat.close()
# mixed erasure patterns (MEC_BATCHER_MIX_PATTERNS): four GETs of the one-block object with a different drive offline each (shard 0
# and 5 rebuilt; 13 and 15: parity, nothing rebuilt), then four heals of different stale sets (one and two drives) — each ONE latency
# launch with a decode plan per block
bat = mb.Batcher(k, m, bs, max_batch_blocks=8, max_wait_us=500000, mix_patterns=True)
offl = [0, 5, 13, 15]
gd = [[None if i == offl[t] else mb.pinned_array(want[3][i].size) for i in range(k + m)] for t in range(4)]
for t, r in enumerate(gd):
    for i, f in enumerate(r):
        if f is not None: f[:] = want[3][i]
res = [None] * 4
def get(t): res[t] = bat.decode(gd[t], 0, pin[3].size, pin[3].size, dst=mb.pinned_array(pin[3].size))
th = [threading.Thread(target=get, args=(t,)) for t in range(4)]
[x.start() for x in th]; [x.join() for x in th]
assert all(np.array_equal(r[0], pin[3]) and r[1] == 0 for r in res)
assert bat.stat("batches") == 1 and bat.stat("mixed_batches") == 1 and bat.stat("patterns") == 3
bat.close()
stale = [{0}, {3, 14}, {15}, {7, 8}]
bat = mb.Batcher(k, m, bs, max_batch_blocks=sum(-(-a.size // bs) for a in pin), max_wait_us=500000, mix_patterns=True)
hd = [[None if i in stale[t] else mb.pinned_array(want[t][i].size) for i in range(k + m)] for t in range(4)]
for t, r in enumerate(hd):
    for i, f in enumerate(r):
        if f is not None: f[:] = want[t][i]
def heal(t): res[t] = bat.heal(hd[t], [i in stale[t] for i in range(k + m)], pin[t].size, pinned=True)
th = [threading.Thread(target=heal, args=(t,)) for t in range(4)]
[x.start() for x in th]; [x.join() for x in th]
assert all(r[1] == 0 and all(np.array_equal(r[0][i], want[t][i]) for i in stale[t]) for t, r in enumerate(res))
assert bat.stat("batches") == 1 and bat.stat("mixed_batches") == 1 and bat.stat("patterns") == 4
bat.close()
# one merged batch of pinned PUTs with mixed checksum masks (mec_batcher_encode_crc): segmented CRC kernels over the staged batch;
# the 2 MiB object spans eight 256 KiB regions
objs = pin
masks = [7, 1, 6, 0]
bat = mb.Batcher(k, m, bs, max_batch_blocks=sum(-(-a.size // bs) for a in objs), max_wait_us=500000)
res = [None] * len(objs)
def put(t): res[t] = bat.encode(objs[t], pinned=True, checksums=masks[t]) if masks[t] else (bat.encode(objs[t], pinned=True), None)
th = [threading.Thread(target=put, args=(t,)) for t in range(len(objs))]
[x.start() for x in th]; [x.join() for x in th]
for t, (fs, crc) in enumerate(res):
    if masks[t]:
        w = o.crcs(objs[t])
        assert w[0] == zlib.crc32(objs[t].tobytes())
        assert crc == tuple(v if masks[t] & (1 << i) else 0 for i, v in enumerate(w)), (t, crc, w)
assert all(np.array_equal(x, y) for x, y in zip(res[0][0], want[0]))
assert bat.stat("batches") == 1 and bat.stat("crc_requests") == 3
bat.close()
# one merged transcode round: four moves RS(12,4) -> RS(6,2) with source drive 1 offline in one batch (staging, fused reconstruct,
# batch_transcode_resplit_kernel, the destination's encode and frame scatter)
bat = mb.Batcher(k, m, bs, max_batch_blocks=sum(-(-a.size // bs) for a in pin), max_wait_us=500000, dst=(6, 2))
tw = [o.erasure_encode(6, 2, bs, 3, a)[0] for a in pin]
res = [None] * 4
def move(t): res[t] = bat.transcode(rd[t], pin[t].size, pinned=True)
th = [threading.Thread(target=move, args=(t,)) for t in range(4)]
[x.start() for x in th]; [x.join() for x in th]
assert all(r[1] == 0 and all(np.array_equal(x, y) for x, y in zip(r[0], tw[t])) for t, r in enumerate(res))
assert bat.stat("batches") == 1 and bat.stat("transcodes") == 4
bat.close()
# legacy parts: RS(12,4) at 10 MiB blocks -> RS(6,2) at 1 MiB blocks, one merged batch of two moves (a source block run that
# straddles the edge between full and short destination blocks) and one mec_transcode with source drive 1 offline
lbs = 10 << 20
ldat = [np.random.default_rng(40 + t).integers(0, 256, n, dtype=np.uint8) for t, n in enumerate((lbs + (1 << 19) + 7, 3 << 19))]
lsrc = []
for a in ldat:
    fs = o.erasure_encode(k, m, lbs, 3, a)[0]
    pf = [mb.pinned_array(f.size) for f in fs]
    for x, f in zip(pf, fs): x[:] = f
    lsrc.append(pf)
ltw = [o.erasure_encode(6, 2, 1 << 20, 3, a)[0] for a in ldat]
bat = mb.Batcher(k, m, lbs, max_batch_blocks=3, max_wait_us=500000, dst=(6, 2, 1 << 20))
res = [None] * 2
def lmove(t): res[t] = bat.transcode(lsrc[t], ldat[t].size, pinned=True)
th = [threading.Thread(target=lmove, args=(t,)) for t in range(2)]
[x.start() for x in th]; [x.join() for x in th]
assert all(r[1] == 0 and all(np.array_equal(x, y) for x, y in zip(r[0], ltw[t])) for t, r in enumerate(res))
assert bat.stat("batches") == 1 and bat.stat("transcodes") == 2
bat.close()
lc, ld = mb.Codec(k, m, lbs), mb.Codec(6, 2, 1 << 20)
outs, hint = lc.transcode([None if i == 1 else f for i, f in enumerate(lsrc[0])], ldat[0].size, ld)
assert hint == 0 and all(np.array_equal(x, y) for x, y in zip(outs, ltw[0]))
# whole-file moves (mec_batcher_transcode_whole): four RS(12,4) parts written with SHA256 -> RS(6,2) in one merged batch with
# source drive 1 offline (one batched staging copy, ONE whole_hash_kernel launch over shard files of four lengths,
# batch_whole_rows_kernel, the merged reconstruct without digests, re-split, encode and scatter), then a fifth move whose chosen
# reader 5 has a flipped byte: its merged batch fails the digest check and it is redone on the private pair
wdat = [np.random.default_rng(60 + t).integers(0, 256, n, dtype=np.uint8) for t, n in enumerate((1 << 19, (1 << 20) + 5, 77, 2 * (1 << 20) + 999, 300001))]
wsrc, wsum = [], []
for a in wdat:
    fs, ss = o.erasure_encode(k, m, bs, 1, a)
    pf = [mb.pinned_array(f.size) for f in fs]
    for x, f in zip(pf, fs): x[:] = f
    wsrc.append(pf); wsum.append(ss)
wsrc[4][5][100] ^= 1
wtw = [o.erasure_encode(6, 2, bs, 3, a)[0] for a in wdat]
bat = mb.Batcher(k, m, bs, max_batch_blocks=8, max_wait_us=500000, dst=(6, 2))
res = [None] * 5
def wmove(t): res[t] = bat.transcode_whole([None if i == 1 else f for i, f in enumerate(wsrc[t])], wsum[t], wdat[t].size, 1, pinned=True)
th = [threading.Thread(target=wmove, args=(t,)) for t in range(4)]
[x.start() for x in th]; [x.join() for x in th]
assert all(r[1] == 0 and all(np.array_equal(x, y) for x, y in zip(r[0], wtw[t])) for t, r in enumerate(res[:4]))
assert bat.stat("batches") == 1 and bat.stat("transcodes_whole") == 4 and bat.stat("whole_hash_launches") == 1
res[4] = bat.transcode_whole(wsrc[4], wsum[4], wdat[4].size, 1, pinned=True)
assert res[4][1] == -7 and all(np.array_equal(x, y) for x, y in zip(res[4][0], wtw[4]))
assert bat.stat("redone") == 1 and bat.stat("transcodes_whole_serial") == 1
bat.close()
# mixed GETs and heals of half-healed SHA256 parts (mec_batcher_decode_mixed / mec_batcher_heal_mixed): even drives hold
# HighwayHash256S frames, odd drives raw shard files.  Four GETs share one merged batch (frames of the streaming readers through the
# gather kernel, the whole-file readers' shard files staged whole and hashed in ONE whole_hash_kernel launch over a stream table of
# whole-file readers only, batch_whole_rows_kernel for their positions, the merged reconstruct with drive 2 offline, the GET scatter
# straight into the callers' buffers), then four heals of drive 15 in one merged batch (heal frame scatter)
hdat = [np.random.default_rng(80 + t).integers(0, 256, n, dtype=np.uint8) for t, n in enumerate((1 << 19, (1 << 20) + 5, 77, 2 * (1 << 20) + 999))]
hsrc, hsum, hwant = [], [], []
for a in hdat:
    sf, _ = o.erasure_encode(k, m, bs, 3, a)
    wf, ss = o.erasure_encode(k, m, bs, 1, a)
    fs = [sf[i] if i % 2 == 0 else wf[i] for i in range(k + m)]
    pf = [mb.pinned_array(max(f.size, 1))[:f.size] for f in fs]
    for x, f in zip(pf, fs): x[:] = f
    hsrc.append(pf); hsum.append([None if i % 2 == 0 else ss[i] for i in range(k + m)]); hwant.append(sf)
halg = [3 if i % 2 == 0 else 1 for i in range(k + m)]
bat = mb.Batcher(k, m, bs, max_batch_blocks=16, max_wait_us=500000)
res = [None] * 8
def hget(t): res[t] = bat.decode_mixed([None if i == 2 else f for i, f in enumerate(hsrc[t])], halg, hsum[t], 0, hdat[t].size, hdat[t].size, dst=mb.pinned_array(hdat[t].size))
def hheal(t): res[4 + t] = bat.heal_mixed(hsrc[t], halg, hsum[t], [i == 15 for i in range(k + m)], hdat[t].size, pinned=True)
for fn in (hget, hheal):
    th = [threading.Thread(target=fn, args=(t,)) for t in range(4)]
    [x.start() for x in th]; [x.join() for x in th]
assert all(r[1] == 0 and np.array_equal(r[0], hdat[t]) for t, r in enumerate(res[:4]))
assert all(np.array_equal(r[15], hwant[t][15]) for t, r in enumerate(res[4:]))
assert bat.stat("batches") == 2 and bat.stat("reads_whole") == 8 and bat.stat("whole_hash_launches") == 2 and bat.stat("redone") == 0
bat.close()
print("sanitizer case ok")
PY
echo "== memcheck"; timeout 1200 compute-sanitizer --tool memcheck --print-limit 20 python /tmp/san_case.py > gpurun_out/memcheck.txt 2>&1; echo rc=$?; grep -E "ERROR SUMMARY|sanitizer case ok|Invalid|out of bounds|misaligned" gpurun_out/memcheck.txt | head -12
echo "== racecheck"; timeout 1200 compute-sanitizer --tool racecheck --print-limit 20 python /tmp/san_case.py > gpurun_out/racecheck.txt 2>&1; echo rc=$?; grep -E "RACECHECK SUMMARY|sanitizer case ok|hazard" gpurun_out/racecheck.txt | head -12
echo "== synccheck"; timeout 1200 compute-sanitizer --tool synccheck --print-limit 20 python /tmp/san_case.py > gpurun_out/synccheck.txt 2>&1; echo rc=$?; grep -E "ERROR SUMMARY|sanitizer case ok|Barrier" gpurun_out/synccheck.txt | head -8

# The latency kernel (ec_small.cuh) at its pipeline edges: one stage + 1 and seven stages on one 3- and one 4-GF-warp geometry,
# 1-byte shards, a 1-byte last block, and RS(8,8) rebuilding 8 shards.  Every object has an allocation of exactly its length
# (PYTORCH_NO_CUDA_MEMORY_CACHING=1), so that memcheck sees any read past its last byte, including the zero-byte cp.async of a
# shard row that is all padding.
cat > /tmp/san_small.py <<'PY'
import sys, numpy as np, torch
sys.path.insert(0, '.'); sys.path.insert(0, 'tests')
import minio_b200 as mb, oracle_lib as o
st = torch.cuda.current_stream().cuda_stream
g = torch.Generator(device="cuda:0"); g.manual_seed(5)
rnd = lambda n: torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda:0", generator=g)
for k, m, sup in ((12, 4, 768), (16, 4, 1024)):
    for S in (1, sup + 1, 6 * sup + 29):
        bs = k * S if k * S % 2 else k * S - 1
        for length in (3 * bs + 1, 2 * bs + bs // 2):
            nb, pitch = -(-length // bs), (S + 15) // 16 * 16
            src = rnd(length)
            par = torch.zeros((nb * m, pitch), dtype=torch.uint8, device="cuda:0")
            dig = torch.zeros((nb, k + m, 32), dtype=torch.uint8, device="cuda:0")
            c = mb.Codec(k, m, bs)
            c.encode_blocks_device(src.data_ptr(), length, par.data_ptr(), pitch, dig.data_ptr(), st)
            torch.cuda.synchronize()
            assert c.stat("form_small") == c.launches == 1, (k, m, S, length)
            h, hp, hd = src.cpu().numpy(), par.cpu().numpy(), dig.cpu().numpy()
            for b in range(nb):
                sh = o.encode_data(k, m, h[b * bs:(b + 1) * bs])
                assert all(np.array_equal(hp[b * m + j, :sh[0].size], sh[k + j]) for j in range(m)), (k, m, S, length, b)
                assert all(hd[b, i].tobytes() == o.hh256(sh[i]) for i in range(k + m)), (k, m, S, length, b)
            c.close()
k, m, S, nb = 8, 8, 769, 3
erased = [0, 2, 4, 6, 9, 11, 13, 15]
src = np.random.default_rng(6).integers(0, 256, nb * k * S, dtype=np.uint8)
shards = [o.encode_data(k, m, src[b * k * S:(b + 1) * k * S]) for b in range(nb)]
fp = (32 + S + 15) // 16 * 16
frames = {}
for i in range(k + m):
    if i in erased: continue
    f = np.zeros((nb, fp), dtype=np.uint8)
    for b in range(nb):
        f[b, :32] = np.frombuffer(o.hh256(shards[b][i]), dtype=np.uint8); f[b, 32:32 + S] = shards[b][i]
    frames[i] = torch.from_numpy(f).to("cuda:0")
out = torch.zeros((nb * 8, (S + 15) // 16 * 16), dtype=torch.uint8, device="cuda:0")
dig = torch.zeros((nb, k + 8, 32), dtype=torch.uint8, device="cuda:0")
cor = torch.zeros((nb, k), dtype=torch.uint8, device="cuda:0")
c = mb.Codec(k, m, k * S)
c.reconstruct_device([frames[i].data_ptr() if i in frames else 0 for i in range(k + m)], fp, nb, [int(i in erased) for i in range(k + m)],
                     0, out.data_ptr(), out.shape[1], dig.data_ptr(), cor.data_ptr(), st)
torch.cuda.synchronize()
assert c.stat("form_small") == c.launches == 1 and int(cor.sum()) == 0
ho = out.cpu().numpy()
assert all(np.array_equal(ho[b * 8 + q, :S], shards[b][i]) for b in range(nb) for q, i in enumerate(erased))
c.close()
print("latency-kernel sanitizer case ok")
PY
logs=${SANITIZE_LOGS:-/tmp}   # full sanitizer reports of this stanza: small_<tool>.txt
for tool in memcheck racecheck synccheck; do
  echo "== $tool (latency kernel): $logs/small_$tool.txt"
  PYTORCH_NO_CUDA_MEMORY_CACHING=1 timeout 1200 compute-sanitizer --tool $tool --print-limit 20 python /tmp/san_small.py > "$logs/small_$tool.txt" 2>&1
  echo rc=$?; grep -E "ERROR SUMMARY|RACECHECK SUMMARY|sanitizer case ok|Invalid|out of bounds|hazard|Barrier" "$logs/small_$tool.txt" | head -12
done
