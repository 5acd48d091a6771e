"""Object hashes of PUTs through the cross-request coalescer (mec_batcher_encode_sums): MD5, SHA-1 and SHA-256 of every caller's
object, computed by ONE stream_sums_kernel per merged batch on the bytes the batch staged, on every staging path, against hashlib;
the CRCs of the same call against zlib and the CPU oracle; every part-file byte against the oracle.

As in test_gpu_batcher_checksums.py, each staging configuration runs in a child process of its own (the library reads MEC_BATCHER_*
once per batcher, and the pinned / pageable choice is per process here): this file run as a script.  Callers are released together by
a barrier; with MEC_BATCHER_DEPTH=0 and each batcher capped at exactly its round's blocks, a round is one batch.  A round mixes callers
of the new entry point with every subset of the six mask bits (complete part files and scatter-gather outputs) and callers of
mec_batcher_encode / _sg / _crc, over objects whose bytes sit in two segments of the staged buffer (full blocks, short last block):
at RS(10,1) with a block of MiB - 1 bytes every full-block segment after the first starts misaligned and is not a multiple of 64
bytes long, so the block across the segment boundary is assembled bytewise.  The CRC triple and the 96-byte digest record of every
caller live in the guarded output arena at odd offsets: bytes the mask does not ask for must keep their guard values.  The child
prints one JSON line with the mismatches and the batcher's counters per round; the parent asserts on it."""
import hashlib
import json
import os
import subprocess
import sys
import zlib

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MiB, KiB = 1 << 20, 1 << 10
GEOMS = (("rs12_4", 12, 4, MiB), ("rs7_5", 7, 5, MiB), ("rs10_1", 10, 1, MiB - 1))
CONFIGS = {
    "put-dma": ("pinned", {"MEC_BATCHER_DEPTH": "0"}),
    "put-gather": ("pinned", {"MEC_BATCHER_GATHER": "1", "MEC_BATCHER_DEPTH": "0"}),
    "put-hybrid": ("pinned", {"MEC_BATCHER_GATHER_PCT": "50", "MEC_BATCHER_DEPTH": "0"}),
    "put-memcpy": ("pageable", {"MEC_BATCHER_DEPTH": "0"}),
}
CHILD_TIMEOUT_S = 300
GUARD = 64
MAX_WAIT_US = 500_000
CRC_MASK, SUM_MASK = 7, 56
SLOTS = ((8, "md5", 0, 16), (16, "sha1", 32, 20), (32, "sha256", 64, 32))


def digests(data, mask):
    """{offset in the record: digest} of the MEC_SUM_* bits of mask"""
    return {o: hashlib.new(name, data).digest() for bit, name, o, _ in SLOTS if mask & bit}


# ---- child ----------------------------------------------------------------------------------------------------------------------

def _child(config, cache_dir):
    import ctypes as C
    import threading

    import numpy as np

    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import minio_b200 as mb
    import oracle_lib as oracle

    how, _ = CONFIGS[config]
    L = mb.lib()
    out = {"config": config, "rounds": [], "mismatches": [], "errors": {}}

    def rand(n, seed):
        return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)

    def cached(key, fn):
        path = os.path.join(cache_dir, key + ".npy")
        if os.path.exists(path):
            return np.load(path)
        v = np.asarray(fn())
        tmp = f"{path}.{os.getpid()}.npy"
        np.save(tmp, v)
        os.replace(tmp, path)
        return v

    class Arena:
        """one host buffer of many regions, each GUARD bytes clear of the previous one at a chosen misalignment, filled with a
        non-zero pattern; after the round it must equal the pattern plus the expected regions"""

        def __init__(self):
            self.size, self.regions = 0, []

        def reserve(self, nbytes, mis):
            off = (self.size + GUARD + 63) // 64 * 64 + mis
            self.size = off + nbytes
            return off

        def alloc(self, seed):
            total = self.size + GUARD
            self.buf = mb.pinned_array(total) if how == "pinned" else np.empty(total, dtype=np.uint8)
            self.buf[:] = rand(total, seed) | 1
            self.ref = self.buf.copy()
            self.base = self.buf.ctypes.data

        def expect(self, off, want, label):
            self.regions.append((off, np.asarray(want, dtype=np.uint8), label))

        def check(self, rnd):
            for off, want, label in self.regions:
                got = self.buf[off:off + want.size]
                if not np.array_equal(got, want):
                    bad = np.flatnonzero(got != want)
                    out["mismatches"].append(dict(label, round=rnd, bytes=int(bad.size), first=int(bad[0])))
                self.ref[off:off + want.size] = want
            bad = np.flatnonzero(self.buf != self.ref)
            if bad.size:
                out["mismatches"].append({"round": rnd, "guard": True, "bytes": int(bad.size), "first": int(bad[0])})

        def free(self):
            if how == "pinned":
                L.mec_free_pinned(self.base)

    stat_names = ["batches", "requests", "blocks", "kernel_batches", "crc_requests", "sum_requests", "launches"]

    def run_round(bat, calls, rnd, info):
        bar = threading.Barrier(len(calls))
        res = [None] * len(calls)

        def worker(q):
            try:
                bar.wait()
                res[q] = calls[q]()
            except Exception as e:  # noqa: BLE001
                res[q] = repr(e)
        before = {s: bat.stat(s) for s in stat_names}
        th = [threading.Thread(target=worker, args=(q,)) for q in range(len(calls))]
        [t.start() for t in th]
        [t.join() for t in th]
        out["rounds"].append(dict(info, round=rnd, d={s: bat.stat(s) - before[s] for s in stat_names}))
        return res

    def make_objs(geom, sizes, seed0):
        name, k, m, bs = geom
        objs = []
        for o, size in enumerate(sizes):
            key = f"{k}_{m}_{bs}_{size}_{seed0 + o}"
            d = rand(size, seed0 + o)
            files = list(cached("files_" + key, lambda: np.stack(oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, d)[0])))
            crcs = tuple(int(v) for v in cached("crc_" + key, lambda: np.array(oracle.crcs(d), dtype=np.uint64)))
            if crcs[0] != zlib.crc32(d.tobytes()):
                out["mismatches"].append({"what": "oracle crc32 != zlib", "size": size})
            objs.append((d, files, crcs, digests(d.tobytes(), SUM_MASK)))
        return objs

    def put_round(bat, geom, objs, plan, rnd, info):
        """plan: list of (object, api, mask); api one of sums / sums_sg (mec_batcher_encode_sums without / with data digests),
        enc / sg / crc (mec_batcher_encode / _sg / _crc), wrap / wrap_sg (Batcher.encode / encode_sg with checksums= and hashes=)"""
        name, k, m, bs = geom
        n, S = k + m, oracle.shard_size(bs, k)
        src_ar, out_ar = Arena(), Arena()
        lay = []
        for q, (o, api, mask) in enumerate(plan):
            data = objs[o][0]
            sg = api in ("sums_sg", "sg")
            nb = -(-data.size // bs)
            files = [None if (sg and i < k) else out_ar.reserve(objs[o][1][i].size, (2 * (q + i) + 1) % 16) for i in range(n)]
            dd = out_ar.reserve(max(nb, 1) * k * 32, (2 * q + 3) % 16) if sg else None
            crc = out_ar.reserve(24, 0) if api in ("sums", "sums_sg", "crc") else None  # uint64 triple: 8-byte aligned
            rec = out_ar.reserve(96, (q * 5 + 1) % 16) if api in ("sums", "sums_sg") else None
            lay.append((src_ar.reserve(max(data.size, 1), 1 + q % 15), files, dd, crc, rec))
        src_ar.alloc(1000)
        out_ar.alloc(1001)
        marker = np.zeros(1, dtype=np.uint8)
        calls, wrapped = [], {}
        nonempty = 0
        for q, ((o, api, mask), (so, files, dd, crc, rec)) in enumerate(zip(plan, lay)):
            data, want, crcs, sums = objs[o]
            nonempty += data.size > 0
            src_ar.buf[so:so + data.size] = data
            src_ar.expect(so, data, {"request": q, "what": "src"})
            if api.startswith("wrap"):
                wsrc = src_ar.buf[so:so + data.size]
                calls.append(lambda q=q, w=wsrc, sg=api == "wrap_sg", mask=mask, ln=data.size: (
                    wrapped.__setitem__(q, (bat.encode_sg if sg else bat.encode)(w, pinned=how == "pinned", checksums=mask & CRC_MASK,
                                                                                  hashes=mask & SUM_MASK)), ln)[1])
                continue
            fp = (C.c_void_p * n)(*[(marker.ctypes.data if dd is not None and i < k else None) if f is None else out_ar.base + f
                                    for i, f in enumerate(files)])
            for i, f in enumerate(files):
                if f is not None:
                    out_ar.expect(f, want[i], {"request": q, "drive": i})
            dp = None
            if dd is not None:
                nb = -(-data.size // bs)
                if nb:
                    out_ar.expect(dd, np.stack([want[i][b * (32 + S):b * (32 + S) + 32] for b in range(nb) for i in range(k)]).reshape(-1),
                                  {"request": q, "what": "data_digests"})
                dp = out_ar.base + dd
            if crc is not None and mask & CRC_MASK:
                w3 = [v if mask & (1 << t) else 0 for t, v in enumerate(crcs)]
                out_ar.expect(crc, np.array(w3, dtype=np.uint64).view(np.uint8), {"request": q, "what": "crc3", "mask": mask})
            if rec is not None:
                for off, dg in sums.items():
                    if mask & {0: 8, 32: 16, 64: 32}[off]:
                        out_ar.expect(rec + off, np.frombuffer(dg, dtype=np.uint8), {"request": q, "what": "sums", "mask": mask,
                                                                                     "slot": off, "size": int(data.size)})
            s = src_ar.base + so
            cp = out_ar.base + crc if crc is not None else None
            rp = out_ar.base + rec if rec is not None else None
            if api in ("sums", "sums_sg"):
                calls.append(lambda s=s, ln=data.size, fp=fp, dp=dp, mask=mask, cp=cp, rp=rp:
                             L.mec_batcher_encode_sums(bat.h, s, ln, fp, dp, 0, mask, cp if mask & CRC_MASK else None,
                                                       rp if mask & SUM_MASK else None))
            elif api == "crc":
                calls.append(lambda s=s, ln=data.size, fp=fp, mask=mask, cp=cp:
                             L.mec_batcher_encode_crc(bat.h, s, ln, fp, None, 0, mask, cp if mask else None))
            elif api == "sg":
                calls.append(lambda s=s, ln=data.size, fp=fp, dp=dp: L.mec_batcher_encode_sg(bat.h, s, ln, fp, dp, 0))
            else:
                calls.append(lambda s=s, ln=data.size, fp=fp: L.mec_batcher_encode(bat.h, s, ln, fp, 0))
        rec_info = dict(info, geom=name, requests=nonempty,
                        crc_masked=sum(1 for _, _, mk in plan if mk & CRC_MASK),
                        sum_masked=sum(1 for _, _, mk in plan if mk & SUM_MASK))
        res = run_round(bat, calls, rnd, rec_info)
        for q, ((o, api, mask), r) in enumerate(zip(plan, res)):
            data, want, crcs, sums = objs[o]
            if r != data.size:
                out["mismatches"].append({"round": rnd, "request": q, "rc": r if isinstance(r, int) else str(r)})
                continue
            if api.startswith("wrap"):
                w = wrapped[q]
                files = w[0]
                for i in range(k if api == "wrap_sg" else 0, n):
                    if not np.array_equal(files[i], want[i]):
                        out["mismatches"].append({"round": rnd, "request": q, "what": api, "drive": i})
                got = w[-1]
                want_d = {nm: sums[o2] for bit, nm, o2, _ in SLOTS if mask & bit}
                if got != want_d:
                    out["mismatches"].append({"round": rnd, "request": q, "what": api + " hashes", "mask": mask})
                if mask & CRC_MASK:
                    got3 = w[-2]
                    if got3 != tuple(v if mask & (1 << t) else 0 for t, v in enumerate(crcs)):
                        out["mismatches"].append({"round": rnd, "request": q, "what": api + " crcs", "mask": mask})
                if how == "pinned":
                    for f in files:
                        if f is not None:
                            L.mec_free_pinned(f.ctypes.data)
                    if api == "wrap_sg":
                        L.mec_free_pinned(w[1].ctypes.data)
        src_ar.check(rnd)
        out_ar.check(rnd)
        src_ar.free()
        out_ar.free()

    def cap_of(objs, plan, bs):
        return max(1, sum(-(-objs[o][0].size // bs) for o, _, _ in plan))

    for gi, geom in enumerate(GEOMS):
        name, k, m, bs = geom
        sizes = [0, 1, 55, 56, 64, 1000, 262145, bs - 1, bs, bs + 1, 3 * bs + 4321]
        objs = make_objs(geom, sizes, 7000 + 100 * gi)
        # every subset of the six bits through the new entry point (objects cycling, both output forms), every object also through
        # an old entry point, and the Python binding twice
        plan = [(mask % len(objs), "sums_sg" if mask % 2 else "sums", mask) for mask in range(64)]
        plan += [(o, ("enc", "sg", "crc")[o % 3], 7 if o % 3 == 2 else 0) for o in range(len(objs))]
        plan += [(len(objs) - 1, "wrap", 63), (7, "wrap_sg", 40)]
        cap = cap_of(objs, plan, bs)
        bat = mb.Batcher(k, m, bs, max_batch_blocks=cap, max_wait_us=MAX_WAIT_US)
        put_round(bat, geom, objs, plan, f"{name}/main", {"name": "main", "cap": cap})
        bat.close()
        # a request above max_batch_blocks leads a batch of its own; the slot's buffers grow for it
        bat = mb.Batcher(k, m, bs, max_batch_blocks=2, max_wait_us=MAX_WAIT_US)
        put_round(bat, geom, objs, [(len(objs) - 1, "sums_sg", 63)], f"{name}/big", {"name": "big"})
        bat.close()

    if config == "put-dma":
        # the launches the hashes add: the same rounds without and with MEC_SUM_* bits (CRC bits alike in both)
        geom = GEOMS[0]
        name, k, m, bs = geom
        objs = make_objs(geom, [1000 + 37 * q for q in range(64)], 8000)
        bat = mb.Batcher(k, m, bs, max_batch_blocks=64, max_wait_us=MAX_WAIT_US)
        put_round(bat, geom, objs, [(5, "sums", 0)], "launch/one-0", {"name": "one-0"})
        put_round(bat, geom, objs, [(5, "sums", 8)], "launch/one-8", {"name": "one-8"})
        put_round(bat, geom, objs, [(q, "sums_sg", q % 8) for q in range(64)], "launch/many-crc", {"name": "many-crc"})
        put_round(bat, geom, objs, [(q, "sums_sg", q % 8 | (8 * (q % 7 + 1))) for q in range(64)], "launch/many-sums",
                  {"name": "many-sums"})
        # refusals with a real batcher: nothing is queued
        n = k + m
        data = mb.pinned_array(5000)
        data[:] = rand(5000, 1)
        files = [mb.pinned_array(1 << 20) for _ in range(n)]
        fp = (C.c_void_p * n)(*[f.ctypes.data for f in files])
        rec = (C.c_uint8 * 96)(*([0x5A] * 96))
        crc3 = (C.c_uint64 * 3)(11, 22, 33)
        r0 = bat.stat("requests")
        e = out["errors"]
        e["unknown_bit"] = L.mec_batcher_encode_sums(bat.h, data.ctypes.data, 5000, fp, None, 0, 64 | 8, crc3, rec)
        e["high_bit"] = L.mec_batcher_encode_sums(bat.h, data.ctypes.data, 5000, fp, None, 0, 1 << 30, crc3, rec)
        e["null_sums"] = L.mec_batcher_encode_sums(bat.h, data.ctypes.data, 5000, fp, None, 0, 7 | 32, crc3, None)
        e["null_crc3"] = L.mec_batcher_encode_sums(bat.h, data.ctypes.data, 5000, fp, None, 0, 1 | 8, None, rec)
        e["refused_requests"] = bat.stat("requests") - r0
        fq = (C.c_void_p * n)(*([files[0].ctypes.data] + [None] * (n - 1)))
        e["quorum"] = L.mec_batcher_encode_sums(bat.h, data.ctypes.data, 5000, fq, None, n, 63, crc3, rec)
        e["untouched"] = bytes(rec) == bytes([0x5A] * 96) and list(crc3) == [11, 22, 33]
        s0 = bat.stat("sum_requests")
        e["empty"] = L.mec_batcher_encode_sums(bat.h, None, 0, fp, None, 0, 56 | 7, crc3, rec)
        e["empty_rec"] = bytes(rec).hex()
        e["empty_crc3"] = [int(v) for v in crc3]
        e["empty_sum_requests"] = bat.stat("sum_requests") - s0
        e["empty_requests"] = bat.stat("requests") - r0
        bat.close()
        for f in files + [data]:
            L.mec_free_pinned(f.ctypes.data)
    print(json.dumps(out))


# ---- parent ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def oracle_cache(tmp_path_factory):
    return str(tmp_path_factory.mktemp("batcher_sums_oracle"))


def _run_child(config, cache_dir):
    env = {key: v for key, v in os.environ.items() if not key.startswith(("MEC_BATCHER_", "MEC_NO_BATCH_COPY"))}
    env.update(CONFIGS[config][1])
    p = subprocess.run([sys.executable, os.path.abspath(__file__), config, cache_dir], env=env, capture_output=True, text=True,
                       timeout=CHILD_TIMEOUT_S, cwd=ROOT)
    assert p.returncode == 0, f"child {config} exited {p.returncode}:\n{p.stderr[-4000:]}"
    return json.loads(p.stdout.strip().split("\n")[-1])


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
def test_batcher_sums(oracle, oracle_cache, config):
    res = _run_child(config, oracle_cache)
    assert not res["mismatches"], res["mismatches"][:10]
    rounds = {r["round"]: r for r in res["rounds"]}
    for g in GEOMS:
        assert g[0] + "/main" in rounds and g[0] + "/big" in rounds
    for r in res["rounds"]:
        d, ctx = r["d"], (r["round"], r["d"])
        assert d["batches"] == 1 and d["requests"] == r["requests"], ctx
        assert d["crc_requests"] == r["crc_masked"] and d["sum_requests"] == r["sum_masked"], ctx
        assert d["kernel_batches"] == (1 if CONFIGS[config][0] == "pinned" else 0), ctx
    if config != "put-dma":
        return
    launches = {name: rounds["launch/" + name]["d"]["launches"] for name in ("one-0", "one-8", "many-crc", "many-sums")}
    assert launches["one-8"] == launches["one-0"] + 1, launches
    assert launches["many-sums"] == launches["many-crc"] + 1, launches
    e = res["errors"]
    assert e["unknown_bit"] == e["high_bit"] == e["null_sums"] == e["null_crc3"] == -12, e
    assert e["refused_requests"] == 0, e
    assert e["quorum"] == -11 and e["untouched"], e
    empty = bytes.fromhex(e["empty_rec"])
    assert empty[:16] == hashlib.md5(b"").digest() and empty[16:32] == bytes([0x5A] * 16), e
    assert empty[32:52] == hashlib.sha1(b"").digest() and empty[52:64] == bytes([0x5A] * 12), e
    assert empty[64:] == hashlib.sha256(b"").digest(), e
    assert e["empty"] == 0 and e["empty_crc3"] == [0, 0, 0] and e["empty_sum_requests"] == 1 and e["empty_requests"] == 0, e


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])
