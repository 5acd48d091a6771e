"""Object checksums of PUTs through the cross-request coalescer (mec_batcher_encode_crc): CRC32 / CRC32C / CRC64NVME of every
caller's object, computed on the bytes the merged batch staged, on every staging path, against zlib and the CPU oracle.

As in test_gpu_batcher.py, each staging configuration runs in a child process of its own (the library reads MEC_BATCHER_* once per
process): this file run as a script.  Callers are released together by a barrier; with MEC_BATCHER_DEPTH=0 and each batcher capped
at exactly its round's blocks, a round is one batch.  Every round mixes callers of the new entry point with masks 0..7 (complete
part files and scatter-gather outputs) and callers of the old entry points, over objects whose bytes sit in two segments of the
staged buffer (full blocks, short last block) at every alignment.  The child checks every output byte, every guard byte and every
checksum itself and prints one JSON line with the mismatches and the batcher's counters per round; the parent asserts on it."""
import json
import os
import subprocess
import sys
import zlib

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MiB, KiB = 1 << 20, 1 << 10
# RS(12,4); RS(7,5) with odd S; RS(10,1) at an odd block size: every full-block segment after the first starts misaligned
GEOMS = (("rs12_4", 12, 4, MiB), ("rs7_5", 7, 5, MiB), ("rs10_1", 10, 1, MiB - 1))
# id -> (how the callers' buffers are allocated, environment of the child)
CONFIGS = {
    "put-dma": ("pinned", {"MEC_BATCHER_DEPTH": "0"}),
    "put-gather": ("pinned", {"MEC_BATCHER_GATHER": "1", "MEC_BATCHER_DEPTH": "0"}),
    "put-hybrid": ("pinned", {"MEC_BATCHER_GATHER_PCT": "50", "MEC_BATCHER_DEPTH": "0"}),
    "put-memcpy": ("pageable", {"MEC_BATCHER_DEPTH": "0"}),
}
CHILD_TIMEOUT_S = 240
GUARD = 64
MAX_WAIT_US = 500_000
BIG_CRC = 8 * MiB   # above this the oracle's CRC32C / CRC64NVME are taken over two halves and merged


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

    def want_files(k, m, bs, data, key):
        return list(cached(f"files_{k}_{m}_{bs}_{key}", lambda: np.stack(oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, data)[0])))

    def want_crcs(data, key):
        """(CRC32, CRC32C, CRC64NVME): CRC32 from zlib always; the others from the oracle, over two merged halves for long objects"""
        c32 = zlib.crc32(data.tobytes())
        if data.size <= BIG_CRC:
            w = oracle.crcs(data)
            if w[0] != c32:
                out["mismatches"].append({"what": "oracle crc32 != zlib", "size": int(data.size)})
            return (c32, int(w[1]), int(w[2]))
        h = data.size // 2
        a, b = cached(f"crc_{key}_a", lambda: np.array(oracle.crcs(data[:h]), dtype=np.uint64)), \
            cached(f"crc_{key}_b", lambda: np.array(oracle.crcs(data[h:]), dtype=np.uint64))
        return (c32,) + tuple(int(L.mec_checksum_combine(ty, int(a[t]), int(b[t]), data.size - h)) for t, ty in ((1, 2), (2, 4)))

    class Arena:
        """one host buffer holding many regions, each GUARD bytes clear of the previous one at a chosen misalignment; filled with a
        non-zero pattern, compared as a whole with the pattern plus the expected regions after the round"""

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
            self.regions.append((off, want, label))

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

    stat_names = ["batches", "requests", "blocks", "kernel_batches", "crc_requests", "launches", "small_launches"]

    def snap(bat):
        return {s: bat.stat(s) for s in stat_names}

    def run_round(bat, calls, rnd, info):
        bar = threading.Barrier(len(calls))
        res = [None] * len(calls)

        def worker(q):
            try:
                bar.wait()
                res[q] = calls[q]()
            except Exception as e:  # noqa: BLE001
                res[q] = repr(e)
        before = snap(bat)
        th = [threading.Thread(target=worker, args=(q,)) for q in range(len(calls))]
        [t.start() for t in th]
        [t.join() for t in th]
        after = snap(bat)
        out["rounds"].append(dict(info, round=rnd, requests=len(calls), d={s: after[s] - before[s] for s in stat_names}))
        return res

    def put_round(bat, geom, objs, plan, rnd, info):
        """plan: list of (object, api, mask), api one of crc / crc_sg (mec_batcher_encode_crc without / with data digests), enc / sg
        (mec_batcher_encode / mec_batcher_encode_sg), wrap / wrap_sg (Batcher.encode / Batcher.encode_sg with checksums=mask)"""
        name, k, m, bs = geom
        n, S = k + m, oracle.shard_size(bs, k)
        src_ar, out_ar = Arena(), Arena()
        lay = []
        for q, (o, api, mask) in enumerate(plan):
            data = objs[o][0]
            sg = api in ("crc_sg", "sg")
            nb = -(-data.size // bs)
            files = [None if (sg and i < k) else out_ar.reserve(objs[o][1][i].size, (2 * (q + i) + 1) % 16) for i in range(n)]
            dd = out_ar.reserve(nb * k * 32, (2 * q + 3) % 16) if sg else None
            lay.append((src_ar.reserve(data.size, 1 + q % 15), files, dd))
        src_ar.alloc(1000)
        out_ar.alloc(1001)
        marker = np.zeros(1, dtype=np.uint8)
        calls, outs3, wrapped = [], [], {}
        for q, ((o, api, mask), (so, files, dd)) in enumerate(zip(plan, lay)):
            data, want = objs[o][0], objs[o][1]
            src_ar.buf[so:so + data.size] = data
            src_ar.expect(so, data, {"request": q, "what": "src"})
            o3 = (C.c_uint64 * 3)(0x5eed, 0x5eed, 0x5eed)
            outs3.append(o3)
            if api.startswith("wrap"):
                wsrc = src_ar.buf[so:so + data.size]
                calls.append(lambda q=q, w=wsrc, sg=api == "wrap_sg", mask=mask, ln=data.size: (
                    wrapped.__setitem__(q, (bat.encode_sg if sg else bat.encode)(w, pinned=how == "pinned", checksums=mask)), ln)[1])
                continue
            fp = (C.c_void_p * n)(*[(marker.ctypes.data if dd is not None and i < k else None) if f is None else out_ar.base + f
                                    for i, f in enumerate(files)])
            for i, f in enumerate(files):
                if f is not None:
                    out_ar.expect(f, want[i], {"request": q, "drive": i})
            dp = None
            if dd is not None:
                nb = -(-data.size // bs)
                out_ar.expect(dd, np.stack([want[i][b * (32 + S):b * (32 + S) + 32] for b in range(nb) for i in range(k)]).reshape(-1),
                              {"request": q, "what": "data_digests"})
                dp = out_ar.base + dd
            s = src_ar.base + so
            if api in ("crc", "crc_sg"):
                calls.append(lambda s=s, ln=data.size, fp=fp, dp=dp, mask=mask, o3=o3:
                             L.mec_batcher_encode_crc(bat.h, s, ln, fp, dp, 0, mask, o3 if mask else None))
            elif api == "sg":
                calls.append(lambda s=s, ln=data.size, fp=fp, dp=dp: L.mec_batcher_encode_sg(bat.h, s, ln, fp, dp, 0))
            else:
                calls.append(lambda s=s, ln=data.size, fp=fp: L.mec_batcher_encode(bat.h, s, ln, fp, 0))
        blocks = sum(-(-objs[o][0].size // bs) for o, _, _ in plan)
        rec = dict(info, geom=name, blocks=blocks, ntails=sum(1 for o, _, _ in plan if objs[o][0].size % bs),
                   masked=sum(1 for _, _, mk in plan if mk))
        res = run_round(bat, calls, rnd, rec)
        for q, ((o, api, mask), r) in enumerate(zip(plan, res)):
            data = objs[o][0]
            if r != data.size:
                out["mismatches"].append({"round": rnd, "request": q, "rc": r if isinstance(r, int) else str(r)})
                continue
            want3 = tuple(v if mask & (1 << t) else 0 for t, v in enumerate(objs[o][2]))
            if api.startswith("wrap"):
                w = wrapped[q]
                got3, files = w[-1], w[0]
                for i in range(k if api == "wrap_sg" else 0, n):
                    if not np.array_equal(files[i], objs[o][1][i]):
                        out["mismatches"].append({"round": rnd, "request": q, "what": api, "drive": i})
                if api == "wrap_sg":
                    for b in range(w[1].shape[0]):
                        for i in range(k):
                            if not np.array_equal(w[1][b, i], objs[o][1][i][b * (32 + S):b * (32 + S) + 32]):
                                out["mismatches"].append({"round": rnd, "request": q, "what": "wrap_sg digest", "block": b})
                if how == "pinned":
                    for f in files:
                        if f is not None:
                            L.mec_free_pinned(f.ctypes.data)
                    if api == "wrap_sg":
                        L.mec_free_pinned(w[1].ctypes.data)
            elif api in ("crc", "crc_sg") and mask:
                got3 = tuple(int(v) for v in outs3[q])
            else:
                got3 = want3 = None
            if got3 != want3:
                out["mismatches"].append({"round": rnd, "request": q, "size": int(data.size), "mask": mask, "got": got3, "want": want3})
        src_ar.check(rnd)
        out_ar.check(rnd)
        src_ar.free()
        out_ar.free()
        return rec

    def make_objs(geom, sizes, seed0):
        name, k, m, bs = geom
        objs = []
        for o, size in enumerate(sizes):
            key = f"{size}_{seed0 + o}"
            d = rand(size, seed0 + o)
            objs.append((d, want_files(k, m, bs, d, key), want_crcs(d, key)))
        return objs

    def main_plan(nobj):
        """every object through the new entry point (masks 0..7, the long object with all three) and through an old one; the Python
        binding on two objects"""
        masks = [(5 * o + 7) % 8 for o in range(nobj)]
        masks[-1] = 7
        plan = []
        for o in range(nobj):
            plan.append((o, "crc_sg" if o % 2 else "crc", masks[o]))
            plan.append((o, "enc" if o % 2 else "sg", 0))
        return plan + [(nobj - 2, "wrap", 7), (2, "wrap_sg", 5)]

    for gi, geom in enumerate(GEOMS):
        name, k, m, bs = geom
        sizes = [1, 15, 1023, 1024, 1025, 262143, 262144, 262145, bs - 1, bs, bs + 1, 3 * bs + 4321, 64 * bs + 777]
        objs = make_objs(geom, sizes, 7000 + 100 * gi)
        plan = main_plan(len(objs))
        cap = sum(-(-objs[o][0].size // bs) for o, _, _ in plan)
        bat = mb.Batcher(k, m, bs, max_batch_blocks=cap, max_wait_us=MAX_WAIT_US)
        num_sms = bat.stat("num_sms")
        put_round(bat, geom, objs, plan, f"{name}/main", {"name": "main", "cap": cap})
        bat.close()
        if config != "put-dma" or name == "rs7_5":
            continue
        # more than 5 x SMs blocks in ONE batch: the throughput kernel over the full blocks plus one launch per short block
        bs64 = 64 * KiB - (1 if bs % 2 else 0)
        limit = 5 * num_sms
        nblk = limit // 4 + 4
        g64 = (name + "@64k", k, m, bs64)
        big = make_objs(g64, [nblk * bs64 + 1 + 997 * q for q in range(2)], 9000 + 100 * gi)
        plan = [(0, "crc", 7), (0, "sg", 0), (1, "crc_sg", 6), (1, "enc", 0)]
        cap64 = sum(-(-big[o][0].size // bs64) for o, _, _ in plan)
        bat = mb.Batcher(k, m, bs64, max_batch_blocks=cap64, max_wait_us=MAX_WAIT_US)
        put_round(bat, g64, big, plan, f"{g64[0]}/overlimit", {"name": "overlimit", "cap": cap64, "limit": limit})
        bat.close()

    if config == "put-dma":
        # launches added by the checksums: one request, then 64 requests, each round once without and once with masks; the same
        # 64 objects through mec_batcher_encode_sg
        geom = GEOMS[0]
        name, k, m, bs = geom
        objs = make_objs(geom, [1000 + 37 * q for q in range(64)], 8000)
        bat = mb.Batcher(k, m, bs, max_batch_blocks=64, max_wait_us=MAX_WAIT_US)
        put_round(bat, geom, objs, [(5, "crc", 0)], "launch/one-0", {"name": "one-0"})
        put_round(bat, geom, objs, [(5, "crc", 7)], "launch/one-7", {"name": "one-7"})
        put_round(bat, geom, objs, [(q, "crc_sg", 0) for q in range(64)], "launch/many-0", {"name": "many-0"})
        put_round(bat, geom, objs, [(q, "sg", 0) for q in range(64)], "launch/many-sg", {"name": "many-sg"})
        put_round(bat, geom, objs, [(q, "crc_sg", q % 7 + 1) for q in range(64)], "launch/many-mix", {"name": "many-mix"})
        # argument errors with a real batcher
        n = k + m
        data = mb.pinned_array(5000)
        data[:] = rand(5000, 1)
        files = [mb.pinned_array(1 << 20) for _ in range(n)]
        fp = (C.c_void_p * n)(*[f.ctypes.data for f in files])
        r0 = bat.stat("requests")
        out["errors"]["null_out3"] = L.mec_batcher_encode_crc(bat.h, data.ctypes.data, 5000, fp, None, 0, 7, None)
        out["errors"]["null_out3_requests"] = bat.stat("requests") - r0
        o3 = (C.c_uint64 * 3)(11, 22, 33)
        fq = (C.c_void_p * n)(*([files[0].ctypes.data] + [None] * (n - 1)))
        out["errors"]["quorum"] = L.mec_batcher_encode_crc(bat.h, data.ctypes.data, 5000, fq, None, n, 7, o3)
        out["errors"]["quorum_out3"] = [int(v) for v in o3]
        o3 = (C.c_uint64 * 3)(11, 22, 33)
        out["errors"]["empty"] = L.mec_batcher_encode_crc(bat.h, None, 0, fp, None, 0, 7, o3)
        out["errors"]["empty_out3"] = [int(v) for v in o3]
        bat.close()
        for f in files + [data]:
            L.mec_free_pinned(f.ctypes.data)
    out["limit"] = 5 * num_sms
    print(json.dumps(out))


# ---- parent ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def oracle_cache(tmp_path_factory):
    return str(tmp_path_factory.mktemp("batcher_crc_oracle"))


def _run_child(config, cache_dir):
    env = {key: v for key, v in os.environ.items() if not key.startswith(("MEC_BATCHER_", "MEC_NO_BATCH_COPY"))}
    env.update(CONFIGS[config][1])
    p = subprocess.run([sys.executable, os.path.abspath(__file__), config, cache_dir], env=env, capture_output=True, text=True,
                       timeout=CHILD_TIMEOUT_S, cwd=ROOT)
    assert p.returncode == 0, f"child {config} exited {p.returncode}:\n{p.stderr[-4000:]}"
    return json.loads(p.stdout.strip().split("\n")[-1])


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
def test_batcher_checksums(oracle, oracle_cache, config):
    res = _run_child(config, oracle_cache)
    assert not res["mismatches"], res["mismatches"][:10]
    rounds = {r["round"]: r for r in res["rounds"]}
    for g in GEOMS:
        assert g[0] + "/main" in rounds
    for r in res["rounds"]:
        d, ctx = r["d"], (r["round"], r["d"])
        assert d["batches"] == 1 and d["requests"] == r["requests"], ctx
        assert d["crc_requests"] == r["masked"], ctx
        assert d["kernel_batches"] == (1 if CONFIGS[config][0] == "pinned" else 0), ctx
        if r["name"] == "overlimit":
            # the full blocks in ONE throughput launch, every short block in a latency launch of its own
            assert r["blocks"] > r["limit"] and d["small_launches"] == r["ntails"], ctx
    if config != "put-dma":
        return
    assert "rs12_4@64k/overlimit" in rounds and "rs10_1@64k/overlimit" in rounds
    launches = {name: rounds["launch/" + name]["d"]["launches"] for name in ("one-0", "one-7", "many-0", "many-sg", "many-mix")}
    extra = launches["one-7"] - launches["one-0"]
    assert 0 < extra <= 2 and launches["many-mix"] - launches["many-0"] == extra, launches
    assert launches["many-0"] == launches["many-sg"], launches
    e = res["errors"]
    assert e["null_out3"] == -12 and e["null_out3_requests"] == 0, e
    assert e["quorum"] == -11 and e["quorum_out3"] == [11, 22, 33], e
    assert e["empty"] == 0 and e["empty_out3"] == [0, 0, 0], e


def test_encode_crc_rejects_null_batcher():
    import ctypes as C

    sys.path.insert(0, ROOT)
    import minio_b200 as mb
    out3 = (C.c_uint64 * 3)()
    files = (C.c_void_p * 16)()
    assert mb.lib().mec_batcher_encode_crc(None, None, 0, files, None, 0, 7, out3) == -12
    assert mb.lib().mec_batcher_encode_crc(None, None, 0, files, None, 0, 0, None) == -12


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])
