"""GPU tests of the cross-request coalescer (mec_batcher_*): every staging path, geometry and frame alignment, byte for byte
against the CPU oracle.

The staging and output paths are picked by environment switches that the library reads once per process (MEC_BATCHER_GATHER,
MEC_BATCHER_DMA_BLOCKS, MEC_BATCHER_GET_OUT, ...), so every configuration runs in a child process of its own: this file run as a
script.  The child drives concurrent callers through the batcher, released together by a barrier, checks every byte of every
caller's output and of the guard bytes around it itself, and prints one JSON line with the mismatches and the batcher's counters
per round.  The parent asserts on that line which batches, kernels and kernel forms ran.

Every caller's part files (PUT) and destination (GET) sit between guard bytes at an odd offset of their own, in a buffer filled
with a non-zero pattern: a skipped byte, a missing zero pad or a store past the end shows up.  With MEC_BATCHER_DEPTH=0 and a
0.5 s max_wait_us the merging is deterministic: each geometry's batcher is capped at exactly its main round's blocks (counted as
the worker counts them: ceil(len / bs) per PUT, length / bs + 2 per GET), so that round is one batch and the same round plus one
more small request is two.  A second batcher with 64 KiB blocks runs one round of more than 5 x SMs blocks in a single batch, which
takes the throughput kernel plus one launch per short last block instead of the latency kernel."""
import json
import os
import subprocess
import sys
import time

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MiB, KiB = 1 << 20, 1 << 10
FORMS = ("small", "fast3d", "fast3d_auto", "fast3d_semi", "fast", "fast_auto", "aligned", "aligned_auto", "runtime", "bytewise",
         "dyn_aligned", "dyn_runtime", "dyn_bytewise", "jit")
# (name, k, m, block size): compiled RS(12,4) with even S; RS(7,5) with odd S = 149797 (frames at every alignment mod 4) and the
# runtime-matrix kernel in two row passes of 4; RS(16,4), 20 streams: four GF warps and two hash warps; RS(20,12), n = 32 =
# kBatchMaxFiles, three row passes, S % 16 = 4; RS(10,1) at an odd block size, row chunk 1, every short block's input misaligned;
# RS(20,13), n = 33: too many drives for the mapped path
GEOMS = (("rs12_4", 12, 4, MiB), ("rs7_5", 7, 5, MiB), ("rs16_4", 16, 4, MiB), ("rs20_12", 20, 12, 256 * KiB),
         ("rs10_1", 10, 1, MiB - 1), ("rs20_13", 20, 13, 256 * KiB))
# id -> (PUT or GET, environment of the child)
CONFIGS = {
    "put-dma": ("put", {}),
    "put-dma-depth0": ("put", {"MEC_BATCHER_DEPTH": "0"}),
    "put-gather": ("put", {"MEC_BATCHER_GATHER": "1", "MEC_BATCHER_DEPTH": "0"}),
    "put-hybrid": ("put", {"MEC_BATCHER_GATHER_PCT": "50", "MEC_BATCHER_DEPTH": "0"}),
    "put-memcpy": ("put", {"MEC_BATCHER_MEMCPY": "1"}),
    "get-dma": ("get", {}),
    "get-dma-depth0": ("get", {"MEC_BATCHER_DEPTH": "0"}),
    "get-gather": ("get", {"MEC_BATCHER_DMA_BLOCKS": "1000000", "MEC_BATCHER_DEPTH": "0"}),
    "get-mixed": ("get", {"MEC_BATCHER_DMA_BLOCKS": "2", "MEC_NO_BATCH_COPY": "1", "MEC_BATCHER_DEPTH": "0"}),
    "get-out1": ("get", {"MEC_BATCHER_GET_OUT": "1", "MEC_BATCHER_DEPTH": "0"}),
    "get-out2": ("get", {"MEC_BATCHER_GET_OUT": "2", "MEC_BATCHER_DEPTH": "0"}),
}
CHILD_TIMEOUT_S = 120
GUARD = 64
MAX_WAIT_US = 500_000


# ---- child ----------------------------------------------------------------------------------------------------------------------

def _child(config, cache_dir):
    import ctypes as C
    import threading

    import numpy as np

    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import minio_b200 as mb
    import oracle_lib as oracle

    kind, env = CONFIGS[config]
    depth0 = env.get("MEC_BATCHER_DEPTH") == "0"
    L = mb.lib()
    out = {"config": config, "rounds": [], "mismatches": [], "init_s": [], "oracle_s": 0.0}
    t_start = time.time()

    def rand(n, seed):
        return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)

    def oracle_files(k, m, bs, data, key):
        """oracle.erasure_encode, cached on disk across the children (every child encodes the same seeded objects)"""
        path = os.path.join(cache_dir, f"{k}_{m}_{bs}_{key}.npy")
        if os.path.exists(path):
            return list(np.load(path))
        t0 = time.time()
        files, _ = oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, data)
        out["oracle_s"] += time.time() - t0
        tmp = f"{path}.{os.getpid()}.npy"
        np.save(tmp, np.stack(files))
        os.replace(tmp, path)
        return files

    class Arena:
        """one host buffer holding many regions, each GUARD bytes clear of the previous one at a chosen misalignment; filled with
        a non-zero pattern before the round, compared as a whole with the pattern plus the expected regions after it"""

        def __init__(self, how):
            self.how, self.size, self.regions = how, 0, []

        def reserve(self, nbytes, mis):
            off = (self.size + GUARD + 63) // 64 * 64 + mis
            self.size = off + nbytes
            return off

        def alloc(self, seed):
            total = self.size + GUARD
            if self.how == "pinned":
                self.buf = mb.pinned_array(total)
            elif self.how == "numa":
                self.buf = mb.pinned_array(total, device=0)
            else:
                self.buf = np.empty(total, dtype=np.uint8)
            self.buf[:] = rand(total, seed) | 1
            self.ref = self.buf.copy()
            self.base = self.buf.ctypes.data

        def view(self, off, n):
            return self.buf[off:off + n]

        def expect(self, off, want, label, frame=None):
            self.regions.append((off, want, label, frame))

        def check(self, rnd):
            for off, want, label, frame in self.regions:
                got = self.buf[off:off + want.size]
                if not np.array_equal(got, want):
                    bad = np.flatnonzero(got != want)
                    rec = dict(label, round=rnd, bytes=int(bad.size), first=int(bad[0]))
                    if frame:
                        rec["block"] = int(bad[0]) // frame
                    out["mismatches"].append(rec)
                self.ref[off:off + want.size] = want
            bad = np.flatnonzero(self.buf != self.ref)
            if bad.size:
                out["mismatches"].append({"round": rnd, "guard": self.how, "bytes": int(bad.size), "first": int(bad[0])})

        def free(self):
            if self.how != "pageable":
                L.mec_free_pinned(self.base)

    stat_names = ["batches", "requests", "blocks", "kernel_batches", "redone", "launches", "small_launches"] + ["form_" + f for f in FORMS]

    def snap(bat):
        return {s: bat.stat(s) for s in stat_names}

    def run_round(bat, calls, rnd, info):
        """all callers released together; -> per-call results; appends the round's counter deltas to the JSON"""
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
        t0 = time.time()
        [t.start() for t in th]
        [t.join() for t in th]
        after = snap(bat)
        d = {s: after[s] - before[s] for s in stat_names}
        out["rounds"].append(dict(info, round=rnd, requests=len(calls), d=d, wall_s=round(time.time() - t0, 3)))
        return res

    def new_batcher(k, m, bs, cap):
        t0 = time.time()
        bat = mb.Batcher(k, m, bs, max_batch_blocks=cap, max_wait_us=MAX_WAIT_US)
        out["init_s"].append(round(time.time() - t0, 3))
        return bat

    def sizes_of(k, bs):
        nfull = max(3, 3 * MiB // bs)
        # pure padding; one block +- 1 (bs - 1 still has shard length S); a short last block of full shard length; one byte into
        # a block; a few MiB plus a tail whose shard length (1001) is odd
        return [1, k - 1, k, bs - 1, bs, 3 * bs + bs - 1, 2 * bs + 1, nfull * bs + 1001 * k - 1]

    def check_rc(res, want, rnd):
        for q, (r, w) in enumerate(zip(res, want)):
            if r != w:
                out["mismatches"].append({"round": rnd, "request": q, "rc": r if isinstance(r, int) else str(r), "want": w})

    # a registered (cudaHostRegister) buffer may be dereferenced by the batcher's kernels only at its host address
    def numa_precondition():
        import ctypes.util
        import glob
        cands = [ctypes.util.find_library("cudart"), "libcudart.so", "libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so"]
        for p in sys.path:
            cands += sorted(glob.glob(os.path.join(p, "nvidia", "cuda_runtime", "lib", "libcudart.so*")))
        rt = None
        for c in cands:
            if not c:
                continue
            try:
                rt = C.CDLL(c)
                break
            except OSError:
                continue
        assert rt is not None, "libcudart not found"
        rt.cudaHostGetDevicePointer.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_uint]
        rt.cudaDeviceGetAttribute.argtypes = [C.POINTER(C.c_int), C.c_int, C.c_int]
        rt.cudaSetDevice(0)
        res = {}
        for how in ("numa", "pinned"):
            a = mb.pinned_array(4 * MiB, device=0 if how == "numa" else None)
            dp = C.c_void_p()
            rc = rt.cudaHostGetDevicePointer(C.byref(dp), C.c_void_p(a.ctypes.data), 0)
            res[how] = {"rc": rc, "same": rc == 0 and dp.value == a.ctypes.data}
            L.mec_free_pinned(a.ctypes.data)
        v = C.c_int(-1)
        rt.cudaDeviceGetAttribute(C.byref(v), 91, 0)  # cudaDevAttrCanUseHostPointerForRegisteredMem
        res["can_use_host_pointer_for_registered_mem"] = v.value
        return res

    num_sms = None

    # ---- PUT ----------------------------------------------------------------------------------------------------------------
    def put_round(bat, geom, objs, rnd, how="pinned", pageable_every=0, extra_one=False, wrapper=True, info=None):
        name, k, m, bs = geom
        n, S = k + m, oracle.shard_size(bs, k)
        src_ar, out_ar = Arena(how), Arena(how)
        pag_src, pag_out = Arena("pageable"), Arena("pageable")
        reqs = []
        # every object as mec_batcher_encode (complete images) and as mec_batcher_encode_sg (parity images + data digests);
        # one encode with a data drive offline, one with a parity drive offline, one encode_sg with a parity drive offline
        plan = [(o, sg) for o in range(len(objs)) for sg in (False, True)]
        if extra_one:
            plan.append((0, False))
        for q, (o, sg) in enumerate(plan):
            data, want = objs[o]
            pageable = pageable_every and q % pageable_every == 1
            sa, oa = (pag_src, pag_out) if pageable else (src_ar, out_ar)
            offline = {1} if (o == 3 and not sg) else {k} if (o == 5 and not sg) else {n - 1} if (o == 6 and sg) else set()
            files = [None if i in offline or (sg and i < k) else oa.reserve(want[i].size, (2 * (q + i) + 1) % 16) for i in range(n)]
            nb = -(-data.size // bs)
            dd = oa.reserve(nb * k * 32, (2 * q + 3) % 16) if sg else None
            reqs.append(dict(o=o, sg=sg, sa=sa, oa=oa, src=sa.reserve(data.size, 1 + q % 15), files=files, dd=dd, nb=nb))
        for i, ar in enumerate((src_ar, out_ar, pag_src, pag_out)):
            ar.alloc(1000 + i)
        marker = np.zeros(1, dtype=np.uint8)
        calls, want_rc = [], []
        for q, r in enumerate(reqs):
            data, want = objs[r["o"]]
            r["sa"].view(r["src"], data.size)[:] = data
            r["sa"].expect(r["src"], data, {"request": q, "what": "src"})
            fp = (C.c_void_p * n)(*[None if f is None else r["oa"].base + f for f in r["files"]])
            for i, f in enumerate(r["files"]):
                if f is not None:
                    r["oa"].expect(f, want[i], {"request": q, "drive": i}, frame=32 + S)
            if r["sg"]:
                # data drives: only NULL / non-NULL is looked at
                fp = (C.c_void_p * n)(*[marker.ctypes.data if i < k else (None if r["files"][i] is None else r["oa"].base + r["files"][i])
                                        for i in range(n)])
                dd_want = np.stack([want[i][b * (32 + S):b * (32 + S) + 32] for b in range(r["nb"]) for i in range(k)]).reshape(-1)
                r["oa"].expect(r["dd"], dd_want, {"request": q, "what": "data_digests"}, frame=k * 32)
                dd_ptr = r["oa"].base + r["dd"]
                calls.append(lambda h=bat.h, s=r["sa"].base + r["src"], ln=data.size, fp=fp, dp=dd_ptr: L.mec_batcher_encode_sg(h, s, ln, fp, dp, 0))
            else:
                calls.append(lambda h=bat.h, s=r["sa"].base + r["src"], ln=data.size, fp=fp: L.mec_batcher_encode(h, s, ln, fp, 0))
            want_rc.append(data.size)
        # the Python binding's own pinned outputs (Batcher.encode / Batcher.encode_sg), on the object with an odd shard tail
        wrap = []
        wdata, wwant = objs[-1]
        if wrapper:
            wsrc = mb.pinned_array(wdata.size)
            wsrc[:] = wdata
            for sg in (False, True):
                slot = {}
                wrap.append(slot)
                calls.append(lambda sg=sg, slot=slot: (slot.setdefault("r", (bat.encode_sg if sg else bat.encode)(wsrc, pinned=True)), wdata.size)[1])
                want_rc.append(wdata.size)
        sizes = [objs[r["o"]][0].size for r in reqs] + ([wdata.size] * 2 if wrapper else [])
        nslots = sum(-(-s // bs) for s in sizes)   # = the worker's count of a PUT's blocks
        ntails = sum(1 for s in sizes if s % bs)
        rec = dict(info or {}, geom=name, kind="put", n=n, worker_blocks=nslots, nslots=nslots, ntails=ntails,
                   nfull=nslots - ntails, mapped=n <= 32 and not pageable_every and config != "put-memcpy")
        res = run_round(bat, calls, rnd, rec)
        check_rc(res, want_rc, rnd)
        for ar in (src_ar, out_ar, pag_src, pag_out):
            ar.check(rnd)
        for slot in wrap:
            r = slot.get("r")
            if r is None:
                continue
            if isinstance(r, tuple):
                files, dd = r
                assert files[:k] == [None] * k and dd.shape == (-(-wdata.size // bs), k, 32)
                for i in range(k, n):
                    if not np.array_equal(files[i], wwant[i]):
                        out["mismatches"].append({"round": rnd, "what": "Batcher.encode_sg", "drive": i})
                for b in range(dd.shape[0]):
                    for i in range(k):
                        if not np.array_equal(dd[b, i], wwant[i][b * (32 + S):b * (32 + S) + 32]):
                            out["mismatches"].append({"round": rnd, "what": "Batcher.encode_sg digest", "block": b, "drive": i})
                for f in files[k:]:
                    L.mec_free_pinned(f.ctypes.data)
                L.mec_free_pinned(dd.ctypes.data)
            else:
                for i in range(n):
                    if not np.array_equal(r[i], wwant[i]):
                        out["mismatches"].append({"round": rnd, "what": "Batcher.encode", "drive": i})
                    L.mec_free_pinned(r[i].ctypes.data)
        if wrapper:
            L.mec_free_pinned(wsrc.ctypes.data)
        for ar in (src_ar, out_ar, pag_src, pag_out):
            if hasattr(ar, "buf"):
                ar.free()
        return rec

    def put_blocks(objs, bs, wrapper=True):
        nb = [-(-d.size // bs) for d, _ in objs]
        return 2 * sum(nb) + (2 * nb[-1] if wrapper else 0)

    # ---- GET ----------------------------------------------------------------------------------------------------------------
    def reader_sets(k, m):
        sets = [("r0", {k + m - 1}), ("r1", {1})]
        if m >= 4:
            sets.append(("r4", {0, 2, 5, 6}))
        if m >= 12:
            sets.append(("r12", set(range(12))))
        return sets

    def ranges_of(size, bs, S):
        rs = [(0, size)]
        a = min(size - 1, S // 2 + 3)                        # starts and ends mid-shard
        rs.append((a, min(size - a, bs + S)))
        if size >= 2 * bs:
            rs.append((bs, bs))                              # exactly one block, on block edges
        t = size % bs
        if size > bs and t > 2:
            rs.append((size - t + t // 3, t - t // 3 - 1))   # inside the short last block only
        return sorted({r for r in rs if r[1] > 0})

    def get_round(bat, geom, objs, rnd, plan, info=None):
        """plan: list of (object, offline set, offset, length)"""
        name, k, m, bs = geom
        n, S = k + m, oracle.shard_size(bs, k)
        fil, dst = Arena("pinned"), Arena("pinned")
        used = sorted({o for o, _, _, _ in plan})
        fpos = {o: [fil.reserve(objs[o][1][i].size, (5 * o + 3 * i) % 16) for i in range(n)] for o in used}
        dpos = [dst.reserve(ln, (2 * q + 1) % 16) for q, (_, _, _, ln) in enumerate(plan)]
        fil.alloc(2000)
        dst.alloc(2001)
        for o in used:
            for i in range(n):
                fil.view(fpos[o][i], objs[o][1][i].size)[:] = objs[o][1][i]
                fil.expect(fpos[o][i], objs[o][1][i], {"object": o, "drive": i, "what": "part file"})
        calls, want_rc, hints = [], [], []
        for q, (o, offl, off, ln) in enumerate(plan):
            data = objs[o][0]
            fp = (C.c_void_p * n)(*[None if i in offl else fil.base + fpos[o][i] for i in range(n)])
            dst.expect(dpos[q], data[off:off + ln], {"request": q, "object": o, "offset": off, "length": ln, "offline": sorted(offl)})
            hint = C.c_int(-1)
            hints.append(hint)
            calls.append(lambda h=bat.h, fp=fp, off=off, ln=ln, tot=data.size, d=dst.base + dpos[q], hint=hint:
                         L.mec_batcher_decode(h, fp, off, ln, tot, d, C.byref(hint)))
            want_rc.append(ln)
        groups = {}
        for o, offl, off, ln in plan:
            size = objs[o][0].size
            sfs = oracle.shard_file_size(bs, k, size)
            nbt = -(-sfs // S)
            b0, b1 = off // bs, (off + ln) // bs - (1 if (off + ln) % bs == 0 else 0)
            b1 = min(b1, nbt - 1)
            tail = min(S, sfs - b1 * S) != S
            g = groups.setdefault(tuple(sorted(offl)), [0, 0, 0])
            g[0] += b1 - b0 + 1
            g[1] += 1 if tail else 0
            g[2] += ln // bs + 2
        rec = dict(info or {}, geom=name, kind="get", n=n, groups=len(groups), worker_blocks=sum(g[2] for g in groups.values()),
                   nslots=sum(g[0] for g in groups.values()), ntails=sum(g[1] for g in groups.values()),
                   group_tails=[g[1] for g in groups.values()], mapped=n <= 32)
        rec["nfull"] = rec["nslots"] - rec["ntails"]
        res = run_round(bat, calls, rnd, rec)
        check_rc(res, want_rc, rnd)
        for q, h in enumerate(hints):
            if h.value != 0:
                out["mismatches"].append({"round": rnd, "request": q, "heal_hint": h.value})
        fil.check(rnd)
        dst.check(rnd)
        fil.free()
        dst.free()
        return rec

    def get_main_plan(k, m, bs, S, objs, sets):
        return [(o, offl, a, ln) for _, offl in sets for o in range(len(objs)) for a, ln in ranges_of(objs[o][0].size, bs, S)]

    def get_blocks(plan, bs):
        return sum(ln // bs + 2 for _, _, _, ln in plan)

    # ---- the rounds ---------------------------------------------------------------------------------------------------------
    if kind == "put":
        pre = numa_precondition() if config.startswith("put-dma") else None
        out["numa_precondition"] = pre
    for gi, geom in enumerate(GEOMS):
        name, k, m, bs = geom
        n, S = k + m, oracle.shard_size(bs, k)
        objs = []
        for o, size in enumerate(sizes_of(k, bs)):
            d = rand(size, 7000 + 100 * gi + o)
            objs.append((d, oracle_files(k, m, bs, d, f"{size}_{7000 + 100 * gi + o}")))
        if kind == "put":
            cap = put_blocks(objs, bs)
            bat = new_batcher(k, m, bs, cap)
            if num_sms is None:
                num_sms = bat.stat("num_sms")
            put_round(bat, geom, objs, f"{name}/main", info={"name": "main", "cap": cap})
            if depth0:
                put_round(bat, geom, objs, f"{name}/overcap", extra_one=True, info={"name": "overcap", "cap": cap})
            if config.startswith("put-dma"):
                # pinned and pageable callers in one batch: no gather / scatter kernels for any of them
                put_round(bat, geom, objs, f"{name}/pageable-mix", pageable_every=3, info={"name": "pageable-mix", "cap": cap})
                if pre and pre["numa"]["same"]:
                    put_round(bat, geom, objs, f"{name}/numa", how="numa", info={"name": "numa", "cap": cap})
            bat.close()
        else:
            sets = reader_sets(k, m)
            plan = get_main_plan(k, m, bs, S, objs, sets)
            cap = get_blocks(plan, bs)
            bat = new_batcher(k, m, bs, cap)
            if num_sms is None:
                num_sms = bat.stat("num_sms")
            get_round(bat, geom, objs, f"{name}/main", plan, info={"name": "main", "cap": cap})
            if depth0:
                # one reader set of cap + 2 worker blocks: two batches
                one = [(o, {1}, a, ln) for o in range(len(objs)) for a, ln in ranges_of(objs[o][0].size, bs, S)]
                whole = (len(objs) - 1, {1}, 0, objs[-1][0].size)
                while get_blocks(one + [whole], bs) <= cap:
                    one.append(whole)
                one += [(0, {1}, 0, 1)] * ((cap - get_blocks(one, bs)) // 2 + 1)   # 1-byte GETs count 2 blocks each
                get_round(bat, geom, objs, f"{name}/overcap", one, info={"name": "overcap", "cap": cap})
            bat.close()
        if depth0:
            # more than 5 x SMs blocks in ONE batch: the throughput kernel over the full blocks plus one launch per short block
            bs64 = 64 * KiB - (1 if bs % 2 else 0)
            limit = 5 * num_sms
            nblk = limit // 8 + 4   # eight requests: four objects, each as encode and encode_sg (GET: whole and inner range)
            big = []
            for q in range(4):
                size = nblk * bs64 + 1 + 997 * q
                d = rand(size, 9000 + 100 * gi + q)
                big.append((d, oracle_files(k, m, bs64, d, f"{size}_{9000 + 100 * gi + q}")))
            g64 = (name + "@64k", k, m, bs64)
            if kind == "put":
                cap64 = put_blocks(big, bs64, wrapper=False)
                bat = new_batcher(k, m, bs64, cap64)
                put_round(bat, g64, big, f"{g64[0]}/overlimit", wrapper=False, info={"name": "overlimit", "cap": cap64, "limit": limit})
            else:
                plan = [(q, {1}, 0, big[q][0].size) for q in range(4)] + [(q, {1}, 1 + q, big[q][0].size - 2 - q) for q in range(4)]
                cap64 = get_blocks(plan, bs64)
                bat = new_batcher(k, m, bs64, cap64)
                get_round(bat, g64, big, f"{g64[0]}/overlimit", plan, info={"name": "overlimit", "cap": cap64, "limit": limit})
            bat.close()
    out["num_sms"] = num_sms
    out["limit"] = 5 * num_sms
    out["child_s"] = round(time.time() - t_start, 2)
    out["oracle_s"] = round(out["oracle_s"], 2)
    print(json.dumps(out))


# ---- parent ---------------------------------------------------------------------------------------------------------------------

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oracle_cache(tmp_path_factory):
    return str(tmp_path_factory.mktemp("batcher_oracle"))


def _run_child(config, cache_dir):
    env = {key: v for key, v in os.environ.items() if not key.startswith(("MEC_BATCHER_", "MEC_NO_BATCH_COPY"))}
    env.update(CONFIGS[config][1])
    t0 = time.time()
    p = subprocess.run([sys.executable, os.path.abspath(__file__), config, cache_dir], env=env, capture_output=True, text=True,
                       timeout=CHILD_TIMEOUT_S, cwd=ROOT)
    assert p.returncode == 0, f"child {config} exited {p.returncode}:\n{p.stderr[-4000:]}"
    res = json.loads(p.stdout.strip().split("\n")[-1])
    res["wall_s"] = round(time.time() - t0, 2)
    return res


def _forms(d):
    return {f: d["form_" + f] for f in FORMS if d["form_" + f]}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_batcher_config(oracle, oracle_cache, config):
    kind, env = CONFIGS[config]
    depth0 = env.get("MEC_BATCHER_DEPTH") == "0"
    res = _run_child(config, oracle_cache)
    print(json.dumps({"config": config, "wall_s": res["wall_s"], "child_s": res["child_s"], "init_s": res["init_s"],
                      "oracle_s": res["oracle_s"], "numa_precondition": res.get("numa_precondition")}))
    assert not res["mismatches"], res["mismatches"][:10]
    limit = res["limit"]
    gather = config == "put-gather" or config == "put-hybrid"   # hybrid: every round here has >= 8 callers
    if config.startswith("put-dma"):
        pre = res["numa_precondition"]
        assert pre["numa"]["same"], f"registered buffers are not device-addressable at their host address: {pre}"
        assert any(r["name"] == "numa" for r in res["rounds"])
    names = {(r["geom"], r["name"]) for r in res["rounds"]}
    for g in GEOMS:
        assert (g[0], "main") in names
        if depth0:
            assert (g[0], "overcap") in names and (g[0] + "@64k", "overlimit") in names
    for r in res["rounds"]:
        d, ctx = r["d"], (r["round"], r["d"])
        forms = _forms(d)
        other = sum(v for f, v in forms.items() if f != "small")
        # no frame is corrupt here: a merged GET redone on its own would hide a mis-staged frame behind exact bytes
        assert d["redone"] == 0, ctx
        if kind == "put":
            assert d["requests"] == r["requests"], ctx
            if depth0:
                assert d["batches"] == (2 if r["name"] == "overcap" else 1), ctx
            else:
                assert 0 < d["batches"] < d["requests"], ctx
            if r["mapped"]:
                assert d["kernel_batches"] == d["batches"], ctx
            elif r["name"] == "pageable-mix" and not depth0:
                assert d["kernel_batches"] < d["batches"], ctx   # batches cut short may hold pinned callers only
            else:
                assert d["kernel_batches"] == 0, ctx
            if r["name"] == "overcap" or not depth0:
                continue
            if r["name"] == "overlimit":
                # the full blocks in ONE throughput launch, every short block in one latency launch of its own
                assert r["nfull"] > limit and r["nslots"] > limit, ctx
                assert other == 1 and forms.get("small", 0) == r["ntails"], ctx
                if r["mapped"]:
                    assert d["launches"] == (1 if gather else 0) + 1 + r["ntails"] + 1, ctx
            elif r["mapped"]:
                # the whole batch, full and short blocks, is ONE latency launch with a per-block table
                assert r["nslots"] <= limit and forms == {"small": 1}, ctx
                assert d["launches"] == (3 if gather else 2), ctx
            else:
                # per-request copies: one launch over every caller's full blocks, one per short block
                assert other == 0 and forms.get("small", 0) == (1 if r["nfull"] else 0) + r["ntails"], ctx
        else:
            if not r["mapped"]:
                # more drives than the kernels' descriptor holds: every GET runs on its own, outside any batch
                assert d["batches"] == 0 and d["kernel_batches"] == 0, ctx
                continue
            assert d["requests"] == r["requests"] and d["kernel_batches"] == d["batches"], ctx
            if not depth0:
                assert r["groups"] <= d["batches"] < d["requests"], ctx
                continue
            want = {"main": r["groups"], "overcap": 2, "overlimit": 1}[r["name"]]
            assert d["batches"] == want, ctx
            if r["name"] == "overcap":
                continue
            g = 1 if config in ("get-gather", "get-mixed") and r["name"] == "main" else 0
            sc = 0 if config == "get-out2" else 1
            if r["name"] == "overlimit":
                g = 1 if config == "get-gather" else 0
                assert r["nfull"] > limit and other == 1 and forms.get("small", 0) == r["ntails"], ctx
                assert d["launches"] == g + 1 + r["ntails"] + sc, ctx
            else:
                # one latency launch per reader set; every set has short last blocks, so each ran with the per-block length table
                assert all(t > 0 for t in r["group_tails"]) and forms == {"small": r["groups"]}, ctx
                assert d["launches"] == r["groups"] * (g + 1 + sc), ctx


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])
