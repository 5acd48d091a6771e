"""GPU tests of heals through the cross-request coalescer (mec_batcher_heal): every staging path, geometry, stale set and frame
alignment, byte for byte against the CPU oracle and against mec_heal_prefer on the same inputs.

The staging switches are read once per process (MEC_BATCHER_DMA_BLOCKS, MEC_BATCHER_DEPTH), so every configuration runs in a child
process of its own: this file run as a script.  The child drives concurrent heals through the batcher, released together by a
barrier, checks every healed part file, every reader and every guard byte itself, and prints one JSON line with the mismatches and
the batcher's counters per round.  The parent asserts on that line which batches, kernels and kernel forms ran.

Every caller has its own copy of the surviving part files and its own out files, each between guard bytes at an offset of its own
(out files at odd offsets) in a page-locked buffer filled with a non-zero pattern: a skipped byte, a frame written at the wrong place
or a store past the end of a frame shows up.  With MEC_BATCHER_DEPTH=0 and a 0.5 s max_wait_us the merging is deterministic: the
batcher is capped at exactly one round's blocks (ceil(total / bs) per heal), so a round of one key (reader set + stale set) is one
batch, and a round of two stale sets is two.  A second batcher with 64 KiB blocks heals more than 5 x SMs blocks in one batch, which
takes the throughput kernel plus one launch per short last block."""
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
# (name, k, m, block size, m stale drives of data and parity mixed); RS(7,5): odd S, frames at every alignment mod 4; RS(20,12):
# n = 32 = kBatchMaxFiles; RS(10,1) at an odd block size; RS(20,13), n = 33: too many drives for the merged path
GEOMS = (("rs12_4", 12, 4, MiB, {1, 5, 12, 15}), ("rs7_5", 7, 5, MiB, {0, 3, 6, 8, 11}), ("rs16_4", 16, 4, MiB, {2, 9, 16, 19}),
         ("rs20_12", 20, 12, 256 * KiB, {1, 4, 7, 10, 13, 19, 20, 22, 24, 27, 30, 31}), ("rs10_1", 10, 1, MiB - 1, {4}),
         ("rs20_13", 20, 13, 256 * KiB, None))
CONFIGS = {
    "heal-dma": {},
    "heal-dma-depth0": {"MEC_BATCHER_DEPTH": "0"},
    "heal-gather": {"MEC_BATCHER_DMA_BLOCKS": "1000000", "MEC_BATCHER_DEPTH": "0"},
}
CHILD_TIMEOUT_S = 300
GUARD = 64
MAX_WAIT_US = 500_000
FILE_CORRUPT, READ_QUORUM, INVALID_ARGUMENT = -7, -10, -12


# ---- child ----------------------------------------------------------------------------------------------------------------------

def _child(config, cache_dir):
    import ctypes as C
    import threading

    import numpy as np

    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import minio_b200 as mb
    import oracle_lib as oracle

    env = CONFIGS[config]
    depth0 = env.get("MEC_BATCHER_DEPTH") == "0"
    L = mb.lib()
    out = {"config": config, "rounds": [], "mismatches": [], "checks": 0}
    t_start = time.time()

    def rand(n, seed):
        return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)

    def oracle_files(k, m, bs, data, key):
        """oracle.erasure_encode, cached on disk across the children (every child encodes the same seeded objects)"""
        path = os.path.join(cache_dir, f"{k}_{m}_{bs}_{key}.npy")
        if os.path.exists(path):
            return list(np.load(path))
        files, _ = oracle.erasure_encode(k, m, bs, oracle.HIGHWAYHASH256S, data)
        tmp = f"{path}.{os.getpid()}.npy"
        np.save(tmp, np.stack(files))
        os.replace(tmp, path)
        return files

    def mismatch(rec):
        out["mismatches"].append(rec)

    class Arena:
        """one host buffer holding many regions, each GUARD bytes clear of the previous one at a chosen misalignment; filled with
        a non-zero pattern, compared as a whole with the pattern plus the expected regions after the round"""

        def __init__(self, how="pinned"):
            self.how, self.size, self.regions = how, 0, []

        def reserve(self, nbytes, mis):
            off = (self.size + GUARD + 63) // 64 * 64 + mis
            self.size = off + nbytes
            return off

        def alloc(self, seed):
            total = self.size + GUARD
            self.buf = mb.pinned_array(total) if self.how == "pinned" else np.empty(total, dtype=np.uint8)
            self.buf[:] = rand(total, seed) | 1
            self.ref = self.buf.copy()
            self.base = self.buf.ctypes.data

        def view(self, off, n):
            return self.buf[off:off + n]

        def expect(self, off, want, label):
            self.regions.append((off, want, label))

        def check(self, rnd):
            for off, want, label in self.regions:
                got = self.buf[off:off + want.size]
                if not np.array_equal(got, want):
                    bad = np.flatnonzero(got != want)
                    mismatch(dict(label, round=rnd, bytes=int(bad.size), first=int(bad[0])))
                self.ref[off:off + want.size] = want
            bad = np.flatnonzero(self.buf != self.ref)
            if bad.size:
                mismatch({"round": rnd, "guard": self.how, "bytes": int(bad.size), "first": int(bad[0])})

        def free(self):
            if self.how == "pinned":
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
        [t.start() for t in th]
        [t.join() for t in th]
        after = snap(bat)
        out["rounds"].append(dict(info, round=rnd, requests=len(calls), d={s: after[s] - before[s] for s in stat_names}))
        return res

    def new_batcher(k, m, bs, cap):
        return mb.Batcher(k, m, bs, max_batch_blocks=cap, max_wait_us=MAX_WAIT_US)

    def sizes_of(bs):
        return [1, 4321, bs - 1, bs, 3 * bs + 777]

    def heal_round(bat, geom, objs, rnd, plan, how="pinned", flip=None, compare_codec=None, info=None):
        """plan: list of (object, stale set, offline set, prefer set or None, reader-and-stale drive or None).  Every request reads
        its own copies of the surviving part files.  flip = (request, drive, byte offset in the file): one byte of that reader is
        changed before the round.  compare_codec: a Codec whose mec_heal_prefer must give the same bytes, results and corrupt[]."""
        name, k, m, bs = geom[:4]
        n = k + m
        fil, outa = Arena(how), Arena(how)
        reqs = []
        for q, (o, stale, offl, pref, both) in enumerate(plan):
            want = objs[o][1]
            readers = [None if (i in stale and i != both) or i in offl else fil.reserve(want[i].size, (5 * q + 3 * i) % 16)
                       for i in range(n)]
            outs = [outa.reserve(want[i].size, (2 * (q + i) + 1) % 16) if (i in stale or i == both) else None for i in range(n)]
            reqs.append((readers, outs))
        fil.alloc(3000 + len(rnd))
        outa.alloc(3001 + len(rnd))
        calls, want_rc, corrupts, keep = [], [], [], []
        for q, ((o, stale, offl, pref, both), (readers, outs)) in enumerate(zip(plan, reqs)):
            data, want = objs[o]
            for i, f in enumerate(readers):
                if f is None:
                    continue
                fil.view(f, want[i].size)[:] = want[i]
                exp = want[i]
                if flip and flip[0] == q and flip[1] == i:
                    fil.view(f + flip[2], 1)[:] ^= 0x5A
                    exp = fil.view(f, want[i].size).copy()
                fil.expect(f, exp, {"request": q, "drive": i, "what": "reader"})
            for i, f in enumerate(outs):
                if f is not None:
                    outa.expect(f, want[i], {"request": q, "drive": i, "what": "healed part file", "size": data.size})
            fp = (C.c_void_p * n)(*[None if f is None else fil.base + f for f in readers])
            op = (C.c_void_p * n)(*[None if f is None else outa.base + f for f in outs])
            pf = None if pref is None else np.array([1 if i in pref else 0 for i in range(n)], dtype=np.uint8)
            cor = np.full(n, 0xEE, dtype=np.uint8)
            keep += [fp, op, pf]
            corrupts.append(cor)
            calls.append(lambda h=bat.h, fp=fp, pf=pf, tot=data.size, op=op, cor=cor:
                         L.mec_batcher_heal(h, fp, None if pf is None else pf.ctypes.data, tot, op, cor.ctypes.data))
            want_rc.append(FILE_CORRUPT if flip and flip[0] == q else 0)
        nslots = sum(-(-objs[o][0].size // bs) for o, *_ in plan)
        ntails = sum(1 for o, *_ in plan if oracle.shard_file_size(bs, k, objs[o][0].size) % oracle.shard_size(bs, k))
        keys = {(tuple(sorted(st)), tuple(sorted(off)), None if pr is None else tuple(sorted(pr))) for _, st, off, pr, _ in plan}
        rec = dict(info or {}, geom=name, keys=len(keys), nslots=nslots, ntails=ntails, nfull=nslots - ntails)
        res = run_round(bat, calls, rnd, rec)
        for q, (r, w) in enumerate(zip(res, want_rc)):
            if r != w:
                mismatch({"round": rnd, "request": q, "rc": r if isinstance(r, int) else str(r), "want": w})
            want_cor = np.zeros(n, dtype=np.uint8)
            if flip and flip[0] == q:
                want_cor[flip[1]] = 1
            if not np.array_equal(corrupts[q], want_cor):
                mismatch({"round": rnd, "request": q, "corrupt": corrupts[q].tolist()})
        if compare_codec is not None:
            # mec_heal_prefer on the very same inputs: same bytes, result and corrupt[]
            for q, ((o, stale, offl, pref, both), (readers, outs)) in enumerate(zip(plan, reqs)):
                files = [None if f is None else fil.view(f, objs[o][1][i].size) for i, f in enumerate(readers)]
                pf = None if pref is None else [1 if i in pref else 0 for i in range(n)]
                got, rc, cor = compare_codec.heal(files, [f is not None for f in outs], objs[o][0].size, prefer=pf, report=True)
                out["checks"] += 1
                if rc != res[q] or not np.array_equal(cor, corrupts[q]):
                    mismatch({"round": rnd, "request": q, "mec_heal_prefer": rc, "corrupt": cor.tolist()})
                for i, f in enumerate(outs):
                    if f is not None and not np.array_equal(got[i], outa.view(f, got[i].size)):
                        mismatch({"round": rnd, "request": q, "drive": i, "what": "differs from mec_heal_prefer"})
        fil.check(rnd)
        outa.check(rnd)
        fil.free()
        outa.free()
        return rec

    def codes(bat, codec, geom, objs):
        """host-side checks: the same codes, corrupt[] and untouched outputs as mec_heal_prefer"""
        name, k, m, bs = geom[:4]
        n = k + m
        data, want = objs[-1]
        files = [mb.pinned_array(want[i].size) for i in range(n)]
        for i in range(n):
            files[i][:] = want[i]
        fsz = want[0].size
        cases = []
        full = (C.c_void_p * n)(*[f.ctypes.data for f in files])
        short = (C.c_void_p * n)(*[files[i].ctypes.data if i < k - 1 else None for i in range(n)])
        for label, hb, fp, tot, with_out in (("null handle", False, full, data.size, True), ("null files", True, None, data.size, True),
                                             ("null out_files", True, full, data.size, False), ("total 0", True, full, 0, True),
                                             ("total < 0", True, full, -5, True), ("read quorum", True, short, data.size, True)):
            got = []
            for which in ("batcher", "codec"):
                o = mb.pinned_array(fsz)
                o[:] = 0x5A
                op = (C.c_void_p * n)(*[o.ctypes.data if i == 1 else None for i in range(n)]) if with_out else None
                cor = np.full(n, 0xEE, dtype=np.uint8)
                if which == "batcher":
                    rc = L.mec_batcher_heal(bat.h if hb else None, fp, None, tot, op, cor.ctypes.data)
                else:
                    rc = L.mec_heal_prefer(codec.h if hb else None, fp, None, tot, op, cor.ctypes.data)
                got.append((rc, cor.tolist(), bool((o == 0x5A).all())))
                L.mec_free_pinned(o.ctypes.data)
            out["checks"] += 1
            want_rc = {"total 0": 0, "total < 0": 0, "read quorum": READ_QUORUM}.get(label, INVALID_ARGUMENT)
            if got[0] != got[1] or got[0][0] != want_rc or not got[0][2]:
                mismatch({"geom": name, "case": label, "batcher": got[0], "mec_heal_prefer": got[1], "want": want_rc})
        for f in files:
            L.mec_free_pinned(f.ctypes.data)

    def wrapper(bat, geom, objs):
        """Batcher.heal with page-locked out files (merged) and with pageable ones (private path): the oracle's bytes"""
        name, k, m, bs = geom[:4]
        n = k + m
        data, want = objs[-1]
        files = [None if i == 1 else mb.pinned_array(want[i].size) for i in range(n)]
        for i, f in enumerate(files):
            if f is not None:
                f[:] = want[i]
        for pinned in (True, False):
            outs, rc, cor = bat.heal(files, [i == 1 for i in range(n)], data.size, pinned=pinned)
            out["checks"] += 1
            if rc != 0 or cor.any() or not np.array_equal(outs[1], want[1]) or any(outs[i] is not None for i in range(n) if i != 1):
                mismatch({"geom": name, "what": "Batcher.heal", "pinned": pinned, "rc": rc})
            if pinned:
                L.mec_free_pinned(outs[1].ctypes.data)
        for f in files:
            if f is not None:
                L.mec_free_pinned(f.ctypes.data)

    def mixed_kinds(geom, objs):
        """one heal (drive 1 stale), one PUT and one degraded GET (drive 1 offline) of every object, queued together on a batcher
        capped at their blocks: heals never share a batch with the others, and every output is exact"""
        name, k, m, bs = geom[:4]
        n = k + m
        ar = Arena()
        heals = [(o, [None if i == 1 else ar.reserve(objs[o][1][i].size, (3 * o + i) % 16) for i in range(n)],
                  ar.reserve(objs[o][1][1].size, (2 * o + 1) % 16)) for o in range(len(objs))]
        puts = [(o, ar.reserve(objs[o][0].size, (o + 5) % 16), [ar.reserve(objs[o][1][i].size, (2 * (o + i) + 1) % 16) for i in range(n)])
                for o in range(len(objs))]
        gets = [(o, [None if i == 1 else ar.reserve(objs[o][1][i].size, (7 * o + i) % 16) for i in range(n)],
                 ar.reserve(objs[o][0].size, (2 * o + 3) % 16)) for o in range(len(objs))]
        ar.alloc(4000)

        def place(off, arr, label):
            ar.view(off, arr.size)[:] = arr
            ar.expect(off, arr, label)

        def ptrs(offs):
            return (C.c_void_p * n)(*[None if f is None else ar.base + f for f in offs])
        calls, want_rc, blocks = [], [], 0
        for o, rd, od in heals:
            data, want = objs[o]
            for i, f in enumerate(rd):
                if f is not None:
                    place(f, want[i], {"kind": "heal", "object": o, "drive": i, "what": "reader"})
            ar.expect(od, want[1], {"kind": "heal", "object": o, "drive": 1})
            calls.append(lambda fp=ptrs(rd), op=ptrs([od if i == 1 else None for i in range(n)]), tot=data.size:
                         L.mec_batcher_heal(bat.h, fp, None, tot, op, None))
            want_rc.append(0)
            blocks += -(-data.size // bs)
        for o, so, fo in puts:
            data, want = objs[o]
            place(so, data, {"kind": "put", "object": o, "what": "src"})
            for i, f in enumerate(fo):
                ar.expect(f, want[i], {"kind": "put", "object": o, "drive": i})
            calls.append(lambda s=ar.base + so, ln=data.size, fp=ptrs(fo): L.mec_batcher_encode(bat.h, s, ln, fp, 0))
            want_rc.append(data.size)
            blocks += -(-data.size // bs)
        for o, rd, do in gets:
            data, want = objs[o]
            for i, f in enumerate(rd):
                if f is not None:
                    place(f, want[i], {"kind": "get", "object": o, "drive": i, "what": "reader"})
            ar.expect(do, data, {"kind": "get", "object": o})
            calls.append(lambda fp=ptrs(rd), ln=data.size, d=ar.base + do: L.mec_batcher_decode(bat.h, fp, 0, ln, ln, d, None))
            want_rc.append(data.size)
            blocks += data.size // bs + 2
        bat = new_batcher(k, m, bs, blocks)
        rnd = f"{name}/mixed-kinds"
        res = run_round(bat, calls, rnd, {"geom": name, "name": "mixed-kinds", "cap": blocks})
        for q, (r, w) in enumerate(zip(res, want_rc)):
            if r != w:
                mismatch({"round": rnd, "request": q, "rc": r if isinstance(r, int) else str(r), "want": w})
        ar.check(rnd)
        ar.free()
        bat.close()

    # ---- the rounds ---------------------------------------------------------------------------------------------------------
    num_sms = None
    for gi, geom in enumerate(GEOMS):
        name, k, m, bs, mixed = geom
        n = k + m
        objs = []
        for o, size in enumerate(sizes_of(bs)):
            d = rand(size, 8000 + 100 * gi + o)
            objs.append((d, oracle_files(k, m, bs, d, f"{size}_{8000 + 100 * gi + o}")))
        codec = mb.Codec(k, m, bs)

        def plan_of(stale, offl=frozenset(), pref=None, both=None):
            return [(o, stale, offl, pref, both) for _ in range(2) for o in range(len(objs))]

        main = plan_of({1})
        cap = sum(-(-objs[o][0].size // bs) for o, *_ in main)
        bat = new_batcher(k, m, bs, cap)
        if num_sms is None:
            num_sms = bat.stat("num_sms")
        if mixed is None:
            # more drives than the kernels' tables hold: every heal runs on its own, outside any batch
            heal_round(bat, geom, objs, f"{name}/serial-n", main, compare_codec=codec, info={"name": "serial", "cap": cap})
            codes(bat, codec, geom, objs)
            bat.close()
            codec.close()
            continue
        sets = [("data1", {1}, frozenset()), ("parity1", {n - 1}, frozenset()), ("mixed", mixed, frozenset())]
        if m >= 3:
            sets.append(("offline", {1}, frozenset({0, 3})))   # the reader set skips drives 0, 1 and 3
        for sname, stale, offl in sets:
            heal_round(bat, geom, objs, f"{name}/{sname}", plan_of(stale, offl), info={"name": "merged", "set": sname, "cap": cap})
        # preferReaders: the last k drives first, a reader set that is not the first k
        pref = set(range(n - k, n)) - {1}
        heal_round(bat, geom, objs, f"{name}/prefer", plan_of({1}, pref=pref), compare_codec=codec,
                   info={"name": "merged", "set": "prefer", "cap": cap})
        if m >= 2:
            # bitrot in drive 0 (a chosen reader) of request 4 (3 blocks + 777 bytes), block 1; k + 1 readers online
            S = oracle.shard_size(bs, k)
            heal_round(bat, geom, objs, f"{name}/bitrot", main, flip=(4, 0, (32 + S) + 32 + 7), compare_codec=codec,
                       info={"name": "bitrot", "cap": cap})
        # the private path: pageable buffers, and a drive that is both a reader and stale (passed through unchanged)
        heal_round(bat, geom, objs, f"{name}/pageable", main, how="pageable", compare_codec=codec, info={"name": "serial", "cap": cap})
        heal_round(bat, geom, objs, f"{name}/reader-stale", plan_of({1}, both=0), compare_codec=codec,
                   info={"name": "serial", "cap": cap})
        if depth0:
            # two stale sets queued together: two batches
            half = [(o, {1} if q < len(objs) else {n - 1}, frozenset(), None, None) for q, o in enumerate([*range(len(objs))] * 2)]
            heal_round(bat, geom, objs, f"{name}/two-sets", half, info={"name": "two-sets", "cap": cap})
        codes(bat, codec, geom, objs)
        wrapper(bat, geom, objs)
        bat.close()
        if depth0:
            mixed_kinds(geom, objs)
            # more than 5 x SMs blocks in ONE batch: the throughput kernel over the full blocks plus one launch per short block
            bs64 = 64 * KiB - (1 if bs % 2 else 0)
            limit = 5 * num_sms
            nblk = limit // 4 + 4
            big = []
            for q in range(4):
                size = nblk * bs64 + 1 + 997 * q
                d = rand(size, 9500 + 100 * gi + q)
                big.append((d, oracle_files(k, m, bs64, d, f"{size}_{9500 + 100 * gi + q}")))
            plan = [(q, {1}, frozenset(), None, None) for q in range(4)]
            cap64 = sum(-(-d.size // bs64) for d, _ in big)
            bat = new_batcher(k, m, bs64, cap64)
            heal_round(bat, (name + "@64k", k, m, bs64), big, f"{name}@64k/overlimit", plan,
                       info={"name": "overlimit", "cap": cap64, "limit": limit})
            bat.close()
        codec.close()
    out["num_sms"] = num_sms
    out["limit"] = 5 * num_sms
    out["child_s"] = round(time.time() - t_start, 2)
    print(json.dumps(out))


# ---- parent ---------------------------------------------------------------------------------------------------------------------

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oracle_cache(tmp_path_factory):
    return str(tmp_path_factory.mktemp("batcher_heal_oracle"))


def _run_child(config, cache_dir):
    env = {key: v for key, v in os.environ.items() if not key.startswith(("MEC_BATCHER_", "MEC_NO_BATCH_COPY"))}
    env.update(CONFIGS[config])
    p = subprocess.run([sys.executable, os.path.abspath(__file__), config, cache_dir], env=env, capture_output=True, text=True,
                       timeout=CHILD_TIMEOUT_S, cwd=ROOT)
    assert p.returncode == 0, f"child {config} exited {p.returncode}:\n{p.stderr[-4000:]}"
    return json.loads(p.stdout.strip().split("\n")[-1])


def _forms(d):
    return {f: d["form_" + f] for f in FORMS if d["form_" + f]}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_batcher_heal_config(oracle, oracle_cache, config):
    env = CONFIGS[config]
    depth0 = env.get("MEC_BATCHER_DEPTH") == "0"
    g = 1 if config == "heal-gather" else 0   # the gather kernel stages every request
    res = _run_child(config, oracle_cache)
    print(json.dumps({"config": config, "child_s": res["child_s"], "checks": res["checks"], "rounds": len(res["rounds"])}))
    assert not res["mismatches"], res["mismatches"][:10]
    limit = res["limit"]
    names = {(r["geom"], r["name"]) for r in res["rounds"]}
    for geom in GEOMS:
        if geom[4] is None:
            assert (geom[0], "serial") in names
            continue
        assert (geom[0], "merged") in names and (geom[0], "serial") in names
        if geom[2] >= 2:
            assert (geom[0], "bitrot") in names
        if depth0:
            assert (geom[0], "two-sets") in names and (geom[0], "mixed-kinds") in names and (geom[0] + "@64k", "overlimit") in names
    for r in res["rounds"]:
        d, ctx = r["d"], (r["round"], r["d"])
        forms = _forms(d)
        other = sum(v for f, v in forms.items() if f != "small")
        if r["name"] == "serial":
            # mec_heal_prefer on the private handle: nothing is queued, the batcher's codec launches nothing
            assert d["batches"] == 0 and d["kernel_batches"] == 0 and d["requests"] == 0 and d["launches"] == 0, ctx
            continue
        if r["name"] == "mixed-kinds":
            # heals, PUTs and GETs queued together: one batch per kind, every one through the gather / scatter kernels
            assert d["requests"] == r["requests"] and d["batches"] == 3 and d["kernel_batches"] == 3 and d["redone"] == 0, ctx
            continue
        assert d["requests"] == r["requests"] and d["kernel_batches"] == d["batches"], ctx
        assert d["redone"] == (1 if r["name"] == "bitrot" else 0), ctx
        if r["name"] == "overlimit":
            # the full blocks in ONE throughput launch, every short block in one latency launch of its own, one scatter
            assert d["batches"] == 1 and r["nfull"] > limit, ctx
            assert other == 1 and forms.get("small", 0) == r["ntails"], ctx
            assert d["launches"] == g + 1 + r["ntails"] + 1, ctx
            continue
        assert r["nslots"] <= limit, ctx
        want_batches = {"two-sets": 2}.get(r["name"], 1)
        if depth0:
            assert d["batches"] == want_batches, ctx
        else:
            assert want_batches <= d["batches"] <= d["requests"], ctx
        # per batch: ONE latency launch over every block (short last blocks with their own shard length) and one heal scatter
        assert forms == {"small": d["batches"]}, ctx
        assert d["launches"] == d["batches"] * (g + 2), ctx


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])
