"""GPU tests of reads of mixed erasure patterns through the cross-request coalescer (mec_batcher_new_ex with
MEC_BATCHER_MIX_PATTERNS, mec_batcher_decode_prefer): GETs and heals whose reader and stale sets differ from object to object, as
MinIO's per-object rotation of shard indices over the drives makes them (hashOrder, cmd/erasure-metadata-utils.go:178), merged
into ONE latency launch with a decode matrix per erasure block — byte for byte against the CPU oracle and against
mec_decode_prefer / mec_heal_prefer on a plain codec, on every staging path, geometry and frame alignment.

The staging switches are read once per process (MEC_BATCHER_DMA_BLOCKS, MEC_BATCHER_GET_OUT, MEC_BATCHER_DEPTH), so every
configuration runs in a child process of its own: this file run as a script.  The child releases concurrent callers together
with a barrier, checks every output, reader and guard byte itself and prints one JSON line with the mismatches and the batcher's
counters per round; the parent asserts which batches, patterns, launches and kernel forms ran.  With MEC_BATCHER_DEPTH=0, a
0.5 s max_wait_us and a batcher capped at exactly one round's blocks, the merging is deterministic."""
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
# RS(12,4): the default set; RS(4,2): the fewest streams; RS(8,8): up to eight rebuilt rows in two row passes; RS(6,3) at an odd
# block size: odd shard sizes, so frames in the part files and in the arena sit at every alignment
GEOMS = (("rs12_4", 12, 4, MiB), ("rs4_2", 4, 2, MiB), ("rs8_8", 8, 8, 256 * KiB), ("rs6_3", 6, 3, MiB - 1))
CONFIGS = {
    "pat-dma": {"MEC_BATCHER_DEPTH": "0"},
    "pat-gather": {"MEC_BATCHER_DMA_BLOCKS": "1000000", "MEC_BATCHER_DEPTH": "0"},
    "pat-out1": {"MEC_BATCHER_GET_OUT": "1", "MEC_BATCHER_DEPTH": "0"},
    "pat-out2": {"MEC_BATCHER_GET_OUT": "2", "MEC_BATCHER_DEPTH": "0"},
}
CHILD_TIMEOUT_S = 300
GUARD = 64
MAX_WAIT_US = 500_000
MIX = 1  # MEC_BATCHER_MIX_PATTERNS
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
        """one page-locked buffer holding many regions, each GUARD bytes clear of the previous one at a chosen misalignment;
        filled with a non-zero pattern, compared as a whole with the pattern plus the expected regions after the round"""

        def __init__(self):
            self.size, self.regions = 0, []

        def reserve(self, nbytes, mis):
            off = (self.size + GUARD + 63) // 64 * 64 + mis
            self.size = off + nbytes
            return off

        def alloc(self, seed):
            total = self.size + GUARD
            self.buf = mb.pinned_array(total)
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
                mismatch({"round": rnd, "guard": True, "bytes": int(bad.size), "first": int(bad[0])})

        def free(self):
            L.mec_free_pinned(self.base)

    stat_names = ["batches", "requests", "blocks", "kernel_batches", "redone", "launches", "small_launches", "patterns",
                  "mixed_batches"] + ["form_" + f for f in FORMS]

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

    def new_batcher(k, m, bs, cap, mix):
        return mb.Batcher(k, m, bs, max_batch_blocks=cap, max_wait_us=MAX_WAIT_US, mix_patterns=mix)

    def rotated(n, rho, drives):
        """shard indices that the physical drives `drives` hold for an object rotated by rho"""
        return {(d - rho) % n for d in drives}

    def chosen_of(n, k, offl, pref):
        """parallelReader's readers: with `pref` (at least k drives, all online here) the first k preferred ones, else the first
        k online"""
        if pref is not None:
            return sorted(pref)[:k]
        return [i for i in range(n) if i not in offl][:k]

    def read_slots(bs, S, k, size, off, ln):
        sfs = oracle.shard_file_size(bs, k, size)
        b0, b1 = off // bs, (off + ln) // bs - (1 if (off + ln) % bs == 0 else 0)
        return min(b1, -(-sfs // S) - 1) - b0 + 1

    def get_round(bat, geom, objs, rnd, plan, codec, flip=None, info=None):
        """plan: list of (object, offline shard set, offset, length, prefer set or None).  Every request reads its own copy of
        the part files.  flip = (request, shard, byte offset in the file): one byte of that copy is changed before the round.
        Every result is compared with the oracle's bytes and with mec_decode_prefer on `codec` over the same inputs."""
        name, k, m, bs = geom
        n, S = k + m, oracle.shard_size(bs, k)
        fil, dst = Arena(), Arena()
        fpos = [[None if i in offl else fil.reserve(objs[o][1][i].size, (5 * q + 3 * i) % 16) for i in range(n)]
                for q, (o, offl, _, _, _) in enumerate(plan)]
        dpos = [dst.reserve(ln, (2 * q + 1) % 16) for q, (_, _, _, ln, _) in enumerate(plan)]
        fil.alloc(2000 + len(rnd))
        dst.alloc(2001 + len(rnd))
        calls, hints, keep, keys = [], [], [], set()
        for q, (o, offl, off, ln, pref) in enumerate(plan):
            data, want = objs[o]
            for i, f in enumerate(fpos[q]):
                if f is None:
                    continue
                fil.view(f, want[i].size)[:] = want[i]
                exp = want[i]
                if flip and flip[0] == q and flip[1] == i:
                    fil.view(f + flip[2], 1)[:] ^= 0x5A
                    exp = fil.view(f, want[i].size).copy()
                fil.expect(f, exp, {"request": q, "drive": i, "what": "part file"})
            dst.expect(dpos[q], data[off:off + ln], {"request": q, "object": o, "offset": off, "length": ln})
            fp = (C.c_void_p * n)(*[None if f is None else fil.base + f for f in fpos[q]])
            pf = None if pref is None else np.array([1 if i in pref else 0 for i in range(n)], dtype=np.uint8)
            hint = C.c_int(-1)
            keep += [fp, pf]
            hints.append(hint)
            calls.append(lambda h=bat.h, fp=fp, pf=pf, off=off, ln=ln, tot=data.size, d=dst.base + dpos[q], hint=hint:
                         L.mec_batcher_decode_prefer(h, fp, None if pf is None else pf.ctypes.data, off, ln, tot, d, C.byref(hint)))
            ch = chosen_of(n, k, offl, pref)
            keys.add((tuple(ch), tuple(i for i in range(k) if i not in ch)))
        nslots = sum(read_slots(bs, S, k, objs[o][0].size, off, ln) for o, _, off, ln, _ in plan)
        alive_keys = {tuple(sorted(offl)) if pref is None else ("p",) + tuple(chosen_of(n, k, offl, pref)) for _, offl, _, _, pref in plan}
        rec = dict(info or {}, geom=name, kind="get", patterns=len(keys), keys=len(alive_keys), nslots=nslots,
                   rmax=max(len(t) for _, t in keys))
        res = run_round(bat, calls, rnd, rec)
        for q, (o, offl, off, ln, pref) in enumerate(plan):
            want_hint = FILE_CORRUPT if flip and flip[0] == q and flip[1] in chosen_of(n, k, offl, pref) else 0
            if res[q] != ln or hints[q].value != want_hint:
                mismatch({"round": rnd, "request": q, "rc": str(res[q]), "hint": hints[q].value, "want_hint": want_hint})
        # mec_decode_prefer on a plain codec, same inputs: same result, heal hint and bytes
        for q, (o, offl, off, ln, pref) in enumerate(plan):
            fp = (C.c_void_p * n)(*[None if f is None else fil.base + f for f in fpos[q]])
            pf = None if pref is None else np.array([1 if i in pref else 0 for i in range(n)], dtype=np.uint8)
            got = mb.pinned_array(max(ln, 1))
            hint = C.c_int(-1)
            rc = L.mec_decode_prefer(codec.h, fp, None if pf is None else pf.ctypes.data, off, ln, objs[o][0].size, got.ctypes.data,
                                     C.byref(hint))
            out["checks"] += 1
            if rc != res[q] or hint.value != hints[q].value or not np.array_equal(got[:ln], dst.view(dpos[q], ln)):
                mismatch({"round": rnd, "request": q, "mec_decode_prefer": rc, "hint": hint.value})
            L.mec_free_pinned(got.ctypes.data)
        fil.check(rnd)
        dst.check(rnd)
        fil.free()
        dst.free()
        return rec

    def heal_round(bat, geom, objs, rnd, plan, codec, info=None):
        """plan: list of (object, stale shard set); stale drives are offline readers too"""
        name, k, m, bs = geom
        n = k + m
        fil, outa = Arena(), Arena()
        fpos = [[None if i in st else fil.reserve(objs[o][1][i].size, (5 * q + 3 * i) % 16) for i in range(n)]
                for q, (o, st) in enumerate(plan)]
        opos = [[outa.reserve(objs[o][1][i].size, (2 * (q + i) + 1) % 16) if i in st else None for i in range(n)]
                for q, (o, st) in enumerate(plan)]
        fil.alloc(3000 + len(rnd))
        outa.alloc(3001 + len(rnd))
        calls, corrupts, keep, keys = [], [], [], set()
        for q, (o, st) in enumerate(plan):
            data, want = objs[o]
            for i, f in enumerate(fpos[q]):
                if f is not None:
                    fil.view(f, want[i].size)[:] = want[i]
                    fil.expect(f, want[i], {"request": q, "drive": i, "what": "reader"})
            for i, f in enumerate(opos[q]):
                if f is not None:
                    outa.expect(f, want[i], {"request": q, "drive": i, "what": "healed part file"})
            fp = (C.c_void_p * n)(*[None if f is None else fil.base + f for f in fpos[q]])
            op = (C.c_void_p * n)(*[None if f is None else outa.base + f for f in opos[q]])
            cor = np.full(n, 0xEE, dtype=np.uint8)
            keep += [fp, op]
            corrupts.append(cor)
            calls.append(lambda h=bat.h, fp=fp, op=op, tot=data.size, cor=cor: L.mec_batcher_heal(h, fp, None, tot, op, cor.ctypes.data))
            keys.add((tuple(chosen_of(n, k, st, None)), tuple(sorted(st))))
        rec = dict(info or {}, geom=name, kind="heal", patterns=len(keys), keys=len({tuple(sorted(st)) for _, st in plan}),
                   nslots=sum(-(-objs[o][0].size // bs) for o, _ in plan), rmax=max(len(st) for _, st in plan))
        res = run_round(bat, calls, rnd, rec)
        for q, (o, st) in enumerate(plan):
            if res[q] != 0 or corrupts[q].any():
                mismatch({"round": rnd, "request": q, "rc": str(res[q]), "corrupt": corrupts[q].tolist()})
            files = [None if f is None else fil.view(f, objs[o][1][i].size) for i, f in enumerate(fpos[q])]
            got, rc, cor = codec.heal(files, [i in st for i in range(n)], objs[o][0].size, report=True)
            out["checks"] += 1
            if rc != res[q] or cor.any():
                mismatch({"round": rnd, "request": q, "mec_heal_prefer": rc})
            for i, f in enumerate(opos[q]):
                if f is not None and not np.array_equal(got[i], outa.view(f, got[i].size)):
                    mismatch({"round": rnd, "request": q, "drive": i, "what": "differs from mec_heal_prefer"})
        fil.check(rnd)
        outa.check(rnd)
        fil.free()
        outa.free()
        return rec

    def get_cap(plan, bs):
        return sum(ln // bs + 2 for _, _, _, ln, _ in plan)

    def host_side(geom, objs, codec):
        """flags, prefer == NULL against mec_batcher_decode, and the error codes of mec_decode_prefer"""
        name, k, m, bs = geom
        n = k + m
        h = C.c_void_p()
        for flags in (2, MIX | 4, -1):
            rc = L.mec_batcher_new_ex(k, m, bs, 0, 16, 0, flags, C.byref(h))
            out["checks"] += 1
            if rc != INVALID_ARGUMENT or h.value:
                mismatch({"geom": name, "case": "flags", "flags": flags, "rc": rc})
        data, want = objs[-1]
        files = [mb.pinned_array(want[i].size) for i in range(n)]
        for i in range(n):
            files[i][:] = want[i]
        full = (C.c_void_p * n)(*[None if i == 1 else files[i].ctypes.data for i in range(n)])
        short = (C.c_void_p * n)(*[files[i].ctypes.data if i < k - 1 else None for i in range(n)])
        pref = np.array([1 if i >= n - k else 0 for i in range(n)], dtype=np.uint8)
        for mix in (False, True):
            bat = new_batcher(k, m, bs, 64, mix)
            # prefer == NULL: exactly mec_batcher_decode
            for off, ln in ((0, data.size), (7, data.size // 2)):
                got = []
                for fn in ("prefer", "plain"):
                    d = mb.pinned_array(max(ln, 1))
                    hint = C.c_int(-1)
                    if fn == "prefer":
                        rc = L.mec_batcher_decode_prefer(bat.h, full, None, off, ln, data.size, d.ctypes.data, C.byref(hint))
                    else:
                        rc = L.mec_batcher_decode(bat.h, full, off, ln, data.size, d.ctypes.data, C.byref(hint))
                    got.append((rc, hint.value, d[:ln].tobytes()))
                    L.mec_free_pinned(d.ctypes.data)
                out["checks"] += 1
                if got[0] != got[1] or got[0][0] != ln or got[0][2] != data[off:off + ln].tobytes():
                    mismatch({"geom": name, "case": "prefer NULL", "mix": mix, "rc": [g[0] for g in got]})
            cases = (("null handle", False, full, 0, data.size, data.size, True), ("null files", True, None, 0, data.size, data.size, True),
                     ("offset < 0", True, full, -1, 5, data.size, True), ("length < 0", True, full, 0, -1, data.size, True),
                     ("past total", True, full, 1, data.size, data.size, True), ("length 0", True, full, 0, 0, data.size, True),
                     ("null dst", True, full, 0, data.size, data.size, False),
                     ("read quorum", True, short, 0, data.size, data.size, True))
            for label, hb, fp, off, ln, tot, with_dst in cases:
                for pf in (None, pref):
                    got = []
                    for which in ("batcher", "codec"):
                        d = mb.pinned_array(max(data.size, 1))
                        d[:] = 0x5A
                        hint = C.c_int(-1)
                        dp = d.ctypes.data if with_dst else None
                        pp = None if pf is None else pf.ctypes.data
                        if which == "batcher":
                            rc = L.mec_batcher_decode_prefer(bat.h if hb else None, fp, pp, off, ln, tot, dp, C.byref(hint))
                        else:
                            rc = L.mec_decode_prefer(codec.h if hb else None, fp, pp, off, ln, tot, dp, C.byref(hint))
                        got.append((rc, hint.value, bool((d == 0x5A).all())))
                        L.mec_free_pinned(d.ctypes.data)
                    out["checks"] += 1
                    want_rc = {"length 0": 0, "read quorum": READ_QUORUM}.get(label, INVALID_ARGUMENT)
                    if got[0] != got[1] or got[0][0] != want_rc or not got[0][2]:
                        mismatch({"geom": name, "case": label, "prefer": pf is not None, "mix": mix, "batcher": got[0],
                                  "mec_decode_prefer": got[1], "want": want_rc})
            bat.close()
        for f in files:
            L.mec_free_pinned(f.ctypes.data)

    # ---- the rounds ---------------------------------------------------------------------------------------------------------
    num_sms = None
    for gi, geom in enumerate(GEOMS):
        name, k, m, bs = geom
        n, S = k + m, oracle.shard_size(bs, k)
        objs = []
        for o, size in enumerate((4321, bs - 1, bs, 2 * bs + 777)):
            d = rand(size, 6000 + 100 * gi + o)
            objs.append((d, oracle_files(k, m, bs, d, f"{size}_{6000 + 100 * gi + o}")))
        codec = mb.Codec(k, m, bs)
        nob = len(objs)

        def ranged(q, o):
            size = objs[o][0].size
            if q % 3 == 1 and size > 2 * S:
                a = S // 2 + 3                  # starts and ends mid-shard
                return a, min(size - a, bs + S)
            return 0, size

        # rotated GETs: physical drive 0 offline, request q's object rotated by q % n — its offline shard index rotates; a
        # parity shard offline reads the k data shards (r = 0), a data shard offline rebuilds it (r = 1)
        gplan = [(q % nob, rotated(n, q % n, {0}), *ranged(q, q % nob), None) for q in range(n)]
        cap = get_cap(gplan, bs)
        for mix in (True, False):
            bat = new_batcher(k, m, bs, cap, mix)
            if num_sms is None:
                num_sms = bat.stat("num_sms")
            get_round(bat, geom, objs, f"{name}/get-rot/mix{int(mix)}", gplan, codec, info={"name": "get-rot", "mix": mix})
            bat.close()
        # rotated heals: one stale drive, and every third request two (drives 0 and 1), so r differs within the batch
        hplan = [(q % nob, rotated(n, q % n, {0, 1} if q % 3 == 2 and m >= 2 else {0})) for q in range(n)]
        hcap = sum(-(-objs[o][0].size // bs) for o, _ in hplan)
        for mix in (True, False):
            bat = new_batcher(k, m, bs, hcap, mix)
            heal_round(bat, geom, objs, f"{name}/heal-rot/mix{int(mix)}", hplan, codec, info={"name": "heal-rot", "mix": mix})
            bat.close()
        # preferReaders: the k "local" drives 0..k-1, rotated per object; every drive online
        pplan = [(q % nob, set(), 0, objs[q % nob][0].size, rotated(n, q % n, range(k))) for q in range(n)]
        pcap = get_cap(pplan, bs)
        bat = new_batcher(k, m, bs, pcap, True)
        get_round(bat, geom, objs, f"{name}/prefer", pplan, codec, info={"name": "prefer", "mix": True})
        # a corrupt frame (block 0 of the shard) on a drive request 2 does not read: never read, nothing redone
        big = [q for q in range(n) if objs[pplan[q][0]][0].size > bs][0]
        o, _, _, _, pref = pplan[big]
        other = [i for i in range(n) if i not in pref][0]
        get_round(bat, geom, objs, f"{name}/prefer-unread", pplan, codec, flip=(big, other, 32 + 7),
                  info={"name": "prefer-unread", "mix": True})
        # ... and on a chosen drive, block 1: that request alone is redone (parallelReader's fail-over), the others are exact
        get_round(bat, geom, objs, f"{name}/prefer-bitrot", pplan, codec, flip=(big, sorted(pref)[0], (32 + S) + 32 + 7),
                  info={"name": "prefer-bitrot", "mix": True})
        bat.close()
        if config == "pat-dma":
            host_side(geom, objs, codec)
        codec.close()
        if gi == 0:
            # more blocks of mixed patterns than one latency launch takes: batches cut at that limit, each one latency launch;
            # then one request larger than the limit alone: a batch of its own through today's single-pattern path
            bs64 = 64 * KiB
            limit = 5 * num_sms
            nblk = limit // 8 + 3
            lobjs = []
            for o in range(4):
                size = nblk * bs64 + 1 + 997 * o
                d = rand(size, 9600 + o)
                lobjs.append((d, oracle_files(k, m, bs64, d, f"{size}_{9600 + o}")))
            size = (limit + 10) * bs64 + 333
            d = rand(size, 9700)
            lobjs.append((d, oracle_files(k, m, bs64, d, f"{size}_9700")))
            codec = mb.Codec(k, m, bs64)
            g64 = (name + "@64k", k, m, bs64)
            lplan = [(q % 4, rotated(n, q % n, {0}), 0, lobjs[q % 4][0].size, None) for q in range(16)]
            lcap = get_cap(lplan, bs64)
            bat = new_batcher(k, m, bs64, lcap, True)
            get_round(bat, g64, lobjs, f"{name}@64k/overlimit", lplan, codec, info={"name": "overlimit", "mix": True, "limit": limit})
            bat.close()
            one = [(4, {3}, 0, lobjs[4][0].size, None)]
            bat = new_batcher(k, m, bs64, get_cap(one, bs64), True)
            get_round(bat, g64, lobjs, f"{name}@64k/lone", one, codec, info={"name": "lone", "mix": True, "limit": limit})
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
    return str(tmp_path_factory.mktemp("batcher_patterns_oracle"))


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
def test_batcher_patterns_config(oracle, oracle_cache, config):
    env = CONFIGS[config]
    g = 1 if "MEC_BATCHER_DMA_BLOCKS" in env else 0     # the gather kernel stages every request
    sc = 0 if env.get("MEC_BATCHER_GET_OUT") == "2" else 1  # GET_OUT=2: the copy engine writes the callers' buffers
    res = _run_child(config, oracle_cache)
    print(json.dumps({"config": config, "child_s": res["child_s"], "checks": res["checks"], "rounds": len(res["rounds"])}))
    assert not res["mismatches"], res["mismatches"][:10]
    limit = res["limit"]
    names = {(r["geom"], r["name"], r["mix"]) for r in res["rounds"]}
    for geom in GEOMS:
        for nm in ("get-rot", "heal-rot"):
            assert (geom[0], nm, True) in names and (geom[0], nm, False) in names
        assert all((geom[0], nm, True) in names for nm in ("prefer", "prefer-unread", "prefer-bitrot"))
    assert (GEOMS[0][0] + "@64k", "overlimit", True) in names and (GEOMS[0][0] + "@64k", "lone", True) in names
    for r in res["rounds"]:
        d, ctx = r["d"], (r["round"], r["d"], {x: r[x] for x in ("patterns", "keys", "nslots", "rmax") if x in r})
        forms = _forms(d)
        heal = r["kind"] == "heal"
        tail = 1 if heal and r["rmax"] > 0 else (0 if heal else sc)   # heal scatter / GET scatter kernel per batch
        assert d["requests"] == r["requests"] and d["kernel_batches"] == d["batches"], ctx
        assert d["redone"] == (1 if r["name"] == "prefer-bitrot" else 0), ctx
        if r["name"] == "overlimit":
            # cut at the latency kernel's limit: every batch fits ONE latency launch
            assert r["nslots"] > limit and d["batches"] >= -(-r["nslots"] // limit), ctx
            assert forms == {"small": d["batches"]} and d["launches"] == d["batches"] * (g + 1 + tail), ctx
            assert d["mixed_batches"] >= 1, ctx
            continue
        if r["name"] == "lone":
            # one pattern, more blocks than one latency launch takes: the throughput kernel and one launch for the short block
            assert d["batches"] == 1 and d["mixed_batches"] == 0 and d["patterns"] == 1, ctx
            assert forms.get("small", 0) == 1 and sum(forms.values()) == 2, ctx
            continue
        assert r["nslots"] <= limit, ctx
        if r["mix"]:
            # ONE batch, ONE latency launch with a decode plan per block
            assert d["batches"] == 1 and d["patterns"] == r["patterns"], ctx
            assert d["mixed_batches"] == (1 if r["patterns"] > 1 else 0), ctx
            assert forms == {"small": 1} and d["launches"] == g + 1 + tail, ctx
            if r["name"] in ("get-rot", "heal-rot"):
                assert r["patterns"] > 1, ctx
        else:
            # one batch (and one latency launch) per reader set / stale set, as before
            assert d["batches"] == r["keys"] and d["mixed_batches"] == 0 and d["patterns"] == r["keys"], ctx
            assert forms == {"small": r["keys"]} and d["launches"] == r["keys"] * (g + 1 + tail), ctx


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])
