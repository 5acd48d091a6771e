"""GPU tests of moves between pools through the cross-request coalescer (mec_batcher_new_transcode, mec_batcher_transcode): many
concurrent parts read from one erasure geometry, rebuilt where drives are missing, re-split and encoded to another geometry in
merged batches — byte for byte against the CPU oracle's Erasure.Encode of the destination geometry and against mec_transcode on a
plain codec pair, on every staging path and both kernel forms.

The staging switches are read once per process (MEC_BATCHER_DMA_BLOCKS, MEC_BATCHER_DEPTH, MEC_SMALL_BLOCKS), so every
configuration runs in a child process of its own: this file run as a script.  The child releases concurrent callers together with
a barrier, checks every output, source file and guard byte itself and prints one JSON line with the mismatches and the batcher's
counters per round; the parent asserts which batches, launches and kernel forms ran.  With MEC_BATCHER_DEPTH=0, a 0.5 s
max_wait_us and a batcher capped at exactly one round's blocks, the merging is deterministic."""
import json
import os
import subprocess
import sys
import time

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MiB = 1 << 20
BS = MiB - 1  # odd shard sizes on both sides: frames in the part files and in the staging at every alignment
FORMS = ("small", "fast3d", "fast3d_auto", "fast3d_semi", "fast", "fast_auto", "aligned", "aligned_auto", "runtime", "bytewise",
         "dyn_aligned", "dyn_runtime", "dyn_bytewise", "jit")
CONFIGS = {
    "tc-dma": {"MEC_BATCHER_DEPTH": "0"},
    "tc-gather": {"MEC_BATCHER_DMA_BLOCKS": "1000000", "MEC_BATCHER_DEPTH": "0"},
    "tc-small0": {"MEC_SMALL_BLOCKS": "0", "MEC_BATCHER_DEPTH": "0"},
}
CHILD_TIMEOUT_S = 600
GUARD = 64
MAX_WAIT_US = 500_000
MIX = 1  # MEC_BATCHER_MIX_PATTERNS
FILE_CORRUPT, WRITE_QUORUM, READ_QUORUM, INVALID_ARGUMENT = -7, -11, -10, -12


def lengths(bs):
    """one byte, a sub-block, one block, three blocks and a tail"""
    return (1, bs // 2 + 13, bs, 3 * bs + 12345)


# ---- child ----------------------------------------------------------------------------------------------------------------------

def _child(config, cache_dir):
    import ctypes as C
    import threading

    import numpy as np

    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import minio_b200 as mb
    import oracle_lib as oracle
    from test_gpu_transcode import PAIRS

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

    stat_names = (["batches", "requests", "blocks", "kernel_batches", "redone", "launches", "patterns", "mixed_batches",
                   "transcodes", "transcodes_serial", "blocks_read", "bytes_h2d", "dst_blocks_encoded", "dst_launches"]
                  + ["form_" + f for f in FORMS] + ["dst_form_" + f for f in FORMS])

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

    class Obj:
        def __init__(self, pair, size, seed):
            k1, m1, k2, m2 = pair
            self.data = rand(size, seed)
            self.src = oracle_files(k1, m1, BS, self.data, f"{size}_{seed}")
            self.dst = oracle_files(k2, m2, BS, self.data, f"{size}_{seed}")

    def src_layout(k, size):
        """(slots, short slots) of a whole-part read: a block is a short slot when its shard length is not S"""
        S, sfs = oracle.shard_size(BS, k), oracle.shard_file_size(BS, k, size)
        nb = -(-size // BS)
        return nb, (1 if sfs - (nb - 1) * S != S else 0)

    def chosen_of(n, k, offl, pref):
        """parallelReader's readers: preferred online drives first, then index order; ascending"""
        order = [i for i in range(n) if pref and i in pref] + [i for i in range(n) if not (pref and i in pref)]
        return sorted([i for i in order if i not in offl][:k])

    def move_round(bat, pair, plan, rnd, info, ref=None, flip=None, wq=0):
        """plan: list of (Obj, offline source shards, prefer set or None, offline destination writers).  Every request reads its
        own copy of the part files.  flip = (request, shard, byte offset in the file).  ref = (src Codec, dst Codec): every result
        is compared with mec_transcode on that pair over the same inputs."""
        k1, m1, k2, m2 = pair
        n1, n2 = k1 + m1, k2 + m2
        fil, outa = Arena(), Arena()
        fpos = [[None if i in offl else fil.reserve(o.src[i].size, (5 * q + 3 * i) % 16) for i in range(n1)]
                for q, (o, offl, _, _) in enumerate(plan)]
        opos = [[None if i in doff else outa.reserve(o.dst[i].size, (2 * (q + i) + 1) % 16) for i in range(n2)]
                for q, (o, _, _, doff) in enumerate(plan)]
        fil.alloc(4000 + len(rnd))
        outa.alloc(4001 + len(rnd))
        calls, hints, keep, keys = [], [], [], set()
        for q, (o, offl, pref, doff) in enumerate(plan):
            for i, f in enumerate(fpos[q]):
                if f is None:
                    continue
                fil.view(f, o.src[i].size)[:] = o.src[i]
                exp = o.src[i]
                if flip and flip[0] == q and flip[1] == i:
                    fil.view(f + flip[2], 1)[:] ^= 0x5A
                    exp = fil.view(f, o.src[i].size).copy()
                fil.expect(f, exp, {"request": q, "drive": i, "what": "source part file"})
            for i, f in enumerate(opos[q]):
                if f is not None:
                    outa.expect(f, o.dst[i], {"request": q, "drive": i, "what": "destination part file"})
            fp = (C.c_void_p * n1)(*[None if f is None else fil.base + f for f in fpos[q]])
            op = (C.c_void_p * n2)(*[None if f is None else outa.base + f for f in opos[q]])
            pf = None if pref is None else np.array([1 if i in pref else 0 for i in range(n1)], dtype=np.uint8)
            hint = C.c_int(-1)
            keep += [fp, op, pf]
            hints.append(hint)
            calls.append(lambda h=bat.h, fp=fp, pf=pf, tot=o.data.size, op=op, hint=hint:
                         L.mec_batcher_transcode(h, fp, None if pf is None else pf.ctypes.data, tot, op, wq, C.byref(hint)))
            keys.add(tuple(chosen_of(n1, k1, offl, pref)))
        lay = [src_layout(k1, o.data.size) for o, _, _, _ in plan]
        sizes = [o.data.size for o, _, _, _ in plan]
        rec = dict(info, pair=list(pair), keys=len(keys), nslots=sum(a for a, _ in lay), src_tails=sum(b for _, b in lay),
                   nblocks=sum(-(-s // BS) for s in sizes), dst_tails=sum(1 for s in sizes if s % BS),
                   h2d=k1 * sum(oracle.bitrot_shard_file_size(oracle.shard_file_size(BS, k1, s), oracle.shard_size(BS, k1),
                                                              oracle.HIGHWAYHASH256S) for s in sizes))
        res = run_round(bat, calls, rnd, rec)
        for q, (o, offl, pref, _) in enumerate(plan):
            want_hint = FILE_CORRUPT if flip and flip[0] == q and flip[1] in chosen_of(n1, k1, offl, pref) else 0
            out["checks"] += 1
            if res[q] != o.data.size or hints[q].value != want_hint:
                mismatch({"round": rnd, "request": q, "rc": str(res[q]), "hint": hints[q].value, "want_hint": want_hint})
        if ref is not None:
            for q, (o, offl, pref, doff) in enumerate(plan):
                fp = (C.c_void_p * n1)(*[None if f is None else fil.base + f for f in fpos[q]])
                pf = None if pref is None else np.array([1 if i in pref else 0 for i in range(n1)], dtype=np.uint8)
                got = [None if i in doff else np.zeros(o.dst[i].size, dtype=np.uint8) for i in range(n2)]
                hint = C.c_int(-1)
                rc = L.mec_transcode(ref[0].h, fp, None if pf is None else pf.ctypes.data, o.data.size, ref[1].h, mb.capi._ptrs(got),
                                     wq, C.byref(hint))
                out["checks"] += 1
                if rc != res[q] or hint.value != hints[q].value or any(
                        g is not None and not np.array_equal(g, outa.view(opos[q][i], g.size)) for i, g in enumerate(got)):
                    mismatch({"round": rnd, "request": q, "mec_transcode": rc, "hint": hint.value})
        fil.check(rnd)
        outa.check(rnd)
        fil.free()
        outa.free()
        return rec

    def new_batcher(pair, cap, mix):
        k1, m1, k2, m2 = pair
        return mb.Batcher(k1, m1, BS, max_batch_blocks=cap, max_wait_us=MAX_WAIT_US, mix_patterns=mix, dst=(k2, m2))

    def cap_of(plan):
        return sum(-(-o.data.size // BS) for o, _, _, _ in plan)

    def host_side(pair, objs, refs):
        """refusals before queueing, the private paths, and a plain batcher"""
        k1, m1, k2, m2 = pair
        n1, n2 = k1 + m1, k2 + m2
        big = objs[3]
        bat = new_batcher(pair, 64, False)
        src = [mb.pinned_array(f.size) for f in big.src]
        for a, f in zip(src, big.src):
            a[:] = f
        fsz = big.dst[0].size
        outs = [mb.pinned_array(fsz) for _ in range(n2)]
        for a in outs:
            a[:] = 0xA5
        fp = mb.capi._ptrs(src)

        def call(files, total, wq, online=range(n2), pref=None):
            op = (C.c_void_p * n2)(*[outs[i].ctypes.data if i in online else None for i in range(n2)])
            hint = C.c_int(-1)
            before = bat.stat("requests"), bat.stat("transcodes_serial")
            rc = L.mec_batcher_transcode(bat.h, files, None, total, op, wq, C.byref(hint))
            return rc, hint.value, bat.stat("requests") - before[0], bat.stat("transcodes_serial") - before[1]

        cases = {
            "write quorum": (call(fp, big.data.size, n2, online=range(n2 - 1)), (WRITE_QUORUM, 0, 0, 0)),
            "read quorum": (call((C.c_void_p * n1)(*[src[i].ctypes.data if i > m1 else None for i in range(n1)]), big.data.size, 0),
                            (READ_QUORUM, 0, 0, 0)),
            "total 0": (call(fp, 0, k2), (0, 0, 0, 0)),
            "total < 0": (call(fp, -1, 0), (INVALID_ARGUMENT, 0, 0, 0)),
            "null files": (call(None, big.data.size, 0), (INVALID_ARGUMENT, 0, 0, 0)),
        }
        for label, (got, want) in cases.items():
            out["checks"] += 1
            if got != want:
                mismatch({"pair": pair, "case": label, "got": got, "want": want})
        if any(not (a == 0xA5).all() for a in outs):
            mismatch({"pair": pair, "case": "refusals wrote out files"})
        # pageable out files and a part larger than max_batch_blocks: the private pair, same bytes
        before = bat.stat("requests"), bat.stat("transcodes_serial")
        got, hint = bat.transcode(src, big.data.size, pinned=False)
        out["checks"] += 1
        if hint != 0 or any(not np.array_equal(g, w) for g, w in zip(got, big.dst)) or \
                (bat.stat("requests") - before[0], bat.stat("transcodes_serial") - before[1]) != (0, 1):
            mismatch({"pair": pair, "case": "pageable out files"})
        bat.close()
        small = new_batcher(pair, 2, False)
        got, hint = small.transcode(src, big.data.size, pinned=True)
        out["checks"] += 1
        if hint != 0 or any(not np.array_equal(g, w) for g, w in zip(got, big.dst)) or \
                (small.stat("requests"), small.stat("transcodes_serial")) != (0, 1):
            mismatch({"pair": pair, "case": "part above max_batch_blocks"})
        for g in got:
            L.mec_free_pinned(g.ctypes.data)
        small.close()
        # a batcher without a destination geometry
        plain = mb.Batcher(k1, m1, BS, max_batch_blocks=16, max_wait_us=0)
        hint = C.c_int(-1)
        rc = L.mec_batcher_transcode(plain.h, fp, None, big.data.size, mb.capi._ptrs(outs), 0, C.byref(hint))
        out["checks"] += 1
        if rc != INVALID_ARGUMENT or hint.value != 0:
            mismatch({"pair": pair, "case": "plain batcher", "rc": rc})
        plain.close()
        for a in src + outs:
            L.mec_free_pinned(a.ctypes.data)

    def kinds_round(pair, objs):
        """transcodes, PUTs and GETs of the source geometry issued at once on one transcode batcher: one batch per kind"""
        k1, m1, k2, m2 = pair
        n1 = k1 + m1
        puts = [mb.pinned_array(o.data.size) for o in objs]
        for a, o in zip(puts, objs):
            a[:] = o.data
        pfiles = [[mb.pinned_array(f.size) for f in o.src] for o in objs]
        gsrc = [[mb.pinned_array(f.size) for f in o.src] for o in objs]
        for fs, o in zip(gsrc, objs):
            for a, f in zip(fs, o.src):
                a[:] = f
        gdst = [mb.pinned_array(o.data.size) for o in objs]
        tsrc = [[mb.pinned_array(f.size) for f in o.src] for o in objs]
        for fs, o in zip(tsrc, objs):
            for a, f in zip(fs, o.src):
                a[:] = f
        touts = [[mb.pinned_array(f.size) for f in o.dst] for o in objs]
        keep, calls, tr_hints = [], [], []
        for q, o in enumerate(objs):
            pp = mb.capi._ptrs(pfiles[q])
            gp = mb.capi._ptrs(gsrc[q])
            tp, op = mb.capi._ptrs(tsrc[q]), mb.capi._ptrs(touts[q])
            gh, th = C.c_int(-1), C.c_int(-1)
            keep += [pp, gp, tp, op, gh, th]
            tr_hints.append(th)
            calls.append(lambda pp=pp, s=puts[q], n=o.data.size: L.mec_batcher_encode(bat.h, s.ctypes.data, n, pp, 0))
            calls.append(lambda gp=gp, d=gdst[q], n=o.data.size, h=gh: L.mec_batcher_decode(bat.h, gp, 0, n, n, d.ctypes.data, C.byref(h)))
            calls.append(lambda tp=tp, op=op, n=o.data.size, h=th: L.mec_batcher_transcode(bat.h, tp, None, n, op, 0, C.byref(h)))
        cap = sum(-(-o.data.size // BS) for o in objs) * 2 + sum(o.data.size // BS + 2 for o in objs)
        bat = new_batcher(pair, cap, False)
        res = run_round(bat, calls, f"{pair}/kinds", {"name": "kinds", "pair": list(pair), "nobj": len(objs)})
        for q, o in enumerate(objs):
            out["checks"] += 1
            if res[3 * q:3 * q + 3] != [o.data.size] * 3 or tr_hints[q].value != 0:
                mismatch({"case": "kinds", "request": q, "rc": [str(x) for x in res[3 * q:3 * q + 3]]})
            if any(not np.array_equal(a, w) for a, w in zip(pfiles[q], o.src)):
                mismatch({"case": "kinds", "request": q, "what": "PUT part files"})
            if not np.array_equal(gdst[q], o.data):
                mismatch({"case": "kinds", "request": q, "what": "GET bytes"})
            if any(not np.array_equal(a, w) for a, w in zip(touts[q], o.dst)):
                mismatch({"case": "kinds", "request": q, "what": "transcode out files"})
        bat.close()
        for a in puts + gdst + [x for fs in pfiles + gsrc + tsrc + touts for x in fs]:
            L.mec_free_pinned(a.ctypes.data)

    # ---- the rounds ---------------------------------------------------------------------------------------------------------
    num_sms = None
    for pi, (k1, m1, k2, m2, _) in enumerate(PAIRS):
        pair = (k1, m1, k2, m2)
        n1 = k1 + m1
        name = f"rs{k1}_{m1}-rs{k2}_{m2}"
        objs = [Obj(pair, size, 7000 + 100 * pi + o) for o, size in enumerate(lengths(BS))]
        refs = (mb.Codec(k1, m1, BS), mb.Codec(k2, m2, BS))
        # every length twice, all drives online: exactly one merged batch
        plan = [(objs[q % 4], set(), None, set()) for q in range(8)]
        bat = new_batcher(pair, cap_of(plan), False)
        if num_sms is None:
            num_sms = bat.stat("num_sms")
        move_round(bat, pair, plan, f"{name}/healthy", {"name": "healthy", "mix": False}, ref=refs)
        # data and parity drives offline, with and without `prefer`; an offline destination writer
        offl = {1, k1} if m1 >= 2 else {1}
        pref = set(range(n1 - k1, n1))
        dplan = [(objs[q % 4], offl, None, {k2}) for q in range(8)]
        move_round(bat, pair, dplan, f"{name}/degraded", {"name": "degraded", "mix": False}, ref=refs)
        pplan = [(objs[q % 4], offl, pref, set()) for q in range(8)]
        move_round(bat, pair, pplan, f"{name}/prefer", {"name": "prefer", "mix": False}, ref=refs)
        # a corrupt frame of a chosen reader (block 1 of shard 0) in one request of eight: that one is redone alone
        S = oracle.shard_size(BS, k1)
        move_round(bat, pair, plan, f"{name}/bitrot", {"name": "bitrot", "mix": False}, ref=refs, flip=(3, 0, (32 + S) + 32 + 7))
        bat.close()
        # rotated objects: physical drive 0 offline, request q's object rotated by q % n — its offline shard index rotates
        rplan = [(objs[q % 4], {(0 - q) % n1}, None, set()) for q in range(n1)]
        for mix in (True, False):
            bat = new_batcher(pair, cap_of(rplan), mix)
            move_round(bat, pair, rplan, f"{name}/rot/mix{int(mix)}", {"name": "rot", "mix": mix}, ref=refs)
            bat.close()
        if config == "tc-dma":
            host_side(pair, objs, refs)
        if pi == 0:
            kinds_round(pair, objs)
        for c in refs:
            c.close()
    out["num_sms"] = num_sms
    out["child_s"] = round(time.time() - t_start, 2)
    print(json.dumps(out))


# ---- parent ---------------------------------------------------------------------------------------------------------------------

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oracle_cache(tmp_path_factory):
    return str(tmp_path_factory.mktemp("batcher_transcode_oracle"))


def _run_child(config, cache_dir):
    env = {key: v for key, v in os.environ.items() if not key.startswith(("MEC_BATCHER_", "MEC_SMALL_BLOCKS"))}
    env.update(CONFIGS[config])
    p = subprocess.run([sys.executable, os.path.abspath(__file__), config, cache_dir], env=env, capture_output=True, text=True,
                       timeout=CHILD_TIMEOUT_S, cwd=ROOT)
    assert p.returncode == 0, f"child {config} exited {p.returncode}:\n{p.stderr[-4000:]}"
    return json.loads(p.stdout.strip().split("\n")[-1])


def _forms(d, prefix=""):
    return {f: d[prefix + "form_" + f] for f in FORMS if d[prefix + "form_" + f]}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_batcher_transcode_config(oracle, oracle_cache, config):
    env = CONFIGS[config]
    g = 1 if "MEC_BATCHER_DMA_BLOCKS" in env else 0   # the gather kernel stages every request
    small = "MEC_SMALL_BLOCKS" not in env               # latency kernel on both sides; MEC_SMALL_BLOCKS=0 also turns MIX off
    res = _run_child(config, oracle_cache)
    print(json.dumps({"config": config, "child_s": res["child_s"], "checks": res["checks"], "rounds": len(res["rounds"])}))
    assert not res["mismatches"], res["mismatches"][:10]
    names = {(tuple(r["pair"]), r["name"], r["mix"]) for r in res["rounds"] if "mix" in r}
    from test_gpu_transcode import PAIRS
    for k1, m1, k2, m2, _ in PAIRS:
        p = (k1, m1, k2, m2)
        assert all((p, nm, False) in names for nm in ("healthy", "degraded", "prefer", "bitrot", "rot"))
        assert (p, "rot", True) in names
    kinds = [r for r in res["rounds"] if r["name"] == "kinds"]
    assert len(kinds) == 1
    d = kinds[0]["d"]
    # one batch per kind: PUTs, GETs and transcodes never share one
    assert d["batches"] == 3 and d["requests"] == 3 * kinds[0]["nobj"] and d["transcodes"] == kinds[0]["nobj"], d
    for r in res["rounds"]:
        if r["name"] == "kinds":
            continue
        d, ctx = r["d"], (r["round"], r["d"], {x: r[x] for x in ("keys", "nslots", "src_tails", "nblocks", "dst_tails")})
        bitrot = r["name"] == "bitrot"
        assert d["requests"] == r["requests"] and d["kernel_batches"] == d["batches"], ctx
        assert d["redone"] == (1 if bitrot else 0) and d["transcodes_serial"] == d["redone"], ctx
        assert d["transcodes"] == r["requests"] - d["redone"], ctx
        mix = r["mix"] and small
        nb = 1 if mix else r["keys"]
        assert d["batches"] == nb and d["patterns"] == r["keys"], ctx
        assert d["mixed_batches"] == (1 if mix and r["keys"] > 1 else 0), ctx
        # the blocks moved: read on the source, encoded on the destination (a redo runs on the private pair, not counted here)
        assert d["blocks_read"] == r["nslots"] and d["blocks"] == r["nslots"] and d["dst_blocks_encoded"] == r["nblocks"], ctx
        assert d["bytes_h2d"] == r["h2d"], ctx
        forms, dforms = _forms(d), _forms(d, "dst_")
        if nb == 1:
            # source: [gather] + reconstruct + resplit; destination: encode + scatter
            if small:
                assert forms == {"small": 1} and dforms == {"small": 1}, ctx
                assert d["launches"] == g + 1 + 1 and d["dst_launches"] == 1 + 1, ctx
            else:
                assert "small" not in forms and "small" not in dforms, ctx
                nsrc = (1 if r["nslots"] > r["src_tails"] else 0) + r["src_tails"]
                ndst = (1 if r["nblocks"] > r["dst_tails"] else 0) + r["dst_tails"]
                assert sum(forms.values()) == nsrc and d["launches"] == g + nsrc + 1, ctx
                assert sum(dforms.values()) == ndst and d["dst_launches"] == ndst + 1, ctx
        elif small:
            assert forms == {"small": nb} and dforms == {"small": nb}, ctx
            assert d["launches"] == nb * (g + 2) and d["dst_launches"] == 2 * nb, ctx


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])
