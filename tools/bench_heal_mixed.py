#!/usr/bin/env python
"""Heal and GET of legacy parts whose drives mix bitrot formats: mec_heal_mixed / mec_decode_mixed against what a binding can
compose without them, on the same pinned, NUMA-local buffers.

Modes, per workload:
  heal_mixed_1 / heal_mixed_2     mec_heal_mixed of an all-whole-file part, 1 and 2 stale drives (written as HighwayHash256S frames)
  compose_1 / compose_2           mec_decode_whole of the whole part into a host buffer, then mec_encode of it on a HighwayHash256S
                                  codec, keeping the stale drives' images; must write the same files as the mode above
  decode_mixed_streaming          mec_decode_mixed of an all-streaming part (every drive HighwayHash256S), whole part ...
  decode_prefer_streaming         ... against mec_decode_prefer of the same part: the overhead check
  decode_mixed_whole              mec_decode_mixed of an all-whole-file part ...
  decode_whole                    ... against mec_decode_whole
  decode_mixed_half               mec_decode_mixed of a half-healed part (every other drive streams)
Workloads: SHA256 and HighwayHash256; RS(12,4) at 10 MiB and at 1 MiB blocks; parts of 64 MiB and 1 MiB.  After a warm-up the modes
run alternately, three timed runs each.  Prints one JSON line: GiB/s of part bytes per mode (median and the three runs), bytes moved
per direction per part byte (from the codecs' counters), and the card with its power limit and clock ceiling, read in the same call.

    python tools/bench_heal_mixed.py
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np

import minio_b200 as mb
from minio_b200 import capi

MiB, GiB = 1 << 20, 1 << 30
DEV = 0
ALGO_NAMES = {mb.HIGHWAYHASH256: "HighwayHash256", mb.SHA256: "SHA256"}


def card():
    """name, power limit and max SM clock, read-only"""
    try:
        return subprocess.run(["nvidia-smi", "-i", str(DEV), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def ptrs(arrs):
    return (C.c_void_p * len(arrs))(*[(a.ctypes.data if a is not None else None) for a in arrs])


class Workload:
    def __init__(self, k, m, bs, algo, total):
        L = capi.lib()
        self.pinned = []
        pin = lambda n: self.pinned.append(mb.pinned_array(max(n, 1), device=DEV)) or self.pinned[-1]
        self.k, self.m, self.n, self.bs, self.algo, self.total = k, m, k + m, bs, algo, total
        n = self.n
        self.c = mb.Codec(k, m, bs, device=DEV)              # HighwayHash256S: the mixed calls and the compose's encode
        self.w = mb.Codec(k, m, bs, algo, device=DEV)        # the part's whole-file algorithm
        self.data = pin(total)
        self.data[:] = np.random.default_rng(total + k + algo).integers(0, 256, total, dtype=np.uint8)
        self.wfiles = [pin(self.w.shard_file_size(total)) for _ in range(n)]
        self.sums = np.zeros((n, 64), dtype=np.uint8)
        assert L.mec_encode_whole(self.w.h, self.data.ctypes.data, total, ptrs(self.wfiles), self.sums.ctypes.data, 0) == total
        fsz = self.c.bitrot_file_size(total)
        self.sfiles = [pin(fsz) for _ in range(n)]
        assert L.mec_encode(self.c.h, self.data.ctypes.data, total, ptrs(self.sfiles), 0) == total
        self.whole_algos = (C.c_int32 * n)(*[algo] * n)
        self.stream_algos = (C.c_int32 * n)(*[mb.HIGHWAYHASH256S] * n)
        self.half_algos = (C.c_int32 * n)(*[mb.HIGHWAYHASH256S if i % 2 == 0 else algo for i in range(n)])
        self.half_files = ptrs([self.sfiles[i] if i % 2 == 0 else self.wfiles[i] for i in range(n)])
        self.wptrs, self.sptrs = ptrs(self.wfiles), ptrs(self.sfiles)
        self.heal_outs = {s: [pin(fsz) if i < s else None for i in range(n)] for s in (1, 2)}
        self.enc_outs = [pin(fsz) for _ in range(n)]
        self.obj = pin(total)
        self.corrupt = np.zeros(n, dtype=np.uint8)
        self.hint = C.c_int(0)

    def close(self):
        self.c.close()
        self.w.close()
        for a in self.pinned:
            capi.lib().mec_free_pinned(a.ctypes.data)

    def heal_mixed(self, stale):
        # the stale drives are not read: their files stay in `files`, out_files marks them
        rc = capi.lib().mec_heal_mixed(self.c.h, self.whole_algos, self.wptrs, self.sums.ctypes.data, None, self.total,
                                       ptrs(self.heal_outs[stale]), self.corrupt.ctypes.data)
        assert rc == 0, rc

    def compose(self, stale):
        L = capi.lib()
        files = ptrs([None if i < stale else f for i, f in enumerate(self.wfiles)])
        rc = L.mec_decode_whole(self.w.h, files, self.sums.ctypes.data, 0, self.total, self.total, self.obj.ctypes.data, C.byref(self.hint))
        assert rc == self.total, rc
        # Erasure.Encode writes every drive; a binding keeps the stale drives' images
        assert L.mec_encode(self.c.h, self.obj.ctypes.data, self.total, ptrs(self.enc_outs), 0) == self.total

    def decode_mixed(self, algos, files):
        rc = capi.lib().mec_decode_mixed(self.c.h, algos, files, self.sums.ctypes.data, None, 0, self.total, self.total,
                                         self.obj.ctypes.data, C.byref(self.hint))
        assert rc == self.total and self.hint.value == 0, rc

    def decode_prefer(self):
        rc = capi.lib().mec_decode_prefer(self.c.h, self.sptrs, None, 0, self.total, self.total, self.obj.ctypes.data, C.byref(self.hint))
        assert rc == self.total, rc

    def decode_whole(self):
        rc = capi.lib().mec_decode_whole(self.w.h, self.wptrs, self.sums.ctypes.data, 0, self.total, self.total, self.obj.ctypes.data,
                                         C.byref(self.hint))
        assert rc == self.total, rc

    def modes(self):
        return {
            "heal_mixed_1": lambda: self.heal_mixed(1),
            "compose_1": lambda: self.compose(1),
            "heal_mixed_2": lambda: self.heal_mixed(2),
            "compose_2": lambda: self.compose(2),
            "decode_mixed_streaming": lambda: self.decode_mixed(self.stream_algos, self.sptrs),
            "decode_prefer_streaming": self.decode_prefer,
            "decode_mixed_whole": lambda: self.decode_mixed(self.whole_algos, self.wptrs),
            "decode_whole": self.decode_whole,
            "decode_mixed_half": lambda: self.decode_mixed(self.half_algos, self.half_files),
        }

    def same_heals(self):
        """each heal wrote, for every stale drive, what the compose's encode wrote for it, and both are mec_encode's images"""
        ok = True
        for s in (1, 2):
            self.heal_mixed(s)
            self.compose(s)
            ok &= all(np.array_equal(self.heal_outs[s][i], self.enc_outs[i]) and np.array_equal(self.enc_outs[i], self.sfiles[i])
                      for i in range(s))
        self.decode_mixed(self.half_algos, self.half_files)
        return bool(ok and np.array_equal(self.obj, self.data))

    def counters(self):
        return {d: self.c.stat("bytes_" + d) + self.w.stat("bytes_" + d) for d in ("h2d", "d2h")}

    def name(self):
        return f"{ALGO_NAMES[self.algo]} RS({self.k},{self.m}) {self.bs // MiB} MiB blocks, {self.total // MiB} MiB part"


def timed(fn, calls):
    t = time.perf_counter()
    for _ in range(calls):
        fn()
    return time.perf_counter() - t  # every call returns after its streams drained


def measure(w, calls):
    row = {"workload": w.name(), "part_bytes": w.total, "calls_per_run": calls}
    modes = w.modes()
    for fn in modes.values():
        fn()
    for name, fn in modes.items():  # bytes per call from the counters, one call
        c0 = w.counters()
        fn()
        c1 = w.counters()
        row[name] = {"h2d_per_part_byte": round((c1["h2d"] - c0["h2d"]) / w.total, 3),
                     "d2h_per_part_byte": round((c1["d2h"] - c0["d2h"]) / w.total, 3), "runs_gib_s": []}
    row["same_outputs"] = w.same_heals()
    for _ in range(3):  # alternate the modes
        for name, fn in modes.items():
            dt = timed(fn, calls)
            row[name]["runs_gib_s"].append(round(calls * w.total / dt / GiB, 3))
    for name in modes:
        row[name]["gib_s"] = round(float(np.median(row[name]["runs_gib_s"])), 3)
        row[name]["ms_per_call"] = round(w.total / (row[name]["gib_s"] * GiB) * 1e3, 2)
    row["heal_speedup_1"] = round(row["heal_mixed_1"]["gib_s"] / row["compose_1"]["gib_s"], 3)
    row["heal_speedup_2"] = round(row["heal_mixed_2"]["gib_s"] / row["compose_2"]["gib_s"], 3)
    return row


def main():
    assert mb.device_count() > 0, "no CUDA device"
    capi.lib().mec_bind_thread_to_device(DEV)
    result = {"card": card(), "runs": 3, "results": []}
    for bs in (10 * MiB, MiB):
        for algo in (mb.HIGHWAYHASH256, mb.SHA256):
            for total, calls in ((64 * MiB, 1), (MiB, 10)):
                w = Workload(12, 4, bs, algo, total)
                result["results"].append(measure(w, calls))
                w.close()
    result["card_after"] = card()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
