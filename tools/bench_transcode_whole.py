#!/usr/bin/env python
"""Data movement of parts written with a whole-file bitrot algorithm: mec_transcode_whole against the Decode -> Encode pipe it
replaces (mec_decode_whole into a host buffer, then mec_encode_sg) on the same pinned, NUMA-local buffers.

Workloads: RS(12,4) at 10 MiB blocks (blockSizeV1) into RS(6,2) at 1 MiB, and RS(12,4) into RS(12,4) at 1 MiB; HighwayHash256 and
SHA256 sources; parts of 1 MiB and 64 MiB; sources healthy and with two data drives offline.  After a warm-up the two modes run
alternately, three timed runs each.  Both modes must write the same part files (parity drives byte for byte, data drives' digests).
Prints one JSON line: GiB/s of part bytes per mode, bytes moved per direction per call (from the codecs' counters), the card with
its power limit and clock ceiling, and, from a separate profiled run of each 64 MiB workload, the time of the whole-file hash: the
fused call's one whole_hash_kernel launch over the k files against the pipe's k launches, one per file, back to back on one stream.

    python tools/bench_transcode_whole.py [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
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
    def __init__(self, k1, m1, bs1, k2, m2, bs2, algo, total, offline):
        L = capi.lib()
        self.pinned = []
        pin = lambda n: self.pinned.append(mb.pinned_array(n, device=DEV)) or self.pinned[-1]
        self.k1, self.m1, self.bs1, self.k2, self.m2, self.bs2 = k1, m1, bs1, k2, m2, bs2
        self.algo, self.total, self.offline = algo, total, offline
        self.src, self.dst = mb.Codec(k1, m1, bs1, algo, device=DEV), mb.Codec(k2, m2, bs2, device=DEV)
        data = pin(total)
        data[:] = np.random.default_rng(total + k2 + algo).integers(0, 256, total, dtype=np.uint8)
        files = [pin(self.src.shard_file_size(total)) for _ in range(k1 + m1)]
        self.sums = np.zeros((k1 + m1, 64), dtype=np.uint8)
        rc = L.mec_encode_whole(self.src.h, data.ctypes.data, total, ptrs(files), self.sums.ctypes.data, 0)
        assert rc == total, rc
        self.files = ptrs([None if i in offline else f for i, f in enumerate(files)])
        dsz = self.dst.bitrot_file_size(total)
        self.outs = [pin(dsz) for _ in range(k2 + m2)]
        self.out_ptrs = ptrs(self.outs)
        # decode + encode_sg: the object lands in host memory, the data drives' frames are the caller's slices of it
        self.obj = data  # overwritten by every decode with the same bytes
        self.sg_files = [pin(dsz) if i >= k2 else None for i in range(k2 + m2)]
        self.marker = np.zeros(1, dtype=np.uint8)
        self.sg_ptrs = ptrs([f if f is not None else self.marker for f in self.sg_files])
        self.dd = pin(-(-total // bs2) * k2 * 32)
        self.hint = C.c_int(0)

    def close(self):
        self.src.close()
        self.dst.close()
        for a in self.pinned:
            capi.lib().mec_free_pinned(a.ctypes.data)

    def transcode_whole(self):
        rc = capi.lib().mec_transcode_whole(self.src.h, self.files, self.sums.ctypes.data, None, self.total, self.dst.h, self.out_ptrs,
                                            0, C.byref(self.hint))
        assert rc == self.total and self.hint.value == 0, rc

    def decode_encode_sg(self):
        L = capi.lib()
        rc = L.mec_decode_whole(self.src.h, self.files, self.sums.ctypes.data, 0, self.total, self.total, self.obj.ctypes.data,
                                C.byref(self.hint))
        assert rc == self.total and self.hint.value == 0, rc
        rc = L.mec_encode_sg(self.dst.h, self.obj.ctypes.data, self.total, self.sg_ptrs, self.dd.ctypes.data, 0)
        assert rc == self.total, rc

    def same_outputs(self):
        """parity drives byte for byte, data drives' digests: both modes wrote the same part files"""
        k2, S = self.k2, self.dst.shard_size()
        nb = -(-self.total // self.bs2)
        dd = self.dd.reshape(nb, k2, 32)
        if not all(np.array_equal(self.outs[i], self.sg_files[i]) for i in range(k2, k2 + self.m2)):
            return False
        return all(np.array_equal(self.outs[i][b * (32 + S):b * (32 + S) + 32], dd[b, i]) for i in range(k2) for b in range(nb))

    def counters(self):
        return {d: self.src.stat("bytes_" + d) + self.dst.stat("bytes_" + d) for d in ("h2d", "d2h")}

    def name(self):
        bs = f"{self.bs1 // MiB} MiB blocks -> {self.bs2 // MiB} MiB blocks"
        return (f"{ALGO_NAMES[self.algo]} RS({self.k1},{self.m1})->RS({self.k2},{self.m2}) {bs}, {self.total // MiB} MiB, "
                + ("healthy" if not self.offline else f"data drives {sorted(self.offline)} offline"))


def timed(fn, calls):
    t = time.perf_counter()
    for _ in range(calls):
        fn()
    return time.perf_counter() - t  # every call returns after its streams drained


def measure(w, calls):
    row = {"workload": w.name(), "part_bytes": w.total, "calls_per_run": calls}
    modes = {"transcode_whole": w.transcode_whole, "decode_whole_encode_sg": w.decode_encode_sg}
    for fn in modes.values():
        fn()
    for name, fn in modes.items():  # bytes per call from the counters, one call
        c0 = w.counters()
        fn()
        c1 = w.counters()
        row[name] = {"h2d_per_part_byte": round((c1["h2d"] - c0["h2d"]) / w.total, 3),
                     "d2h_per_part_byte": round((c1["d2h"] - c0["d2h"]) / w.total, 3), "runs_gib_s": []}
    row["same_outputs"] = w.same_outputs()
    for _ in range(3):  # alternate the modes
        for name, fn in modes.items():
            dt = timed(fn, calls)
            row[name]["runs_gib_s"].append(round(calls * w.total / dt / GiB, 3))
    for name in modes:
        row[name]["gib_s"] = round(float(np.median(row[name]["runs_gib_s"])), 3)
        row[name]["ms_per_call"] = round(w.total / (row[name]["gib_s"] * GiB) * 1e3, 2)
    row["speedup"] = round(row["transcode_whole"]["gib_s"] / row["decode_whole_encode_sg"]["gib_s"], 3)
    return row


def hash_times(w, out_dir):
    """whole_hash_kernel time in one call of each mode, from a profiled run of its own (CUDA activity trace)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    res = {"workload": w.name()}
    for name, fn in (("transcode_whole", w.transcode_whole), ("decode_whole_encode_sg", w.decode_encode_sg)):
        fn()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
        path = os.path.join(out_dir or tempfile.mkdtemp(), f"whole_{name}_trace.json")
        prof.export_chrome_trace(path)
        ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
        hh = sorted((e for e in ev if "whole_hash_kernel" in e["name"]), key=lambda e: e["ts"])
        res[name] = {"hash_launches": len(hh), "hash_ms": round(sum(e["dur"] for e in hh) / 1e3, 2),
                     "hash_span_ms": round((hh[-1]["ts"] + hh[-1]["dur"] - hh[0]["ts"]) / 1e3, 2) if hh else 0.0,
                     "other_kernels_ms": round(sum(e["dur"] for e in ev if "whole_hash_kernel" not in e["name"]) / 1e3, 2)}
        if not out_dir:
            os.remove(path)
            os.rmdir(os.path.dirname(path))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for the profiler traces (default: temporary ones, removed)")
    args = ap.parse_args()
    assert mb.device_count() > 0, "no CUDA device"
    capi.lib().mec_bind_thread_to_device(DEV)
    result = {"card": card(), "runs": 3, "results": [], "hash_times": []}
    # (k1, m1, source block size, k2, m2, destination block size): a decommissioned pool's legacy 10 MiB-block parts, and equal pools
    pairs = [(12, 4, 10 * MiB, 6, 2, MiB), (12, 4, MiB, 12, 4, MiB)]
    for pair in pairs:
        for algo in (mb.HIGHWAYHASH256, mb.SHA256):
            for total, calls in ((64 * MiB, 2), (MiB, 20)):
                for offline in ((), (0, 1)):
                    w = Workload(*pair, algo, total, set(offline))
                    result["results"].append(measure(w, calls))
                    if total == 64 * MiB and not offline:
                        result["hash_times"].append(hash_times(w, args.out))
                    w.close()
    result["card_after"] = card()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
