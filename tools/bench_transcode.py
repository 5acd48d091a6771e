#!/usr/bin/env python
"""Data movement between pools: mec_transcode against mec_decode_prefer + mec_encode_sg on the same pinned, NUMA-local buffers.

Workloads: RS(12,4) -> RS(6,2) and RS(12,4) -> RS(12,4) at 1 MiB blocks, and legacy parts written with 10 MiB blocks (blockSizeV1)
moved from RS(12,4) into RS(6,2) at 1 MiB; parts of 64 MiB and 1 MiB, source healthy and with two data drives offline.
After a warm-up the two modes run alternately, three timed runs each.  Prints one JSON line: GiB/s of part bytes and calls/s per
mode, bytes moved per direction per call (from the codecs' counters), the card with its power limit and clock ceiling, and, from a
separate profiled run, the kernel time per chunk of reconstruct, re-split and encode (CUDA activity trace).

    python tools/bench_transcode.py [--out DIR] [--legacy-only]
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
    def __init__(self, k1, m1, k2, m2, total, offline, bs1=MiB, bs2=MiB):
        L = capi.lib()
        self.pinned = []
        pin = lambda n: self.pinned.append(mb.pinned_array(n, device=DEV)) or self.pinned[-1]
        self.k1, self.m1, self.k2, self.m2, self.total, self.offline = k1, m1, k2, m2, total, offline
        self.bs1, self.bs2 = bs1, bs2
        self.src, self.dst = mb.Codec(k1, m1, bs1, device=DEV), mb.Codec(k2, m2, bs2, device=DEV)
        data = pin(total)
        data[:] = np.random.default_rng(total + k2).integers(0, 256, total, dtype=np.uint8)
        fsz = self.src.bitrot_file_size(total)
        files = [pin(fsz) for _ in range(k1 + m1)]
        rc = L.mec_encode(self.src.h, data.ctypes.data, total, ptrs(files), 0)
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
        nb = -(-total // bs2)
        self.dd = pin(nb * k2 * 32)
        self.hint = C.c_int(0)

    def close(self):
        self.src.close()
        self.dst.close()
        for a in self.pinned:
            capi.lib().mec_free_pinned(a.ctypes.data)

    def transcode(self):
        rc = capi.lib().mec_transcode(self.src.h, self.files, None, self.total, self.dst.h, self.out_ptrs, 0, C.byref(self.hint))
        assert rc == self.total, rc

    def decode_encode_sg(self):
        L = capi.lib()
        rc = L.mec_decode_prefer(self.src.h, self.files, None, 0, self.total, self.total, self.obj.ctypes.data, C.byref(self.hint))
        assert rc == self.total, rc
        rc = L.mec_encode_sg(self.dst.h, self.obj.ctypes.data, self.total, self.sg_ptrs, self.dd.ctypes.data, 0)
        assert rc == self.total, rc

    def same_outputs(self):
        """parity drives byte for byte, data drives' digests: both modes wrote the same part files"""
        k2, S = self.k2, self.dst.shard_size()
        nb = -(-self.total // self.bs2)
        dd = self.dd.reshape(nb, k2, 32)
        for i in range(k2, k2 + self.m2):
            if not np.array_equal(self.outs[i], self.sg_files[i]):
                return False
        for i in range(k2):
            frames = [self.outs[i][b * (32 + S):b * (32 + S) + 32] for b in range(nb)]
            if not all(np.array_equal(frames[b], dd[b, i]) for b in range(nb)):
                return False
        return True

    def counters(self):
        return {d: self.src.stat("bytes_" + d) + self.dst.stat("bytes_" + d) for d in ("h2d", "d2h")}

    def name(self):
        bs = "" if self.bs1 == self.bs2 else f" {self.bs1 // MiB} MiB blocks -> {self.bs2 // MiB} MiB blocks,"
        return (f"RS({self.k1},{self.m1})->RS({self.k2},{self.m2}){bs} {self.total // MiB} MiB "
                + ("healthy" if not self.offline else f"data drives {sorted(self.offline)} offline"))


def timed(fn, calls):
    t = time.perf_counter()
    for _ in range(calls):
        fn()
    return time.perf_counter() - t  # every call returns after its streams drained


def measure(w, calls):
    row = {"workload": w.name(), "part_bytes": w.total, "src_block_size": w.bs1, "dst_block_size": w.bs2, "calls_per_run": calls}
    modes = {"transcode": w.transcode, "decode_encode_sg": w.decode_encode_sg}
    for fn in modes.values():
        for _ in range(3):
            fn()
    for name, fn in modes.items():  # bytes per call from the counters, one call
        c0 = w.counters()
        fn()
        c1 = w.counters()
        row[name] = {"h2d_bytes_per_call": c1["h2d"] - c0["h2d"], "d2h_bytes_per_call": c1["d2h"] - c0["d2h"],
                     "h2d_per_part_byte": round((c1["h2d"] - c0["h2d"]) / w.total, 3),
                     "d2h_per_part_byte": round((c1["d2h"] - c0["d2h"]) / w.total, 3), "runs_gib_s": []}
    row["same_outputs"] = w.same_outputs()
    for _ in range(3):  # alternate the modes
        for name, fn in modes.items():
            dt = timed(fn, calls)
            row[name]["runs_gib_s"].append(round(calls * w.total / dt / GiB, 2))
    for name in modes:
        r = row[name]
        r["gib_s"] = round(float(np.median(r["runs_gib_s"])), 2)
        r["calls_s"] = round(r["gib_s"] * GiB / w.total, 1)
    row["speedup"] = round(row["transcode"]["gib_s"] / row["decode_encode_sg"]["gib_s"], 3)
    return row


def kernel_times(w, calls, out_dir):
    """Kernel time per chunk of the transcode, from a profiled run of its own.  Under default options every chunk on a slot stream
    is three launches: the fused reconstruct (verify only when the source is healthy), the re-split, the fused encode."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    w.transcode()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            w.transcode()
    path = os.path.join(out_dir or tempfile.mkdtemp(), "transcode_trace.json")
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
    per_stream = {}
    for e in ev:
        per_stream.setdefault(e["args"].get("stream"), []).append(e)
    rec, rsp, enc = [], [], []
    for lst in per_stream.values():
        lst.sort(key=lambda e: e["ts"])
        for j, e in enumerate(lst):
            if "transcode_resplit" in e["name"]:
                rsp.append(e["dur"])
                if j > 0:
                    rec.append(lst[j - 1]["dur"])
                if j + 1 < len(lst):
                    enc.append(lst[j + 1]["dur"])
    res = {"workload": w.name(), "chunks": len(rsp), "kernels": len(ev), "three_per_chunk": len(ev) == 3 * len(rsp)}
    if rsp:
        res.update({"reconstruct_us_per_chunk": round(float(np.mean(rec)), 1), "resplit_us_per_chunk": round(float(np.mean(rsp)), 1),
                    "encode_us_per_chunk": round(float(np.mean(enc)), 1),
                    "part_kernel_us": round(float(np.sum(rec) + np.sum(rsp) + np.sum(enc)) / calls, 1)})
    if not out_dir:
        os.remove(path)
        os.rmdir(os.path.dirname(path))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for the profiler trace (default: a temporary one, removed)")
    ap.add_argument("--legacy-only", action="store_true", help="only the workloads whose source block size differs")
    args = ap.parse_args()
    assert mb.device_count() > 0, "no CUDA device"
    capi.lib().mec_bind_thread_to_device(DEV)
    result = {"card": card(), "runs": 3, "results": [], "kernel_times": []}
    # (k1, m1, source block size, k2, m2, destination block size): equal pools, and a decommissioned pool's legacy 10 MiB-block parts
    pairs = [(12, 4, MiB, 6, 2, MiB), (12, 4, MiB, 12, 4, MiB), (12, 4, 10 * MiB, 6, 2, MiB)]
    for (k1, m1, bs1, k2, m2, bs2) in pairs[2:] if args.legacy_only else pairs:
        for total, calls in ((64 * MiB, 24), (MiB, 400)):
            for offline in ((), (0, 1)):
                w = Workload(k1, m1, k2, m2, total, set(offline), bs1, bs2)
                result["results"].append(measure(w, calls))
                if total == 64 * MiB and (k1, m1, k2, m2) == (12, 4, 6, 2):
                    result["kernel_times"].append(kernel_times(w, 4, args.out))
                w.close()
    result["card_after"] = card()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
