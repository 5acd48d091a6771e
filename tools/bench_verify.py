"""VerifyFile-shaped bitrot verification on one codec (mec_bitrot_verify_parts) against the calls it replaces.

  (a) kernel: whole_hash_kernel time of ONE grouped launch over a mixed set of whole-file streams (SHA256, HighwayHash256,
      BLAKE2b512) against one launch per algorithm over the same streams (kernel durations from a CUDA activity trace;
      torch.profiler, run of its own)
  (b) a legacy object of P parts: one mec_bitrot_verify_parts call against P x mec_bitrot_verify_whole (host clock around calls
      that end in a device synchronise)
  (c) streaming parts: mec_bitrot_verify_parts against mec_bitrot_verify_batch over the same files (they should be equal)

Prints one JSON line per measurement, each with the card name and power limit read in the same run.  Needs a GPU.
Usage: python tools/bench_verify.py [--reps N] [--parts P] [--part-mib M]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
SHA256, HIGHWAYHASH256, HIGHWAYHASH256S, BLAKE2B512 = 1, 2, 3, 4
MiB = 1 << 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return float(np.median(t)) * 1e3


def kernel_ms(fn):
    """whole_hash_kernel durations (ms) of one call of fn, from a CUDA activity trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.device_time / 1e3 for e in prof.events() if "whole_hash_kernel" in e.name]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--parts", type=int, default=16)
    ap.add_argument("--part-mib", type=float, default=1.0)
    a = ap.parse_args()
    import minio_b200 as mb
    import oracle_lib as o
    assert mb.device_count() > 0, "no CUDA device"
    gpu = card()
    c = mb.Codec(12, 4, MiB)
    S = c.shard_size()
    rng = np.random.default_rng(0)

    # (a) one grouped launch against one launch per algorithm, same streams: 3 x 64 shard files of one 12-drive object's size
    flen = int(a.part_mib * MiB) // 12
    streams = {al: [rng.integers(0, 256, flen, dtype=np.uint8) for _ in range(64)] for al in (SHA256, HIGHWAYHASH256, BLAKE2B512)}
    sums = {al: [o.bitrot_hash(al, f) for f in fs] for al, fs in streams.items()}
    mixed = [(al, f, s) for q in range(64) for al in streams for f, s in [(streams[al][q], sums[al][q])]]

    def grouped():
        assert c.bitrot_verify_parts([x[1] for x in mixed], [x[0] for x in mixed], [0] * len(mixed), [x[2] for x in mixed]) == [0] * len(mixed)

    def per_algo():
        for al in streams:
            assert c.bitrot_verify_parts(streams[al], [al] * 64, [0] * 64, sums[al]) == [0] * 64
    kg, kp = kernel_ms(grouped), kernel_ms(per_algo)
    print(json.dumps({"bench": "grouped_kernel", "gpu": gpu, "streams": len(mixed), "file_bytes": flen, "grouped_launches": len(kg),
                      "grouped_kernel_ms": round(sum(kg), 3), "per_algo_launches": len(kp), "per_algo_kernel_ms": round(sum(kp), 3)}))

    # (b) VerifyFile of a legacy object of P parts on one drive
    for al in (SHA256, HIGHWAYHASH256, BLAKE2B512):
        files = [rng.integers(0, 256, flen, dtype=np.uint8) for _ in range(a.parts)]
        want = [o.bitrot_hash(al, f) for f in files]
        wants = [np.frombuffer(w, dtype=np.uint8) for w in want]
        t_parts = timed(lambda: c.bitrot_verify_parts(files, [al] * a.parts, [0] * a.parts, want), a.reps)
        t_whole = timed(lambda: [c.bitrot_verify_whole(al, f, w) for f, w in zip(files, wants)], a.reps)
        print(json.dumps({"bench": "legacy_object", "gpu": gpu, "algo": al, "parts": a.parts, "file_bytes": flen,
                          "verify_parts_ms": round(t_parts, 3), "verify_whole_x_parts_ms": round(t_whole, 3),
                          "speedup": round(t_whole / t_parts, 2)}))

    # (c) streaming parts: the same files through both calls
    plen = flen
    data = [rng.integers(0, 256, plen, dtype=np.uint8) for _ in range(a.parts)]
    sfiles = []
    for d in data:
        img = bytearray()
        for off in range(0, plen, S):
            img += o.hh256(bytes(d[off:off + S])) + bytes(d[off:off + S])
        sfiles.append(np.frombuffer(bytes(img), dtype=np.uint8))
    t_parts = timed(lambda: c.bitrot_verify_parts(sfiles, [HIGHWAYHASH256S] * a.parts, [plen] * a.parts), a.reps)
    t_batch = timed(lambda: c.bitrot_verify_batch(sfiles, [plen] * a.parts), a.reps)
    print(json.dumps({"bench": "streaming_parts", "gpu": gpu, "parts": a.parts, "part_bytes": plen, "verify_parts_ms": round(t_parts, 3),
                      "verify_batch_ms": round(t_batch, 3)}))
    c.close()


if __name__ == "__main__":
    main()
