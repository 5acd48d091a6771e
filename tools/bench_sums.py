"""Object-hash rates: stream_sums_kernel through mec_sums_device against hashlib on one CPU core, in one run.

For each algorithm (MD5, SHA-1, SHA-256), stream count (1 and 4096) and message size (4 KiB .. 4 MiB) the kernel hashes `streams`
messages of `size` bytes in ONE launch, timed with CUDA events over several launches after a warm-up launch; reported as per-stream
MB/s (size / launch time) and aggregate GB/s (streams x size / launch time).  Messages start at odd offsets (every one misaligned, as
in a merged batch at an odd block size).  Their bytes come from one device buffer of at most 4 GiB: 4096 streams of 4 MiB share it
(stream i and stream i + 1024 read the same bytes), which does not help a kernel that is bound by one thread's compression chain.
The same sizes through hashlib's MD5, SHA-1 and SHA-256 on the calling thread give the single-core CPU rate.  The card's name, power
limit and SM clocks are read with nvidia-smi in the same run.  Prints one JSON object; --out also writes it to a file.

Usage: python tools/bench_sums.py [--reps 5] [--out bench_out/bench_sums.json]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KiB, MiB = 1 << 10, 1 << 20
SIZES = [4 * KiB, 64 * KiB, 256 * KiB, MiB, 4 * MiB]
STREAMS = [1, 4096]
ALGOS = {"md5": 8, "sha1": 16, "sha256": 32}
SUM_BYTES = 96


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        return {"error": r.stderr.strip()}
    f = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return dict(zip(q.split(","), f))


def cpu_rates(min_seconds=0.3):
    out = {}
    for name in ALGOS:
        for size in SIZES:
            data = np.random.default_rng(size).integers(0, 256, size, dtype=np.uint8).tobytes()
            n, t0 = 0, time.perf_counter()
            while True:
                hashlib.new(name, data).digest()
                n += 1
                dt = time.perf_counter() - t0
                if dt >= min_seconds:
                    break
            out[f"{name}/{size}"] = size * n / dt / 1e6
    return out


def gpu_rates(reps):
    import torch
    import minio_b200 as mb
    c = mb.Codec(12, 4)
    cap = 4 << 30
    buf = torch.randint(0, 256, (cap + 4096,), dtype=torch.uint8, device="cuda")
    out = torch.empty(max(STREAMS) * SUM_BYTES, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream()
    res = []
    for name, bit in ALGOS.items():
        for streams in STREAMS:
            for size in SIZES:
                span = min(streams * size, cap)
                offs = [(i * size) % span + 1 + 2 * (i % 8) for i in range(streams)]
                lens = [size] * streams
                c.sums_device(buf.data_ptr(), offs, lens, bit, out.data_ptr(), st.cuda_stream)  # warm-up
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                for _ in range(reps):
                    c.sums_device(buf.data_ptr(), offs, lens, bit, out.data_ptr(), st.cuda_stream)
                e1.record(st)
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / reps
                res.append({"algo": name, "streams": streams, "size": size, "ms_per_launch": round(ms, 4),
                            "per_stream_MBps": round(size / (ms * 1e-3) / 1e6, 2),
                            "aggregate_GBps": round(streams * size / (ms * 1e-3) / 1e9, 3)})
                # spot check of the timed launches' output: the first and the last stream against hashlib
                slot = 32 * list(ALGOS).index(name)
                got = out[:streams * SUM_BYTES].cpu().numpy()
                for i in (0, streams - 1):
                    want = hashlib.new(name, buf[offs[i]:offs[i] + size].cpu().numpy().tobytes()).digest()
                    assert got[i * SUM_BYTES + slot:i * SUM_BYTES + slot + len(want)].tobytes() == want, (name, streams, size, i)
    c.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_sums.py needs a CUDA device")
    info = gpu_info()
    gpu = gpu_rates(a.reps)
    result = {"gpu": info, "gpu_after": gpu_info(), "kernel": gpu, "cpu_one_core_MBps": {k: round(v, 1) for k, v in cpu_rates().items()}}
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
