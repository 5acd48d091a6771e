"""Server-side encryption (DARE 2.0, AES-256-GCM) on the GPU against the plain erasure path and the host cipher.

  (a) mec_dare_device seal and open: GiB/s of plaintext per call (CUDA events around the call, which includes the key setup and
      ends in a synchronise), at 1 GiB in one stream and at 4096 streams of 64 KiB and of 1 MiB
  (b) mec_encode_sse vs mec_encode, and mec_decode_sse vs mec_decode with 0 and 4 drives offline, for 1 MiB, 64 MiB and 1 GiB
      RS(12,4) objects at 1 MiB blocks, page-locked host buffers (host clock around calls that end in a synchronise; median)
  (c) the host alternative: Python `cryptography` AESGCM sealing 64 KiB DARE packages on one thread (one sio stream) and on every
      core (one stream per process); "not measured" when `cryptography` is missing

Prints one JSON line per measurement, each with the card name and power limit read in the same run.  Needs a GPU: without one it
fails.  Usage: python tools/bench_sse.py [--reps N] [--max-mib M] [--streams S]"""
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
MiB, GiB = 1 << 20, 1 << 30
KEY, NONCE = bytes(range(32)), bytes(range(12))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def emit(rec, gpu):
    rec["card"] = gpu
    print(json.dumps(rec), flush=True)


def timed(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def dare_device(mb, gpu, reps, streams, total_mib):
    import torch
    import dare_ref as d
    c = mb.Codec(12, 4, MiB)
    shapes = [(1, total_mib * MiB), (streams, 64 << 10), (streams, MiB)]
    for ns, n in shapes:
        src = torch.randint(0, 256, (ns * n,), dtype=torch.uint8, device="cuda")
        enc = d.encrypted_size(n)
        sealed = torch.empty(ns * enc, dtype=torch.uint8, device="cuda")
        plain = torch.empty(ns * n, dtype=torch.uint8, device="cuda")
        keys = np.frombuffer(np.random.default_rng(ns).bytes(32 * ns), np.uint8)
        nonces = np.frombuffer(np.random.default_rng(ns + 1).bytes(12 * ns), np.uint8)
        in_off, out_off = np.arange(ns, dtype=np.int64) * n, np.arange(ns, dtype=np.int64) * enc
        st = torch.cuda.current_stream()
        ops = {"seal": lambda: c.dare_device(1, keys, src.data_ptr(), in_off, [n] * ns, sealed.data_ptr(), out_off, nonces=nonces,
                                             stream=st.cuda_stream),
               "open": lambda: c.dare_device(2, keys, sealed.data_ptr(), out_off, [enc] * ns, plain.data_ptr(), in_off,
                                             enc_totals=[enc] * ns, stream=st.cuda_stream)}
        for name in ("seal", "open"):
            ops[name]()
            times = []
            for _ in range(reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(st)
                ops[name]()
                b.record(st)
                b.synchronize()
                times.append(a.elapsed_time(b) / 1e3)
            t = float(np.median(times))
            emit({"bench": "dare_device", "op": name, "streams": ns, "stream_bytes": n, "ms": round(t * 1e3, 3),
                  "gib_s": round(ns * n / t / GiB, 2)}, gpu)
        assert torch.equal(plain, src), "open did not give the sealed bytes back"
        del src, sealed, plain
        torch.cuda.empty_cache()
    c.close()


def pipelines(mb, gpu, reps, max_mib):
    import ctypes as C
    import dare_ref as d
    L = mb.lib()
    c = mb.Codec(12, 4, MiB)
    for size in [s for s in (MiB, 64 * MiB, GiB) if s <= max_mib * MiB]:
        src = mb.pinned_array(size)
        src[:] = np.random.default_rng(size).integers(0, 256, size, dtype=np.uint8)
        enc = d.encrypted_size(size)
        files = {}
        for name, ln in (("plain", size), ("sse", enc)):
            fsz = c.bitrot_file_size(ln)
            files[name] = [mb.pinned_array(fsz) for _ in range(16)]
        ptr = {k: (C.c_void_p * 16)(*[f.ctypes.data for f in v]) for k, v in files.items()}
        key, nonce = np.frombuffer(KEY, np.uint8), np.frombuffer(NONCE, np.uint8)
        t_plain = timed(lambda: L.mec_encode(c.h, src.ctypes.data, size, ptr["plain"], 0), reps)
        t_sse = timed(lambda: L.mec_encode_sse(c.h, src.ctypes.data, size, key.ctypes.data, nonce.ctypes.data, ptr["sse"], 0), reps)
        emit({"bench": "encode", "object_bytes": size, "encode_ms": round(t_plain * 1e3, 3), "encode_sse_ms": round(t_sse * 1e3, 3),
              "encode_gib_s": round(size / t_plain / GiB, 2), "encode_sse_gib_s": round(size / t_sse / GiB, 2)}, gpu)
        dst = mb.pinned_array(size)
        hint = C.c_int(0)
        for offline in (0, 4):
            fp = {k: (C.c_void_p * 16)(*[None if i < offline else f.ctypes.data for i, f in enumerate(v)]) for k, v in files.items()}
            t_plain = timed(lambda: L.mec_decode(c.h, fp["plain"], 0, size, size, dst.ctypes.data, C.byref(hint)), reps)
            t_sse = timed(lambda: L.mec_decode_sse(c.h, fp["sse"], None, 0, size, enc, key.ctypes.data, dst.ctypes.data, C.byref(hint)),
                          reps)
            assert np.array_equal(dst, src), "decode_sse did not give the object back"
            emit({"bench": "decode", "object_bytes": size, "offline": offline, "decode_ms": round(t_plain * 1e3, 3),
                  "decode_sse_ms": round(t_sse * 1e3, 3), "decode_gib_s": round(size / t_plain / GiB, 2),
                  "decode_sse_gib_s": round(size / t_sse / GiB, 2)}, gpu)
    c.close()


def _host_seal(n):
    import dare_ref as d
    pt = np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8).tobytes()
    t0 = time.perf_counter()
    d.seal(KEY, NONCE, pt)
    return time.perf_counter() - t0


def host(gpu, total_mib):
    try:
        import cryptography  # noqa: F401
    except ImportError:
        emit({"bench": "host_aesgcm", "result": "not measured: cryptography is not installed"}, gpu)
        return
    from concurrent.futures import ProcessPoolExecutor
    n = total_mib * MiB
    _host_seal(MiB)
    t = min(_host_seal(n) for _ in range(3))
    emit({"bench": "host_aesgcm", "threads": 1, "gib_s": round(n / t / GiB, 2)}, gpu)
    cores = os.cpu_count() or 1
    with ProcessPoolExecutor(cores) as ex:
        list(ex.map(_host_seal, [MiB] * cores))
        t0 = time.perf_counter()
        list(ex.map(_host_seal, [n] * cores))
        t = time.perf_counter() - t0
    emit({"bench": "host_aesgcm", "threads": cores, "gib_s": round(cores * n / t / GiB, 2)}, gpu)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-mib", type=int, default=1024, help="largest object of (a) one-stream and (b)")
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--host-mib", type=int, default=256)
    a = ap.parse_args()
    import minio_b200 as mb
    if mb.device_count() == 0:
        sys.exit("bench_sse: no CUDA device (the numbers here are GPU numbers; there is nothing to fall back to)")
    gpu = card()
    dare_device(mb, gpu, a.reps, a.streams, a.max_mib)
    pipelines(mb, gpu, a.reps, a.max_mib)
    host(gpu, a.host_mib)


if __name__ == "__main__":
    main()
