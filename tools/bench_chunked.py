"""Signature V4 streaming bodies (aws-chunked, STREAMING-AWS4-HMAC-SHA256-PAYLOAD) on the GPU against the plain encode and the host.

  (a) mec_chunk_signatures_device: one launch over R rows of 8 KiB, 64 KiB and 1 MiB chunks, R = 16 .. 4096 (host clock around
      the call, which ends in a synchronise; median): call time, time per row and aggregate GiB/s of payload hashed
  (b) mec_encode_chunked against mec_encode of the same decoded bytes, RS(12,4) at 1 MiB blocks, 1, 64 and 1024 MiB objects
      in 64 KiB and 1 MiB aws-chunks, page-locked body, object and part files, the two calls alternated (median)
  (c) the host alternative: hashlib + hmac verifying the same bodies' chunk signatures on one core (what the serial reader
      spends besides its copies)

Prints one JSON line per measurement, each with the card name, power limit and max SM clock read in the same run.  Needs a GPU:
without one it fails.  Usage: python tools/bench_chunked.py [--reps N] [--max-mib M]"""
import argparse
import ctypes as C
import hashlib
import hmac
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30


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


def kernel(mb, ref, gpu, reps):
    import torch
    c = mb.Codec(12, 4, MiB)
    key = ref.signing_key("bench")
    scope = ref.scope_of()
    for size in (8 * KiB, 64 * KiB, MiB):
        for rows in (16, 64, 256, 1024, 4096):
            buf = torch.randint(0, 256, (rows * size,), dtype=torch.uint8, device="cuda")
            offs = [i * size for i in range(rows)]
            sig = [b"0" * 64] * rows
            fn = lambda: c.chunk_signatures_device(key, ref.DATE, scope, buf.data_ptr(), offs, [size] * rows, sig, sig, [0] * rows)
            t = timed(fn, reps)
            emit({"bench": "chunk_signatures_device", "chunk_bytes": size, "rows": rows, "call_ms": round(t * 1e3, 3),
                  "us_per_row": round(t * 1e6 / rows, 3), "GiB_s": round(rows * size / t / GiB, 2)}, gpu)
            del buf
    c.close()


def host_verify(body, spans, key, scope, seed):
    """the chunk signatures of a body on one core: sha256 of each payload, then the HMAC of the string to sign"""
    mv = memoryview(body)
    prev = seed
    head = b"AWS4-HMAC-SHA256-PAYLOAD\n" + b"20130524T000000Z\n" + scope.encode() + b"\n"
    tail = b"\n" + hashlib.sha256(b"").hexdigest().encode() + b"\n"
    for s, n, claim in spans:
        d = hashlib.sha256(mv[s:s + n]).hexdigest().encode()
        sig = hmac.new(key, head + prev + tail + d, hashlib.sha256).hexdigest().encode()
        if not hmac.compare_digest(sig, claim):
            raise RuntimeError("host verify failed")
        prev = claim


def end_to_end(mb, ref, gpu, reps, max_mib):
    L = mb.lib()
    k, m, bs = 12, 4, MiB
    c = mb.Codec(k, m, bs)
    key = ref.signing_key("bench")
    seed = b"4f232c4386841ef735655705268965c44a0e4690baa4adea153f7db9fa80a0a9"
    scope = ref.scope_of()
    for mib in (1, 64, 1024):
        if mib > max_mib:
            continue
        D = mib * MiB
        data = mb.pinned_array(D)[:D]
        data[:] = np.random.default_rng(mib).integers(0, 256, D, dtype=np.uint8)
        fsz = c.bitrot_file_size(D)
        files = [mb.pinned_array(fsz)[:fsz] for _ in range(k + m)]
        fp = (C.c_void_p * (k + m))(*[f.ctypes.data for f in files])
        for csize in (64 * KiB, MiB):
            sizes = [min(csize, D - o) for o in range(0, D, csize)]
            b = ref.build(data, sizes, key, seed)
            body = mb.pinned_array(len(b.data))[:len(b.data)]
            body[:] = np.frombuffer(bytes(b.data), dtype=np.uint8)
            spans = [(f["payload"][0], f["payload"][1] - f["payload"][0], f["sigval"]) for f in b.chunks]
            del b
            tl = C.c_int64(0)

            def chunked():
                rc = L.mec_encode_chunked(c.h, body.ctypes.data, body.size, D, key, seed, ref.DATE.encode(), scope.encode(), 0, fp, 0,
                                          None, 0, C.byref(tl))
                assert rc == D, rc

            def plain():
                rc = L.mec_encode(c.h, data.ctypes.data, D, fp, 0)
                assert rc == D, rc
            chunked()
            want = [f.copy() for f in files]
            plain()
            assert all(np.array_equal(a, w) for a, w in zip(files, want)), "mec_encode_chunked differs from mec_encode"
            tc, tp = [], []
            for _ in range(reps):
                tc.append(timed(chunked, 1))
                tp.append(timed(plain, 1))
            tc, tp = float(np.median(tc)), float(np.median(tp))
            th = timed(lambda: host_verify(body, spans, key, scope, seed), max(1, min(reps, 3)))
            emit({"bench": "encode_chunked", "object_mib": mib, "chunk_bytes": csize, "chunks": len(spans),
                  "chunked_ms": round(tc * 1e3, 3), "encode_ms": round(tp * 1e3, 3), "extra_ms": round((tc - tp) * 1e3, 3),
                  "chunked_GiB_s": round(D / tc / GiB, 2), "encode_GiB_s": round(D / tp / GiB, 2),
                  "host_verify_ms_1core": round(th * 1e3, 3), "host_verify_MB_s": round(D / th / 1e6, 1)}, gpu)
    c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--max-mib", type=int, default=1024)
    a = ap.parse_args()
    import minio_b200 as mb
    import sigv4_ref as ref
    assert mb.device_count() > 0, "no CUDA device: this benchmark measures the GPU"
    gpu = card()
    kernel(mb, ref, gpu, a.reps)
    end_to_end(mb, ref, gpu, a.reps, a.max_mib)


if __name__ == "__main__":
    main()
