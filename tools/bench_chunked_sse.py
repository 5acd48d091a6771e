"""Streaming-signed PUT bodies of encrypted buckets (aws-chunked + DARE 2.0) on the GPU against the two ways a binding has without it.

  (a) mec_encode_chunked_sse: de-framing and signature checks on the device, sealed and encoded in the same pipeline
  (b) mec_encode_sse of the already de-framed plaintext: the lower bound (no signature work at all)
  (c) hashlib + hmac verifying the body's chunk signatures on one host core, then mec_encode_sse: what a binding does without (a)

RS(12,4) at 1 MiB blocks, 1, 4, 64 and 1024 MiB objects in 64 KiB and 1 MiB aws-chunks, page-locked body, plaintext and part
files; the three alternated, medians of --reps.  The part files of (a) are checked against (b) before timing.  Prints one JSON line
per measurement with the card name, power limit and max SM clock read in the same run.  Needs a GPU: without one it fails.
Usage: python tools/bench_chunked_sse.py [--reps N] [--max-mib M]"""
import argparse
import ctypes as C
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_chunked import KiB, MiB, GiB, card, emit, host_verify  # noqa: E402  (bench_chunked puts the repository on sys.path)


def once(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def run(mb, ref, gpu, reps, max_mib):
    L = mb.lib()
    k, m, bs = 12, 4, MiB
    c = mb.Codec(k, m, bs)
    key = ref.signing_key("bench")
    seed = b"4f232c4386841ef735655705268965c44a0e4690baa4adea153f7db9fa80a0a9"
    scope = ref.scope_of()
    sse_key, nonce = bytes(range(32)), bytes.fromhex("0123456789abcdeffedcba98")
    for mib in (1, 4, 64, 1024):
        if mib > max_mib:
            continue
        D = mib * MiB
        data = mb.pinned_array(D)[:D]
        data[:] = np.random.default_rng(mib).integers(0, 256, D, dtype=np.uint8)
        fsz = c.bitrot_file_size(mb.capi.dare_encrypted_size(D))
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

            def fused():
                rc = L.mec_encode_chunked_sse(c.h, body.ctypes.data, body.size, D, key, seed, ref.DATE.encode(), scope.encode(), 0,
                                              sse_key, nonce, fp, 0, None, 0, C.byref(tl))
                assert rc == D, rc

            def sse():
                rc = L.mec_encode_sse(c.h, data.ctypes.data, D, sse_key, nonce, fp, 0)
                assert rc == D, rc

            def host_then_sse():
                host_verify(body, spans, key, scope, seed)
                sse()
            fused()
            want = [f.copy() for f in files]
            sse()
            assert all(np.array_equal(a, w) for a, w in zip(files, want)), "mec_encode_chunked_sse differs from mec_encode_sse"
            del want
            host_then_sse()
            ta, tb, tc = [], [], []
            for _ in range(reps):
                ta.append(once(fused))
                tb.append(once(sse))
                tc.append(once(host_then_sse))
            ta, tb, tc = (float(np.median(t)) for t in (ta, tb, tc))
            emit({"bench": "encode_chunked_sse", "object_mib": mib, "chunk_bytes": csize, "chunks": len(spans),
                  "a_chunked_sse_ms": round(ta * 1e3, 3), "b_encode_sse_ms": round(tb * 1e3, 3),
                  "c_host_verify_then_sse_ms": round(tc * 1e3, 3), "a_minus_b_ms": round((ta - tb) * 1e3, 3),
                  "a_GiB_s": round(D / ta / GiB, 2), "b_GiB_s": round(D / tb / GiB, 2), "c_GiB_s": round(D / tc / GiB, 2)}, gpu)
            del body
        del files, data
    c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-mib", type=int, default=1024)
    a = ap.parse_args()
    import minio_b200 as mb
    import sigv4_ref as ref
    assert mb.device_count() > 0, "no CUDA device: this benchmark measures the GPU"
    run(mb, ref, card(), a.reps, a.max_mib)


if __name__ == "__main__":
    main()
