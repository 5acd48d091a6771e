"""DARE 2.0 ChaCha20-Poly1305 (option "dare_chacha20") against AES-256-GCM on the GPU, in one session on one card.

  (a) mec_dare_device seal and open: GiB/s of plaintext per call (CUDA events around the call, which includes any key setup and ends
      in a synchronise) for one 1 GiB stream, 4096 x 1 MiB and 4096 x 64 KiB; median of --reps, the two ciphers alternated rep by
      rep.  AES seals at option 0 and opens at 0 and at 1 (the extra ChaCha20 launch over AES rows); ChaCha20 seals at 2, opens at 1.
  (b) mec_decode_sse of a ChaCha20 part (option 1) against an AES part (option 0), RS(12,4) at 1 MiB blocks, 1 MiB / 64 MiB / 1 GiB,
      0 and 4 drives offline, page-locked buffers (host clock; median, alternated)
  (c) the coalescer: --threads concurrent 1 MiB encrypted GETs per round through one batcher, ChaCha20 parts at option 1 against AES
      parts at option 0 (host clock per round; median, alternated)

Prints one JSON line per measurement, each with the card name, power limit and max SM clock read in the same run.  Needs a GPU.
Usage: python tools/bench_sse_chacha.py [--reps N] [--max-mib M] [--streams S] [--threads T]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

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


def alternated(fns, reps):
    """{name: median seconds} of host-clocked calls, every name once per rep in turn, after one warm-up each"""
    for f in fns.values():
        f()
    t = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            t0 = time.perf_counter()
            f()
            t[k].append(time.perf_counter() - t0)
    return {k: float(np.median(v)) for k, v in t.items()}


def dare_device(mb, gpu, reps, streams, total_mib):
    import torch
    import dare_ref as d
    cs = {v: mb.Codec(12, 4, MiB) for v in (0, 1, 2)}
    for v, c in cs.items():
        c.set_option("dare_chacha20", v)
    st = torch.cuda.current_stream()
    for ns, n in [(1, total_mib * MiB), (streams, MiB), (streams, 64 << 10)]:
        src = torch.randint(0, 256, (ns * n,), dtype=torch.uint8, device="cuda")
        enc = d.encrypted_size(n)
        sealed = {x: torch.empty(ns * enc, dtype=torch.uint8, device="cuda") for x in ("aes", "chacha")}
        plain = torch.empty(ns * n, dtype=torch.uint8, device="cuda")
        keys = np.frombuffer(np.random.default_rng(ns).bytes(32 * ns), np.uint8)
        nonces = np.frombuffer(np.random.default_rng(ns + 1).bytes(12 * ns), np.uint8)
        in_off, out_off = np.arange(ns, dtype=np.int64) * n, np.arange(ns, dtype=np.int64) * enc

        def seal(c, x):
            return lambda: c.dare_device(1, keys, src.data_ptr(), in_off, [n] * ns, sealed[x].data_ptr(), out_off, nonces=nonces,
                                         stream=st.cuda_stream)

        def open_(c, x):
            return lambda: c.dare_device(2, keys, sealed[x].data_ptr(), out_off, [enc] * ns, plain.data_ptr(), in_off,
                                         enc_totals=[enc] * ns, stream=st.cuda_stream)

        ops = {"seal_aes": seal(cs[0], "aes"), "seal_chacha": seal(cs[2], "chacha"), "open_aes": open_(cs[0], "aes"),
               "open_aes_at_1": open_(cs[1], "aes"), "open_chacha": open_(cs[1], "chacha")}
        for f in ops.values():
            f()
        times = {k: [] for k in ops}
        for _ in range(reps):
            for k, f in ops.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(st)
                f()
                b.record(st)
                b.synchronize()
                times[k].append(a.elapsed_time(b) / 1e3)
        assert torch.equal(plain, src), "open did not give the sealed bytes back"
        rec = {"bench": "dare_device", "streams": ns, "stream_bytes": n}
        for k, v in times.items():
            rec[k + "_gib_s"] = round(ns * n / float(np.median(v)) / GiB, 2)
        emit(rec, gpu)
        del src, sealed, plain
        torch.cuda.empty_cache()
    for c in cs.values():
        c.close()


def decode(mb, gpu, reps, max_mib):
    L = mb.lib()
    c0, c1, c2 = (mb.Codec(12, 4, MiB) for _ in range(3))
    c1.set_option("dare_chacha20", 1)
    c2.set_option("dare_chacha20", 2)
    key, nonce = np.frombuffer(KEY, np.uint8), np.frombuffer(NONCE, np.uint8)
    for size in [s for s in (MiB, 64 * MiB, GiB) if s <= max_mib * MiB]:
        src = mb.pinned_array(size)
        src[:] = np.random.default_rng(size).integers(0, 256, size, dtype=np.uint8)
        enc = mb.capi.dare_encrypted_size(size)
        fsz = c0.bitrot_file_size(enc)
        files = {x: [mb.pinned_array(fsz) for _ in range(16)] for x in ("aes", "chacha")}
        for x, c in (("aes", c0), ("chacha", c2)):
            ptr = (C.c_void_p * 16)(*[f.ctypes.data for f in files[x]])
            assert L.mec_encode_sse(c.h, src.ctypes.data, size, key.ctypes.data, nonce.ctypes.data, ptr, 0) == size
        assert files["aes"][0][33] == 0 and files["chacha"][0][33] == 1  # header byte 1 of the first package: the cipher
        dst = mb.pinned_array(size)
        hint = C.c_int(0)
        for offline in (0, 4):
            fp = {x: (C.c_void_p * 16)(*[None if i < offline else f.ctypes.data for i, f in enumerate(v)]) for x, v in files.items()}
            t = alternated({
                "aes": lambda: L.mec_decode_sse(c0.h, fp["aes"], None, 0, size, enc, key.ctypes.data, dst.ctypes.data, C.byref(hint)),
                "chacha": lambda: L.mec_decode_sse(c1.h, fp["chacha"], None, 0, size, enc, key.ctypes.data, dst.ctypes.data,
                                                   C.byref(hint))}, reps)
            assert np.array_equal(dst, src), "decode_sse did not give the object back"
            emit({"bench": "decode_sse", "object_bytes": size, "offline": offline, "aes_ms": round(t["aes"] * 1e3, 3),
                  "chacha_ms": round(t["chacha"] * 1e3, 3), "aes_gib_s": round(size / t["aes"] / GiB, 2),
                  "chacha_gib_s": round(size / t["chacha"] / GiB, 2)}, gpu)
        for v in files.values():
            for f in v:
                L.mec_free_pinned(f.ctypes.data)
        L.mec_free_pinned(src.ctypes.data)
        L.mec_free_pinned(dst.ctypes.data)
    for c in (c0, c1, c2):
        c.close()


def batcher(mb, gpu, reps, threads):
    c0, c2 = mb.Codec(12, 4, MiB), mb.Codec(12, 4, MiB)
    c2.set_option("dare_chacha20", 2)
    size = MiB
    parts = {}
    for x, c in (("aes", c0), ("chacha", c2)):
        parts[x] = []
        for i in range(threads):
            pt = np.random.default_rng(i).integers(0, 256, size, dtype=np.uint8)
            files = [mb.pinned_array(f.size) for f in c.encode_sse(pt, KEY, NONCE)]
            for f, g in zip(files, c.encode_sse(pt, KEY, NONCE)):
                f[:] = g
            parts[x].append((pt, files))
    enc = mb.capi.dare_encrypted_size(size)
    bs = {x: mb.Batcher(12, 4, MiB) for x in parts}
    bs["chacha"].set_option("dare_chacha20", 1)
    dsts = [mb.pinned_array(size) for _ in range(threads)]
    ex = ThreadPoolExecutor(threads)

    def round_(x):
        def one(i):
            out, _ = bs[x].decode_sse(parts[x][i][1], 0, size, enc, KEY, dst=dsts[i])
            return np.array_equal(out, parts[x][i][0])
        return lambda: all(ex.map(one, range(threads)))

    t = alternated({x: round_(x) for x in parts}, reps)
    assert round_("aes")() and round_("chacha")()
    emit({"bench": "batcher_decode_sse", "threads": threads, "object_bytes": size,
          "aes_ms": round(t["aes"] * 1e3, 3), "chacha_ms": round(t["chacha"] * 1e3, 3),
          "aes_gib_s": round(threads * size / t["aes"] / GiB, 2), "chacha_gib_s": round(threads * size / t["chacha"] / GiB, 2),
          "aes_batches": bs["aes"].stat("batches"), "chacha_batches": bs["chacha"].stat("batches"),
          "serial": bs["aes"].stat("sse_serial") + bs["chacha"].stat("sse_serial")}, gpu)
    ex.shutdown()
    for b in bs.values():
        b.close()
    c0.close(); c2.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-mib", type=int, default=1024, help="largest object of (a) one-stream and (b)")
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--threads", type=int, default=64)
    a = ap.parse_args()
    import minio_b200 as mb
    if mb.device_count() == 0:
        sys.exit("bench_sse_chacha: no CUDA device (the numbers here are GPU numbers; there is nothing to fall back to)")
    gpu = card()
    dare_device(mb, gpu, a.reps, a.streams, a.max_mib)
    decode(mb, gpu, a.reps, a.max_mib)
    batcher(mb, gpu, a.reps, a.threads)


if __name__ == "__main__":
    main()
