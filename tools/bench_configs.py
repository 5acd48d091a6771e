#!/usr/bin/env python
"""Device-resident timings of the other BASELINE.json configs (3: reconstruct, 4: heal shape, 5: block-size
sweep) — parity-checked against the encode outputs; one JSON object per line.  bench.py stays the headline."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import minio_b200 as mb  # noqa: E402

GiB = float(1 << 30)
PEAK = 3350.0  # GB/s: H100 SXM data-sheet HBM3 bandwidth; frac_of_hbm_peak is of this nominal figure
dev = torch.device("cuda:0")


def set_device(index):
    """bench.py runs one rank per GPU: every case below allocates on and times `dev`."""
    global dev
    dev = torch.device(f"cuda:{index}")
    torch.cuda.set_device(dev)


def timeit(fn, steps=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def make_stream(nbytes, seed):
    g = torch.Generator(device=dev); g.manual_seed(seed)
    out = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    step = 1 << 30
    for o in range(0, nbytes, step):
        n = min(step, nbytes - o)
        out[o:o + n] = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev, generator=g)
    return out


def encode(k, m, bs, nblocks, seed):
    S = -(-bs // k)
    pitch = (S + 15) // 16 * 16
    src = make_stream(nblocks * bs, seed)
    par = torch.zeros((nblocks * m, pitch), dtype=torch.uint8, device=dev)
    dig = torch.zeros((nblocks, k + m, 32), dtype=torch.uint8, device=dev)
    c = mb.Codec(k, m, bs, device=dev.index or 0)
    c.set_option("jit", 1)  # synchronous specialisation: the default (-1) compiles in the background and would be measured half-warm
    st = torch.cuda.current_stream().cuda_stream
    fn = lambda: c.encode_blocks_device(src.data_ptr(), src.numel(), par.data_ptr(), pitch, dig.data_ptr(), st)
    ms = timeit(fn)
    return c, src, par, dig, S, pitch, ms


def frames_from(k, m, bs, nblocks, src, par, dig, S):
    fp = (32 + S + 15) // 16 * 16
    frames = []
    src2 = src.view(nblocks, bs)
    par3 = par.view(nblocks, m, -1)
    arena = torch.zeros((k + m, nblocks, fp), dtype=torch.uint8, device=dev)  # one allocation: shard files at a uniform stride (run-wise 3-D TMA fetch)
    for i in range(k + m):
        f = arena[i]
        f[:, :32] = dig[:, i]
        if i < k:
            lo, hi = i * S, min((i + 1) * S, bs)
            if hi > lo:
                f[:, 32:32 + hi - lo] = src2[:, lo:hi]
        else:
            f[:, 32:32 + S] = par3[:, i - k, :S]
        frames.append(f)
    return frames, fp


def reconstruct_case(name, k, m, bs, nblocks, erased, seed, flags=0, quiet=False, steps=10):
    """flags: MEC_RECONSTRUCT_* bits (3 = GetObject shape: data only, rebuilt shards not hashed; 0 = heal shape)"""
    c, src, par, dig, S, pitch, enc_ms = encode(k, m, bs, nblocks, seed)
    frames, fp = frames_from(k, m, bs, nblocks, src, par, dig, S)
    del src, par
    n = k + m
    r = len(erased)
    want = [1 if i in erased else 0 for i in range(n)]
    ptrs = [0 if i in erased else frames[i].data_ptr() for i in range(n)]
    opitch = (S + 15) // 16 * 16
    out = torch.zeros((nblocks * r, opitch), dtype=torch.uint8, device=dev)
    odig = torch.zeros((nblocks, k + r, 32), dtype=torch.uint8, device=dev)
    cor = torch.zeros((nblocks, k), dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    fn = lambda: c.reconstruct_device(ptrs, fp, nblocks, want, flags, out.data_ptr(), opitch, odig.data_ptr(), cor.data_ptr(), st)
    c.set_option("jit", 0)
    generic_ms = timeit(fn, steps=max(2, steps // 3))
    c.set_option("jit", 1)
    import time
    torch.cuda.synchronize(); t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); first_call_s = time.perf_counter() - t0
    ms = timeit(fn, steps=steps)
    ok = int(cor.sum().item()) == 0
    o3 = out.view(nblocks, r, opitch)
    for q, i in enumerate(sorted(erased)):
        ok &= bool(torch.equal(o3[:, q, :S], frames[i][:, 32:32 + S]))
        if not flags & 2:
            ok &= bool(torch.equal(odig[:, k + q], frames[i][:, :32]))
    algo = k * (S + 32) + r * S + (0 if flags & 2 else r * 32)
    res = {"config": name, "flags": flags, "k": k, "m": m, "block_size": bs, "blocks": nblocks, "erased": sorted(erased), "ms": ms,
           "GiB_per_s_object": nblocks * bs / GiB / (ms / 1e3), "algorithmic_bytes_per_block": algo,
           "achieved_GBps": algo * nblocks / (ms / 1e3) / 1e9, "frac_of_hbm_peak": algo * nblocks / (ms / 1e3) / 1e9 / PEAK,
           "bit_exact_vs_encode": ok, "generic_kernel_ms": generic_ms, "generic_GiB_per_s": nblocks * bs / GiB / (generic_ms / 1e3),
           "first_call_seconds_incl_nvrtc": first_call_s, "encode_ms_same_shape": enc_ms, "encode_GiB_per_s": nblocks * bs / GiB / (enc_ms / 1e3)}
    if not quiet:
        print(json.dumps(res), flush=True)
    c.close()
    return res


def verify_case(k, m, bs, nblocks, seed):
    """deep-scan bitrotVerify shape (SURVEY §8f rank 1): hash k shard files' frames, compare with stored digests, no RS work"""
    c, src, par, dig, S, pitch, enc_ms = encode(k, m, bs, nblocks, seed)
    frames, fp = frames_from(k, m, bs, nblocks, src, par, dig, S)
    del src, par
    n = k + m
    ptrs = [frames[i].data_ptr() for i in range(n)]
    odig = torch.zeros((nblocks, k, 32), dtype=torch.uint8, device=dev)
    cor = torch.zeros((nblocks, k), dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    fn = lambda: c.reconstruct_device(ptrs, fp, nblocks, [0] * n, False, 0, 16, odig.data_ptr(), cor.data_ptr(), st)
    ms = timeit(fn)
    ok = int(cor.sum().item()) == 0 and bool(torch.equal(odig, dig[:, :k]))
    frames[3][5, 100] ^= 1
    fn(); torch.cuda.synchronize()
    ok &= int(cor.sum().item()) == 1 and int(cor[5, 3].item()) == 1
    hashed = nblocks * k * (S + 32)
    print(json.dumps({"config": "verify: deep-scan of %d RS(%d,%d) shard files (hash + compare only)" % (k, k, m), "k": k, "m": m, "block_size": bs,
                      "blocks": nblocks, "ms": ms, "GiB_per_s_object": nblocks * bs / GiB / (ms / 1e3), "hashed_GBps": hashed / (ms / 1e3) / 1e9,
                      "frac_of_hbm_peak": hashed / (ms / 1e3) / 1e9 / PEAK, "bit_exact_vs_encode": ok}), flush=True)
    c.close()


def jit_encode_case(k, m, bs, nblocks):
    """a geometry without a compiled specialisation: generic kernel vs NVRTC-specialised encode"""
    c, src, par, dig, S, pitch, ms = encode(k, m, bs, nblocks, 21)
    ref = par.clone(); refd = dig.clone()
    c.set_option("jit", 0)
    st = torch.cuda.current_stream().cuda_stream
    fn = lambda: c.encode_blocks_device(src.data_ptr(), src.numel(), par.data_ptr(), pitch, dig.data_ptr(), st)
    gms = timeit(fn)
    ok = bool(torch.equal(par, ref)) and bool(torch.equal(dig, refd))
    algo = bs + m * S + (k + m) * 32
    print(json.dumps({"config": "encode RS(%d,%d), no compiled specialisation: NVRTC-specialised vs generic kernel" % (k, m), "k": k, "m": m,
                      "block_size": bs, "blocks": nblocks, "ms": ms, "GiB_per_s_object": nblocks * bs / GiB / (ms / 1e3),
                      "generic_GiB_per_s": nblocks * bs / GiB / (gms / 1e3), "frac_of_hbm_peak": algo * nblocks / (ms / 1e3) / 1e9 / PEAK,
                      "bit_exact_vs_encode": ok}), flush=True)
    c.close()


def sweep(k, m, sizes, total_bytes):
    for bs in sizes:
        nblocks = total_bytes // bs
        c, src, par, dig, S, pitch, ms = encode(k, m, bs, nblocks, 11)
        algo = bs + m * S + (k + m) * 32
        print(json.dumps({"config": "5-sweep with HighwayHash256S instead of SHA256 (block-size sweep of the fused kernel)", "k": k, "m": m,
                          "block_size": bs, "blocks": nblocks, "ms": ms, "GiB_per_s_object": nblocks * bs / GiB / (ms / 1e3),
                          "frac_of_hbm_peak": algo * nblocks / (ms / 1e3) / 1e9 / PEAK}), flush=True)
        c.close()
        del src, par, dig


def sha256_sweep(k, m, sizes, total_bytes, quiet=False):
    """BASELINE config 5: RS(8,8) with SHA256 whole-file bitrot, one-block objects (one digest per shard file), block-size sweep.
    Parity from the fused kernel without hashing, then one SHA-256 stream per shard (`whole_hash.cuh`); checked with hashlib."""
    import hashlib
    out = []
    for bs in sizes:
        nblocks = total_bytes // bs
        S = bs // k
        pitch = (S + 15) // 16 * 16
        src = torch.cat([make_stream(nblocks * bs, 5), torch.zeros(256, dtype=torch.uint8, device=dev)])
        par = torch.zeros((nblocks * m + 1, pitch), dtype=torch.uint8, device=dev)
        dig = torch.zeros((nblocks * (k + m), 64), dtype=torch.uint8, device=dev)
        c = mb.Codec(k, m, bs, algo=mb.SHA256, device=dev.index or 0)
        st = torch.cuda.current_stream().cuda_stream

        def fn():
            c.encode_blocks_device(src.data_ptr(), nblocks * bs, par.data_ptr(), pitch, 0, st)
            c.whole_hash_device(mb.SHA256, src.data_ptr(), S, S, nblocks * k, dig.data_ptr(), st)               # data shard (b, t) = stream b*k+t
            c.whole_hash_device(mb.SHA256, par.data_ptr(), pitch, S, nblocks * m, dig.data_ptr() + nblocks * k * 64, st)
        ms = timeit(fn, steps=5, warm=2)
        h_dig = dig.cpu().numpy()
        ok = True
        for b in sorted({0, nblocks // 2, nblocks - 1}):   # the first, a middle and the last block: k + m digests each
            h_src = src[b * bs:(b + 1) * bs].cpu().numpy().tobytes(); h_par = par[b * m:(b + 1) * m, :S].cpu().numpy()
            ok &= all(hashlib.sha256(h_src[t * S:(t + 1) * S]).digest() == h_dig[b * k + t, :32].tobytes() for t in range(k))
            ok &= all(hashlib.sha256(h_par[j].tobytes()).digest() == h_dig[nblocks * k + b * m + j, :32].tobytes() for j in range(m))
        algo = bs + m * S + (k + m) * 32   # what a single fused pass would move (the implementation makes two passes)
        res = {"config": "5: RS(%d,%d) + SHA256 whole-file bitrot, one-block objects" % (k, m), "k": k, "m": m, "block_size": bs,
               "blocks": nblocks, "ms": ms, "GiB_per_s_object": nblocks * bs / GiB / (ms / 1e3), "algorithmic_bytes_per_block": algo,
               "frac_of_hbm_peak": algo * nblocks / (ms / 1e3) / 1e9 / PEAK, "bit_exact_vs_encode": bool(ok)}
        out.append(res)
        if not quiet:
            print(json.dumps(res), flush=True)
        c.close()
        del src, par, dig
    return out


def heal_batch_case(nobj=32, obj_mib=64, pools=(1, 2, 3, 4), pinned=True):
    """BASELINE config 4 through the HOST boundary (per-GPU slice, scaled to nobj objects): mec_heal_batch over a pool of
    codec handles — frames come from (pinned or pageable) host memory, healed shard files go back to it."""
    import time
    k, m, bs = 16, 4, 1 << 20
    n = k + m
    stale_set = (0, 7, 16, 19)
    size = obj_mib << 20
    enc = mb.Codec(k, m, bs)
    rng = np.random.default_rng(4)
    objects, ref = [], []
    for o in range(nobj):
        data = rng.integers(0, 256, size, dtype=np.uint8)
        files = enc.encode(data)
        stale = [i in stale_set for i in range(n)]
        if pinned:
            src = []
            for i in range(n):
                if stale[i]:
                    src.append(None)
                else:
                    a = mb.pinned_array(files[i].size); a[:] = files[i]; src.append(a)
        else:
            src = [None if stale[i] else files[i] for i in range(n)]
        objects.append((src, stale, size))
        ref.append(files)
    fsz = enc.bitrot_file_size(size)
    enc.close()
    outs_pre = [[mb.pinned_array(fsz) if i in stale_set else None for i in range(n)] for _ in range(nobj)] if pinned else None
    for npool in pools:
        pool = [mb.Codec(k, m, bs) for _ in range(npool)]
        mb.heal_batch(pool, objects[:max(2, npool)], None if outs_pre is None else outs_pre[:max(2, npool)])  # warm: buffers, specialised kernel
        time.sleep(1.0)
        t0 = time.perf_counter()
        outs = mb.heal_batch(pool, objects, outs_pre)
        dt = time.perf_counter() - t0
        ok = all(np.array_equal(outs[o][i], ref[o][i]) for o in range(nobj) for i in stale_set)
        print(json.dumps({"config": "4-host: RS(16,4) heal batch through mec_heal_batch, %d objects x %d MiB, stale %s" % (nobj, obj_mib, list(stale_set)),
                          "pool": npool, "host_memory": "pinned" if pinned else "pageable", "seconds": dt, "GiB_per_s_object": nobj * size / GiB / dt, "bit_exact_vs_encode": bool(ok)}), flush=True)
        for c in pool:
            c.close()


if __name__ == "__main__":
    MiB = 1 << 20
    only = sys.argv[1] if len(sys.argv) > 1 else ""
    if only == "healbatch":
        heal_batch_case(pinned=True)
        heal_batch_case(pools=(2,), pinned=False)
        sys.exit(0)
    if only == "gen":   # generic (runtime-matrix) kernel numbers only
        reconstruct_case("gen r=4", 12, 4, MiB, 3552, {0, 1, 2, 3}, 3, 0)
        reconstruct_case("gen r=2", 12, 4, MiB, 3552, {0, 1}, 3, 0)
        reconstruct_case("gen r=1", 12, 4, MiB, 3552, {3}, 3, 0)
        verify_case(12, 4, MiB, 10240, 9)
        sys.exit(0)
    if only == "jit":
        for _ in range(3):
            jit_encode_case(10, 4, MiB, 4096)
        jit_encode_case(10, 4, MiB, 8192)
        jit_encode_case(7, 5, MiB, 4096)
        jit_encode_case(6, 3, MiB, 4096)
        sys.exit(0)
    if only == "4k":   # one case, e.g. under ncu
        reconstruct_case("4: RS(16,4) heal shape, stale {0,7,16,19}", 16, 4, MiB, int(sys.argv[2]) if len(sys.argv) > 2 else 2960, {0, 7, 16, 19}, 4, 0)
        sys.exit(0)
    if only == "3b":
        reconstruct_case("3b: RS(12,4) heal shape, shards {1,5,12,15} stale", 12, 4, MiB, int(sys.argv[2]) if len(sys.argv) > 2 else 3552, {1, 5, 12, 15}, 3, 0)
        sys.exit(0)
    if only == "3a":   # one case, e.g. under ncu
        reconstruct_case("3a: RS(12,4) GetObject shape, data shards {0,1,2,3} erased", 12, 4, MiB, int(sys.argv[2]) if len(sys.argv) > 2 else 3552, {0, 1, 2, 3}, 3, 3)
        sys.exit(0)
    reconstruct_case("3a: RS(12,4) GetObject shape (data only, rebuilt shards not hashed), data shards {0,1,2,3} erased", 12, 4, MiB, 10240, {0, 1, 2, 3}, 3, 3)
    reconstruct_case("3a': RS(12,4) heal shape (rebuilt shards hashed), shards {0,1,2,3} stale", 12, 4, MiB, 10240, {0, 1, 2, 3}, 3, 0)
    reconstruct_case("3b: RS(12,4) heal shape, shards {1,5,12,15} stale", 12, 4, MiB, 10240, {1, 5, 12, 15}, 3, 0)
    reconstruct_case("3c: RS(12,4) GetObject shape, one data shard erased", 12, 4, MiB, 10240, {3}, 3, 3)
    reconstruct_case("4: RS(16,4) heal shape, stale {0,7,16,19} (per-GPU slice of 1024 x 64 MiB over 8 GPUs: 128 objects)", 16, 4, MiB, 8192, {0, 7, 16, 19}, 4, 0)
    verify_case(12, 4, MiB, 10240, 9)
    jit_encode_case(10, 4, MiB, 4096)
    jit_encode_case(7, 5, MiB, 2048)
    sha256_sweep(8, 8, [64 << 10, 256 << 10, MiB, 4 * MiB], 1 << 30)
    sweep(8, 8, [64 << 10, 128 << 10, 256 << 10, 512 << 10, MiB, 2 * MiB, 4 * MiB], 1 << 30)
