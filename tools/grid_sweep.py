#!/usr/bin/env python3
"""Device-resident encode + bitrot rate of several (k, m, block size) shapes at the engine's default grid and at other CTAs per SM.

For each shape, 8 GiB of seeded random object bytes (rounded down to whole blocks) are encoded with mec_encode_blocks_device;
geometries without a compiled kernel run the NVRTC-specialised one (jit = 1).  The grid settings of one shape are alternated
over --rounds rounds, each timing --launches launches with CUDA events after --warmup untimed ones.  grid_mult = 64 is more CTAs
than ever fit, i.e. the occupancy-sized grid.  One JSON line per (shape, setting) goes to stdout and to <out>/grid_sweep.jsonl.

  python tools/grid_sweep.py [--shapes 12,4,1048576 6,2,1048576] [--grid 0,64] [--rounds 3] [--out bench_out]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["12,4,1048576", "6,2,1048576", "10,4,1048576", "7,5,1048576"])
    ap.add_argument("--grid", default="0,64", help="comma-separated grid_mult values (0 = the engine's default)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--gib", type=float, default=8.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    import torch
    import minio_b200 as mb
    dev = torch.device("cuda:0")
    props = torch.cuda.get_device_properties(0)
    grids = [int(x) for x in args.grid.split(",")]
    stream = torch.cuda.current_stream()
    with open(os.path.join(args.out, "grid_sweep.jsonl"), "w") as log:
        for shape in args.shapes:
            k, m, bs = (int(x) for x in shape.split(","))
            S = -(-bs // k)
            pitch = (S + 15) // 16 * 16
            nblocks = int(args.gib * (1 << 30)) // bs
            nbytes = nblocks * bs
            gen = torch.Generator(device=dev)
            gen.manual_seed(k * 1000 + m)
            src = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            for o0 in range(0, nbytes, 1 << 30):
                n = min(1 << 30, nbytes - o0)
                src[o0:o0 + n] = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev, generator=gen)
            par = torch.empty((nblocks * m, pitch), dtype=torch.uint8, device=dev)
            dig = torch.empty((nblocks, k + m, 32), dtype=torch.uint8, device=dev)
            codecs = {}
            for g in grids:
                c = mb.Codec(k, m, bs, device=0)
                c.set_option("jit", 1)
                c.set_option("grid_mult", g)
                codecs[g] = c
            rates = {g: [] for g in grids}
            for rnd in range(args.rounds):
                for g in grids[rnd % len(grids):] + grids[:rnd % len(grids)]:  # rotated: no setting always runs first
                    c = codecs[g]
                    for _ in range(args.warmup):
                        c.encode_blocks_device(src.data_ptr(), nbytes, par.data_ptr(), pitch, dig.data_ptr(), stream.cuda_stream)
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(stream)
                    for _ in range(args.launches):
                        c.encode_blocks_device(src.data_ptr(), nbytes, par.data_ptr(), pitch, dig.data_ptr(), stream.cuda_stream)
                    b.record(stream)
                    b.synchronize()
                    rates[g].append(nbytes * args.launches / (1 << 30) / (a.elapsed_time(b) / 1e3))
            for g in grids:
                rec = {"gpu": props.name, "k": k, "m": m, "block_size": bs, "S_mod_16": S % 16, "blocks": nblocks, "grid_mult": g,
                       "jit_launches": codecs[g].stat("jit_launches"), "GiB_s_median": statistics.median(rates[g]),
                       "GiB_s_min": min(rates[g]), "GiB_s_max": max(rates[g])}
                print(json.dumps(rec), flush=True)
                log.write(json.dumps(rec) + "\n")
                codecs[g].close()
            del src, par, dig
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
