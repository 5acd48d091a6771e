#!/usr/bin/env python
"""Kernel time of small launches (device-resident encode of N 1 MiB blocks): latency kernel (ec_small.cuh) vs throughput kernel."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import minio_b200 as mb
from minio_b200 import capi


def main():
    k, m, bs = (int(sys.argv[1]), int(sys.argv[2]), 1 << 20) if len(sys.argv) > 2 else (12, 4, 1 << 20)
    torch.cuda.set_device(0)
    out = []
    for nb in (1, 2, 4, 8, 16, 32, 64, 132, 264, 396, 528, 792, 1056, 1848, 3696):
        row = {"blocks": nb}
        src = torch.randint(0, 256, (nb * bs,), dtype=torch.uint8, device="cuda")
        for name, small in (("latency_kernel", 1 << 30), ("throughput_kernel", 0)):
            c = mb.Codec(k, m, bs)
            c.set_option("small_blocks", small)
            S = c.shard_size()
            par = torch.zeros((nb * m * ((S + 15) // 16 * 16),), dtype=torch.uint8, device="cuda")
            dig = torch.zeros((nb * (k + m) * 32,), dtype=torch.uint8, device="cuda")
            run = lambda: c.encode_blocks_device(src.data_ptr(), nb * bs, par.data_ptr(), (S + 15) // 16 * 16, dig.data_ptr(), torch.cuda.current_stream().cuda_stream)
            for _ in range(5):
                run()
            torch.cuda.synchronize()
            ts = []
            for _ in range(20):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(torch.cuda.current_stream())
                run()
                e1.record(torch.cuda.current_stream())
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) * 1e3)
            row[name + "_us"] = round(float(np.median(ts)), 1)
            row[name + "_small_launches"] = c.stat("small_launches")
            if name == "latency_kernel":
                ref = dig.cpu().numpy().copy(), par.cpu().numpy().copy()
            else:
                row["identical"] = bool((ref[0] == dig.cpu().numpy()).all() and (ref[1] == par.cpu().numpy()).all())
        print(json.dumps(row), flush=True)
        out.append(row)


if __name__ == "__main__":
    main()
