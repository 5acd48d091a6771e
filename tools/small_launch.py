#!/usr/bin/env python
"""A handful of latency-kernel launches (RS(12,4) encode of N 1 MiB blocks, device-resident) — the target of the ncu capture in tools/gpu_prof_small.sh."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import minio_b200 as mb
nb = int(sys.argv[1]) if len(sys.argv) > 1 else 132
k, m, bs = 12, 4, 1 << 20
c = mb.Codec(k, m, bs)
S = c.shard_size(); pitch = (S + 15) // 16 * 16
src = torch.randint(0, 256, (nb * bs,), dtype=torch.uint8, device="cuda")
par = torch.zeros((nb * m * pitch,), dtype=torch.uint8, device="cuda")
dig = torch.zeros((nb * (k + m) * 32,), dtype=torch.uint8, device="cuda")
for _ in range(6):
    c.encode_blocks_device(src.data_ptr(), nb * bs, par.data_ptr(), pitch, dig.data_ptr(), torch.cuda.current_stream().cuda_stream)
torch.cuda.synchronize()
print("small launches:", c.stat("small_launches"))
