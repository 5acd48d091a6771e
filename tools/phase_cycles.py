#!/usr/bin/env python3
"""Where the SM cycles of the headline encode go (RS(12,4) + HighwayHash256S, 10 240 x 1 MiB device-resident blocks).

--block-size picks another block size for the same encode: 1 048 704 bytes (12 x 87 392) makes every shard row 16-byte
aligned, which runs the aligned (direct-fetch) form of the kernel at the same work per byte as 1 MiB to within 0.02 %.

One run does three things:
  1. builds libminio_ec.so with -DMEC_PHASE_CYCLES=1 into <out>/phase_lib/ (skipped when it is newer than every source)
     and runs the headline shape through it: per launch, the share of warp cycles in the TMA wait, barrier (A), barrier (B),
     the GF step and the HH step (ec_kernel.cuh PhaseSlot), the SM clock the CTAs really ran at (clock64 over
     %globaltimer), and object bytes per SM clock;
  2. samples power.draw and clocks.sm with nvidia-smi --query-gpu (read-only) while it runs;
  3. builds and runs tools/ubench2.cu: the compute-only ceiling of the kernel's instruction mix per SM clock.
Results go to <out>/phase_cycles.json and a summary to stdout.

  python tools/phase_cycles.py [--out bench_out] [--launches 20] [--warmup 3] [--use-auto 0,2] [--block-size BYTES]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "minio_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
K, M = 12, 4
PHASES = ("tma_wait", "barrier_A", "barrier_B", "gf", "hh")  # PhaseSlot 0..4
SLOT_WARP, SLOT_CTA_CLK, SLOT_CTA_NS, HEADER, MAX_SM = 5, 6, 7, 8, 256


def newer_than_sources(path):
    if not os.path.exists(path):
        return False
    t = os.path.getmtime(path)
    return all(os.path.getmtime(os.path.join(CSRC, f)) < t for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h", ".cc")))


def build_lib(out):
    """The product library with the phase counters compiled in (same flags as minio_b200/csrc/Makefile otherwise)."""
    d = os.path.join(out, "phase_lib")
    so = os.path.join(d, "libminio_ec_phase.so")
    if newer_than_sources(so):
        return so
    os.makedirs(d, exist_ok=True)
    subprocess.check_call(["make", "-s", "-C", CSRC, "jit_headers.inc"])
    fl = ["-std=c++17", "-O3", *ARCH, "-lineinfo", "-Xcompiler", "-fPIC", "-DMEC_PHASE_CYCLES=1"]
    jobs = [[NVCC, *fl, "-c", os.path.join(CSRC, "ec_engine.cu"), "-o", os.path.join(d, "ec_engine.o")],
            [NVCC, *fl, "-c", os.path.join(CSRC, "ec_api.cu"), "-o", os.path.join(d, "ec_api.o")],
            [NVCC, *fl, "-x", "cu", "-c", os.path.join(CSRC, "rs_matrix.cc"), "-o", os.path.join(d, "rs_matrix.o")],
            [NVCC, *fl, "-x", "cu", "-c", os.path.join(CSRC, "ec_numa.cc"), "-o", os.path.join(d, "ec_numa.o")]]
    procs = [subprocess.Popen(j) for j in jobs]
    if any(p.wait() for p in procs):
        sys.exit("phase_cycles: building the instrumented library failed")
    subprocess.check_call([NVCC, *ARCH, "-shared", "-o", so] + [os.path.join(d, o) for o in ("ec_engine.o", "ec_api.o", "rs_matrix.o", "ec_numa.o")]
                          + ["-cudart", "static", "-ldl", "-lpthread"])
    return so


def build_ubench2(out):
    exe = os.path.join(out, "ubench2")
    if not (os.path.exists(exe) and os.path.getmtime(exe) > max(os.path.getmtime(os.path.join(ROOT, "tools", "ubench2.cu")),
                                                                 os.path.getmtime(os.path.join(CSRC, "ec_device.cuh")))):
        subprocess.check_call([NVCC, "-O3", "-std=c++17", *ARCH, "-I", CSRC, "-o", exe, os.path.join(ROOT, "tools", "ubench2.cu")])
    return exe


class SmiSampler:
    """power.draw and clocks.sm every 20 ms (nvidia-smi --query-gpu, read-only); stopped and reaped by stop()."""

    def __init__(self, index):
        self.rows, self.proc = [], None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(index), "--query-gpu=power.draw,clocks.sm,power.limit",
                                          "--format=csv,noheader,nounits", "-lms", "20"], stdout=subprocess.PIPE, text=True)
        except OSError:
            return
        self.t = threading.Thread(target=self._read, daemon=True)
        self.t.start()

    def _read(self):
        for line in self.proc.stdout:
            try:
                self.rows.append((time.monotonic(), [float(x) for x in line.split(",")]))
            except ValueError:
                pass

    def window(self, t0, t1):
        sel = [r for t, r in self.rows if t0 <= t <= t1]
        if not sel:
            return None
        return {"samples": len(sel), "power_W_median": statistics.median(r[0] for r in sel),
                "clocks_sm_MHz_median": statistics.median(r[1] for r in sel), "power_limit_W": sel[0][2]}

    def stop(self):
        if self.proc:
            self.proc.terminate()
            self.proc.wait()
            self.t.join(timeout=2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out"))
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=10240)
    ap.add_argument("--block-size", type=int, default=1 << 20, help="erasure block size in bytes")
    ap.add_argument("--use-auto", default="0", help="comma-separated values of the engine's use_auto option to measure")
    ap.add_argument("--no-ubench", action="store_true")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    so = build_lib(args.out)
    exe = None if args.no_ubench else build_ubench2(args.out)

    os.environ["MEC_LIB"] = so  # minio_b200.capi loads the library named here
    sys.path.insert(0, ROOT)
    import torch
    import minio_b200 as mb
    L = mb.lib()
    L.mec_phase_cycles.restype = C.c_int
    L.mec_phase_cycles.argtypes = [C.POINTER(C.c_ulonglong), C.c_int, C.c_int]
    dev = torch.device("cuda:0")
    props = torch.cuda.get_device_properties(0)
    nsm = props.multi_processor_count
    BS = args.block_size
    S = -(-BS // K)
    pitch = (S + 15) // 16 * 16
    nbytes = args.blocks * BS
    gen = torch.Generator(device=dev)
    gen.manual_seed(0x4D494E494F00 + 2)
    src = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    for o0 in range(0, nbytes, 1 << 30):
        n = min(1 << 30, nbytes - o0)
        src[o0:o0 + n] = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev, generator=gen)
    par = torch.empty((args.blocks * M, pitch), dtype=torch.uint8, device=dev)
    dig = torch.empty((args.blocks, K + M, 32), dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream()
    words = HEADER + 8 * MAX_SM
    buf = (C.c_ulonglong * words)()

    smi = SmiSampler(0)
    result = {"gpu": props.name, "sms": nsm, "block_size": BS, "blocks": args.blocks, "launches": args.launches, "runs": []}
    try:
        for ua in [int(x) for x in args.use_auto.split(",")]:
            codec = mb.Codec(K, M, BS, device=0)
            codec.set_option("use_auto", ua)
            for _ in range(args.warmup):
                codec.encode_blocks_device(src.data_ptr(), nbytes, par.data_ptr(), pitch, dig.data_ptr(), stream.cuda_stream)
            torch.cuda.synchronize()
            if L.mec_phase_cycles(buf, words, 1) < 0:
                sys.exit("phase_cycles: the library has no phase counters (was it built with -DMEC_PHASE_CYCLES=1?)")
            per = []
            t0 = time.monotonic()
            for _ in range(args.launches):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                codec.encode_blocks_device(src.data_ptr(), nbytes, par.data_ptr(), pitch, dig.data_ptr(), stream.cuda_stream)
                b.record(stream)
                L.mec_phase_cycles(buf, words, 1)  # synchronises, reads, clears
                ms = a.elapsed_time(b)
                v = list(buf)
                sm = [v[HEADER + 8 * i:HEADER + 8 * i + 8] for i in range(nsm)]
                tot = [sum(s[j] for s in sm) for j in range(8)]
                warp = tot[SLOT_WARP]
                mhz = 1e3 * tot[SLOT_CTA_CLK] / tot[SLOT_CTA_NS]
                span_ns = v[1] - v[0]
                per.append({"ms": ms, "GiB_s": nbytes / (1 << 30) / (ms / 1e3), "eff_MHz": mhz, "span_ms": span_ns / 1e6,
                            "B_per_clk_SM": nbytes / (span_ns * 1e-3 * mhz) / nsm,
                            "share": {p: tot[i] / warp for i, p in enumerate(PHASES)} | {"other": 1 - sum(tot[:5]) / warp},
                            # CTAs resident on average over the launch: below the grid size, the difference is the tail
                            "mean_ctas": tot[SLOT_CTA_NS] / span_ns})
            t1 = time.monotonic()
            codec.close()
            med = lambda key: statistics.median(r[key] for r in per)
            run = {"use_auto": ua, "GiB_s_median": med("GiB_s"), "GiB_s_min": min(r["GiB_s"] for r in per), "GiB_s_max": max(r["GiB_s"] for r in per),
                   "eff_MHz_median": med("eff_MHz"), "B_per_clk_SM_median": med("B_per_clk_SM"),
                   "share_median": {p: statistics.median(r["share"][p] for r in per) for p in (*PHASES, "other")},
                   "mean_resident_ctas": med("mean_ctas"), "smi": smi.window(t0, t1), "per_launch": per}
            result["runs"].append(run)
            sh = " ".join(f"{p}={100 * v:.1f}%" for p, v in run["share_median"].items())
            print(f"block_size={BS} use_auto={ua}: {run['GiB_s_median']:.1f} GiB/s (instrumented; {run['GiB_s_min']:.1f}-{run['GiB_s_max']:.1f}), "
                  f"effective SM clock {run['eff_MHz_median']:.0f} MHz, {run['B_per_clk_SM_median']:.2f} object B/clk/SM, "
                  f"{run['mean_resident_ctas']:.0f} CTAs resident on average; "
                  f"warp cycles: {sh}; nvidia-smi {run['smi']}", flush=True)
    finally:
        smi.stop()

    if exe:
        txt = subprocess.run([exe], capture_output=True, text=True, timeout=300).stdout
        result["ubench2"] = txt
        print(txt, end="")
    with open(os.path.join(args.out, "phase_cycles.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
