#!/bin/bash
# Coalesced vs pooled GETs and heals of half-healed legacy parts (tools/conc_bench modes bget_mixed / get_mixed and bheal_mixed /
# heal_mixed) at RS(12,4): drives 0-7 healed into HighwayHash256S, drives 8-15 raw shard files of ALGO; heals rebuild drive 8.
# Batched and pool modes alternate inside each shape, RUNS runs each; one JSON line per run on stdout.
# Usage: tools/gpu_conc_mixed.sh [RUNS] [THREADS...]
set -u
cd "$(dirname "$0")/.."
g++ -O2 -std=c++17 tools/conc_bench.cc -o tools/conc_bench -Iinclude -Lminio_b200 -lminio_ec -Loracle -loracle -lpthread || exit 1
export LD_LIBRARY_PATH=$PWD/minio_b200:$PWD/oracle:${LD_LIBRARY_PATH:-}
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader
runs=${1:-3}; shift || true
threads=${*:-64 256}
for algo in 1 2; do
  for size in 256k 1; do
    for t in $threads; do
      for op in get heal; do
        for r in $(seq "$runs"); do
          for mode in b${op}_mixed ${op}_mixed; do
            ALGO=$algo HEALED=8 timeout 300 ./tools/conc_bench "$mode" "$t" "$size" 8 8 0 || echo "{\"mode\": \"$mode\", \"failed\": $?}"
          done
        done
      done
    done
  done
done
