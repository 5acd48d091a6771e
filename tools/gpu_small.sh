#!/bin/bash
# latency-form sweep (one block, one block per SM and a few per SM) and the GPU tests; results go to $OUT (default bench_out/)
cd "$(dirname "$0")/.."
O=${OUT:-bench_out}
mkdir -p "$O"
python tools/bench_small.py 12 4 2>&1 | grep -E "\"blocks\": (1|132|528|792)," | tee "$O/small_12_4_b.jsonl"
python tools/bench_small.py 16 4 2>&1 | grep -E "\"blocks\": (1|132|528)," | tee "$O/small_16_4_b.jsonl"
timeout 1500 python -m pytest tests -q -m gpu --timeout 900 -x > "$O/pytest_gpu.txt" 2>&1; echo "rc=$?"; tail -3 "$O/pytest_gpu.txt"
