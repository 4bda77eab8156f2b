#!/bin/bash
# Evidence for profiles/: launch list of the default bench command, one full capture of the ingest kernel
# (warm caches), one of the GNN layer, SASS proof of the TMA / cp.async / wgmma instructions.
set -u
mkdir -p gpurun_out
echo "== launch list"
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file gpurun_out/r2_launches.csv \
  python bench.py --steps 2 --warmup 3 --no-cpu --no-e2e > gpurun_out/launches_bench.log 2>&1
tail -1 gpurun_out/launches_bench.log | cut -c1-160
echo "== ingest full capture"
timeout 900 ncu --set full --cache-control none --clock-control none --import-source on -k regex:ingest_pairs_v -s 4 -c 1 -o gpurun_out/prof_r2_final_ingest -f \
  python bench.py --steps 2 --warmup 3 --no-cpu --no-e2e --no-gnn --no-verify > gpurun_out/ncu_final_ingest.log 2>&1
tail -1 gpurun_out/ncu_final_ingest.log | cut -c1-160
echo "== gnn full capture"
timeout 900 ncu --set full --cache-control none --clock-control none --import-source on -k regex:sage_layer -c 2 -o gpurun_out/prof_r2_final_gnn -f \
  python bench.py --steps 1 --warmup 1 --no-cpu --no-e2e --no-verify > gpurun_out/ncu_final_gnn.log 2>&1
tail -1 gpurun_out/ncu_final_gnn.log | cut -c1-160
echo "== default bench"
timeout 900 python bench.py 2>&1 | tail -1 > gpurun_out/bench_default_r2.json; cut -c1-400 gpurun_out/bench_default_r2.json
echo "== reference arm"
timeout 900 python bench.py --impl reference --steps 3 --warmup 1 2>&1 | tail -1 > gpurun_out/bench_reference_r2.json; cut -c1-400 gpurun_out/bench_reference_r2.json
