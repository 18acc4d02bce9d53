#!/bin/bash
# Round-end evidence on one GPU: ncu rows per kernel class + launch list (tools/run_ncu_classes.sh), then the bench
# lines the profiles/ directory quotes.  Outputs -> gpurun_out/
TAG=${1:-r02c}
mkdir -p gpurun_out
bash tools/run_ncu_classes.sh $TAG
b() { # name, args...
  name=$1; shift
  timeout 400 python bench.py "$@" > gpurun_out/${TAG}_bench_$name.json 2> gpurun_out/${TAG}_bench_$name.err; rc=$?
  echo "bench $name rc=$rc"; tail -c 400 gpurun_out/${TAG}_bench_$name.json | head -c 400; echo
}
b posenet_bs64 --steps 30 --warmup 5
b mapnet_n32t3 --workload mapnet_n32t3 --steps 30 --warmup 5 --no-modes --no-cpu-baseline
b mapnetpp_n16t10 --workload mapnetpp_n16t10 --steps 30 --warmup 5 --no-modes --no-cpu-baseline
b posenet_bs64_tc_split --precision tc_split --steps 20 --warmup 5 --no-modes --no-cpu-baseline
b posenet_bs64_fp32 --precision fp32 --steps 8 --warmup 3 --no-modes --no-cpu-baseline
b reference --impl reference --steps 3 --warmup 1
timeout 200 python tools/bench_preprocess.py gpurun_out/${TAG}_preprocess_bench.json
timeout 300 python tools/bench_conv.py 64 > gpurun_out/${TAG}_conv_microbench.txt 2>&1; tail -7 gpurun_out/${TAG}_conv_microbench.txt
