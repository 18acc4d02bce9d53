#!/bin/bash
# One `ncu --set full` row per KERNEL CLASS of the training step (VERDICT r1 item 4), exported to CSV on the box -- the
# .ncu-rep files stay there (gpurun returns at most 64 MiB).  Usage (one GPU, ~8 min):
#     gpurun --timeout 1500 -- 'bash tools/run_ncu_classes.sh r02c'
# then here:  python tools/ncu_summary.py --csv gpurun_out/ncu_<tag>_*.csv <tag>
# Each class: skip the first S matching launches (warm-up steps), capture C.  The command under ncu is one eager step of
# the default workload (posenet_bs64) after 3 warm-up steps; its printed numbers are NOT bench values.
TAG=${1:-r02}
mkdir -p gpurun_out
T0=$(date +%s)
CMD="python bench.py --steps 1 --warmup 3 --no-graph --no-cpu-baseline --no-modes"
run() {   # name regex skip count [extra bench args]
  local name=$1 re=$2 skip=$3 cnt=$4; shift 4
  if [ -n "$ONLY" ] && ! echo " $ONLY " | grep -q " $name "; then return; fi
  timeout 170 ncu --set full --clock-control none --import-source on -k regex:"$re" -s $skip -c $cnt -f -o /tmp/ncu_$name \
      $CMD "$@" > gpurun_out/ncu_${TAG}_$name.log 2>&1
  local rc=$?
  ncu -i /tmp/ncu_$name.ncu-rep --page raw --csv > gpurun_out/ncu_${TAG}_$name.csv 2>/dev/null
  echo "[t+$(( $(date +%s) - T0 ))s] $name rc=$rc rows=$(( $(wc -l < gpurun_out/ncu_${TAG}_$name.csv) - 2 ))"
}
# ---- conv engines, bf16 mode (what the bench line runs): the 4th step (3 warm-up steps precede it) ----
# (ncu matches the regex against the function's base name: no return type, namespace or template arguments)
# per step: k_tc_conv 38 launches (13 forward: stem + layer1 two-CTA-per-SM <64,1,2>, layer4 <256,1,1>; then the dgrads),
# k_tc_conv2 30, k_tc_wgrad 7, k_tc_wgrad2 29, k_bn_apply 32, k_bn_bwd_apply 33
run conv1cta      '^k_tc_conv$'   114 10
run conv1cta_bwd  '^k_tc_conv$'   127 6
run conv1cta_l1bw '^k_tc_conv$'   145 5
run conv2cta      '^k_tc_conv2$'  90 5
run conv2cta_bwd  '^k_tc_conv2$'  112 4
run wgrad1        '^k_tc_wgrad$'  21 3
run wgrad2        '^k_tc_wgrad2$' 87 6
# ---- element-wise / reduction / small kernels ----
run bnapply    'k_bn_apply'          100 3
run bnbwdapply 'k_bn_bwd_apply'      100 3
run bnbwdapply_l1 'k_bn_bwd_apply'   126 2
run stempool   '^k_stem_pool$'       3 1
run stempoolb  'k_stem_pool_bwd'     3 1
run pack       'k_pack_weights'      3 1
run transpose  'k_transpose_dg'      3 1
run gap        'k_gap'               6 2
run adam       'k_adam'              9 1
# ---- strict tensor-core mode: the same engines on split operand planes, plus its un-fused BN-backward reduction ----
run split_conv1cta '^k_tc_conv$'  60 3 --precision tc_split
run split_conv2cta '^k_tc_conv2$' 90 3 --precision tc_split
run split_wgrad2   '^k_tc_wgrad2$' 80 3 --precision tc_split
run split_sums     'k_channel_sums'  60 2 --precision tc_split
# plain launch list (durations only) of one eager step, for the per-kernel shares
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 900 --csv --log-file gpurun_out/launches_${TAG}.csv \
    python bench.py --steps 2 --warmup 1 --no-modes --no-cpu-baseline --no-graph > gpurun_out/ncu_${TAG}_launches.log 2>&1
echo "[t+$(( $(date +%s) - T0 ))s] launch list rc=$?"
# source-level stall samples of two conv launches (tools/ncu_stalls.py)
ncu -i /tmp/ncu_conv2cta.ncu-rep --page source --csv > gpurun_out/ncu_${TAG}_conv2cta_source.csv 2>/dev/null
ncu -i /tmp/ncu_conv1cta_l1bw.ncu-rep --page source --csv > gpurun_out/ncu_${TAG}_conv1cta_l1bw_source.csv 2>/dev/null
python - <<'PY'
import os, sys
sys.path.insert(0, os.getcwd())
from geomapnet_b200 import build
open("gpurun_out/ncu_sources_digest.txt", "w").write(build._digest()[:16])
PY
ls -la gpurun_out/ncu_${TAG}_*.csv | awk '{print $5, $9}'; du -sh gpurun_out
echo "[t+$(( $(date +%s) - T0 ))s] done"
