#!/bin/bash
# round-2 final evidence on ONE GPU: GPU tests, smoke, bench lines (all workloads, both directions, reference arm), launch list of the
# bench command, full captures of the kernels of the step.  Everything lands in gpurun_out/ with the tag given as $1.
T=${1:-r02final}
mkdir -p gpurun_out
timeout 1500 python -m pytest tests -m gpu -q --no-header -p no:logging --tb=short -rf 2>&1 | grep -v "^DEBUG" | tail -30 > gpurun_out/${T}_pytest_gpu.log
timeout 300 python __graft_entry__.py smoke > gpurun_out/${T}_smoke.log 2>&1; echo "smoke exit: $?" >> gpurun_out/${T}_smoke.log
timeout 600 python bench.py --steps 20 --warmup 5 > gpurun_out/${T}_bench.json 2> gpurun_out/${T}_bench.err; echo "bench exit: $?" >> gpurun_out/${T}_bench.err
timeout 300 python bench.py --impl reference --steps 3 --warmup 1 > gpurun_out/${T}_bench_reference.json 2>> gpurun_out/${T}_bench.err
timeout 400 python bench.py --workload cfg3_baseline --no-cpu-baseline > gpurun_out/${T}_bench_cfg3_baseline.json 2>> gpurun_out/${T}_bench.err
for w in cfg4_pon cfg2_static_lss; do timeout 300 python bench.py --workload $w --no-cpu-baseline --no-extras > gpurun_out/${T}_bench_$w.json 2>> gpurun_out/${T}_bench.err; done
timeout 300 python bench.py --layout channels_last --no-cpu-baseline --no-extras > gpurun_out/${T}_bench_channels_last.json 2>> gpurun_out/${T}_bench.err
timeout 300 python bench.py --direction fwd_bwd --workload cfg3_baseline --head-dtype f16 > gpurun_out/${T}_bench_train_cfg3_f16.json 2>> gpurun_out/${T}_bench.err
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 300 --csv --log-file gpurun_out/${T}_launches.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-extras > gpurun_out/${T}_ncu_bench.log 2>&1
W=cfg2_static_lss_b8
cap() { timeout 300 ncu --set full --clock-control none --import-source on -k regex:$1 -s $2 -c 1 -f -o gpurun_out/${T}_prof_$3 python tools/ncu_target.py $W $4 >> gpurun_out/${T}_ncu_full.log 2>&1; }
cap lift_forward_cols_kernel 2 fwd_intile tile
cap lift_forward_cols_kernel 2 fwd_planned tile_planned
cap finalize_tma 8 finalize step
cap lift_backward_kernel 1 bwd bwd
cap lift_plan_kernel 1 plan bwd
cap bev_conv7x7s2 2 conv conv
cap depth_layer_kernel 2 depth_layer depth
W=cfg3_baseline
cap finalize_warp_kernel 4 finalize_warp step_warped
cap warp_backward_gather_kernel 1 warp_backward warp_bwd
timeout 200 compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize_target.py > gpurun_out/${T}_memcheck.log 2>&1; echo "memcheck exit: $?" >> gpurun_out/${T}_memcheck.log
tail -4 gpurun_out/${T}_pytest_gpu.log; tail -2 gpurun_out/${T}_memcheck.log; tail -2 gpurun_out/${T}_smoke.log; tail -3 gpurun_out/${T}_bench.err; ls gpurun_out | grep -c ${T}
