# final single-GPU call: GPU suite, full bench, ncu --set full of the level-0 kernels (CSV only)
D=gpurun_out/${1:-final}; mkdir -p $D
( timeout 900 python -m pytest tests -m gpu -q -s > $D/pytest_gpu.log 2>&1; echo "pytest exit $?" >> $D/pytest_gpu.log )
grep -E "passed|failed|error|exit|FAILED|Error|cfg3" $D/pytest_gpu.log | tail -8
timeout 600 python bench.py > $D/bench.json 2> $D/bench.err; echo "bench exit $?"
python tools/show_bench.py $D/bench.json 2>/dev/null | head -20
timeout 500 ncu --set full --clock-control none --import-source on -k 'regex:temporal_fused_kernel|tc_conv3_kernel|gn_apply_kernel' -c 7 -f -o $D/full python tools/profile_step.py 1 > $D/full.out 2>&1
ncu -i $D/full.ncu-rep --page raw --csv > $D/full_raw.csv 2>/dev/null; rm -f $D/full.ncu-rep
tail -1 $D/full.out; du -sh $D
