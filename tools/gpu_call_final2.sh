# final single-GPU evidence call: full bench (device-resident + e2e + cpu baseline + clip line), ncu launch list of one step, ncu --set full
# of the level-0 kernels (CSV only).  The GPU suite runs in the other calls of the same HEAD.
D=gpurun_out/${1:-final2}; mkdir -p $D
timeout 600 python bench.py > $D/bench.json 2> $D/bench.err; echo "bench exit $?"
python tools/show_bench.py $D/bench.json 2>/dev/null | head -20
timeout 400 ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none --csv --log-file $D/launches.csv python tools/profile_step.py 2 > $D/launches.out 2>&1
tail -1 $D/launches.out
timeout 500 ncu --set full --clock-control none --import-source on -k 'regex:temporal_fused_kernel|tc_conv3_kernel|gn_apply_kernel|tc_gemm_kernel' -s 20 -c 9 -f -o $D/full python tools/profile_step.py 1 > $D/full.out 2>&1
ncu -i $D/full.ncu-rep --page raw --csv > $D/full_raw.csv 2>/dev/null; rm -f $D/full.ncu-rep
gzip -f $D/launches.csv; tail -1 $D/full.out; du -sh $D
