# ncu --set full of the first level-0 launches of a step (temporal attention, the two 3x3 convs of the first ResBlock, gn_apply), CSV only
D=gpurun_out/${1:-ncufull}; mkdir -p $D
timeout 500 ncu --set full --clock-control none --import-source on -k 'regex:temporal_fused_kernel|tc_conv3_kernel|gn_apply_kernel' -c 7 -f -o $D/full python tools/profile_step.py 1 > $D/full.out 2>&1
ncu -i $D/full.ncu-rep --page raw --csv > $D/full_raw.csv 2>/dev/null; rm -f $D/full.ncu-rep
tail -1 $D/full.out; du -sh $D
