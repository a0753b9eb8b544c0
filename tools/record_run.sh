#!/bin/bash
# Record run (on the GPU box, from the repo root): both bench arms, the ncu launch list and one ncu --set full capture of the BA kernels.
# Outputs land in gpurun_out/; summarise with tools/ncu_summary.py and copy what is to be judged into profiles/.
mkdir -p gpurun_out
timeout 300 python bench.py --impl reference --steps 5 --warmup 1 2> gpurun_out/rec_ref.err | grep '^{' > gpurun_out/rec_ref.json
timeout 400 python bench.py --steps 20 --warmup 3 2> gpurun_out/rec_ours.err | grep '^{' > gpurun_out/rec_ours.json
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 700 --csv --log-file gpurun_out/launches.csv \
    python bench.py --steps 2 --warmup 3 --no-cpu-baseline > gpurun_out/ncu_launch.log 2>&1
timeout 400 ncu --set full --clock-control none --import-source on -k regex:"k_syrk|k_jac_slab|k_residual_stream|k_ldlt_all|k_ldlt_solve" -c 6 \
    -f -o gpurun_out/prof_r1_ba python bench.py --steps 1 --warmup 3 --no-cpu-baseline > gpurun_out/ncu_full.log 2>&1
ls -la gpurun_out | tail -12
python -c "
import json
for f in ('rec_ref','rec_ours'):
    d=json.load(open('gpurun_out/%s.json'%f)); print(f, d['value'], d.get('e2e',{}).get('value'), d.get('ms_per_step'))"
