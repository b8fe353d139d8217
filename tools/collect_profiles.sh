#!/bin/bash
# Runs on the GPU box (under gpurun): ncu launch list of the bench command + one --set full capture per solver
# kernel at the bench's batch size.  Outputs land in gpurun_out/; tools/summarise_profiles.py turns them
# into the tracked files under profiles/.
set -u
R=${1:-r01}
B=${2:-528}
mkdir -p gpurun_out
ncu --metrics gpu__time_duration.sum --clock-control none -c 700 --csv --log-file gpurun_out/${R}_launches_bench.csv \
    python bench.py --steps 2 --warmup 3 --skip-cpu > gpurun_out/${R}_bench_under_ncu.log 2>&1
for k in k_landmarks k_schur k_solve k_imu k_quality; do
  skip=6; [ $k = k_quality ] && skip=1
  ncu --set full --clock-control none --import-source on -k regex:"^$k" -s $skip -c 1 -f -o gpurun_out/${R}_$k \
      python tools/prof_small.py $B 4 > /dev/null 2>&1
  ncu -i gpurun_out/${R}_$k.ncu-rep --page details --csv > gpurun_out/${R}_${k}_details.csv 2>/dev/null
  ncu -i gpurun_out/${R}_$k.ncu-rep --page raw --csv --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum,smsp__inst_executed.sum,sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active,sm__warps_active.avg.pct_of_peak_sustained_active > gpurun_out/${R}_${k}_raw.csv 2>/dev/null
  rm -f gpurun_out/${R}_$k.ncu-rep
done
# frontend kernels (cfg-3 shape and OKVIS' production parameters) and the marginalisation kernel: launch list + one full capture each
ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/${R}_launches_frontend.csv \
    python tools/prof_frontend.py > /dev/null 2>&1
for k in k_uniformity k_hamming_topk k_harris k_describe; do
  ncu --set full --clock-control none --import-source on -k regex:"$k" -s 1 -c 1 -f -o gpurun_out/${R}_$k python tools/prof_frontend.py > /dev/null 2>&1
  ncu -i gpurun_out/${R}_$k.ncu-rep --page details --csv > gpurun_out/${R}_${k}_details.csv 2>/dev/null
  rm -f gpurun_out/${R}_$k.ncu-rep
done
ncu --set full --clock-control none --import-source on -k regex:"k_marginalize" -c 1 -f -o gpurun_out/${R}_k_marginalize python tools/sanitize_run.py > /dev/null 2>&1
ncu -i gpurun_out/${R}_k_marginalize.ncu-rep --page details --csv > gpurun_out/${R}_k_marginalize_details.csv 2>/dev/null
rm -f gpurun_out/${R}_k_marginalize.ncu-rep
# compute-sanitizer over every product kernel (tools/sanitize_run.py)
compute-sanitizer --tool memcheck --print-limit 20 python tools/sanitize_run.py > gpurun_out/${R}_sanitizer_memcheck.txt 2>&1
compute-sanitizer --tool racecheck --print-limit 20 python tools/sanitize_run.py > gpurun_out/${R}_sanitizer_racecheck.txt 2>&1
compute-sanitizer --tool synccheck --print-limit 20 python tools/sanitize_run.py > gpurun_out/${R}_sanitizer_synccheck.txt 2>&1
tail -3 gpurun_out/${R}_sanitizer_*.txt
ls -la gpurun_out | tail -30
