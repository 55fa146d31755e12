#!/bin/bash
# end-of-round measurement set on one GPU: tests, smoke, both bench arms, B = 32, train step, ncu launch lists
mkdir -p gpurun_out
timeout 900 python -m pytest tests -q -m gpu --no-header 2>&1 | tail -15 > gpurun_out/fin_gputests.log
python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/fin_smoke.log 2>&1
timeout 400 python bench.py --dump-launches gpurun_out/fin_launches_strict.json > gpurun_out/fin_bench.json 2> gpurun_out/fin_bench.err
timeout 300 python bench.py --no-cpu-baseline --steps 20 --precision fast --dump-launches gpurun_out/fin_launches_fast.json > gpurun_out/fin_bench_fast.json 2> gpurun_out/fin_bench_fast.err
timeout 300 python bench.py --no-cpu-baseline --batch 32 --steps 10 > gpurun_out/fin_bench_b32.json 2> gpurun_out/fin_bench_b32.err
timeout 400 python bench.py --train --steps 10 --warmup 3 > gpurun_out/fin_train.json 2> gpurun_out/fin_train.err
timeout 300 python bench.py --impl reference --steps 2 --warmup 1 > gpurun_out/fin_ref.json 2> gpurun_out/fin_ref.err
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv --log-file gpurun_out/fin_infer_launches_strict.csv python tools/profile_infer_step.py > gpurun_out/fin_prof_strict.log 2>&1
MF_PRECISION=fast timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv --log-file gpurun_out/fin_infer_launches_fast.csv python tools/profile_infer_step.py > gpurun_out/fin_prof_fast.log 2>&1
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv --log-file gpurun_out/fin_train_launches.csv python tools/profile_train_step.py > gpurun_out/fin_train_prof.log 2>&1
