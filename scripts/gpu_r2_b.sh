#!/bin/bash
# round 2, run B: all GPU tests; staggered / lock-step x wait / hand-over with pre-generated episodes
mkdir -p gpurun_out
python -m pytest tests -m gpu -q 2>&1 | tail -40 > gpurun_out/r2b_pytest.txt
cat gpurun_out/r2b_pytest.txt
B="--no-extras --no-cpu-baseline --e2e-steps 10"
rm -f gpurun_out/r2b_ab.txt
run() { name=$1; shift; echo "== $name: $*" | tee -a gpurun_out/r2b_ab.txt; timeout 300 env "$@" 2>&1 | tail -1 | python -c "
import sys,json
l=sys.stdin.read().strip()
try:
    d=json.loads(l); print(round(d['ms_per_step']*1e3,3),'us/step frac',round(d['roofline']['frac'],4),'blocks',d['timing']['blocks'],'step min/max',round(d['timing']['step_ms_min']*1e3,3),round(d['timing']['step_ms_max']*1e3,3))
except Exception as e: print('FAILED', l[-600:])
" | tee -a gpurun_out/r2b_ab.txt; }
run stag_wait python bench.py --steps 20 --warmup 5 $B
run lock_wait python bench.py --steps 20 --warmup 5 --lockstep $B
run stag_ho QS_PDL=3 python bench.py --steps 20 --warmup 5 $B
run lock_ho QS_PDL=3 python bench.py --steps 20 --warmup 5 --lockstep $B
run stag_nopregen QS_PREGEN=0 python bench.py --steps 20 --warmup 5 $B
run stag_pregen64 QS_PREGEN=64 python bench.py --steps 20 --warmup 5 $B
run stag_long python bench.py --steps 20000 --warmup 64 $B
run c2_stag python bench.py --config c2 --steps 20 --warmup 5 $B
run c2_lock python bench.py --config c2 --steps 20 --warmup 5 --lockstep $B
run c4_stag python bench.py --config c4 --steps 20 --warmup 5 $B
run c4_lock python bench.py --config c4 --steps 20 --warmup 5 --lockstep $B
run c5_stag python bench.py --config c5 --steps 20 --warmup 5 $B
run c5_lock python bench.py --config c5 --steps 20 --warmup 5 --lockstep $B
