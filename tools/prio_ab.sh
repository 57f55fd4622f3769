#!/bin/bash
# A/B of the prover's stream layout with the stage timeline of one proof.  CS_PRIO="side,acc,wm" = CUDA priorities of the
# MSM streams (sort / fold / reduce), of the accumulation streams and of the witness-map -> H stream; CS_MSM_SPLIT=0 keeps
# each MSM on one stream.  usage: bash tools/prio_ab.sh > prio_ab.log
run() {
  echo "== $*"
  env "$@" timeout 300 python bench.py --steps 10 --warmup 3 --no-rep3 --no-cpu-baseline --timeline 2>&1 \
    | python -c "
import sys, json
for line in sys.stdin:
    if line.startswith('timeline '): print(line.strip())
    elif line.startswith('{'):
        d = json.loads(line); print('ms_per_step', round(d['ms_per_step'], 3), 'e2e_ms', round(d['e2e']['ms_per_step'], 3), 'msm_stage', {k: round(v, 3) for k, v in d['msm']['stage_ms'].items()})
"
}
run CS_DEFAULT=1
run CS_MSM_SPLIT=0 CS_PRIO=0,0,0
run CS_MSM_SPLIT=0 CS_PRIO=0,0,-3
run CS_PRIO=-1,0,-2
run CS_PRIO=-2,0,-1
run CS_PRIO=-1,0,-1
