#!/bin/bash
# sweep the k_eval_obs tuning knobs (256-observation tiles per CTA, CTAs per SM) on the bench workload
for cfg in "8 2 8" "4 2 8" "16 2 8" "8 3 8" "8 2 4" "8 2 16"; do
  set -- $cfg
  out=$(KBA_EVAL_TILES_JAC=$1 KBA_EVAL_MIN_BLOCKS=$2 KBA_EVAL_TILES_COST=$3 python bench.py --steps 2 --warmup 3 --batch 132 --cpu-sample 0 2>&1 | tail -1)
  echo "jac_tiles=$1 min_blocks=$2 cost_tiles=$3 :: $(echo "$out" | python -c "import json,sys; d=json.loads(sys.stdin.read()); print('value %.1f  jac_ms %.4f  frac %.3f' % (d['value'], d['roofline']['launch_ms_mean'], d['roofline']['frac']))")"
done
