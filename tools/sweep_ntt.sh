#!/bin/bash
# sweeps the NTT tuning hooks; one JSON line per variant on stdout.  usage: bash tools/sweep_ntt.sh > ntt_sweep.jsonl
for tws in 0 1; do
  for thr in 512 256 128; do
    for minb in 1; do
      if [ $minb = 3 ] && [ $thr != 512 ]; then continue; fi
      echo "tws=$tws thr=$thr minb=$minb"
      CS_NTT_TWS=$tws CS_NTT_THREADS=$thr CS_NTT_MINB=$minb timeout 300 python tools/time_ntt.py 2>&1
    done
  done
done
