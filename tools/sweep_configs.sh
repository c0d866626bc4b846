#!/bin/bash
# SURVEY.md §8(d): K sweep of config 2 and a config-4-sized batch (one deneb block's signature set: ~215 tuples, K=512).
# Usage (on the GPU box): bash tools/sweep_configs.sh > sweep.jsonl
for cfg in "4096 1" "4096 64" "4096 128" "4096 512" "1024 2048" "215 512"; do
  set -- $cfg
  python bench.py --tuples $1 --keys $2 --steps 3 --warmup 3 --skip-ssz 2>/dev/null
done
