#!/bin/bash
# A/B of alternate builds on the GPU box: every ethereum_consensus_b200/libb200_consensus*.so gets one strict-mode bench
# run (T=4096, K=512, per-phase trace) and its GPU parity tests.  Build the variants beforehand (no GPU needed), e.g.
#   python -m ethereum_consensus_b200.build --suffix=_o1 --ptxas-opt=bls_g1.cu:1,bls_vm.cu:1
#   python -m ethereum_consensus_b200.build --suffix=_o1g1 --ptxas-opt=bls_g1.cu:1
# then, on the GPU machine:  bash tools/ab_libs.sh > ab.txt 2>&1
for lib in ethereum_consensus_b200/libb200_consensus*.so; do
  echo "== $lib"
  B200_LIB=$PWD/$lib B200_BLS_TRACE=1 python bench.py --steps 3 --warmup 3 --skip-ssz 2> /tmp/ab.err \
    | python -c "import sys,json; d=json.loads(sys.stdin.read()); print('tuples/s', round(d['value']), 'ms/step', round(d['ms_per_step'],2), 'registry', round(d['registry_mode']['tuples_per_s']))"
  grep "b200 bls" /tmp/ab.err | sed -n "5,5p"
  B200_LIB=$PWD/$lib python -m pytest tests/test_bls_gpu.py -x -q 2>&1 | tail -1
done
