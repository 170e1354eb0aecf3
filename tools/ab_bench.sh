#!/bin/bash
# A/B two builds of libcrabml_cuda.so in ONE session on one GPU (shared machines differ between sessions: never compare across sessions).
#   usage:  tools/ab_bench.sh crabml_b200/lib/libcrabml_cuda_A.so crabml_b200/lib/libcrabml_cuda.so [workload] [rounds]
# Build A from another commit here first:  git stash; python crabml_b200/build.py; cp crabml_b200/lib/libcrabml_cuda.so \
#   crabml_b200/lib/libcrabml_cuda_A.so; git stash pop; python crabml_b200/build.py     (*.so stays out of git)
# Prints value / e2e tok/s per run, alternating A B A B, then the in-kernel phase profile of each (stable to ~1 %).
A=$1; B=$2; WL=${3:-llama2-7b-q8_0}; N=${4:-2}
for i in $(seq $N); do
  for v in A B; do
    if [ $v = A ]; then lib=$A; else lib=$B; fi
    echo -n "$v "
    CRABML_CUDA_LIB=$PWD/$lib timeout 200 python bench.py --steps 64 --warmup 8 --no-cpu-baseline --workload $WL 2>/dev/null | tail -1 |
      python -c "import json,sys; d=json.loads(sys.stdin.read()); print(round(d['value'],1), round(d['e2e']['value'],1), d['gpu_launches'])"
  done
done
for v in A B; do
  if [ $v = A ]; then lib=$A; else lib=$B; fi
  echo "== $v: phase profile"
  CRABML_CUDA_LIB=$PWD/$lib timeout 120 python tools/mega_profile.py Q8_0 2>/dev/null | tail -11 | head -8
done
