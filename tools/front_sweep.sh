#!/bin/bash
# register/occupancy sweep of the two OFDM front-end kernels on the GPU box: rebuild with -DSB_FRONT_MINB / -DSB_FRONT11N_MINB
# (resident CTAs per SM that __launch_bounds__ asks for) and print the per-kernel times
cd "$(dirname "$0")/.."
F="-O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC"
for b in ${A_LIST:-4 5 6}; do
  touch sora_b200/csrc/sb200.cu; make -C sora_b200/csrc NVFLAGS="$F -DSB_FRONT_MINB=$b" >/dev/null 2>&1
  echo "11a MINB=$b"; python bench.py --steps 3 --warmup 2 2>/dev/null | python -c "import sys,json; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); print(d['value'], d['ms_per_step'], d.get('kernel_ms'))"
done
for b in ${N_LIST:-4 5 6}; do
  touch sora_b200/csrc/sb200.cu; make -C sora_b200/csrc NVFLAGS="$F -DSB_FRONT11N_MINB=$b" >/dev/null 2>&1
  echo "11n MINB=$b"; python bench_extra.py --config 11n --steps 3 2>/dev/null | python -c "
import sys,json
for l in sys.stdin.read().strip().splitlines():
    if l.startswith('{'): d=json.loads(l); print(d['mcs'], round(d['value']), d['kernel_ms']['ofdm_front_end'])"
done
