#!/bin/bash
# A/B of kernel variants built by tools/build_variant.sh: default bench line (device + e2e) per variant
cd "$(dirname "$0")/.."
for lib in build/variants/libdfm_*.so; do
  n=$(basename $lib .so)
  DFM_BENCH_LIB=$lib timeout 200 python bench.py --no-cpu --steps 5 --warmup 3 2>/dev/null | python -c "
import sys,json; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); print('$n', 'value', round(d['value']), 'ms', round(d['ms_per_step'],3), 'frac', round(d['roofline']['frac'],3), 'e2e', round(d['e2e']['value']), 'ok', d['config']['all_status_ok'])"
done
