#!/bin/bash
mkdir -p gpurun_out
timeout 900 compute-sanitizer --tool memcheck python -m pytest tests/test_gpu_ffat.py -m gpu -q -x -k "golden or small" > gpurun_out/san.log 2>&1; echo "sanitizer rc=$?"; tail -3 gpurun_out/san.log
timeout 900 python -m pytest tests -m gpu -q -x > gpurun_out/pytest.log 2>&1; echo "pytest rc=$?"; tail -3 gpurun_out/pytest.log
run() { tag=$1; shift
  env "$@" timeout 300 python bench.py --steps 20 --warmup 3 --cpu-seconds 0.2 --e2e-steps 2 > gpurun_out/exp_$tag.json 2>gpurun_out/exp_$tag.err
  python -c "
import json; d=json.load(open('gpurun_out/exp_$tag.json')); p=d['roofline']['phase_ms_per_step']; print('$tag', round(d['value']/1e9,2),'GT/s ms/step', round(d['ms_per_step'],3), {k:round(v,3) for k,v in p.items()}, d['gpu_launches'])" || tail -5 gpurun_out/exp_$tag.err
}
run buckets
run buckets_move WFB_BUCKET_MOVE=1
WFB_LIB=$PWD/windflow_b200/variants/lib_trace.so timeout 300 python tools/bk_trace.py
