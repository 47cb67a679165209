#!/bin/bash
mkdir -p gpurun_out
timeout 1800 python -m pytest tests -m gpu -q 2>&1 | cut -c1-300 > gpurun_out/final_pytest.txt
tail -6 gpurun_out/final_pytest.txt
timeout 900 python bench.py 2>gpurun_out/final_bench.err > gpurun_out/final_bench.json
python - <<'PY'
import json
d=json.loads(open('gpurun_out/final_bench.json').read().strip().splitlines()[-1])
for k in ('value','ms_per_step','iterations_per_step','phase_ms_per_iteration','host_syncs_per_iteration','gpu_launches','clocks','e2e','roofline','roofline_assembly','roofline_jacobian_fill','config5','cpu_baseline'): print(k, str(d.get(k))[:900])
PY
tail -3 gpurun_out/final_bench.err
timeout 120 python scripts/spine_stamps.py 1270 > gpurun_out/spine_stamps.txt; tail -3 gpurun_out/spine_stamps.txt
