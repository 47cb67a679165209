#!/bin/bash
# a quick look after a kernel change: the assembly / solve / dense Cholesky tests, then BASELINE configs 3 and 5 with their phase times
mkdir -p gpurun_out
timeout 900 python -m pytest tests/test_normal_gpu.py tests/test_optimize_gpu.py tests/test_solve_golden.py tests/test_factorization_gpu.py -m gpu -q 2>&1 | cut -c1-300 > gpurun_out/quick_pytest.txt
tail -4 gpurun_out/quick_pytest.txt
# the dense Cholesky kernels one by one (factorizations, solves, the not-positive-definite report): the summary only
timeout 900 python -m pytest tests/test_cholesky_gpu.py -m gpu -q 2>&1 | tail -4 | cut -c1-300
timeout 200 python scripts/solve_config.py 3 300 3 2>&1 | tail -1 | cut -c1-700
timeout 300 python scripts/solve_config.py 5 60 2 2>&1 | tail -1 | cut -c1-700
