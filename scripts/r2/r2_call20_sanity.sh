#!/bin/bash
# sanity run of HEAD: gpu tests, smoke, bench (both arms)
mkdir -p gpurun_out/c20
python -m pytest tests -m gpu -x -q > gpurun_out/c20/gputest.log 2>&1; echo "pytest rc=$?" >> gpurun_out/c20/gputest.log
python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/c20/smoke.log 2>&1; echo "smoke rc=$?" >> gpurun_out/c20/smoke.log
python bench.py > gpurun_out/c20/bench.json 2> gpurun_out/c20/bench.err; echo "bench rc=$?" >> gpurun_out/c20/bench.err
python bench.py --impl reference --steps 2 --warmup 1 > gpurun_out/c20/bench_ref.json 2> gpurun_out/c20/bench_ref.err
python scripts/bench_kernels.py > gpurun_out/c20/kernels.jsonl 2> gpurun_out/c20/kernels.err
tail -3 gpurun_out/c20/gputest.log; tail -2 gpurun_out/c20/smoke.log; cut -c1-300 gpurun_out/c20/bench.json
