# Validation on one H100 (run from the repository root):
#   full GPU suite, smoke(), device-resident timings of every bench workload, the non-power-of-two front ends,
#   bench.py (our arm), launch lists of the two headline kernels.
set -x
export PYTHONUNBUFFERED=1
mkdir -p gpurun_out
timeout 1500 python -m pytest tests -m gpu -q > gpurun_out/v_tests.log 2>&1; echo "rc=$?" >> gpurun_out/v_tests.log
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/v_smoke.log 2>&1; echo "rc=$?" >> gpurun_out/v_smoke.log
rm -f gpurun_out/v_ab.jsonl
timeout 300 python tools/ab_time.py --tag final cfg2 cfg3 cfg4 cfg5 stats speech400 >> gpurun_out/v_ab.jsonl 2>> gpurun_out/v_ab.err
timeout 300 python tools/time_nonpow2.py > gpurun_out/v_nonpow2.jsonl 2> gpurun_out/v_nonpow2.err
timeout 900 python bench.py > gpurun_out/v_bench.json 2> gpurun_out/v_bench.err
tail -n 3 gpurun_out/v_tests.log gpurun_out/v_smoke.log; cut -c1-110 gpurun_out/v_ab.jsonl; head -c 300 gpurun_out/v_bench.json
