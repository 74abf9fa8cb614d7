#!/bin/bash
# H100 80GB HBM3 at a 700 W power limit (gpu.txt, read in the same session).  _parent/ is the parent commit's tree,
# built beside this one; bench.py runs alternate between the two builds.
set -u
O=profiles/h100_late
python -c "import __graft_entry__ as g; g.build(); g.smoke()" > $O/smoke.txt 2>&1
(cd _parent && python -c "import __graft_entry__ as g; g.build()")
python -m pytest -q -m gpu tests/test_gpu_late_ticks.py tests/test_gpu_late_samples.py tests/test_gpu_daemon.py \
  tests/test_gpu_query_slices.py tests/test_gpu_daemon_snapshot.py tests/test_gpu_daemon_reshape.py 2>&1 | tail -60 > $O/pytest_gpu.txt
nvidia-smi --query-gpu=name,power.limit --format=csv > $O/gpu.txt
for r in 1 2; do
  (cd _parent && python bench.py --gpus 1 --steps 2000 --warmup 20 --dump-outputs /tmp/dump_par | tail -1) > $O/bench_par_$r.json
  python bench.py --gpus 1 --steps 2000 --warmup 20 --dump-outputs /tmp/dump_new | tail -1 > $O/bench_new_$r.json
done
diff -r /tmp/dump_par /tmp/dump_new > $O/dump_compare.txt 2>&1; echo "diff rc=$?" >> $O/dump_compare.txt

# The re-ask's cost at C2 through the binary (late_bench.json, late_bench_runs.txt), and the GPU suites after the
# patched-bucket fix (pytest_gpu_r2.txt, smoke_r2.txt); gpu_r2.txt was read before and after in the same session.
O=profiles/h100_late
python -c "import __graft_entry__ as g; g.build(); g.smoke()" > $O/smoke_r2.txt 2>&1
nvidia-smi --query-gpu=name,power.limit --format=csv > $O/gpu_r2.txt
python -m pytest -q -m gpu tests/test_gpu_late_ticks.py tests/test_gpu_late_samples.py tests/test_gpu_daemon.py \
  tests/test_gpu_query_slices.py tests/test_gpu_daemon_snapshot.py tests/test_gpu_daemon_reshape.py \
  tests/test_gpu_session_ring.py 2>&1 | tail -40 > $O/pytest_gpu_r2.txt
python tools/late_bench.py > $O/late_bench.json 2> $O/late_bench_runs.txt
nvidia-smi --query-gpu=name,power.limit --format=csv >> $O/gpu_r2.txt
