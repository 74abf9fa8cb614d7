#!/bin/bash
# Run from the repository root after __graft_entry__.build(), on one H100.  $PARENT holds the parent commit's tree
# (git archive HEAD~ | tar -x -C $PARENT), built the same way.  gpu*.txt is read in the same run as the numbers.
set -u
OUT=${OUT:-out}; mkdir -p $OUT
PARENT=${PARENT:-_parent}
# ---- run 1: bench.py, parent and this change, alternated; the outputs of the last timed step compared
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee $OUT/gpu.txt
for i in 1 2; do
  for b in par new; do
    d=.; [ $b = par ] && d=$PARENT
    (cd $d && python bench.py --gpus 1 --steps 2000 --warmup 20 --dump-outputs /tmp/dump_${b}_$i) \
      > $OUT/bench_${b}_$i.json 2> /dev/null
    tail -1 $OUT/bench_${b}_$i.json | cut -c1-200
  done
done
python - <<'PY' | tee $OUT/dump_compare.txt
import numpy as np
for f in ("decision_bits", "counts"):
    a = [np.load(f"/tmp/dump_{b}_{i}/{f}.npy") for b in ("par", "new") for i in (1, 2)]
    print(f, "identical" if all(np.array_equal(a[0], x) for x in a) else "DIFFER")
PY
rm -rf /tmp/dump_par_* /tmp/dump_new_*
# ---- run 2: the snapshot tests and the suites they build on, smoke, and the snapshot numbers at C2 with power
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee $OUT/gpu_r2.txt
python -m pytest -q -m gpu tests/test_gpu_daemon_snapshot.py tests/test_gpu_daemon.py tests/test_gpu_resident_export.py \
  tests/test_gpu_chunks.py tests/test_gpu_groups.py tests/test_gpu_host_e2e.py tests/test_gpu_resident.py \
  > $OUT/pytest_gpu_named.txt 2>&1
tail -2 $OUT/pytest_gpu_named.txt
python -c "import __graft_entry__ as g; g.smoke()" > $OUT/smoke.txt 2>&1; tail -1 $OUT/smoke.txt
python tools/snapshot_bench.py --repeats 3 > $OUT/snapshot_bench.json 2> $OUT/snapshot_bench.err
cut -c1-300 $OUT/snapshot_bench.json
# ---- run 3, on the final tree (the snapshot emulator moved to tests/cpp/snapshot_emul.cpp; TextDevice's snapshot
# methods given refusing defaults): the suites that build the host units or run the binary
python -m pytest -q -m gpu tests/test_gpu_daemon_snapshot.py tests/test_gpu_daemon.py tests/test_gpu_groups.py \
  tests/test_gpu_host_e2e.py tests/test_gpu_resident_export.py > $OUT/pytest_gpu_final.txt 2>&1
tail -2 $OUT/pytest_gpu_final.txt
