#!/bin/bash
# Run from the repository root on one H100:  bash commands.sh STAGE   (OUT: the output directory).  $PARENT holds the
# parent commit's tree (git archive HEAD~ | tar -x -C $PARENT).  The GPU's name and power limit are read in the same
# run as the numbers.
set -u
OUT=${OUT:-out}; mkdir -p $OUT
PARENT=${PARENT:-_parent}
STAGE=${1:-1}
python -c "import __graft_entry__ as g; g.build()" > $OUT/build.txt 2>&1 || { tail -20 $OUT/build.txt; exit 1; }
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee $OUT/gpu_r$STAGE.txt
case $STAGE in
1)  # the new GPU tests and the suites they build on, and smoke
    python -m pytest -q -m gpu tests/test_gpu_resident_live_rows.py tests/test_gpu_daemon_reshape.py tests/test_gpu_daemon.py \
      tests/test_gpu_resident_remap.py tests/test_gpu_daemon_snapshot.py tests/test_gpu_resident.py tests/test_api_launch_path.py \
      > $OUT/pytest_gpu_named.txt 2>&1
    tail -15 $OUT/pytest_gpu_named.txt
    python -c "import __graft_entry__ as g; g.smoke()" > $OUT/smoke.txt 2>&1; tail -3 $OUT/smoke.txt ;;
2)  # bench.py, parent and this change, alternated; the outputs of the last timed step compared
    (cd $PARENT && python -c "import __graft_entry__ as g; g.build()") > $OUT/build_parent.txt 2>&1 || exit 1
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
    rm -rf /tmp/dump_par_* /tmp/dump_new_* ;;
3)  # the reshape numbers at C2: the reshaping tick against the rebuild it replaces (fixtures consistent between the
    # two), and gpr_resident_live_rows alone
    python tools/reshape_bench.py --repeats 3 > $OUT/reshape_bench.json 2> $OUT/reshape_bench.err
    cut -c1-600 $OUT/reshape_bench.json; tail -5 $OUT/reshape_bench.err ;;
4)  # the rest of the GPU suite, first half
    ls tests/test_*.py | sort | awk 'NR % 2 == 1' > $OUT/files4.txt
    python -m pytest -q -m gpu $(cat $OUT/files4.txt) > $OUT/pytest_gpu_4.txt 2>&1; tail -5 $OUT/pytest_gpu_4.txt ;;
5)  # the rest of the GPU suite, second half
    ls tests/test_*.py | sort | awk 'NR % 2 == 0' > $OUT/files5.txt
    python -m pytest -q -m gpu $(cat $OUT/files5.txt) > $OUT/pytest_gpu_5.txt 2>&1; tail -5 $OUT/pytest_gpu_5.txt ;;
6)  # on the final tree: the new GPU tests and the suites they build on, and smoke
    python -m pytest -q -m gpu tests/test_gpu_resident_live_rows.py tests/test_gpu_daemon_reshape.py tests/test_gpu_daemon.py \
      tests/test_gpu_daemon_snapshot.py tests/test_gpu_resident_remap.py > $OUT/pytest_gpu_final.txt 2>&1
    tail -3 $OUT/pytest_gpu_final.txt
    python -c "import __graft_entry__ as g; g.smoke()" > $OUT/smoke_final.txt 2>&1; tail -3 $OUT/smoke_final.txt ;;
esac
