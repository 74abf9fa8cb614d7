#!/bin/bash
# Run from the repository root on one H100:  bash profiles/h100_retime/commands.sh STAGE   (OUT: the output directory).
# $PARENT holds the parent commit's tree (git archive HEAD | tar -x -C $PARENT, before this change is committed).  The
# GPU's name and power limit are read in the same run as the numbers.
set -u
OUT=${OUT:-out}; mkdir -p $OUT
PARENT=${PARENT:-_parent}
STAGE=${1:-1}
python -c "import __graft_entry__ as g; g.build()" > $OUT/build.txt 2>&1 || { tail -20 $OUT/build.txt; exit 1; }
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee $OUT/gpu_r$STAGE.txt
case $STAGE in
1)  # the new GPU test and the suites it builds on, smoke, the retime numbers, and bench.py against the parent
    python -m pytest -q -m gpu tests/test_gpu_resident_retime.py tests/test_gpu_resident_remap.py \
      tests/test_gpu_resident_live_rows.py tests/test_api_launch_path.py tests/test_gpu_daemon_reshape.py \
      > $OUT/pytest_gpu_named.txt 2>&1
    tail -15 $OUT/pytest_gpu_named.txt
    python -c "import __graft_entry__ as g; g.smoke()" > $OUT/smoke.txt 2>&1; tail -3 $OUT/smoke.txt
    python tools/retime_bench.py > $OUT/retime_bench.json 2> $OUT/retime_bench.err
    cut -c1-1500 $OUT/retime_bench.json; tail -5 $OUT/retime_bench.err
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
3)  # the binary with --retime-ring, the ABI test, the daemon and snapshot suites they build on, and smoke
    python -m pytest -q -m gpu tests/test_gpu_daemon_retime.py tests/test_gpu_resident_retime.py \
      tests/test_gpu_daemon_snapshot.py tests/test_gpu_daemon.py > $OUT/pytest_gpu_daemon_retime.txt 2>&1
    tail -15 $OUT/pytest_gpu_daemon_retime.txt
    python -c "import __graft_entry__ as g; g.smoke()" > $OUT/smoke_r3.txt 2>&1; tail -3 $OUT/smoke_r3.txt ;;
2)  # the rest of the GPU suite
    python -m pytest -q -m gpu tests/ > $OUT/pytest_gpu_all.txt 2>&1; tail -8 $OUT/pytest_gpu_all.txt ;;
esac
