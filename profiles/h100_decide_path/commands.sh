#!/bin/bash
# Run from the repository root after __graft_entry__.build(), on one H100.  $PARENT holds the parent commit's tree
# (git archive HEAD~ | tar -x -C $PARENT), built the same way.  gpu.txt is read in the same run as the numbers.
set -u
OUT=${OUT:-out}; mkdir -p $OUT
PARENT=${PARENT:-_parent}
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee $OUT/gpu.txt
# bench.py, parent and this change, alternated; the outputs of the last timed step compared
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
# bench_r2_{new,par}.jsonl, gpu_r2.txt: a second run on another H100 of the same model and power limit, after
# pytest -m gpu over the decision suites (pytest_gpu_named.txt); the same bench.py line in the order new, par, new, par
