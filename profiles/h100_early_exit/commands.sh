#!/bin/bash
# Alternating parent / new measurements on one H100, in one session.  _parent/ holds the parent commit's tree
# (git archive HEAD~ | tar -x -C _parent), built like this one with __graft_entry__.build().
set -u
OUT=out; mkdir -p $OUT
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee $OUT/gpu.txt
for i in 1 2 3; do
  for b in par new; do
    d=.; [ $b = par ] && d=_parent
    (cd $d && python bench.py --gpus 1 --dump-outputs /tmp/dump_${b}_$i) > $OUT/bench_${b}_$i.json 2> $OUT/bench_${b}_$i.err
    tail -1 $OUT/bench_${b}_$i.json | cut -c1-400
  done
done
python - <<'PY'
import numpy as np
for f in ("decision_bits", "counts"):
    a = [np.load(f"/tmp/dump_{b}_{i}/{f}.npy") for b in ("par", "new") for i in (1, 2, 3)]
    print(f, "identical" if all(np.array_equal(a[0], x) for x in a) else "DIFFER")
PY
for args in "--configs c2,c3" "--configs c2,c3 --fill idle --no-power-row" "--configs c2,c3 --fill late --no-power-row" "--configs c2 --series-max" "--configs c2 --fill busy --no-power-row"; do
  for r in 1 2; do
    for b in par new; do
      d=.; [ $b = par ] && d=_parent
      echo "== $b $args" ; (cd $d && python tools/kbench.py $args) 2>&1 | tail -6
    done
  done
done 2>&1 | tee $OUT/kbench.txt
