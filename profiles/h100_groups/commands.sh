#!/bin/bash
# Alternating parent / new measurements on one H100, in one session.  _parent/ holds the parent commit's tree
# (git archive HEAD~ | tar -x -C _parent), built like this one with __graft_entry__.build().
set -u
OUT=out; mkdir -p $OUT
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > $OUT/gpu.txt
for i in 1 2 3; do
  for b in par new; do
    d=.; [ $b = par ] && d=_parent
    (cd $d && python bench.py --gpus 1 --dump-outputs /tmp/dump_${b}_$i) > $OUT/bench_${b}_$i.json 2> $OUT/bench_${b}_$i.err
  done
done
python - > $OUT/dump_compare.txt <<'PY'
import glob, os
import numpy as np
for f in sorted(os.path.basename(f) for f in glob.glob("/tmp/dump_par_1/*.npy")):
    a = [np.load(f"/tmp/dump_{b}_{i}/{f}") for b in ("par", "new") for i in (1, 2, 3)]
    print(f, "identical" if all(np.array_equal(a[0], x) for x in a) else "DIFFER")
PY
python tools/groups_bench.py > $OUT/groups_bench.txt
