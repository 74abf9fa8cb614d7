#!/bin/bash
# Alternating parent / new measurements on one H100, in one session.  _parent/ holds the parent commit's tree
# (git archive HEAD~ | tar -x -C _parent), built like this one with __graft_entry__.build().
# usage: commands.sh bench|kbench|short   (run as consecutive jobs on the same machine; short_runs.txt is from
# earlier builds of this change, see its header)
#   short: tools-free timing of bench.py's call pattern at 5, 20 and 200 decisions per run, and of one isolated
#   blocking decision (short_runs.py beside this file)
set -u
OUT=${OUT:-out}; mkdir -p $OUT
PARENT=${PARENT:-_parent}
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee $OUT/gpu.txt
if [ "$1" = bench ]; then
  for i in 1 2 3; do
    for b in par new; do
      d=.; [ $b = par ] && d=$PARENT
      (cd $d && python bench.py --gpus 1 --dump-outputs /tmp/dump_${b}_$i) > $OUT/bench_${b}_$i.json 2> $OUT/bench_${b}_$i.err
      tail -1 $OUT/bench_${b}_$i.json | cut -c1-300
    done
  done
  python - <<'PY' | tee $OUT/dump_compare.txt
import numpy as np
for f in ("decision_bits", "counts"):
    a = [np.load(f"/tmp/dump_{b}_{i}/{f}.npy") for b in ("par", "new") for i in (1, 2, 3)]
    print(f, "identical" if all(np.array_equal(a[0], x) for x in a) else "DIFFER")
PY
  rm -rf /tmp/dump_par_* /tmp/dump_new_*
elif [ "$1" = short ]; then
  for r in 1 2; do
    for b in par new; do
      d=.; [ $b = par ] && d=$PARENT
      (cd $d && python "$OLDPWD/profiles/h100_probe/short_runs.py" $b) 2>&1 | grep -v Warning
    done
  done | tee $OUT/short_runs.txt
else
  for args in "--configs c2,c3" "--configs c2 --fill idle --no-power-row" "--configs c2 --fill late --no-power-row" \
              "--configs c2 --series-max" "--configs c2 --fill busy --no-power-row"; do
    for r in 1 2; do
      for b in par new; do
        d=.; [ $b = par ] && d=$PARENT
        echo "== $b $args" ; (cd $d && python tools/kbench.py --variants auto $args) 2>&1 | tail -3
      done
    done
  done 2>&1 | tee $OUT/kbench.txt
fi
